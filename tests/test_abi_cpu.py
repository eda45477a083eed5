"""CPU-only checks of the boundary: the C-ABI library loads and exports every symbol include/ddpm_b200.h declares,
the engine's parameter inventory equals the reference's state_dict (names, shapes, order), the compiled plan's
algorithmic FLOPs equal the reference model's, and the product path refuses to run without a GPU (no fallback)."""
import ctypes as C
import math
import os
import re

import pytest
import torch

from oracle import ddpm_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def test_library_exports_every_declared_symbol(L):
    hdr = open(os.path.join(ROOT, "include", "ddpm_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(ddpm_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 20
    for n in sorted(names):
        assert hasattr(L, n), f"{n} declared in include/ddpm_b200.h but not exported"
    from ddpm_torch_b200 import _lib
    assert set(_lib.EXPORTS) == names


def test_struct_layouts_match_header():
    from ddpm_torch_b200 import _lib
    src = ('#include "include/ddpm_b200.h"\n#include <stdio.h>\n#include <stddef.h>\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu", '
           'sizeof(ddpm_gemm_desc), sizeof(ddpm_unet_cfg), sizeof(ddpm_opt_cfg), sizeof(ddpm_halo_desc), sizeof(ddpm_gn_epi), '
           'offsetof(ddpm_gemm_desc, gn), offsetof(ddpm_halo_desc, gn), sizeof(ddpm_gn_desc), sizeof(ddpm_gn_bwd_desc), '
           'offsetof(ddpm_gn_desc, seed), offsetof(ddpm_gn_bwd_desc, scratch));}')
    import subprocess, tempfile
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c"); open(c, "w").write(src)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", ROOT, c, "-o", exe], cwd=ROOT)
        a, b, c_, hd, ge, og, oh, gd, gbd, o_seed, o_scr = map(int, subprocess.check_output([exe]).split())
    assert a == C.sizeof(_lib.GemmDesc) and b == C.sizeof(_lib.UnetCfg) and c_ == C.sizeof(_lib.OptCfg)
    assert hd == C.sizeof(_lib.HaloDesc) and ge == C.sizeof(_lib.GnEpi)
    assert og == _lib.GemmDesc.gn.offset and oh == _lib.HaloDesc.gn.offset
    assert gd == C.sizeof(_lib.GnDesc) and gbd == C.sizeof(_lib.GnBwdDesc)
    assert o_seed == _lib.GnDesc.seed.offset and o_scr == _lib.GnBwdDesc.scratch.offset


def test_no_gpu_means_error_not_fallback(L):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert L.ddpm_runtime_check() != 0
    assert b"CUDA" in L.ddpm_last_error() or b"device" in L.ddpm_last_error()
    import ddpm_torch_b200 as D
    m = D.UNet(3, 32, 3, (1, 2), 1, (False, True))
    with pytest.raises(RuntimeError, match="no CPU"):
        m(torch.zeros(1, 3, 16, 16), torch.zeros(1, dtype=torch.long))


def _handle(L, cfg):
    from ddpm_torch_b200 import _lib
    c = R.normalize_cfg(cfg)
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = c["in_channels"], c["hid_channels"], c["out_channels"]
    u.levels, u.num_res_blocks, u.temb_dim, u.drop_rate = len(c["ch_multipliers"]), c["num_res_blocks"], 0, c["drop_rate"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    h = C.c_void_p()
    assert L.ddpm_unet_create(C.byref(u), C.byref(h)) == 0, L.ddpm_last_error()
    return h


@pytest.mark.parametrize("cfg,n_params", [(R.CIFAR10_CFG, 35_746_307), (R.CELEBAHQ_CFG, 113_673_219), (R.TINY_CFG, None)])
def test_param_inventory_is_the_reference_state_dict(L, cfg, n_params):
    h = _handle(L, cfg)
    shapes = R.param_shapes(cfg)
    assert L.ddpm_unet_num_params(h) == len(shapes)
    total, ranges = 0, []
    for i, (k, s) in enumerate(shapes.items()):
        nm, nd, dims, off = C.c_char_p(), C.c_int(), (C.c_int * 4)(), C.c_longlong()
        assert L.ddpm_unet_param_info(h, i, C.byref(nm), C.byref(nd), C.byref(dims), C.byref(off)) == 0
        assert nm.value.decode() == k and tuple(dims[:nd.value]) == tuple(s)           # the LIST is the reference's state_dict order
        assert off.value % 64 == 0
        ranges.append((off.value, off.value + math.prod(s), k)); total += math.prod(s)
    if n_params:
        assert total == n_params
    # memory placement: registration order, except that the embedding MLP and the fc.weight tensors (whose gradients only exist
    # at the very end of the backward pass) sit behind everything else, so the rest completes in contiguous per-level chunks
    ranges.sort()
    for (a0, a1, _), (b0, b1, _) in zip(ranges, ranges[1:]):
        assert a1 <= b0
    assert L.ddpm_unet_flat_elems(h) >= ranges[-1][1]
    late = [k for _, _, k in ranges if k.startswith("embed.") or k.endswith(".fc.weight")]
    assert [k for _, _, k in ranges][-len(late):] == late
    main = [k for _, _, k in ranges][:-len(late)]
    assert main == [k for k in shapes if k not in set(late)]
    L.ddpm_unet_destroy(h)


@pytest.mark.parametrize("cfg,B,HW", [(R.CIFAR10_CFG, 128, 32), (R.CELEBAHQ_CFG, 4, 256), (R.SMALL64_CFG, 4, 32)])
def test_plan_flops_equal_reference_model(L, cfg, B, HW):
    h = _handle(L, cfg)
    need = L.ddpm_unet_workspace_bytes(h, B, HW, HW, 1)
    assert need > 0, L.ddpm_last_error()
    nf, nb, ntc, ng = C.c_int(), C.c_int(), C.c_int(), C.c_int(); ff, bf = C.c_double(), C.c_double()
    L.ddpm_unet_plan_stats(h, C.byref(nf), C.byref(nb), C.byref(ntc), C.byref(ng), C.byref(ff), C.byref(bf))
    ref = R.fwd_flops_per_image(cfg, HW, HW)
    assert abs(ff.value / B - ref) / ref < 1e-6          # 12.444 / 497.03 GFLOP per image
    assert 1.9 < bf.value / ff.value < 2.2               # dgrad + wgrad
    assert ntc.value > 5 * ng.value                      # the contraction work is on the tensor-core engine
    L.ddpm_unet_destroy(h)


def test_bad_configs_return_errors_not_aborts(L):
    from ddpm_torch_b200 import _lib
    u = _lib.UnetCfg(); u.in_channels = 3; u.hid_channels = 48; u.out_channels = 3; u.levels = 2; u.num_res_blocks = 1
    h = C.c_void_p()
    assert L.ddpm_unet_create(C.byref(u), C.byref(h)) != 0 and b"32" in L.ddpm_last_error()
    h = _handle(L, R.TINY_CFG)
    assert L.ddpm_unet_workspace_bytes(h, 2, 15, 15, 0) < 0          # not divisible by 2^(levels-1)
    assert L.ddpm_unet_repack(h, None) != 0                          # no plan yet
    L.ddpm_unet_destroy(h)


def test_graph_epoch_moves_with_every_dry_plan(L):
    h = _handle(L, R.TINY_CFG)
    e = L.ddpm_unet_graph_epoch(h)
    assert e >= 0, L.ddpm_last_error()
    for _ in range(2):
        assert L.ddpm_unet_workspace_bytes(h, 2, 16, 16, 0) > 0
        assert L.ddpm_unet_graph_epoch(h) > e
        e = L.ddpm_unet_graph_epoch(h)
    assert L.ddpm_unet_graph_epoch(None) < 0 and b"null" in L.ddpm_last_error()
    L.ddpm_unet_destroy(h)


def test_python_module_mirrors_reference_surface():
    import inspect
    import ddpm_torch_b200 as D
    sig = inspect.signature(D.UNet.__init__)
    assert list(sig.parameters)[1:] == ["in_channels", "hid_channels", "out_channels", "ch_multipliers", "num_res_blocks",
                                        "apply_attn", "time_embedding_dim", "drop_rate", "resample_with_conv"]   # unet.py:96-107
    for name in ("q_sample", "train_losses", "p_sample", "p_sample_step", "p_mean_var", "q_posterior_mean_var", "p_sample_progressive"):
        assert hasattr(D.GaussianDiffusion, name)
    assert list(inspect.signature(D.DDIM.__init__).parameters)[1:] == ["betas", "model_mean_type", "model_var_type", "loss_type", "eta", "subsequence"]
    m = D.UNet(3, 32, 3, (1, 2), 1, (False, True))
    sd = R.make_state_dict(R.TINY_CFG, 1)
    assert list(m.state_dict().keys()) == list(sd.keys())
    m.load_state_dict(sd)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items()) and m._views_ok()


def test_opt_step_validates_arguments_before_touching_the_device(L):
    """ddpm_opt_step (clip + Adam + EMA, utils/train.py:159-165): argument errors are reported through the C ABI."""
    from ddpm_torch_b200 import _lib
    cfg = _lib.OptCfg(); cfg.lr, cfg.beta1, cfg.beta2, cfg.eps, cfg.max_grad_norm, cfg.ema_decay, cfg.step = 2e-4, .9, .999, 1e-8, 1., .9999, 1
    assert L.ddpm_opt_step(None, None, None, None, None, 16, C.byref(cfg), None, None, None) != 0
    assert b"null" in L.ddpm_last_error()
    buf = (C.c_float * 64)()
    a = C.addressof(buf)
    a16 = (a + 15) // 16 * 16
    assert L.ddpm_opt_step(a16, a16, a16, a16, a16, 6, C.byref(cfg), a16, a16, None) != 0          # n % 4 != 0
    assert b"multiple of 4" in L.ddpm_last_error()
    cfg.step = 0
    assert L.ddpm_opt_step(a16, a16, a16, a16, a16, 8, C.byref(cfg), a16, a16, None) != 0
    assert b"1-based" in L.ddpm_last_error()
    cfg.step = 1
    assert L.ddpm_opt_step(a16, a16, a16, a16, None, 8, C.byref(cfg), a16, a16, None) != 0         # EMA on, no shadow
    assert L.ddpm_opt_step(a16 + 4, a16, a16, a16, a16, 8, C.byref(cfg), a16, a16, None) != 0      # misaligned
    assert b"aligned" in L.ddpm_last_error()
