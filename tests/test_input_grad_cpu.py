"""Gradients of the UNet with respect to its input x (model(x, t) under autograd, ddpm_unet_backward_ex), without a GPU:

1. The oracle (torch.autograd through oracle/ddpm_ref.py::unet_forward, tests/noresample_ref.py for resample_with_conv=False)
   against the UNMODIFIED reference (tests/golden/unet_input_grad.pt, tools/gen_golden_input_grad.py): dx rel-L2 < 1e-5 in
   every case, and the x_t-gradient of the guidance loss.  tests/test_input_grad_gpu.py leans on it.
2. The C ABI: argument refusals of ddpm_unet_backward_ex / ddpm_unet_backward_launches, and both entry points declared in the
   header and listed in _lib.EXPORTS (which tests/test_abi_cpu.py then holds to the library's symbols).
3. Dry plans: the default backward keeps its launch counts, the input-only backward is strictly smaller by exactly the
   parameter-only launches derived below, and the dx op takes the tensor-core route exactly where out_conv's forward does."""
import ctypes as C
import os
import re

import pytest
import torch

import noresample_ref as N
from oracle import ddpm_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = "unet_input_grad.pt"
NAMES = ["tiny_c1", "tiny_c3", "tiny_c4", "small64_c1", "small64_c2", "small64_c3", "cifar10", "small64_c1to2", "small64_noresample"]


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def oracle_fn(fx):
    """(x, t) -> eps of the oracle over the case's weights (fp32, no dropout)."""
    cfg = fx["cfg"]
    if fx["resample_with_conv"]:
        sd = R.make_state_dict(cfg, fx["seed"])
        return lambda x, t: R.unet_forward(sd, cfg, x, t)
    sd = N.make_state_dict(cfg, fx["seed"])
    return lambda x, t: N.unet_forward(sd, cfg, x, t)


# ------------------------------------------------------------------------------------------------ oracle vs reference
def test_fixture_covers_the_cases(golden):
    assert sorted(golden(FIXTURE)["models"]) == sorted(NAMES)
    assert os.path.getsize(os.path.join(ROOT, "tests", "golden", FIXTURE)) < 1.5e6


@pytest.mark.parametrize("name", NAMES)
def test_oracle_dx_matches_reference(golden, name):
    fx = golden(FIXTURE)["models"][name]
    fn = oracle_fn(fx)
    x = fx["x"].clone().requires_grad_(True)
    (dx,) = torch.autograd.grad((fn(x, fx["t"]) * fx["g"]).sum(), x)
    assert rel_l2(dx, fx["dx"]) < 1e-5
    torch.testing.assert_close(dx.flatten(1).norm(dim=1), fx["dx_norm"], rtol=1e-5, atol=0)


def test_oracle_guidance_gradient_matches_reference(golden):
    """d/dx_t of sum(mask * (x0_hat(x_t) - y)^2), x0_hat from eps, through the mirror's GaussianDiffusion.p_mean_var."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"]["cifar10"]
    gd = fx["guide"]
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    x = fx["x"].clone().requires_grad_(True)
    pred = d.p_mean_var(oracle_fn(fx), x, gd["t"], clip_denoised=False, return_pred=True)[-1]
    loss = (gd["mask"] * (pred - gd["y"])).pow(2).sum()
    (gx,) = torch.autograd.grad(loss, x)
    assert abs(loss.item() - gd["loss"]) <= 1e-5 * gd["loss"]
    assert rel_l2(gx, gd["grad"]) < 1e-5


# ------------------------------------------------------------------------------------------------ C ABI
def test_entry_points_declared_and_exported():
    from ddpm_torch_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ddpm_b200.h")).read(), flags=re.S)
    for name in ("ddpm_unet_backward_ex", "ddpm_unet_backward_launches"):
        assert re.search(rf"\b{name}\s*\(", hdr) and name in _lib.EXPORTS


def _norm(cfg):
    """R.normalize_cfg for either resampler (the engine takes the flag separately)."""
    return R.normalize_cfg(dict(cfg, resample_with_conv=True))


def _cfg_struct(cfg):
    from ddpm_torch_b200 import _lib
    c = _norm(cfg)
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = c["in_channels"], c["hid_channels"], c["out_channels"]
    u.levels, u.num_res_blocks, u.temb_dim, u.drop_rate = len(c["ch_multipliers"]), c["num_res_blocks"], 0, c["drop_rate"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    return u


def _handle(L, cfg, resample_with_conv=1):
    h = C.c_void_p()
    assert L.ddpm_unet_create_ex(C.byref(_cfg_struct(cfg)), resample_with_conv, C.byref(h)) == 0, L.ddpm_last_error()
    return h


def test_backward_ex_refusals(L):
    """Refused before any launch: param_grads not 0 / 1, nothing to compute, no (training) plan."""
    h = _handle(L, R.TINY_CFG)
    try:
        buf = (C.c_float * 64)()
        for bad in (-1, 2, 7):
            assert L.ddpm_unet_backward_ex(h, buf, buf, bad, None) != 0
            assert b"param_grads must be 0 or 1" in L.ddpm_last_error()
        assert L.ddpm_unet_backward_ex(h, buf, None, 0, None) != 0
        assert b"nothing to compute" in L.ddpm_last_error()
        for dx, pg in ((buf, 1), (None, 1), (buf, 0)):
            assert L.ddpm_unet_backward_ex(h, buf, dx, pg, None) != 0
            assert b"ddpm_unet_plan has not been called" in L.ddpm_last_error()
        # an inference (dry) plan has no backward: neither a variant count nor a backward
        assert L.ddpm_unet_workspace_bytes(h, 2, 16, 16, 0) > 0
        assert L.ddpm_unet_backward_launches(h, 1, 0) < 0
        assert b"no training plan" in L.ddpm_last_error()
        assert L.ddpm_unet_workspace_bytes(h, 2, 16, 16, 1) > 0
        assert L.ddpm_unet_backward_launches(h, 0, 0) < 0 and b"nothing to compute" in L.ddpm_last_error()
        for a, b in ((2, 1), (1, 2), (-1, 1)):
            assert L.ddpm_unet_backward_launches(h, a, b) < 0 and b"must be 0 or 1" in L.ddpm_last_error()
        assert L.ddpm_unet_backward_launches(None, 1, 1) < 0
    finally:
        L.ddpm_unet_destroy(h)


# ------------------------------------------------------------------------------------------------ dry plans
def _counts(L, cfg, B, HW, resample_with_conv=1):
    """(forward, default backward, repack) launches and the backward launches of every variant (want_dx, param_grads)."""
    h = _handle(L, cfg, resample_with_conv)
    try:
        assert L.ddpm_unet_workspace_bytes(h, B, HW, HW, 1) > 0, L.ddpm_last_error()
        f, b, p = C.c_int(), C.c_int(), C.c_int()
        L.ddpm_unet_launch_counts(h, C.byref(f), C.byref(b), C.byref(p))
        var = {(dx, pg): L.ddpm_unet_backward_launches(h, dx, pg) for dx, pg in ((0, 1), (1, 1), (1, 0))}
        return (f.value, b.value, p.value), var
    finally:
        L.ddpm_unet_destroy(h)


def test_cifar10_default_backward_unchanged_and_input_only_derived(L):
    """CIFAR-10, bs = 128.  The default backward keeps 146 / 378 / 5 launches.  The dx op is the tensor-core route: the operand pack,
    one KK GEMM and one k_out_gather<3> (3 launches).  The input-only backward drops exactly the parameter-only launches:
        41  bias column sums: 22 ResidualBlock conv2 + 6 AttentionBlocks x (project_out + project_in) + 3 down + 3 up resample
            convs + in_conv
        87  weight-gradient GEMMs: 22 x (conv1 + conv2) + 13 skips (the down block 128 -> 256 and the 12 up blocks, whose
            concat input makes two GEMMs each: 1 + 24) + 6 x 2 attention projections + 6 resample convs
         6  gradient-chunk unpacks
         5  image convs: in_conv weight-gradient GEMM + unpack; out_conv bias sum + weight-gradient GEMM + unpack
        11  timestep MLP: dTP cast, projection backward (3), MLP backward (7)
       150  = 378 + 3 - 231
    The GroupNorm backward pairs stay (their dgamma / dbeta and fused column sums are dropped inside the same launches)."""
    (f, b, p), var = _counts(L, R.CIFAR10_CFG, 128, 32)
    assert (f, b, p) == (146, 378, 5)
    assert var[(0, 1)] == b
    assert var[(1, 1)] == b + 3
    assert var[(1, 0)] == b + 3 - 150 == 231


# (cfg, B, H/W, resample_with_conv): (default backward, input-only + dx, dx launches)
VARIANTS = {
    "tiny_c3": (R.TINY_CFG, 2, 16, 1),
    "tiny_c4": (dict(R.TINY_CFG, in_channels=4, out_channels=4), 2, 16, 1),
    "small64_c1": (dict(R.SMALL64_CFG, in_channels=1, out_channels=1), 2, 32, 1),
    "small64_c3": (R.SMALL64_CFG, 2, 32, 1),
    "small64_c4": (dict(R.SMALL64_CFG, in_channels=4, out_channels=4), 2, 32, 1),
    "small64_c1to2": (dict(R.SMALL64_CFG, in_channels=1, out_channels=2), 2, 32, 1),
    "cifar10_b16": (R.CIFAR10_CFG, 16, 32, 1),
    "cifar10_noresample": (N.CIFAR10_CFG, 128, 32, 0),
}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_input_only_backward_is_strictly_smaller(L, name):
    cfg, B, HW, flag = VARIANTS[name]
    (_, b, _), var = _counts(L, cfg, B, HW, flag)
    assert var[(0, 1)] == b
    assert var[(1, 1)] - b in (2, 3)                     # the dx op: pack + k_out_conv, or pack + GEMM + k_out_gather
    assert 0 < var[(1, 0)] < b


def test_noresample_default_backward_unchanged(L):
    (f, b, p), _ = _counts(L, N.CIFAR10_CFG, 128, 32, 0)
    assert (f, b, p) == (142, 354, 5)


def _out_conv_on_tensor_cores(L, cfg, B, HW, flag):
    """out_conv's forward route, read from the plan: the tensor-core route is a GEMM plus a gather, one forward launch more
    than k_out_conv.  Compared with the same config at out_channels = 4 (9 * 4 > 32: never on the tensor cores)."""
    (f, _, _), _ = _counts(L, cfg, B, HW, flag)
    (f4, _, _), _ = _counts(L, dict(cfg, out_channels=4), B, HW, flag)
    return f == f4 + 1


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_dx_route_follows_out_conv_route(L, name):
    """With in_channels = out_channels, the dx op is on the tensor cores exactly where out_conv's forward is (same rule:
    hid % 64 == 0, a tensor-core geometry, 9 * C <= 32); a 1 -> 2 model follows its in_channels."""
    cfg, B, HW, flag = VARIANTS[name]
    (_, b, _), var = _counts(L, cfg, B, HW, flag)
    tc_dx = var[(1, 1)] - b == 3
    c = _norm(cfg)
    twin = dict(cfg, out_channels=c["in_channels"])
    assert tc_dx == _out_conv_on_tensor_cores(L, twin, B, HW, flag)
    assert tc_dx == (c["hid_channels"] % 64 == 0 and 9 * c["in_channels"] <= 32)
