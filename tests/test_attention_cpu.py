"""CPU-only checks of the attention-core operators of the C ABI and of the attention routes of the planner: every argument error is
reported before any device work, the scratch query sizes each route, and the dry plans of the reference configs (and of configs
with attention at a 4x4 level, C = 128 and C = 512) keep the launch counts they had before the attention launches moved into the
shared route builders."""
import ctypes as C
import os
import re

import pytest

from oracle import ddpm_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20          # a 16-byte aligned non-null address: every call below fails on the host before it could be used


@pytest.fixture(scope="module")
def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _fwd(**kw):
    from ddpm_torch_b200 import _lib
    d = _lib.AttnDesc()
    d.route, d.NB, d.T, d.C = 3, 2, 64, 64
    d.qkv = d.out = d.probs = d.scratch = FAKE
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _bwd(**kw):
    from ddpm_torch_b200 import _lib
    d = _lib.AttnBwdDesc()
    d.route, d.NB, d.T, d.C = 3, 2, 64, 64
    d.qkv = d.d_out = d.probs = d.d_qkv = d.d_scores = d.scratch = FAKE
    for k, v in kw.items():
        setattr(d, k, v)
    return d


COMMON = [
    (dict(route=0), b"route must be 1 (fused), 2 (t16) or 3"),
    (dict(route=4), b"route must be 1 (fused), 2 (t16) or 3"),
    (dict(NB=0), b"need NB >= 1, T >= 1 and C >= 1"),
    (dict(T=-16), b"need NB >= 1, T >= 1 and C >= 1"),
    (dict(C=0), b"need NB >= 1, T >= 1 and C >= 1"),
    (dict(NB=65536), b"exceeds 65535"),
    (dict(C=100), b"C must be a multiple of 8"),
    (dict(route=1, T=128, C=256), b"route 1 (fused) needs T = 256 and C = 256"),
    (dict(route=1, T=256, C=128), b"route 1 (fused) needs T = 256 and C = 256"),
    (dict(route=2, T=16, C=64), b"route 2 (t16) needs T = 16 and C in {128, 256, 512}"),
    (dict(route=2, T=32, C=128), b"route 2 (t16) needs T = 16 and C in {128, 256, 512}"),
    (dict(qkv=None), b"null buffer"),
    (dict(qkv=FAKE + 8), b"16-byte aligned"),
    (dict(scratch=None), b"needs a scratch area"),
]


@pytest.mark.parametrize("kw,msg", COMMON + [
    (dict(out=None), b"null buffer"),
    (dict(probs=None), b"route 3 writes the probabilities: probs is required"),
    (dict(out=FAKE + 2), b"16-byte aligned"),
    (dict(probs=FAKE + 4), b"16-byte aligned"),
])
def test_attention_fwd_validates_arguments(L, kw, msg):
    d = _fwd(**kw)
    assert L.ddpm_attention_fwd_run(C.byref(d), None) != 0
    assert msg in L.ddpm_last_error(), L.ddpm_last_error()


@pytest.mark.parametrize("kw,msg", COMMON + [
    (dict(d_out=None), b"null buffer"),
    (dict(d_qkv=None), b"null buffer"),
    (dict(probs=None), b"probs is required"),
    (dict(route=2, T=16, C=128, probs=None), b"probs is required"),
    (dict(route=1, T=256, C=256, probs=None), b"probs is required"),
    (dict(route=1, T=256, C=256, scratch=None), b"needs a scratch area"),
    (dict(d_scores=FAKE + 8), b"16-byte aligned"),
])
def test_attention_bwd_validates_arguments(L, kw, msg):
    d = _bwd(**kw)
    assert L.ddpm_attention_bwd_run(C.byref(d), None) != 0
    assert msg in L.ddpm_last_error(), L.ddpm_last_error()


def test_null_descriptors_are_refused(L):
    assert L.ddpm_attention_fwd_run(None, None) != 0 and b"null descriptor" in L.ddpm_last_error()
    assert L.ddpm_attention_bwd_run(None, None) != 0 and b"null descriptor" in L.ddpm_last_error()


def _al(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize("NB,T,C_", [(1, 16, 128), (3, 64, 64), (2, 1024, 128), (128, 256, 256)])
def test_scratch_bytes(L, NB, T, C_):
    """route 3: fp32 S forward, fp32 dP + bf16 dS backward; route 1: bf16 dS backward; route 2: nothing."""
    tt = NB * T * T
    assert L.ddpm_attn_scratch_bytes(3, NB, T, C_, 0) == _al(4 * tt)
    assert L.ddpm_attn_scratch_bytes(3, NB, T, C_, 1) == _al(4 * tt) + _al(2 * tt)
    if (T, C_) == (256, 256):
        assert L.ddpm_attn_scratch_bytes(1, NB, T, C_, 0) == 0
        assert L.ddpm_attn_scratch_bytes(1, NB, T, C_, 1) == _al(2 * tt)
    if T == 16:
        assert L.ddpm_attn_scratch_bytes(2, NB, T, C_, 0) == 0 and L.ddpm_attn_scratch_bytes(2, NB, T, C_, 1) == 0


def test_scratch_bytes_refusals(L):
    for args, msg in (((0, 1, 16, 128, 0), b"route"), ((2, 1, 64, 128, 0), b"route 2 (t16)"), ((1, 1, 16, 256, 1), b"route 1 (fused)"),
                      ((3, 1, 64, 60, 0), b"multiple of 8"), ((3, 0, 64, 64, 0), b"NB >= 1"), ((3, 1, 64, 64, 2), b"backward must be 0 or 1")):
        assert L.ddpm_attn_scratch_bytes(*args) < 0
        assert msg in L.ddpm_last_error(), (args, L.ddpm_last_error())


def test_entry_points_declared_and_exported(L):
    from ddpm_torch_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ddpm_b200.h")).read(), flags=re.S)
    for name in ("ddpm_attention_fwd_run", "ddpm_attention_bwd_run", "ddpm_attn_scratch_bytes"):
        assert re.search(rf"\b{name}\s*\(", hdr) and name in _lib.EXPORTS and hasattr(L, name)


def test_descriptor_layouts_match_header():
    from ddpm_torch_b200 import _lib
    import subprocess, tempfile
    src = ('#include "include/ddpm_b200.h"\n#include <stdio.h>\n#include <stddef.h>\nint main(){printf("%zu %zu %zu %zu", '
           'sizeof(ddpm_attn_desc), sizeof(ddpm_attn_bwd_desc), offsetof(ddpm_attn_desc, scratch), offsetof(ddpm_attn_bwd_desc, d_scores));}')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c"); open(c, "w").write(src)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", ROOT, c, "-o", exe], cwd=ROOT)
        a, b, o1, o2 = map(int, subprocess.check_output([exe]).split())
    assert (a, b) == (C.sizeof(_lib.AttnDesc), C.sizeof(_lib.AttnBwdDesc))
    assert (o1, o2) == (_lib.AttnDesc.scratch.offset, _lib.AttnBwdDesc.d_scores.offset)


# ------------------------------------------------------------------------------------------------ dry plans
CELEBA64_CFG = dict(in_channels=3, hid_channels=128, out_channels=3, ch_multipliers=(1, 2, 2, 2), num_res_blocks=2,
                    apply_attn=(False, False, True, False), drop_rate=0.0)          # configs/celeba.json
# attention at a 4x4 level (and in the middle block) with C = 128 / C = 512: the t16 route at the two widths no reference config has
ATT4_C128_CFG = dict(in_channels=3, hid_channels=64, out_channels=3, ch_multipliers=(1, 2), num_res_blocks=1,
                     apply_attn=(False, True), drop_rate=0.0)
ATT4_C512_CFG = dict(in_channels=3, hid_channels=128, out_channels=3, ch_multipliers=(1, 4), num_res_blocks=1,
                     apply_attn=(False, True), drop_rate=0.0)

# (cfg, B, H = W): training plan (forward, backward, repack launches, tensor-core ops, CUDA-core ops), inference plan (forward,
# repack, tensor-core ops, CUDA-core ops), as planned by the parent commit of the shared attention route builders
PLANS = {
    "tiny": ((R.TINY_CFG, 2, 16), (78, 158, 1, 52, 61), (78, 1, 15, 19)),
    "small64": ((R.SMALL64_CFG, 4, 32), (76, 168, 4, 124, 0), (76, 3, 36, 0)),
    "cifar10": ((R.CIFAR10_CFG, 128, 32), (146, 378, 5, 266, 2), (152, 4, 79, 1)),
    "celeba64": ((CELEBA64_CFG, 8, 64), (150, 383, 4, 263, 6), (156, 3, 78, 2)),
    "celebahq": ((R.CELEBAHQ_CFG, 4, 256), (206, 522, 4, 366, 6), (214, 3, 110, 2)),
    "att4_c128": ((ATT4_C128_CFG, 4, 8), (72, 163, 4, 100, 8), (72, 3, 28, 4)),
    "att4_c512": ((ATT4_C512_CFG, 4, 8), (78, 175, 4, 100, 8), (79, 3, 31, 4)),
}


def _plan(L, cfg, B, HW, training):
    from ddpm_torch_b200 import _lib
    c = R.normalize_cfg(cfg)
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = c["in_channels"], c["hid_channels"], c["out_channels"]
    u.levels, u.num_res_blocks, u.temb_dim, u.drop_rate = len(c["ch_multipliers"]), c["num_res_blocks"], 0, c["drop_rate"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    h = C.c_void_p()
    assert L.ddpm_unet_create(C.byref(u), C.byref(h)) == 0, L.ddpm_last_error()
    try:
        assert L.ddpm_unet_workspace_bytes(h, B, HW, HW, training) > 0, L.ddpm_last_error()
        f, b, p = C.c_int(), C.c_int(), C.c_int()
        L.ddpm_unet_launch_counts(h, C.byref(f), C.byref(b), C.byref(p))
        ntc, ng = C.c_int(), C.c_int()
        L.ddpm_unet_plan_stats(h, None, None, C.byref(ntc), C.byref(ng), None, None)
        return (f.value, b.value, p.value, ntc.value, ng.value) if training else (f.value, p.value, ntc.value, ng.value)
    finally:
        L.ddpm_unet_destroy(h)


@pytest.mark.parametrize("name", sorted(PLANS))
def test_dry_plan_launch_counts_unchanged(L, name):
    (cfg, B, HW), train_counts, infer_counts = PLANS[name]
    assert _plan(L, cfg, B, HW, 1) == train_counts
    assert _plan(L, cfg, B, HW, 0) == infer_counts
