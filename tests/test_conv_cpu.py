"""CPU-only checks of the convolution operator of the C ABI (ddpm_conv_run / ddpm_conv_scratch_bytes) and of the conv routes of the
planner: every argument error is refused before any device work, the dry report gives each case of tests/test_conv_gpu.py the
route, launches, block_n and split count the planner's rules give its shape, the scratch query sizes each route, the header and
the ctypes layout agree, and dry plans of the reference configs keep the launch counts, op counts, FLOPs and workspace sizes they
had before the conv launches moved into the shared builders of unet_engine.cuh."""
import ctypes as C
import os
import re

import pytest

from oracle import ddpm_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20          # a 16-byte aligned non-null address: every call below fails on the host, or is dry, before it could be used
import test_conv_gpu as G  # noqa: E402  (the case table; importing it needs no GPU)


@pytest.fixture(scope="module")
def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _desc(**kw):
    """a valid forward on the haloed route (CIFAR-10 conv1 at 32x32): every test changes what it refuses"""
    from ddpm_torch_b200 import _lib
    d = _lib.ConvDesc()
    d.op, d.route, d.B, d.H, d.W, d.ksize, d.stride = 0, 1, 2, 32, 32, 3, 1
    d.Cin0, d.Co = 128, 128
    d.x0 = d.w = d.out = d.scratch = FAKE
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _dry(L, d):
    from ddpm_torch_b200 import _lib
    rep = _lib.ConvReport()
    d.dry, d.report = 1, C.pointer(rep)
    rc = L.ddpm_conv_run(C.byref(d), None)
    return rc, rep


def test_valid_descriptor_is_accepted(L):
    rc, rep = _dry(L, _desc())
    assert rc == 0, L.ddpm_last_error()
    assert (rep.route, rep.launches, rep.block_n, rep.splits, rep.zero_bytes) == (1, 2, 128, 1, 0)


REFUSALS = [
    (dict(op=3), b"op must be 0 (forward), 1 (data gradient) or 2"),
    (dict(route=0), b"route must be 1 (halo)"),
    (dict(route=6), b"route must be 1 (halo)"),
    (dict(B=0), b"need B, H and W >= 1"),
    (dict(W=-8), b"need B, H and W >= 1"),
    (dict(ksize=5), b"ksize must be 1 or 3"),
    (dict(stride=3), b"stride must be 1 or 2"),
    (dict(upsample=2), b"upsample must be 0 or 1"),
    (dict(accumulate=2), b"must be 0 or 1"),
    (dict(Cin0=100), b"multiples of 8"),
    (dict(Co=0), b"multiples of 8"),
    (dict(Cs1=64, s1=FAKE), b"a second skip source needs a first"),
    (dict(stride=2, H=31), b"stride 2 needs ksize 3 and an even H and W"),
    (dict(stride=2, Co=256), b"the resample convs need one source with Cin0 = Co"),
    (dict(upsample=1), b"upsample = 1 is the folded route 5"),
    (dict(route=5), b"route 5 (fold) needs upsample = 1"),
    (dict(route=5, upsample=1, H=8, W=8), b"route 5 (fold) needs Co % 256 == 0"),
    (dict(ksize=1, Cs0=128, s0=FAKE, w_skip=FAKE), b"a fused skip needs the forward of a 3x3 stride-1 conv"),
    (dict(identity_skip=1, Cs0=64, s0=FAKE), b"identity_skip needs Cs0 = Co"),
    (dict(skip_bias=FAKE), b"skip_bias needs a 1x1 skip and a bias"),
    (dict(op=1, Cin1=64, dy=FAKE), b"Cin1 must be 0"),
    (dict(op=2, dy=FAKE, bias=FAKE), b"gradients take no bias"),
    (dict(op=2, dy=FAKE, accumulate=1), b"takes no accumulate flag"),
    (dict(rowvec=FAKE, rowvec_ld=64), b"rowvec_ld must be >= Co"),
    (dict(x0=None), b"null buffer"),
    (dict(out=None), b"null buffer"),
    (dict(w=None), b"null buffer"),
    (dict(op=1), b"null buffer"),                                         # no dy
    (dict(Cs0=128, s0=FAKE), b"null buffer"),                            # no w_skip
    (dict(Cin1=64), b"null buffer"),                                      # no x1
    (dict(x0=FAKE + 8), b"16-byte aligned"),
    (dict(bias=FAKE + 4), b"16-byte aligned"),
    (dict(scratch=FAKE + 2), b"16-byte aligned"),
    # routes the planner would not take for the shape
    (dict(route=3), b"it takes route 1"),                                 # (route 2 is accepted here: the plan without the halo)
    (dict(route=1, H=8, W=8), b"it takes route 2"),
    (dict(route=1, Cin1=64, x1=FAKE), b"it takes route 3"),              # concat input
    (dict(route=1, Co=96, Cin0=96), b"it takes route 3"),
    (dict(route=4), b"it takes route 1"),                                 # route 4 is stride 2 only
    (dict(route=1, residual=FAKE, accumulate=1), b"it takes route 3"),
    (dict(op=2, dy=FAKE, route=1), b"it takes route 2"),
    (dict(op=1, dy=FAKE, stride=2, route=3), b"it takes route 4"),
    (dict(qstats=FAKE, H=8, W=8, route=2), b"qstats needs"),             # split-K at 8x8, B = 2
    (dict(scratch=None), b"needs a scratch area"),
]


@pytest.mark.parametrize("kw,msg", REFUSALS)
def test_conv_validates_arguments(L, kw, msg):
    d = _desc(**kw)
    assert L.ddpm_conv_run(C.byref(d), None) != 0
    assert msg in L.ddpm_last_error(), L.ddpm_last_error()


def test_null_descriptor_is_refused(L):
    assert L.ddpm_conv_run(None, None) != 0 and b"null descriptor" in L.ddpm_last_error()
    assert L.ddpm_conv_scratch_bytes(None) < 0 and b"null descriptor" in L.ddpm_last_error()


def test_gemm_route_accepted_where_the_halo_is(L):
    """route 2 at a haloed shape is the plan with the haloed kernel off (DDPM_NO_HALO)"""
    rc, rep = _dry(L, _desc(route=2))
    assert rc == 0, L.ddpm_last_error()
    assert (rep.route, rep.launches, rep.block_n, rep.splits) == (2, 3, 128, 2)     # B = 2: 16 tiles, split in two


def _al(n):
    return (n + 255) // 256 * 256


def test_scratch_bytes(L):
    PE = 88                                        # sizeof(PackEntry): 6 ints, 8 pointers / long longs
    # halo forward: packed [Co][9 Cin] bf16 + a one-row table
    assert L.ddpm_conv_scratch_bytes(C.byref(_desc())) == _al(128 * 9 * 128 * 2) + _al(PE)
    # + 1x1 skip of a 256 + 128 concat and the combined bias: [Co][9 Cin + 384], bias [Co] f32, three rows
    d = _desc(H=16, W=16, Cin0=256, Co=256, Cs0=256, Cs1=128, s0=FAKE, s1=FAKE, w_skip=FAKE, bias=FAKE, skip_bias=FAKE)
    assert L.ddpm_conv_scratch_bytes(C.byref(d)) == _al(256 * (9 * 256 + 384) * 2) + _al(256 * 4) + _al(3 * PE)
    # split-K at 4x4, B = 128: zeroed fp32 [P][Co] first
    d = _desc(route=2, B=128, H=4, W=4, Cin0=256, Co=256)
    assert L.ddpm_conv_scratch_bytes(C.byref(d)) == _al(128 * 16 * 256 * 4) + _al(256 * 9 * 256 * 2) + _al(PE)
    # 3x3 weight gradient on the tensor cores: zeroed fp32 [9][Co][Cin] and the unpack row, no pack
    d = _desc(op=2, route=2, dy=FAKE, w=None)
    assert L.ddpm_conv_scratch_bytes(C.byref(d)) == _al(9 * 128 * 128 * 4) + _al(PE)
    # 1x1 weight gradient on the tensor cores: atomics straight into dW, no scratch at all
    d = _desc(op=2, route=2, ksize=1, H=16, W=16, Cin0=256, Co=768, dy=FAKE, w=None, scratch=None)
    assert L.ddpm_conv_scratch_bytes(C.byref(d)) == 0
    assert _dry(L, d)[0] == 0, L.ddpm_last_error()
    # fold: [C][16 C]
    d = _desc(route=5, upsample=1, H=8, W=8, Cin0=256, Co=256)
    assert L.ddpm_conv_scratch_bytes(C.byref(d)) == _al(256 * 16 * 256 * 2) + _al(PE)
    assert L.ddpm_conv_scratch_bytes(C.byref(_desc(route=3))) < 0 and b"it takes route 1" in L.ddpm_last_error()


def test_entry_points_declared_and_exported(L):
    from ddpm_torch_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ddpm_b200.h")).read(), flags=re.S)
    for name in ("ddpm_conv_run", "ddpm_conv_scratch_bytes"):
        assert re.search(rf"\b{name}\s*\(", hdr) and name in _lib.EXPORTS and hasattr(L, name)


def test_descriptor_layout_matches_header():
    from ddpm_torch_b200 import _lib
    import subprocess, tempfile
    src = ('#include "include/ddpm_b200.h"\n#include <stdio.h>\n#include <stddef.h>\nint main(){printf("%zu %zu %zu %zu %zu %zu", '
           'sizeof(ddpm_conv_desc), sizeof(ddpm_conv_report), offsetof(ddpm_conv_desc, x0), offsetof(ddpm_conv_desc, rowvec_ld), '
           'offsetof(ddpm_conv_desc, report), offsetof(ddpm_conv_report, zero_bytes));}')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c"); open(c, "w").write(src)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", ROOT, c, "-o", exe], cwd=ROOT)
        got = tuple(map(int, subprocess.check_output([exe]).split()))
    assert got == (C.sizeof(_lib.ConvDesc), C.sizeof(_lib.ConvReport), _lib.ConvDesc.x0.offset, _lib.ConvDesc.rowvec_ld.offset,
                   _lib.ConvDesc.report.offset, _lib.ConvReport.zero_bytes.offset)


# ------------------------------------------------------------------------------------------------ the GPU cases, dry
# (route, launches, block_n, splits) of every case of test_conv_gpu.CASES, from the planner's rules: launches count the weight pack
# (one k_pack_table launch), the conv launches (split-K: GEMM + k_splitk_finalize; CUDA cores with a skip: two; s2 data gradient
# and fold: four parity GEMMs; one weight-gradient GEMM per concat source) and the 3x3 tensor-core weight gradient's unpack
EXPECTED = [
    (1, 2, 128, 1),   # fwd-halo-00 CIFAR-10 downsamples.level_0.0.conv1 (B=1)
    (1, 2, 128, 1),   # fwd-halo-01 CIFAR-10 downsamples.level_0.0.conv1 (B=3)
    (1, 2, 128, 1),   # fwd-halo-02 CIFAR-10 downsamples.level_0.0.conv1 (B=128)
    (1, 2, 256, 1),   # fwd-halo-03 CIFAR-10 downsamples.level_1.1.conv1
    (1, 2, 128, 1),   # fwd-halo-04 CelebA 64x64 downsamples.level_0.0.conv1
    (1, 2, 128, 1),   # fwd-halo-05 CelebA-HQ downsamples.level_0.0.conv1
    (1, 2, 128, 1),   # fwd-halo-06 non-square 16x8 map
    (1, 2, 256, 1),   # fwd-halo-07 CIFAR-10 downsamples.level_1.0.conv2 + skip
    (1, 2, 256, 1),   # fwd-halo-08 CIFAR-10 upsamples.level_1.2.conv2 + skip of the 256+128 concat
    (1, 2, 128, 1),   # fwd-halo-09 CIFAR-10 downsamples.level_0.1.conv2 + identity skip
    (1, 2, 128, 1),   # fwd-halo-10 3x3 conv + residual
    (1, 2, 256, 1),   # fwd-halo-11 3x3 conv accumulating into out
    (1, 2, 128, 1),   # dgrad-halo-12 CIFAR-10 upsamples.level_1.2.conv1.dgrad (into 384)
    (1, 2, 256, 1),   # dgrad-halo-13 CIFAR-10 upsamples.level_1.0.conv1.dgrad (into 512)
    (2, 3, 128, 4),   # fwd-gemm-14 CIFAR-10 downsamples.level_2.0.conv1 (B=3, split-K)
    (2, 3, 128, 4),   # fwd-gemm-15 CIFAR-10 downsamples.level_3.0.conv1 (B=3, split-K)
    (2, 2, 128, 1),   # fwd-gemm-16 CIFAR-10 downsamples.level_2.0.conv1 (B=128, N=128 fill)
    (2, 3, 128, 4),   # fwd-gemm-17 CIFAR-10 middle.0.conv1 (B=128, split-K)
    (2, 3, 128, 4),   # fwd-gemm-18 split-K + bias, row vector and residual
    (2, 3, 128, 4),   # fwd-gemm-19 split-K in place (accumulate)
    (2, 3, 128, 5),   # fwd-gemm-20 CIFAR-10 upsamples.level_2.0.conv2 + skip of the 256+256 concat
    (2, 2, 128, 1),   # fwd-gemm-21 CIFAR-10 downsamples.level_1.0.1.project_in
    (2, 2, 128, 1),   # fwd-gemm-22 small64 attention project_in (128 -> 384)
    (2, 2, 128, 1),   # fwd-gemm-23 CIFAR-10 downsamples.level_1.0.1.project_out + residual
    (2, 3, 128, 2),   # fwd-gemm-24 CIFAR-10 downsamples.level_0.0.conv1 on the GEMM engine (B=3, split-K)
    (2, 3, 128, 4),   # dgrad-gemm-25 CIFAR-10 downsamples.level_2.0.conv1.dgrad
    (2, 3, 128, 4),   # dgrad-gemm-26 CIFAR-10 downsamples.level_3.0.conv1.dgrad
    (2, 2, 128, 1),   # dgrad-gemm-27 CIFAR-10 upsamples.level_2.0.skip.dgrad (into 512)
    (2, 2, 128, 14),   # wgrad-gemm-28 CIFAR-10 downsamples.level_0.0.conv1.wgrad (B=128, bench shape)
    (2, 2, 256, 1),   # wgrad-gemm-29 CIFAR-10 downsamples.level_3.0.conv1.wgrad
    (2, 1, 256, 3),   # wgrad-gemm-30 CIFAR-10 downsamples.level_1.0.1.project_in.wgrad (1x1 into the flat gradient)
    (2, 2, 256, 3),   # wgrad-gemm-31 CIFAR-10 upsamples.level_1.2.skip.wgrad (256+128 concat)
    (3, 2, 64, 1),   # fwd-simt-32 tiny (hid 32) downsamples.level_0.0.conv1
    (3, 2, 64, 1),   # fwd-simt-33 hid-96 downsamples.level_0.0.conv1
    (3, 3, 64, 1),   # fwd-simt-34 tiny upsamples.level_0.1.conv2 + skip of the 32+32 concat
    (3, 2, 64, 1),   # fwd-simt-35 tiny upsamples.level_0.0.conv1 (concat input 64+32)
    (3, 2, 64, 1),   # fwd-simt-36 tiny downsamples.level_0.1.1 (stride 2)
    (3, 2, 64, 1),   # dgrad-simt-37 tiny downsamples.level_0.1.1.dgrad (MAP_TRANSPOSED2)
    (3, 2, 64, 1),   # dgrad-simt-38 tiny downsamples.level_0.1.1.dgrad accumulating
    (3, 2, 64, 1),   # dgrad-simt-39 tiny downsamples.level_0.0.conv1.dgrad
    (3, 1, 64, 1),   # wgrad-simt-40 tiny downsamples.level_0.0.conv1.wgrad
    (3, 1, 64, 1),   # wgrad-simt-41 tiny upsamples.level_0.0.conv1.wgrad (concat 64+32)
    (3, 1, 64, 1),   # wgrad-simt-42 tiny downsamples.level_0.1.1.wgrad (stride 2)
    (4, 3, 128, 2),   # fwd-s2-43 CIFAR-10 downsamples.level_0.2.1 (32 -> 16, B=3, split-K)
    (4, 2, 128, 1),   # fwd-s2-44 CIFAR-10 downsamples.level_0.2.1 (32 -> 16, B=128)
    (4, 3, 128, 4),   # fwd-s2-45 CIFAR-10 downsamples.level_1.2.1 (16 -> 8)
    (4, 3, 128, 4),   # fwd-s2-46 CIFAR-10 downsamples.level_2.2.1 (8 -> 4)
    (4, 3, 128, 4),   # fwd-s2-47 CIFAR-10 downsamples.level_2.2.1 (8 -> 4, B=128, split-K)
    (4, 5, 128, 1),   # dgrad-s2-48 CIFAR-10 downsamples.level_0.2.1.dgrad
    (4, 5, 128, 1),   # dgrad-s2-49 CIFAR-10 downsamples.level_0.2.1.dgrad accumulating
    (4, 5, 256, 1),   # dgrad-s2-50 CIFAR-10 downsamples.level_1.2.1.dgrad accumulating
    (4, 2, 128, 3),   # wgrad-s2-51 CIFAR-10 downsamples.level_0.2.1.wgrad (b_estride)
    (4, 2, 256, 1),   # wgrad-s2-52 CIFAR-10 downsamples.level_1.2.1.wgrad (b_estride)
    (5, 5, 256, 1),   # fwd-fold-53 CIFAR-10 upsamples.level_3.3.1 (4 -> 8)
    (5, 5, 256, 1),   # fwd-fold-54 CIFAR-10 upsamples.level_2.3.1 (8 -> 16)
    (5, 5, 256, 1),   # fwd-fold-55 CelebA-HQ upsamples.level_5.3.1 (512 channels, 8 -> 16)
]


def _case_desc(c):
    d = G.desc_for(c, {}, None, None, None, dry=1)
    for key in ("x0", "w", "out"):
        setattr(d, key, FAKE)
    if c["op"] == 2:
        d.w = None
    if c["Cin1"]:
        d.x1 = FAKE
    if c["op"] != 0:
        d.x0 = FAKE if c["op"] == 2 else None
        d.dy = FAKE
    if c["Cs0"]:
        d.s0 = FAKE
        if c["Cs1"]:
            d.s1 = FAKE
        if not c["ident"]:
            d.w_skip = FAKE
    if c["bias"]:
        d.bias = FAKE
    if c["skip_bias"]:
        d.skip_bias = FAKE
    if c["rowvec"]:
        d.rowvec, d.rowvec_ld = FAKE, c["Co"] + 64
    if c["residual"]:
        d.residual = FAKE
    if c["qstats"]:
        d.qstats = FAKE
    return d


@pytest.mark.parametrize("i", range(len(G.CASES)), ids=G.IDS)
def test_case_dry_report(L, i):
    assert len(EXPECTED) == len(G.CASES)
    c = G.CASES[i]
    rc, rep = _dry(L, _case_desc(c))
    assert rc == 0, L.ddpm_last_error()
    assert (rep.route, rep.launches, rep.block_n, rep.splits) == EXPECTED[i], c["label"]


# ------------------------------------------------------------------------------------------------ dry plans
CELEBA64_CFG = dict(in_channels=3, hid_channels=128, out_channels=3, ch_multipliers=(1, 2, 2, 2), num_res_blocks=2,
                    apply_attn=(False, False, True, False), drop_rate=0.0)
ATT4_C128_CFG = dict(in_channels=3, hid_channels=64, out_channels=3, ch_multipliers=(1, 2), num_res_blocks=1,
                     apply_attn=(False, True), drop_rate=0.0)
ATT4_C512_CFG = dict(in_channels=3, hid_channels=128, out_channels=3, ch_multipliers=(1, 4), num_res_blocks=1,
                     apply_attn=(False, True), drop_rate=0.0)
CFGS = {"tiny": (R.TINY_CFG, 2, 16), "small64": (R.SMALL64_CFG, 4, 32), "cifar10": (R.CIFAR10_CFG, 128, 32),
        "celeba64": (CELEBA64_CFG, 8, 64), "celebahq": (R.CELEBAHQ_CFG, 4, 256), "att4_c128": (ATT4_C128_CFG, 4, 8),
        "att4_c512": (ATT4_C512_CFG, 4, 8)}
# (cfg, resample_with_conv, training) -> (workspace bytes, launches fwd / bwd / repack, ops fwd / bwd, tensor-core / CUDA-core ops,
# fwd / bwd FLOPs), as planned by the parent commit of the shared conv builders.  Inference plans carry the fold (resample_with_conv
# = 1, C % 256 == 0 levels); CIFAR-10 bs = 128 training is 146 / 378 / 5 launches
PLANS = {
    ('att4_c128', 0, 0): (6775816, 70, 0, 3, 60, 0, 26, 4, 436142080.0, 0.0),
    ('att4_c128', 0, 1): (21467392, 70, 154, 4, 60, 120, 91, 8, 436142080.0, 874283008.0),
    ('att4_c128', 1, 0): (7339192, 72, 0, 3, 61, 0, 28, 4, 516358144.0, 0.0),
    ('att4_c128', 1, 1): (23334144, 72, 163, 4, 61, 128, 100, 8, 516358144.0, 1034715136.0),
    ('att4_c512', 0, 0): (70697992, 75, 0, 3, 60, 0, 26, 4, 4741005312.0, 0.0),
    ('att4_c512', 0, 1): (248777984, 75, 166, 4, 60, 123, 91, 8, 4741005312.0, 9483386880.0),
    ('att4_c512', 1, 0): (79406264, 79, 0, 3, 63, 0, 31, 4, 5967839232.0, 0.0),
    ('att4_c512', 1, 1): (270430464, 78, 175, 4, 61, 131, 100, 8, 5967839232.0, 11937054720.0),
    ('celeba64', 0, 0): (480872000, 143, 0, 3, 130, 0, 63, 2, 317756276736.0, 0.0),
    ('celeba64', 0, 1): (1176788736, 143, 359, 4, 130, 292, 236, 6, 317756276736.0, 636349317120.0),
    ('celeba64', 1, 0): (492423760, 156, 0, 3, 141, 0, 78, 2, 373926395904.0, 0.0),
    ('celeba64', 1, 1): (1248210176, 150, 383, 4, 135, 316, 263, 6, 373926395904.0, 748689555456.0),
    ('celebahq', 0, 0): (2809913080, 197, 0, 3, 184, 0, 88, 2, 1758597742592.0, 0.0),
    ('celebahq', 0, 1): (6531414784, 197, 482, 4, 184, 389, 321, 6, 1758597742592.0, 3523968237568.0),
    ('celebahq', 1, 0): (2907518056, 214, 0, 3, 199, 0, 110, 2, 1988110057472.0, 0.0),
    ('celebahq', 1, 1): (6840605952, 206, 522, 4, 191, 429, 366, 6, 1988110057472.0, 3982992867328.0),
    ('cifar10', 0, 0): (2158754192, 142, 0, 4, 129, 0, 64, 1, 1368114855936.0, 0.0),
    ('cifar10', 0, 1): (5116102144, 142, 354, 5, 129, 289, 239, 2, 1368114855936.0, 2739450937344.0),
    ('cifar10', 1, 0): (2169666464, 152, 0, 4, 138, 0, 79, 1, 1592795332608.0, 0.0),
    ('cifar10', 1, 1): (5319134720, 146, 378, 5, 132, 313, 266, 2, 1592795332608.0, 3188811890688.0),
    ('small64', 0, 0): (34391312, 75, 0, 3, 76, 0, 34, 0, 7446200320.0, 0.0),
    ('small64', 0, 1): (79458560, 75, 160, 4, 76, 136, 115, 0, 7446200320.0, 14944043008.0),
    ('small64', 1, 0): (35808704, 76, 0, 3, 77, 0, 36, 0, 8729657344.0, 0.0),
    ('small64', 1, 1): (83031296, 76, 168, 4, 77, 144, 124, 0, 8729657344.0, 17510957056.0),
    ('tiny', 0, 0): (2879240, 77, 0, 1, 77, 0, 14, 18, 225411072.0, 0.0),
    ('tiny', 0, 1): (7253056, 77, 153, 1, 77, 128, 49, 58, 225411072.0, 449773568.0),
    ('tiny', 1, 0): (3036344, 78, 0, 1, 78, 0, 15, 19, 265519104.0, 0.0),
    ('tiny', 1, 1): (7716160, 78, 158, 1, 78, 133, 52, 61, 265519104.0, 537067520.0),
}


def _plan(L, cfg, B, HW, rwc, training):
    from ddpm_torch_b200 import _lib
    c = R.normalize_cfg(cfg)
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = c["in_channels"], c["hid_channels"], c["out_channels"]
    u.levels, u.num_res_blocks, u.temb_dim, u.drop_rate = len(c["ch_multipliers"]), c["num_res_blocks"], 0, c["drop_rate"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    h = C.c_void_p()
    assert L.ddpm_unet_create_ex(C.byref(u), rwc, C.byref(h)) == 0, L.ddpm_last_error()
    try:
        ws = L.ddpm_unet_workspace_bytes(h, B, HW, HW, training)
        assert ws > 0, L.ddpm_last_error()
        f, b, p = C.c_int(), C.c_int(), C.c_int()
        L.ddpm_unet_launch_counts(h, C.byref(f), C.byref(b), C.byref(p))
        nf, nb, ntc, ng = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        ff, bf = C.c_double(), C.c_double()
        L.ddpm_unet_plan_stats(h, C.byref(nf), C.byref(nb), C.byref(ntc), C.byref(ng), C.byref(ff), C.byref(bf))
        return (ws, f.value, b.value, p.value, nf.value, nb.value, ntc.value, ng.value, ff.value, bf.value)
    finally:
        L.ddpm_unet_destroy(h)


@pytest.mark.parametrize("key", sorted(PLANS), ids=lambda k: f"{k[0]}-rwc{k[1]}-{'train' if k[2] else 'infer'}")
def test_dry_plans_unchanged(L, key):
    name, rwc, training = key
    cfg, B, HW = CFGS[name]
    assert _plan(L, cfg, B, HW, rwc, training) == PLANS[key]
