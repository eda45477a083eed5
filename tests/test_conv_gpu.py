"""Every convolution route the UNet engine's planner takes, forward, data gradient and weight gradient, against fp64 torch, through
the C ABI operator ddpm_conv_run (csrc/ddpm_b200.cu), which runs the launch steps the plans run (the same builders in
unet_engine.cuh: same kernels, descriptors, block_n and split counts) over weights packed from fp32 OIHW masters by the plans' own
k_pack_table rows:
  1 halo   conv_halo.cuh                                          2 gemm  GEMM_KK / split-K + k_splitk_finalize / GEMM_MNMN
  3 simt   k_conv_generic (+ skip launch, MAP_TRANSPOSED2), k_wgrad_generic
  4 s2     stride-2 forward, four output-parity data-gradient GEMMs, b_estride weight gradient
  5 fold   nearest-2x upsample folded into the 3x3 conv (PK_UPFOLD, four parity GEMMs)
Every case of CASES names the layer of a reference config it stands for, and runs in two modes.

Exact mode.  Activations and dy are in {-1, 0, 1}, weights in {-1, 0, 1} with about 24 non-zeros per output over the reduction,
bias, skip bias, row vector, residual and a prior dx are integers in [-8, 8].  The test asserts sum |terms| < 2^21 per output, so
every product and partial sum is an integer that fp32 holds exactly, whatever the summation order, split count or atomics; the
outputs are then below 2^8 in magnitude, so bf16 holds them exactly too, and so do the fp32 sums of their squares over a warp
(the quad statistics).  Each route must therefore reproduce the fp64 reference BIT FOR BIT: bf16 outputs equal ref, fp32 weight
gradients equal ref, quad statistics equal the fp64 sums.  The fold's merged weights are sums of at most four integers: exact too.

Random mode.  Activations and dy are N(0.5, 1) (a non-zero mean, so that the zero padding matters), fp32 master weights N(0, 1)
scaled by 1e3 or 1e-3 (not bf16-representable: the pack rounds them), bias / row vector / residual N(0, 1) on the output's scale.
The reference is F.conv2d in fp64 on the bf16 operands and the bf16-rounded weights; S is the same expression over absolute values
(sum over all terms of |a| |w|, plus |bias| + |rowvec| + |residual| + |prior|).  Bounds, element-wise (u = 2^-8, one bf16 rounding;
an fp32 addition on the tensor cores is not guaranteed to round to nearest, so 2^-23 per addition):
  bf16 outputs     |out - ref| <= u |ref| + (1 + u) n 2^-23 S,   n = the terms summed: taps x Cin + skip channels (the K slabs,
                   whatever their split into partials) + 4 epilogue adds (bias, skip bias, row vector, residual / prior)
  fold             the packed weight of each 2x2 tap is bf16(sum of up to four fp32 masters), against the reference's sum of the
                   bf16-rounded masters: at most 2u of the sum of their magnitudes, so + (1 + u) 2u S
  CUDA-core skip   the second launch adds the skip to the bf16-ROUNDED output of the first: + (1 + u) u S
  weight gradient  |dW - ref| <= n 2^-23 S with n = B x Ho x Wo pixel terms + 2 (fp32 output, no rounding to bf16)
The quad statistics are checked in exact mode only.  Each check prints its worst error / bound; teardown prints the worst per route.

Invariants, on every case: outputs prefilled with NaN are fully written (an accumulating weight gradient starts from zeros, a data
gradient with accumulate from a prior dx); guard bands before and after each output (64 elements) and the scratch (256 bytes) are untouched; the
scratch's zero area is all zero after the call (k_splitk_finalize and PK_UNPACK_GRAD clear behind their reads); a second call on
the same scratch gives the identical result (exact mode).  test_routes_agree runs shapes that several routes take and checks them
against each other within the sum of their bounds: halo vs GEMM vs CUDA cores, and fold vs nearest-2x + conv."""
import ctypes as ct
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -8
F23 = 2.0 ** -23
G = 64                      # guard elements (a multiple of 16 bytes for bf16 and fp32)
GB = 256                    # guard bytes around the scratch
SENT_BF16 = -12345.0        # guard sentinel (bf16- and fp32-exact)
HALO, GEMM, SIMT, S2, FOLD = 1, 2, 3, 4, 5
ROUTE_NAME = {HALO: "halo", GEMM: "gemm", SIMT: "simt", S2: "s2", FOLD: "fold"}
OP_NAME = {0: "fwd", 1: "dgrad", 2: "wgrad"}
WORST = {}
T0 = time.time()


def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _p(t):
    return t.data_ptr() if t is not None else None


# ------------------------------------------------------------------------------------------------ cases
def case(label, op, route, B, H, W, Cin0, Co, k=3, stride=1, up=0, Cin1=0, Cs0=0, Cs1=0, ident=0, bias=None, rowvec=False,
         residual=False, acc=False, qstats=False):
    """one conv of a reference config: op 0 fwd / 1 dgrad / 2 wgrad on `route`; bias defaults to the forward having one"""
    return dict(label=label, op=op, route=route, B=B, H=H, W=W, Cin0=Cin0, Cin1=Cin1, Co=Co, k=k, stride=stride, up=up, Cs0=Cs0,
                Cs1=Cs1, ident=ident, bias=(op == 0) if bias is None else bias, skip_bias=Cs0 > 0 and not ident, rowvec=rowvec,
                residual=residual, acc=acc, qstats=qstats)


CASES = [
    # ---- haloed 3x3 (CIFAR-10: hid 128, ch_mult (1, 2, 2, 2), attention at 16x16)
    case("CIFAR-10 downsamples.level_0.0.conv1 (B=1)", 0, HALO, 1, 32, 32, 128, 128, rowvec=True, qstats=True),
    case("CIFAR-10 downsamples.level_0.0.conv1 (B=3)", 0, HALO, 3, 32, 32, 128, 128, rowvec=True, qstats=True),
    case("CIFAR-10 downsamples.level_0.0.conv1 (B=128)", 0, HALO, 128, 32, 32, 128, 128, rowvec=True, qstats=True),
    case("CIFAR-10 downsamples.level_1.1.conv1", 0, HALO, 3, 16, 16, 256, 256, rowvec=True, qstats=True),
    case("CelebA 64x64 downsamples.level_0.0.conv1", 0, HALO, 1, 64, 64, 128, 128, rowvec=True, qstats=True),
    case("CelebA-HQ downsamples.level_0.0.conv1", 0, HALO, 1, 256, 256, 128, 128, rowvec=True),
    case("non-square 16x8 map", 0, HALO, 3, 16, 8, 128, 128, rowvec=True, qstats=True),
    case("CIFAR-10 downsamples.level_1.0.conv2 + skip", 0, HALO, 3, 16, 16, 256, 256, Cs0=128, qstats=True),
    case("CIFAR-10 upsamples.level_1.2.conv2 + skip of the 256+128 concat", 0, HALO, 3, 16, 16, 256, 256, Cs0=256, Cs1=128, qstats=True),
    case("CIFAR-10 downsamples.level_0.1.conv2 + identity skip", 0, HALO, 3, 32, 32, 128, 128, Cs0=128, ident=1, qstats=True),
    case("3x3 conv + residual", 0, HALO, 3, 32, 32, 128, 128, residual=True),
    case("3x3 conv accumulating into out", 0, HALO, 3, 16, 16, 256, 256, acc=True),
    case("CIFAR-10 upsamples.level_1.2.conv1.dgrad (into 384)", 1, HALO, 3, 16, 16, 384, 256),
    case("CIFAR-10 upsamples.level_1.0.conv1.dgrad (into 512)", 1, HALO, 3, 16, 16, 512, 256),
    # ---- tensor-core GEMM
    case("CIFAR-10 downsamples.level_2.0.conv1 (B=3, split-K)", 0, GEMM, 3, 8, 8, 256, 256, rowvec=True),
    case("CIFAR-10 downsamples.level_3.0.conv1 (B=3, split-K)", 0, GEMM, 3, 4, 4, 256, 256, rowvec=True),
    case("CIFAR-10 downsamples.level_2.0.conv1 (B=128, N=128 fill)", 0, GEMM, 128, 8, 8, 256, 256, rowvec=True, qstats=True),
    case("CIFAR-10 middle.0.conv1 (B=128, split-K)", 0, GEMM, 128, 4, 4, 256, 256, rowvec=True),
    case("split-K + bias, row vector and residual", 0, GEMM, 128, 4, 4, 256, 256, rowvec=True, residual=True),
    case("split-K in place (accumulate)", 0, GEMM, 128, 4, 4, 256, 256, acc=True),
    case("CIFAR-10 upsamples.level_2.0.conv2 + skip of the 256+256 concat", 0, GEMM, 3, 8, 8, 256, 256, Cs0=256, Cs1=256),
    case("CIFAR-10 downsamples.level_1.0.1.project_in", 0, GEMM, 3, 16, 16, 256, 768, k=1),
    case("small64 attention project_in (128 -> 384)", 0, GEMM, 3, 16, 16, 128, 384, k=1),
    case("CIFAR-10 downsamples.level_1.0.1.project_out + residual", 0, GEMM, 3, 16, 16, 256, 256, k=1, residual=True, qstats=True),
    case("CIFAR-10 downsamples.level_0.0.conv1 on the GEMM engine (B=3, split-K)", 0, GEMM, 3, 32, 32, 128, 128, rowvec=True),
    case("CIFAR-10 downsamples.level_2.0.conv1.dgrad", 1, GEMM, 3, 8, 8, 256, 256),
    case("CIFAR-10 downsamples.level_3.0.conv1.dgrad", 1, GEMM, 3, 4, 4, 256, 256),
    case("CIFAR-10 upsamples.level_2.0.skip.dgrad (into 512)", 1, GEMM, 3, 8, 8, 512, 256, k=1),
    case("CIFAR-10 downsamples.level_0.0.conv1.wgrad (B=128, bench shape)", 2, GEMM, 128, 32, 32, 128, 128),
    case("CIFAR-10 downsamples.level_3.0.conv1.wgrad", 2, GEMM, 3, 4, 4, 256, 256),
    case("CIFAR-10 downsamples.level_1.0.1.project_in.wgrad (1x1 into the flat gradient)", 2, GEMM, 3, 16, 16, 256, 768, k=1),
    case("CIFAR-10 upsamples.level_1.2.skip.wgrad (256+128 concat)", 2, GEMM, 3, 16, 16, 256, 256, k=1, Cin1=128),
    # ---- CUDA cores
    case("tiny (hid 32) downsamples.level_0.0.conv1", 0, SIMT, 2, 16, 16, 32, 32, rowvec=True),
    case("hid-96 downsamples.level_0.0.conv1", 0, SIMT, 2, 16, 16, 96, 96, rowvec=True),
    case("tiny upsamples.level_0.1.conv2 + skip of the 32+32 concat", 0, SIMT, 2, 16, 16, 32, 32, Cs0=32, Cs1=32),
    case("tiny upsamples.level_0.0.conv1 (concat input 64+32)", 0, SIMT, 2, 16, 16, 64, 32, Cin1=32, rowvec=True),
    case("tiny downsamples.level_0.1.1 (stride 2)", 0, SIMT, 2, 16, 16, 32, 32, stride=2),
    case("tiny downsamples.level_0.1.1.dgrad (MAP_TRANSPOSED2)", 1, SIMT, 2, 16, 16, 32, 32, stride=2),
    case("tiny downsamples.level_0.1.1.dgrad accumulating", 1, SIMT, 2, 16, 16, 32, 32, stride=2, acc=True),
    case("tiny downsamples.level_0.0.conv1.dgrad", 1, SIMT, 2, 16, 16, 32, 32),
    case("tiny downsamples.level_0.0.conv1.wgrad", 2, SIMT, 2, 16, 16, 32, 32),
    case("tiny upsamples.level_0.0.conv1.wgrad (concat 64+32)", 2, SIMT, 2, 16, 16, 64, 32, Cin1=32),
    case("tiny downsamples.level_0.1.1.wgrad (stride 2)", 2, SIMT, 2, 16, 16, 32, 32, stride=2),
    # ---- stride 2 on the tensor cores
    case("CIFAR-10 downsamples.level_0.2.1 (32 -> 16, B=3, split-K)", 0, S2, 3, 32, 32, 128, 128, stride=2),
    case("CIFAR-10 downsamples.level_0.2.1 (32 -> 16, B=128)", 0, S2, 128, 32, 32, 128, 128, qstats=True, stride=2),
    case("CIFAR-10 downsamples.level_1.2.1 (16 -> 8)", 0, S2, 3, 16, 16, 256, 256, stride=2),
    case("CIFAR-10 downsamples.level_2.2.1 (8 -> 4)", 0, S2, 3, 8, 8, 256, 256, stride=2),
    case("CIFAR-10 downsamples.level_2.2.1 (8 -> 4, B=128, split-K)", 0, S2, 128, 8, 8, 256, 256, stride=2),
    case("CIFAR-10 downsamples.level_0.2.1.dgrad", 1, S2, 3, 32, 32, 128, 128, stride=2),
    case("CIFAR-10 downsamples.level_0.2.1.dgrad accumulating", 1, S2, 3, 32, 32, 128, 128, acc=True, stride=2),
    case("CIFAR-10 downsamples.level_1.2.1.dgrad accumulating", 1, S2, 3, 16, 16, 256, 256, acc=True, stride=2),
    case("CIFAR-10 downsamples.level_0.2.1.wgrad (b_estride)", 2, S2, 3, 32, 32, 128, 128, stride=2),
    case("CIFAR-10 downsamples.level_1.2.1.wgrad (b_estride)", 2, S2, 3, 16, 16, 256, 256, stride=2),
    # ---- folded nearest-2x upsample + conv (inference plans)
    case("CIFAR-10 upsamples.level_3.3.1 (4 -> 8)", 0, FOLD, 3, 4, 4, 256, 256, up=1),
    case("CIFAR-10 upsamples.level_2.3.1 (8 -> 16)", 0, FOLD, 3, 8, 8, 256, 256, up=1, qstats=True),
    case("CelebA-HQ upsamples.level_5.3.1 (512 channels, 8 -> 16)", 0, FOLD, 2, 8, 8, 512, 512, up=1),
]
IDS = [f"{OP_NAME[c['op']]}-{ROUTE_NAME[c['route']]}-{i:02d}" for i, c in enumerate(CASES)]


def out_hw(c):
    if c["up"]:
        return 2 * c["H"], 2 * c["W"]
    return c["H"] // c["stride"], c["W"] // c["stride"]


# ------------------------------------------------------------------------------------------------ inputs
def _act(shape, mode, g):
    if mode == "exact":
        return torch.randint(-1, 2, shape, device=DEV, generator=g).to(torch.bfloat16)
    return (torch.randn(shape, device=DEV, generator=g) + 0.5).to(torch.bfloat16)


def _wt(shape, fan, mode, scale, g):
    if mode == "exact":
        w = torch.randint(-1, 2, shape, device=DEV, generator=g).float()
        keep = torch.rand(shape, device=DEV, generator=g) < min(1.0, 24.0 / fan)
        return (w * keep).contiguous()
    return (torch.randn(shape, device=DEV, generator=g) * scale / fan ** 0.5).contiguous()


def _small(shape, mode, scale, g, dtype=torch.float32):
    if mode == "exact":
        return torch.randint(-8, 9, shape, device=DEV, generator=g).to(dtype)
    return (torch.randn(shape, device=DEV, generator=g) * scale).to(dtype)


def make_inputs(c, mode, seed, wscale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    B, H, W, k, Co = c["B"], c["H"], c["W"], c["k"], c["Co"]
    Ho, Wo = out_hw(c)
    Cin = c["Cin0"] + c["Cin1"]
    t = {}
    fan = k * k * Cin + c["Cs0"] + c["Cs1"]
    t["w"] = _wt((Co, Cin, k, k), fan if c["op"] != 1 else k * k * Co, mode, wscale, g)
    osc = wscale * 0.5                      # the output's typical magnitude in random mode
    if c["op"] in (0, 2):
        t["x0"] = _act((B, H, W, c["Cin0"]), mode, g)
        t["x1"] = _act((B, H, W, c["Cin1"]), mode, g) if c["Cin1"] else None
    if c["op"] in (1, 2):
        t["dy"] = _act((B, Ho, Wo, Co), mode, g)
    if c["Cs0"]:
        t["s0"] = _act((B, H, W, c["Cs0"]), mode, g)
        t["s1"] = _act((B, H, W, c["Cs1"]), mode, g) if c["Cs1"] else None
        if not c["ident"]:
            t["w_skip"] = _wt((Co, c["Cs0"] + c["Cs1"]), fan, mode, wscale, g)
    if c["bias"]:
        t["bias"] = _small((Co,), mode, osc, g)
    if c["skip_bias"]:
        t["skip_bias"] = _small((Co,), mode, osc, g)
    if c["rowvec"]:
        t["rowvec"] = _small((B, Co + 64), mode, osc, g)       # rowvec_ld > Co, as the plans' concatenated projections
    if c["residual"]:
        t["residual"] = _small((B, Ho, Wo, Co), mode, osc, g, torch.bfloat16)
    if c["acc"]:
        shp = (B, Ho, Wo, Co) if c["op"] == 0 else (B, H, W, c["Cin0"])
        t["prior"] = _small(shp, mode, osc if c["op"] == 0 else 1.0, g, torch.bfloat16)
    return t


# ------------------------------------------------------------------------------------------------ reference
def _nchw(x):
    return x.permute(0, 3, 1, 2).double()


def _conv(c, x, w):
    if c["up"]:
        x = x.repeat_interleave(2, 2).repeat_interleave(2, 3)
    if c["stride"] == 2:
        return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2)                  # SamePad2d(3, 2): bottom / right only
    return F.conv2d(x, w, padding=c["k"] // 2)


def reference(c, t, absolute=False):
    """fp64 result in the output's layout (NHWC; OIHW for wgrad); absolute=True: the same expression over |terms| (S)"""
    a = (lambda v: v.abs()) if absolute else (lambda v: v)
    w = a(t["w"].bfloat16().double())
    Co = c["Co"]
    if c["op"] == 0:
        x = _nchw(torch.cat([t["x0"]] + ([t["x1"]] if t.get("x1") is not None else []), -1))
        y = _conv(c, a(x), w)
        if c["Cs0"]:
            s = a(_nchw(torch.cat([t["s0"]] + ([t["s1"]] if t.get("s1") is not None else []), -1)))
            y = y + (s if c["ident"] else F.conv2d(s, a(t["w_skip"].bfloat16().double())[:, :, None, None]))
        y = y.permute(0, 2, 3, 1)
        for key in ("bias", "skip_bias"):
            if key in t:
                y = y + a(t[key].double())
        if "rowvec" in t:
            y = y + a(t["rowvec"][:, :Co].double())[:, None, None, :]
        if "residual" in t:
            y = y + a(t["residual"].double())
        if "prior" in t:
            y = y + a(t["prior"].double())
        return y.contiguous()
    dy = a(_nchw(t["dy"]))
    if c["op"] == 1:
        x = torch.zeros(c["B"], c["Cin0"], c["H"], c["W"], dtype=torch.float64, device=DEV, requires_grad=True)
        _conv(c, x, w).backward(dy)
        dx = x.grad.permute(0, 2, 3, 1)
        if "prior" in t:
            dx = dx + a(t["prior"].double())
        return dx.contiguous()
    x = a(_nchw(torch.cat([t["x0"]] + ([t["x1"]] if t.get("x1") is not None else []), -1)))
    ww = torch.zeros_like(w, requires_grad=True)
    _conv(c, x, ww).backward(dy)
    return ww.grad.contiguous()


def n_terms(c):
    Ho, Wo = out_hw(c)
    taps = c["k"] * c["k"]
    if c["op"] == 0:
        return (4 if c["up"] else taps) * (c["Cin0"] + c["Cin1"]) + c["Cs0"] + c["Cs1"] + 4
    if c["op"] == 1:
        return taps * c["Co"] + 4
    return c["B"] * Ho * Wo + 2


def bound(c, ref, S):
    acc = n_terms(c) * F23 * S
    if c["op"] == 2:
        return acc
    if c["up"]:
        acc = acc + 2 * U * S
    if c["route"] == SIMT and c["Cs0"]:
        acc = acc + U * S
    return U * ref.abs() + (1 + U) * acc


# ------------------------------------------------------------------------------------------------ operator
def _guarded(shape, dtype, fill):
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * G,), SENT_BF16, dtype=dtype, device=DEV)
    buf[G:G + n] = fill
    return buf, buf[G:G + n].view(shape)


def desc_for(c, t, out, scratch, qstats, dry=0, report=None):
    from ddpm_torch_b200 import _lib
    d = _lib.ConvDesc()
    d.op, d.route, d.B, d.H, d.W, d.ksize, d.stride, d.upsample = c["op"], c["route"], c["B"], c["H"], c["W"], c["k"], c["stride"], c["up"]
    d.Cin0, d.Cin1, d.Co, d.Cs0, d.Cs1, d.identity_skip = c["Cin0"], c["Cin1"], c["Co"], c["Cs0"], c["Cs1"], c["ident"]
    for key in ("x0", "x1", "s0", "s1", "dy", "w", "w_skip", "bias", "skip_bias", "rowvec", "residual"):
        setattr(d, key, _p(t.get(key)))
    d.rowvec_ld = t["rowvec"].shape[1] if "rowvec" in t else 0
    d.accumulate = 1 if c["acc"] else 0
    d.out, d.qstats, d.scratch, d.dry = _p(out), _p(qstats), _p(scratch), dry
    if report is not None:
        d.report = ct.pointer(report)
    return d


def run(c, t):
    """one call with every invariant checked; returns (out, qstats)"""
    from ddpm_torch_b200 import _lib
    Ho, Wo = out_hw(c)
    if c["op"] == 2:
        shape, dtype = (c["Co"], c["Cin0"] + c["Cin1"], c["k"], c["k"]), torch.float32
    elif c["op"] == 1:
        shape, dtype = (c["B"], c["H"], c["W"], c["Cin0"]), torch.bfloat16
    else:
        shape, dtype = (c["B"], Ho, Wo, c["Co"]), torch.bfloat16
    rep = _lib.ConvReport()
    probe = desc_for(c, t, None, None, None, dry=1, report=rep)
    probe.out = 1 << 20                                    # any aligned address: a dry call does no device work
    _lib.check(L().ddpm_conv_run(ct.byref(probe), None), "conv dry")
    nbytes = L().ddpm_conv_scratch_bytes(ct.byref(probe))
    assert nbytes >= rep.zero_bytes >= 0, L().ddpm_last_error()
    # the tensor-core 1x1 and the CUDA-core weight gradients add into dW: they start from zeros (NaN everywhere else)
    accumulating_wgrad = c["op"] == 2 and (c["k"] == 1 or c["route"] == SIMT)
    fill = 0.0 if accumulating_wgrad else float("nan")
    buf, out = _guarded(shape, dtype, fill)
    if "prior" in t:
        out.copy_(t["prior"])
    sbuf = torch.full((nbytes + 2 * GB,), 0xA5, dtype=torch.uint8, device=DEV)
    sbuf[GB:GB + rep.zero_bytes] = 0
    scratch = sbuf[GB:GB + nbytes]
    qs = torch.zeros(c["B"], c["Co"] // 4, 2, dtype=torch.float64, device=DEV) if c["qstats"] else None
    d = desc_for(c, t, out, scratch if nbytes else None, qs)
    _lib.check(L().ddpm_conv_run(ct.byref(d), _lib.stream_ptr()), "conv")
    torch.cuda.synchronize()
    assert L().ddpm_device_error_flag() == 0
    assert not torch.isnan(out.float()).any(), "output elements left unwritten"
    assert (buf[:G] == SENT_BF16).all() and (buf[G + out.numel():] == SENT_BF16).all(), "output guard band written"
    assert (sbuf[:GB] == 0xA5).all() and (sbuf[GB + nbytes:] == 0xA5).all(), "scratch guard band written"
    assert (sbuf[GB:GB + rep.zero_bytes] == 0).all(), "scratch zero area not cleared behind the reads"
    return out, qs, rep, (d, buf, sbuf, nbytes)


def _note(c, check, ratio):
    key = (OP_NAME[c["op"]], ROUTE_NAME[c["route"]], check)
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    print(f"  {c['label']}: {check} worst error / bound {ratio:.3g}")


def teardown_module():
    print(f"\nworst error / bound per route and check ({time.time() - T0:.0f} s):")
    for (op, route, check), r in sorted(WORST.items()):
        print(f"  {op:5s} {route:4s} {check:10s} {r:.3g}")


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_exact(c):
    t = make_inputs(c, "exact", 1234)
    ref = reference(c, t)
    S = reference(c, t, absolute=True)
    assert S.max().item() < 2 ** 21
    if c["op"] != 2:
        assert ref.abs().max().item() < 256              # bf16 holds every output exactly
    out, qs, rep, (d, buf, sbuf, nbytes) = run(c, t)
    assert rep.route == c["route"]
    expect = ref.float() if c["op"] == 2 else ref.float().bfloat16()
    diff = (out.double() - expect.double()).abs()
    assert torch.equal(out, expect.to(out.dtype)), f"{int((diff > 0).sum())} elements differ, max {diff.max().item()}"
    if qs is not None:
        y = ref.double().reshape(c["B"], -1, c["Co"] // 4, 4)
        want = torch.stack([y.sum((1, 3)), (y * y).sum((1, 3))], -1)
        assert torch.equal(qs, want), (qs - want).abs().max().item()
    # a second call on the same (cleared) scratch: the same bits
    first = out.clone()
    if c["op"] == 2 and (c["k"] == 1 or c["route"] == SIMT):
        out.zero_()
    elif "prior" in t:
        out.copy_(t["prior"])
    else:
        out.fill_(float("nan"))
    if qs is not None:
        qs.zero_()
    from ddpm_torch_b200 import _lib
    _lib.check(L().ddpm_conv_run(ct.byref(d), _lib.stream_ptr()), "conv (second call)")
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    assert (sbuf[GB:GB + rep.zero_bytes] == 0).all()
    _note(c, "exact", 0.0)


@pytest.mark.parametrize("wscale", [1e3, 1e-3], ids=["w1e3", "w1e-3"])
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_random(c, wscale):
    t = make_inputs(c, "random", 99, wscale)
    ref = reference(c, t)
    S = reference(c, t, absolute=True)
    out, _, rep, _ = run(c, t)
    b = bound(c, ref, S)
    err = (out.double() - ref).abs()
    ratio = (err / b).max().item()
    _note(c, "random", ratio)
    assert ratio <= 1.0, f"worst error / bound {ratio:.3g}"


# shapes several routes take: the same inputs through each, against each other within the sum of their bounds
def _split_input(c, t, n0):
    """the same conv with its single-source input split into a two-source concat (the CUDA-core route's form)"""
    c2 = dict(c, route=SIMT, Cin0=n0, Cin1=c["Cin0"] - n0)
    t2 = dict(t, x0=t["x0"][..., :n0].contiguous(), x1=t["x0"][..., n0:].contiguous())
    return c2, t2


AGREE = [
    case("CIFAR-10 downsamples.level_0.0.conv1", 0, HALO, 3, 32, 32, 128, 128, rowvec=True),
    case("CIFAR-10 downsamples.level_1.1.conv1", 0, HALO, 2, 16, 16, 256, 256, rowvec=True),
]


@pytest.mark.parametrize("c", AGREE, ids=["32x32x128", "16x16x256"])
def test_routes_agree(c):
    t = make_inputs(c, "random", 7)
    ref = reference(c, t)
    b = bound(c, ref, reference(c, t, absolute=True))
    outs = {HALO: run(c, t)[0], GEMM: run(dict(c, route=GEMM), t)[0]}
    c3, t3 = _split_input(c, t, 64)
    outs[SIMT] = run(c3, t3)[0]
    for r1, r2 in ((HALO, GEMM), (HALO, SIMT), (GEMM, SIMT)):
        ratio = ((outs[r1].double() - outs[r2].double()).abs() / (2 * b)).max().item()
        print(f"  {c['label']}: {ROUTE_NAME[r1]} vs {ROUTE_NAME[r2]} {ratio:.3g}")
        assert ratio <= 1.0


def test_fold_agrees_with_upsample_then_conv():
    c = case("CIFAR-10 upsamples.level_2.3.1 (8 -> 16)", 0, FOLD, 3, 8, 8, 256, 256, up=1)
    t = make_inputs(c, "random", 11)
    ref = reference(c, t)
    b = bound(c, ref, reference(c, t, absolute=True))
    fold = run(c, t)[0]
    ce = case("the same conv on the materialised 16x16 upsample", 0, HALO, 3, 16, 16, 256, 256)
    te = dict(t, x0=t["x0"].repeat_interleave(2, 1).repeat_interleave(2, 2).contiguous())
    explicit = run(ce, te)[0]
    be = bound(ce, reference(ce, te), reference(ce, te, absolute=True))
    ratio = ((fold.double() - explicit.double()).abs() / (b + be)).max().item()
    print(f"  fold vs nearest-2x + halo conv: {ratio:.3g}")
    assert ratio <= 1.0
