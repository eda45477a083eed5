"""The image-side convolutions of the UNet engine (unet_engine_impl.cuh, plan(): "in_conv", "out_conv.2" and the input gradient),
route by route, against fp64 torch, through the probes ddpm_unet_image_forward / _backward, which run the plan's own ops
("zero.fwd" + the in_conv ops + the out_conv.2 ops; "zero.bwd" + the out_conv.2 backward ops + the in_conv backward ops, with or
without the in_conv.dx ops):
  in_conv     tc: k_pack_in, k_im2col3<Cin> (q_sample prologue, stores x_t), a K = 64 GEMM whose epilogue adds the bias and
              writes h0's quad statistics; simt: k_in_conv<Cin> (same prologue and statistics)
  in wgrad    tc: an MN-major GEMM over the forward's im2col, k_unpack_tap mode 1, the column sum of dh0; simt: k_corr3x3<Cin>
              with the fused bias sum
  out_conv.2  tc: k_pack_tapco, a 1x1 GEMM to the 9*Cout tap outputs, k_out_gather<Cout>; backward k_chansum_nchw, k_im2col3
              with sign -1 over d_eps, a 1x1 dgrad over k_pack_tapco_t, an MN-major wgrad GEMM, k_unpack_tap mode 0;
              simt: k_out_conv<Cout>; backward k_chansum_nchw, k_in_conv<Cout> over the PK_FLIP_T weights, k_corr3x3<Cout> flip_t
  dx          tc: k_pack_tapflip, out_conv's GEMM shape, k_out_gather<Cin> without bias; simt: k_flip_transpose_w,
              k_out_conv<Cin> with a zero bias
The route is read from ddpm_unet_image_layout and asserted against the planner's rules (test_image_conv_cpu.expected_layout),
never assumed.  The cases (test_image_conv_cpu.CASES) reach every route both ways, the tails where B*H*W is not a multiple of
k_in_conv's 64-pixel warp tile or k_corr3x3's 256-pixel block (12x12 at B = 1, 20x12 at B = 3, whose blocks straddle images),
k_out_conv's 4-pixel groups on non-square maps, 96 channels (24 per lane in k_out_conv), the 256-channel limit, and the
CelebA-HQ map.  Each case runs without the prologue and with it, at distinct per-image t.

Exact mode: integer images and noise in [-2, 2], dyadic tables (tab_a, tab_s) in {1, 1/2, 1/4} per t, weights in {-1, 0, 1},
integer biases, a and d_eps in [-2, 2], dh0 in [-1, 1].  x_t is then a multiple of 1/4 with |x_t| <= 2.5, every operand is exact
in bf16, and every sum has Sigma|terms| < 2^21 (asserted), so every partial sum is exact in fp32 whatever the order: each output is
the fp64 result rounded once to its type, bit for bit (h0 and d_a to bf16; eps, dx and the weight and bias gradients in fp32), and
the quad statistics equal the fp64 sums of h0 (|h0| < 90, asserted, keeps each warp's fp32 partial sum of 128 squares below 2^24
sixteenths).  A second call is bit-identical.

Random mode: images uniform in [-1, 1] with some pixels exactly +-1, noise and d_eps N(0, 1), a N(0, 1), dh0 N(0.5, 1), the real
linear schedule's fp32 tables, fp32 weights and biases N(0, 1) x 1e3 on one conv and x 1e-3 on the other (swapped between the two
runs).  The fp64 reference is built on the operands as each route sees them: bf16-rounded x_t, d_eps and weights on the tensor-core
routes (k_im2col3 and the packs round them), fp32 weights and x_t on the CUDA-core routes (which do not).  What is left is
accumulation and output rounding (u = 2^-8 one bf16 rounding; 2^-23 per fp32 addition, which also covers tensor cores that do not
round to nearest):
  bf16 out    |y - ref| <= u|ref| + (1 + u) n 2^-23 S
  fp32 out    |y - ref| <= n 2^-23 S          S = sum |a||w| (+ |bias|) per output element
  n           in_conv 9 Cin + 1; out_conv tc hid + 9 gather adds + 1, simt 9 hid + 1; dx the same with Cin; d_a 9 Cout + 1;
              weight and bias gradients B H W + 1
  qstats      with e_p the fp32 bound of h0 at pixel p (no output rounding: the statistics are taken on the fp32 accumulator):
              |sum - ref| <= sum e_p + 8 2^-23 sum(|ref| + e_p),  |sumsq - ref| <= sum (2|ref| + e_p) e_p + 10 2^-23 sum(|ref| + e_p)^2
              (4 values per lane, five butterfly stages, then fp64 atomics)
x_t is bit-identical to torch's fp32 tab_a[t] * x + tab_s[t] * noise, each operation rounded on its own, on both routes.

Invariants: outputs and the flat gradient buffer are NaN-prefilled and must come back finite where written; after a probe
backward every flat-gradient element outside in_conv.* and out_conv.2.* is exactly zero.  End to end (one case per route mix):
x, noise, t -> fp64 autograd of q_sample + conv2d over the same a, d_eps and dh0 -> every gradient within rel-L2 1e-2 on the
tensor cores and 1e-4 on CUDA cores (bf16 outputs h0 and d_a: 1e-2 on both), which catches a stage that reads the wrong buffer
(say the backward reading x instead of x_t).  Each check prints its worst error / bound under -s; teardown prints the worst per op,
route and mode."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import ddpm_ref as R
import test_image_conv_cpu as IC

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -8
F23 = 2.0 ** -23
NAN = float("nan")
WORST = {}
TS = (999, 0, 500, 1)


def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def ptr(t):
    return None if t is None else t.data_ptr()


@pytest.fixture(scope="module", autouse=True)
def _report():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    print("\n[image conv] worst error / bound per op, route and mode:")
    for k in sorted(WORST):
        print(f"  {k[0]:>7} {k[1]:>5} {k[2]:>6}: {WORST[k]:.3f}")


def rname(r):
    return "tc" if r == 1 else "simt"


def check(op, route, mode, got, ref, bound, what):
    got, ref, bound = got.double(), ref.double(), bound.double()
    assert torch.isfinite(got).all(), f"{op}/{route} {what}: non-finite output (an element left unwritten?)"
    r = ((got - ref).abs() / (bound + 1e-300)).max().item()
    WORST[(op, route, mode)] = max(WORST.get((op, route, mode), 0.0), r)
    print(f"[{op} {route} {mode} {what}] worst error / bound {r:.3f}")
    assert r <= 1.0, f"{op}/{route} {mode} {what}: error / bound {r:.3f}"


def check_exact(op, route, got, ref, what):
    """bit for bit: the engine's output equals the fp64 result rounded once to the output's type"""
    want = ref.to(got.dtype)
    assert torch.isfinite(got.double()).all(), f"{op}/{route} {what}: non-finite output"
    bad = (got != want).sum().item()
    WORST[(op, route, "exact")] = max(WORST.get((op, route, "exact"), 0.0), float(bad))
    assert bad == 0, f"{op}/{route} exact {what}: {bad} elements differ; max |diff| {(got.double() - want.double()).abs().max().item()}"


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def bf(x):
    return x.to(torch.bfloat16).double()


def nchw(t):
    return t.permute(0, 3, 1, 2)


def tables():
    import ddpm_torch_b200 as D
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    return d.sqrt_alphas_bar.to(torch.float32).to(DEV), d.sqrt_one_minus_alphas_bar.to(torch.float32).to(DEV)


def t_rows(B, g):
    t = torch.tensor([TS[i] for i in range(min(B, 4))], dtype=torch.int64)
    if B > 4:
        t = torch.cat([t, torch.randint(0, 1000, (B - 4,), generator=g)])
    return t.to(DEV)


# ------------------------------------------------------------------------------------------------ model + probes
class Case:
    def __init__(self, name):
        import ddpm_torch_b200 as D
        cfg, B, H, W = IC.CASES[name]
        c = R.normalize_cfg(cfg)
        self.name, self.B, self.H, self.W = name, B, H, W
        self.hid, self.cin, self.cout = c["hid_channels"], c["in_channels"], c["out_channels"]
        self.m = D.UNet(c["in_channels"], c["hid_channels"], c["out_channels"], c["ch_multipliers"], c["num_res_blocks"],
                        c["apply_attn"], drop_rate=0.0).to(DEV)
        self.P = dict(self.m.named_parameters())
        self.h = self.m.prepare(B, H, W, True)
        self.lay = IC.layout(L(), self.h)
        assert self.lay == IC.expected_layout(cfg, H, W, 1), (name, self.lay)
        self.r_in, self.r_wg, self.r_out, self.r_dx, self.qs = self.lay

    def set_weights(self, w_in, b_in, w_out, b_out):
        with torch.no_grad():
            self.P["in_conv.weight"].copy_(w_in); self.P["in_conv.bias"].copy_(b_in)
            self.P["out_conv.2.weight"].copy_(w_out); self.P["out_conv.2.bias"].copy_(b_out)
        self.h = self.m.prepare(self.B, self.H, self.W, True)   # the repack stays pending on the side stream: the probe waits

    def grad(self, n):
        for name, shape, off in self.m._meta:
            if name == n:
                return self.m._grads[off:off + math.prod(shape)].view(shape)
        raise KeyError(n)

    def others_zero(self):
        keep = torch.zeros_like(self.m._grads, dtype=torch.bool)
        for name, shape, off in self.m._meta:
            if name.startswith("in_conv.") or name.startswith("out_conv.2."):
                keep[off:off + math.prod(shape)] = True
        return bool((self.m._grads[~keep] == 0).all())

    def run(self, x, a, d_eps, dh0, t=None, noise=None, ta=None, ts=None):
        from ddpm_torch_b200 import _lib
        B, H, W, hid = self.B, self.H, self.W, self.hid
        o = {"xt": torch.full((B, self.cin, H, W), NAN, device=DEV) if noise is not None else None,
             "h0": torch.full((B, H, W, hid), NAN, dtype=torch.bfloat16, device=DEV),
             "qs": torch.full((B, hid // 4, 2), NAN, dtype=torch.float64, device=DEV) if self.qs else None,
             "eps": torch.full((B, self.cout, H, W), NAN, device=DEV),
             "d_a": torch.full((B, H, W, hid), NAN, dtype=torch.bfloat16, device=DEV),
             "dx": torch.full((B, self.cin, H, W), NAN, device=DEV)}
        st = _lib.stream_ptr()
        rc = L().ddpm_unet_image_forward(self.h, x.data_ptr(), ptr(t), ptr(noise), ptr(ta), ptr(ts), a.data_ptr(), ptr(o["xt"]),
                                         o["h0"].data_ptr(), ptr(o["qs"]), o["eps"].data_ptr(), st)
        assert rc == 0, L().ddpm_last_error()
        self.m._grads.fill_(NAN)
        rc = L().ddpm_unet_image_backward(self.h, d_eps.data_ptr(), dh0.data_ptr(), o["dx"].data_ptr(), o["d_a"].data_ptr(), st)
        assert rc == 0, L().ddpm_last_error()
        torch.cuda.synchronize()
        assert L().ddpm_device_error_flag() == 0
        for n in ("in_conv.weight", "in_conv.bias", "out_conv.2.weight", "out_conv.2.bias"):
            o[n] = self.grad(n).clone()
        assert self.others_zero(), "a gradient outside in_conv.* / out_conv.2.* is not exactly zero"
        return o


_CASES = {}


def get_case(name):
    if name not in _CASES:
        _CASES.clear()                 # one model at a time on the device
        torch.cuda.empty_cache()
        _CASES[name] = Case(name)
    return _CASES[name]


# ------------------------------------------------------------------------------------------------ fp64 references
def refs(c, x_t, a, d_eps, dh0, w_in, b_in, w_out, b_out):
    """fp64 references on the operands as each route sees them, and the S = sum |a||w| (+ |bias|) of every output"""
    tc = lambda r: r == 1
    xs = bf(x_t) if tc(c.r_in) else x_t.double()
    wi = bf(w_in) if tc(c.r_in) else w_in.double()
    a64 = nchw(a).double()
    wo = bf(w_out) if tc(c.r_out) else w_out.double()
    de = bf(d_eps) if tc(c.r_out) else d_eps.double()
    dh = nchw(dh0).double()
    xw = bf(x_t) if tc(c.r_wg) else x_t.double()
    wdx = bf(w_in) if tc(c.r_dx) else w_in.double()
    bi, bo = b_in.double(), b_out.double()
    ab = lambda v: v.abs()
    r = {}
    r["h0"] = (F.conv2d(xs, wi, bi, padding=1), F.conv2d(ab(xs), ab(wi), ab(bi), padding=1), 9 * c.cin + 1)
    n_out = c.hid + 10 if tc(c.r_out) else 9 * c.hid + 1
    r["eps"] = (F.conv2d(a64, wo, bo, padding=1), F.conv2d(ab(a64), ab(wo), ab(bo), padding=1), n_out)
    r["d_a"] = (F.conv_transpose2d(de, wo, padding=1), F.conv_transpose2d(ab(de), ab(wo), padding=1), 9 * c.cout + 1)
    n_px = c.B * c.H * c.W + 1
    gw = torch.nn.grad.conv2d_weight
    r["dW_out"] = (gw(a64, w_out.shape, de, padding=1), gw(ab(a64), w_out.shape, ab(de), padding=1), n_px)
    r["db_out"] = (d_eps.double().sum((0, 2, 3)), d_eps.double().abs().sum((0, 2, 3)), n_px)
    r["dW_in"] = (gw(xw, w_in.shape, dh, padding=1), gw(ab(xw), w_in.shape, ab(dh), padding=1), n_px)
    r["db_in"] = (dh.sum((0, 2, 3)), dh.abs().sum((0, 2, 3)), n_px)
    n_dx = c.hid + 10 if tc(c.r_dx) else 9 * c.hid + 1
    r["dx"] = (F.conv_transpose2d(dh, wdx, padding=1), F.conv_transpose2d(ab(dh), ab(wdx), padding=1), n_dx)
    return r


# op -> (engine output key, which route, bf16 output, layout of the engine output)
OPS = {"h0": ("h0", "r_in", True, nchw), "eps": ("eps", "r_out", False, None), "d_a": ("d_a", "r_out", True, nchw),
       "dW_out": ("out_conv.2.weight", "r_out", False, None), "db_out": ("out_conv.2.bias", "r_out", False, None),
       "dW_in": ("in_conv.weight", "r_wg", False, None), "db_in": ("in_conv.bias", "r_wg", False, None),
       "dx": ("dx", "r_dx", False, None)}


def quad_ref(c, h0_ref):
    v = h0_ref.reshape(c.B, c.hid // 4, 4, c.H * c.W)
    return v.sum((2, 3)), (v * v).sum((2, 3))


def inputs(c, mode, prologue, g, flip=False):
    B, H, W, hid, cin, cout = c.B, c.H, c.W, c.hid, c.cin, c.cout
    ri = lambda lo, hi, shape: torch.randint(lo, hi + 1, shape, generator=g).float()
    t = t_rows(B, g)
    if mode == "exact":
        x, noise = ri(-2, 2, (B, cin, H, W)), ri(-2, 2, (B, cin, H, W))
        k = torch.arange(1000) % 7                 # t = 999, 0, 500, 1 get four different (tab_a, tab_s) pairs
        ta = torch.tensor([1.0, 0.5, 0.25, 0.5, 0.25, 0.25, 1.0])[k]
        ts = torch.tensor([0.25, 0.5, 0.25, 0.25, 0.5, 1.0, 0.25])[k]
        w_in, b_in = ri(-1, 1, (hid, cin, 3, 3)), ri(-2, 2, (hid,))
        w_out, b_out = ri(-1, 1, (cout, hid, 3, 3)), ri(-2, 2, (cout,))
        a, d_eps, dh0 = ri(-2, 2, (B, H, W, hid)), ri(-2, 2, (B, cout, H, W)), ri(-1, 1, (B, H, W, hid))
    else:
        x = torch.rand((B, cin, H, W), generator=g) * 2 - 1
        x.view(-1)[::7] = 1.0
        x.view(-1)[3::11] = -1.0
        noise = torch.randn((B, cin, H, W), generator=g)
        ta, ts = None, None
        s_in, s_out = (1e-3, 1e3) if flip else (1e3, 1e-3)
        w_in, b_in = torch.randn((hid, cin, 3, 3), generator=g) * s_in, torch.randn((hid,), generator=g) * s_in
        w_out, b_out = torch.randn((cout, hid, 3, 3), generator=g) * s_out, torch.randn((cout,), generator=g) * s_out
        a = torch.randn((B, H, W, hid), generator=g)
        d_eps = torch.randn((B, cout, H, W), generator=g)
        dh0 = torch.randn((B, H, W, hid), generator=g) + 0.5
    d = dict(x=x, noise=noise, w_in=w_in, b_in=b_in, w_out=w_out, b_out=b_out, a=a.to(torch.bfloat16), d_eps=d_eps,
             dh0=dh0.to(torch.bfloat16))
    d = {k: v.to(DEV) for k, v in d.items()}
    if mode == "exact":
        d["ta"], d["ts"] = ta.to(DEV), ts.to(DEV)
    else:
        d["ta"], d["ts"] = tables()
    d["t"] = t
    if not prologue:
        d["noise"] = None
    return d


def run_case(c, d):
    c.set_weights(d["w_in"], d["b_in"], d["w_out"], d["b_out"])
    pro = d["noise"] is not None
    kw = dict(t=d["t"], noise=d["noise"], ta=d["ta"], ts=d["ts"]) if pro else {}
    o = c.run(d["x"], d["a"], d["d_eps"], d["dh0"], **kw)
    if pro:
        x_t = d["ta"][d["t"]].view(-1, 1, 1, 1) * d["x"] + d["ts"][d["t"]].view(-1, 1, 1, 1) * d["noise"]
        assert torch.equal(o["xt"], x_t), "x_t differs from torch's fp32 tab_a[t] * x + tab_s[t] * noise"
    else:
        x_t = d["x"]
    return o, x_t


CASE_NAMES = sorted(IC.CASES)
# case-major, so that each case's model is built once
RUNS = [(n, m, p) for n in CASE_NAMES for m in ("exact", "random") for p in (False, True)]


@pytest.mark.parametrize("name,mode,prologue", RUNS)
def test_image_convs(name, mode, prologue):
    c = get_case(name)
    g = torch.Generator().manual_seed(RUNS.index((name, mode, prologue)))
    (exact_bit_for_bit if mode == "exact" else random_within_bounds)(c, g, prologue)


def exact_bit_for_bit(c, g, prologue):
    name = c.name
    d = inputs(c, "exact", prologue, g)
    o, x_t = run_case(c, d)
    r = refs(c, x_t, d["a"], d["d_eps"], d["dh0"], d["w_in"], d["b_in"], d["w_out"], d["b_out"])
    for op, (key, rk, is_bf16, lay) in OPS.items():
        ref, S, _ = r[op]
        assert S.max().item() < 2.0 ** 21, f"{op}: exact-mode inputs too large"
        got = o[key] if lay is None else lay(o[key])
        check_exact(op, rname(getattr(c, rk)), got, ref, f"{name} prologue={prologue}")
    if c.qs:
        h0_ref = r["h0"][0]
        assert h0_ref.abs().max().item() < 90, "exact-mode h0 too large for exact fp32 quad statistics"
        s1, s2 = quad_ref(c, h0_ref)
        assert torch.equal(o["qs"][..., 0], s1) and torch.equal(o["qs"][..., 1], s2), "quad statistics differ from the fp64 sums"
        WORST[("qstats", rname(c.r_in), "exact")] = 0.0
    # a second call is bit-identical
    o2, _ = run_case(c, d)
    for k, v in o.items():
        if v is not None:
            assert torch.equal(v, o2[k]), f"{k}: second call differs"


def random_within_bounds(c, g, prologue):
    name = c.name
    d = inputs(c, "random", prologue, g, flip=prologue)
    o, x_t = run_case(c, d)
    r = refs(c, x_t, d["a"], d["d_eps"], d["dh0"], d["w_in"], d["b_in"], d["w_out"], d["b_out"])
    what = f"{name} prologue={prologue}"
    for op, (key, rk, is_bf16, lay) in OPS.items():
        ref, S, n = r[op]
        got = o[key] if lay is None else lay(o[key])
        bound = n * F23 * S
        if is_bf16:
            bound = U * ref.abs() + (1 + U) * bound
        check(op, rname(getattr(c, rk)), "random", got, ref, bound + 1e-300, what)
    if c.qs:
        h0_ref, S, n = r["h0"]
        e = n * F23 * S
        v = lambda z: z.reshape(c.B, c.hid // 4, 4, c.H * c.W).sum((2, 3))
        s1, s2 = quad_ref(c, h0_ref)
        b1 = v(e) + 8 * F23 * v(h0_ref.abs() + e)
        b2 = v((2 * h0_ref.abs() + e) * e) + 10 * F23 * v((h0_ref.abs() + e) ** 2)
        check("qstats", rname(c.r_in), "random", o["qs"][..., 0], s1, b1, what + " sum")
        check("qstats", rname(c.r_in), "random", o["qs"][..., 1], s2, b2, what + " sumsq")


# one case per route mix: all tensor cores, all CUDA cores, tensor-core in_conv with CUDA-core out_conv and dx, and CUDA cores at
# 128 channels on a non-square map
@pytest.mark.parametrize("name", ["small64_c3", "tiny_b3", "small64_c4", "hid128_24x48"])
def test_end_to_end_against_fp64_autograd(name):
    c = get_case(name)
    g = torch.Generator().manual_seed(99)
    B, H, W, hid, cin, cout = c.B, c.H, c.W, c.hid, c.cin, c.cout
    d = inputs(c, "random", True, g)
    with torch.no_grad():                      # weights at the reference's scale
        d["w_in"] /= 1e3 * math.sqrt(9 * cin); d["b_in"] /= 1e3
        d["w_out"] *= 1e3 / math.sqrt(9 * hid); d["b_out"] *= 1e3
    o, _ = run_case(c, d)
    ta, ts = (v.double()[d["t"]].view(-1, 1, 1, 1) for v in (d["ta"], d["ts"]))
    leaf = lambda v: v.double().clone().requires_grad_(True)
    xt = leaf(ta * d["x"].double() + ts * d["noise"].double())
    wi, bi, wo, bo, a64 = leaf(d["w_in"]), leaf(d["b_in"]), leaf(d["w_out"]), leaf(d["b_out"]), leaf(nchw(d["a"]))
    h0 = F.conv2d(xt, wi, bi, padding=1)
    eps = F.conv2d(a64, wo, bo, padding=1)
    ((eps * d["d_eps"].double()).sum() + (h0 * nchw(d["dh0"]).double()).sum()).backward()
    tol = lambda r: 1e-2 if r == 1 else 1e-4
    pairs = [("h0", nchw(o["h0"]), h0.detach(), 1e-2), ("eps", o["eps"], eps.detach(), tol(c.r_out)),
             ("d_a", nchw(o["d_a"]), a64.grad, 1e-2), ("dW_out", o["out_conv.2.weight"], wo.grad, tol(c.r_out)),
             ("db_out", o["out_conv.2.bias"], bo.grad, tol(c.r_out)), ("dW_in", o["in_conv.weight"], wi.grad, tol(c.r_wg)),
             ("db_in", o["in_conv.bias"], bi.grad, tol(c.r_wg)), ("dx", o["dx"], xt.grad, tol(c.r_dx))]
    for op, got, ref, lim in pairs:
        e = rel(got, ref)
        print(f"[e2e {name} {op}] rel-L2 {e:.2e} (limit {lim:g})")
        assert e <= lim, f"{name} {op}: rel-L2 {e:.3e} > {lim:g}"


def test_probe_refusals_on_a_real_plan():
    from ddpm_torch_b200 import _lib
    c = get_case("tail32_12x12")                 # no quad statistics at 12x12
    st = _lib.stream_ptr()
    B, H, W, hid = c.B, c.H, c.W, c.hid
    x = torch.zeros(B, c.cin, H, W, device=DEV)
    a = torch.zeros(B, H, W, hid, dtype=torch.bfloat16, device=DEV)
    eps = torch.zeros(B, c.cout, H, W, device=DEV)
    qs = torch.zeros(B, hid // 4, 2, dtype=torch.float64, device=DEV)
    t = torch.zeros(B, dtype=torch.int64, device=DEV)
    fwd = lambda q=None: L().ddpm_unet_image_forward(c.h, x.data_ptr(), None, None, None, None, a.data_ptr(), None, None, ptr(q),
                                                     eps.data_ptr(), st)
    bwd = lambda: L().ddpm_unet_image_backward(c.h, eps.data_ptr(), a.data_ptr(), None, None, st)
    c.h = c.m.prepare(B, H, W, True)
    assert bwd() != 0 and b"needs a ddpm_unet_image_forward" in L().ddpm_last_error()     # no image forward yet on this plan
    assert fwd(qs) != 0 and b"no quad statistics" in L().ddpm_last_error()
    assert fwd() == 0, L().ddpm_last_error()
    assert L().ddpm_unet_temb_backward(c.h, torch.zeros(B, 1 << 14, device=DEV).data_ptr(), None, None, st) != 0
    assert bwd() == 0, L().ddpm_last_error()
    assert bwd() == 0, L().ddpm_last_error()                       # the image forward stays what the backward reads
    # any other forward of the plan in between is refused
    assert L().ddpm_unet_forward(c.h, x.data_ptr(), t.data_ptr(), eps.data_ptr(), 0, st) == 0, L().ddpm_last_error()
    assert bwd() != 0 and b"needs a ddpm_unet_image_forward" in L().ddpm_last_error()
    assert fwd() == 0
    assert L().ddpm_unet_temb_forward(c.h, t.data_ptr(), 0, None, None, None, None, st) == 0, L().ddpm_last_error()
    assert bwd() != 0 and b"needs a ddpm_unet_image_forward" in L().ddpm_last_error()
    # an inference plan runs the forward probe and refuses the backward
    c.h = c.m.prepare(B, H, W, False)
    assert IC.layout(L(), c.h) == (0, -1, 0, -1, 0)
    assert fwd() == 0, L().ddpm_last_error()
    assert bwd() != 0 and b"without training" in L().ddpm_last_error()
    torch.cuda.synchronize()
    assert L().ddpm_device_error_flag() == 0
    _CASES.clear()
