"""The timestep path of the UNet engine (unet_engine_impl.cuh, plan(): `t` -> sinusoidal embedding -> Linear -> SiLU -> Linear -> the
per-ResBlock projections TP [B][tp_ld] = Linear(SiLU(e1)) that the conv epilogues add as a row vector, and its adjoint), route by
route, against fp64 torch, through the probes ddpm_unet_temb_forward / _backward, which run the plan's own ops ("zero.fwd" + the
OP_TEMB ops, or the one-row ops the sampler swaps in; "zero.bwd" + "temb.dtp_cast" / "temb.proj.bwd" / "temb.mlp.bwd"):
  simt     k_timestep_embedding, k_sgemm fc0, k_sgemm fc1 split-K x4, k_sgemm_table projections split-K x4; backward two
           k_sgemm_table launches (fc weight gradients; d_st with atomics per block) and the MLP adjoint
  tc       B a power of two >= 64: k_cast_bf16 (SiLU) + one wgmma GEMM over Wcat / bias_cat packed by k_pack_fc; backward one
           MN-major GEMM over K = B + k_scatter_fc_grad, a split-K KK GEMM with atomics into d_st over WcatT, the MLP adjoint
  uniform  the one-row SIMT path for row 0 and k_bcast_rows (ddpm_sampler_step), on SIMT and tensor-core plans
The route is read from ddpm_unet_temb_layout and asserted, never assumed.

Each stage is checked element by element against fp64 evaluated on the ENGINE's own input to that stage (e0 on the engine's emb,
e1 on its e0, TP on its e1, the fc weight gradients and d_st on its e1 and the given dTP, embed.2's gradients and d_s0 on its d_st,
embed.0's gradients on its d_s0), so no error propagation has to be bounded.  Bounds (2^-23 per fp32 addition: the tensor cores do
not promise round-to-nearest, and it covers the product roundings of the CUDA-core GEMMs too; u = 2^-8, one bf16 rounding):
  GEMM     |c - ref| <= n 2^-23 S,  S = sum |a||w| + |bias|,  n = the terms summed: K + the bias + the split-K partials (4 in the
           CUDA-core fc1 / projections / d_s0, one per block in the CUDA-core d_st, up to 32 in the tensor-core d_st)
  tc       + (2u + u^2) S: silu(e1) and the packed weights (forward), dTP and silu(e1) (weight gradient), dTP and WcatT (d_st) are
           each rounded to bf16 once
  SiLU     silu_f(y) = y / (1 + __expf(-y)).  __expf(x) is within 2 + 1.173|x| ulp of e^x (CUDA programming guide, intrinsic
           functions), so sigma(y) carries kappa = (1 - sigma)(2 + 1.173|y|) 2^-23 + 2^-23 relative (add and divide included) and
           silu the same; + 1e-30 absolute where __expf overflows (y < -88: silu(y) < 1e-36).  The guide's model is assumed, not
           measured, at |y| ~ 10^3 (the x100 case, where __expf saturates to 0 / inf).  A SiLU on a GEMM operand adds
           sum kappa |silu(a)||w| to that GEMM's bound.
  SiLU'    silu_grad_f(y) = s (1 + y (1 - s)), s as above: |dg| <= s kappa (1 + 2|y|) + 2^-22 (s + s|y|(1 - s)) + 2^-24 s|y|;
           d = dy * g adds one rounding.  Its error e_d enters the next GEMM as sum e_d |w|.
  emb      sin / cos of a = t f_j, f_j = exp(-j k), k = ln(1e4) / (half - 1) formed in fp32 (logf, divide; the constant equals the
           reference's fp64 constant rounded once, for every hid in use): with x = j k, |da| <= |a| (|x| + 1) 5 2^-24, and sinf /
           cosf add 2 ulp: |e - ref| <= |da| + 2^-22 |ref| + 2^-40.  It is also compared with the reference's own fp32 recipe
           (oracle timestep_embedding: fp32 f_j, fp32 products), within the sum of both bounds.
fc.bias gradients are not produced by these ops: they are the GroupNorm column sums, covered by test_groupnorm_gpu.py; the probe's
backward must leave them, and every other non-timestep gradient, exactly zero.

End to end, t -> TP and dTP -> every timestep gradient are compared with fp64 from t itself: rel-L2 <= 1e-2 on the tensor-core
route (bf16 operands) and <= 1e-4 on the CUDA cores.  This catches a stage that reads the wrong buffer, which per-stage checks on
engine inputs would let through.  Route agreement: B = 64 (tensor cores) vs B = 63 (CUDA cores) on the same 63 rows, and the
uniform route vs the per-row route of the same plan, within the sum of both bounds plus the fp64 difference their inputs cause.
Each check prints its worst error / bound under -s; teardown prints the worst per stage and route."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import ddpm_ref as R
import test_temb_cpu as TC

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -8
F23 = 2.0 ** -23
F24 = 2.0 ** -24
WORST = {}

WIDE_CFG = dict(in_channels=3, hid_channels=256, out_channels=3, ch_multipliers=(1, 2, 4), num_res_blocks=2,
                apply_attn=(False, False, True), drop_rate=0.0)
# name -> (cfg, resolution).  The probes run the timestep ops only, so the resolution just has to plan; it is kept small.
CFGS = {"tiny": (R.TINY_CFG, 16), "small64": (R.SMALL64_CFG, 32), "cifar10": (R.CIFAR10_CFG, 32),
        "celebahq": (R.CELEBAHQ_CFG, 64), "wide": (WIDE_CFG, 32)}


def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


@pytest.fixture(scope="module", autouse=True)
def _report():
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    print("\n[temb] worst error / bound per stage and route:")
    for k in sorted(WORST):
        print(f"  {k[0]:>10} {k[1]:>8}: {WORST[k]:.3f}")


def check(stage, route, got, ref, bound, what=""):
    got, ref, bound = got.double(), ref.double(), bound.double()
    assert torch.isfinite(got).all(), f"{stage}/{route} {what}: non-finite output"
    r = ((got - ref).abs() / bound).max().item()
    WORST[(stage, route)] = max(WORST.get((stage, route), 0.0), r)
    print(f"[{stage} {route} {what}] worst error / bound {r:.3f}")
    assert r <= 1.0, f"{stage}/{route} {what}: error / bound {r:.3f}"
    return r


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


# ------------------------------------------------------------------------------------------------ fp64 reference pieces
def sig(y):
    return torch.sigmoid(y)


def silu_kappa(y):
    """relative error of silu_f / sigma through __expf (module docstring)"""
    return (1 - sig(y)) * (2 + 1.173 * y.abs()) * F23 + F23


def silu_err(y):
    return silu_kappa(y) * F.silu(y).abs() + 1e-30


def silu_grad(y):
    s = sig(y)
    return s * (1 + y * (1 - s))


def silu_grad_err(y):
    s = sig(y)
    k = silu_kappa(y)
    return s * k * (1 + 2 * y.abs()) + 2.0 ** -22 * (s + s * y.abs() * (1 - s)) + F24 * s * y.abs() + 1e-30


def emb_ref(t, ch):
    half = ch // 2
    j = torch.arange(half, dtype=torch.float64, device=t.device)
    x = j * (math.log(10000) / (half - 1))
    a = t.double()[:, None] * torch.exp(-x)[None]
    e = torch.cat([torch.sin(a), torch.cos(a)], 1)
    da = a.abs() * (x.abs() + 1)[None] * 5 * F24
    return e, torch.cat([da, da], 1) + 2.0 ** -22 * e.abs() + 2.0 ** -40


def linear_bound(a, w, b, n, a_err=None, tc=False):
    """fp64 a @ w^T + b and its bound (module docstring); a_err = per-element error already in a (SiLU), tc = bf16 operands"""
    S = a.abs() @ w.abs().t() + (b.abs()[None] if b is not None else 0)
    ref = a @ w.t() + (b[None] if b is not None else 0)
    bound = n * F23 * S + (2 * U + U * U) * S * (1 if tc else 0)
    if a_err is not None:
        bound = bound + a_err @ w.abs().t()
    return ref, bound + 1e-30


# ------------------------------------------------------------------------------------------------ model + probe
class Probe:
    def __init__(self, name, B, train, seed=0, scale0=1.0):
        import ddpm_torch_b200 as D
        cfg, HW = CFGS[name]
        c = R.normalize_cfg(cfg)
        self.name, self.B, self.train = name, B, train
        m = D.UNet(c["in_channels"], c["hid_channels"], c["out_channels"], c["ch_multipliers"], c["num_res_blocks"],
                   c["apply_attn"], drop_rate=0.0)
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():       # the reference init, with non-zero biases so that the bias adds and bias_cat are exercised
            for n, p in m.named_parameters():
                if n.startswith("embed.") or ".fc." in n:
                    if n.endswith(".bias"):
                        p.copy_(torch.randn(p.shape, generator=g) * 0.5)
                    if n == "embed.0.weight":
                        p.mul_(scale0)
        self.m = m.to(DEV)
        self.h = self.m.prepare(B, HW, HW, train)       # a training plan leaves its repack pending on the side stream
        (self.route, self.has_uni, self.E, self.tp_ld, self.maxc, self.blocks) = TC.layout(L(), self.h)
        self.ch = c["hid_channels"]
        self.P = dict(self.m.named_parameters())

    @property
    def rname(self):
        return "tc" if self.route == 1 else "simt"

    def w(self, n):
        return self.P[n].detach().double()

    def grad(self, n):
        for name, shape, off in self.m._meta:
            if name == n:
                return self.m._grads[off:off + math.prod(shape)].view(shape)
        raise KeyError(n)

    def forward(self, t, uniform=0):
        B = self.B
        o = {k: torch.full((B, n), float("nan"), device=DEV) for k, n in
             (("emb", self.ch), ("e0", self.E), ("e1", self.E), ("tp", self.tp_ld))}
        from ddpm_torch_b200 import _lib
        st = _lib.stream_ptr()
        rc = L().ddpm_unet_temb_forward(self.h, t.data_ptr(), uniform, o["emb"].data_ptr(), o["e0"].data_ptr(),
                                        o["e1"].data_ptr(), o["tp"].data_ptr(), st)
        assert rc == 0, L().ddpm_last_error()
        torch.cuda.synchronize()
        assert L().ddpm_device_error_flag() == 0
        return o

    def backward(self, dtp):
        o = {k: torch.full((self.B, self.E), float("nan"), device=DEV) for k in ("d_st", "d_s0")}
        from ddpm_torch_b200 import _lib
        # "zero.bwd" clears the whole flat buffer before the timestep ops run, so this NaN fill does not show an element they
        # never wrote: that is left to the element-wise bounds, which reject a stale 0 wherever |ref| exceeds the bound (random
        # dTP keeps the reference away from 0 almost everywhere).  It does show that the memset covers the whole buffer.
        self.m._grads.fill_(float("nan"))
        rc = L().ddpm_unet_temb_backward(self.h, dtp.data_ptr(), o["d_st"].data_ptr(), o["d_s0"].data_ptr(), _lib.stream_ptr())
        assert rc == 0, L().ddpm_last_error()
        torch.cuda.synchronize()
        assert L().ddpm_device_error_flag() == 0
        return o

    def tp_ref(self, e1, tc=None):
        """fp64 TP on the given e1 (rows x tp_ld; pad columns 0) and its bound"""
        tc = self.route == 1 if tc is None else tc
        e1 = e1.double()
        s = F.silu(e1)
        ref = torch.zeros(e1.shape[0], self.tp_ld, dtype=torch.float64, device=DEV)
        bnd = torch.full_like(ref, 1e-30)          # pad columns: exactly zero
        n = self.E + 1 + (0 if tc else 4)
        for b, off, cout in self.blocks:
            r, bd = linear_bound(s, self.w(b + ".fc.weight"), self.w(b + ".fc.bias"), n, silu_err(e1), tc)
            ref[:, off:off + cout] = r; bnd[:, off:off + cout] = bd
        return ref, bnd

    def tp_from_t(self, t):
        """fp64 t -> TP, from nothing the engine computed"""
        e, _ = emb_ref(t, self.ch)
        e0 = e @ self.w("embed.0.weight").t() + self.w("embed.0.bias")
        e1 = F.silu(e0) @ self.w("embed.2.weight").t() + self.w("embed.2.bias")
        return self.tp_ref(e1)[0]


def t_rows(B, seed):
    g = torch.Generator().manual_seed(1000 + seed)
    t = torch.randint(0, 1000, (B,), generator=g)
    fixed = torch.tensor([999, 0, 1])[:B]
    t[:len(fixed)] = fixed
    return t.to(DEV)


def check_forward(p, t, o, rows=None, tag="", route=None):
    route = route or p.rname
    rows = slice(None) if rows is None else rows
    t, emb, e0, e1, tp = t[rows], o["emb"][rows], o["e0"][rows], o["e1"][rows], o["tp"][rows]
    # embedding vs fp64, and vs the reference's own fp32 recipe
    er, eb = emb_ref(t, p.ch)
    check("emb", route, emb, er, eb, tag)
    e32 = R.timestep_embedding(t, p.ch).double()
    check("emb~fp32", route, emb, e32, 2 * eb, tag)
    # MLP, each layer on the engine's input
    r0, b0 = linear_bound(emb.double(), p.w("embed.0.weight"), p.w("embed.0.bias"), p.ch + 1)
    check("e0", route, e0, r0, b0, tag)
    r1, b1 = linear_bound(F.silu(e0.double()), p.w("embed.2.weight"), p.w("embed.2.bias"), p.E + 1 + 4, silu_err(e0.double()))
    check("e1", route, e1, r1, b1, tag)
    rt, bt = p.tp_ref(e1, tc=(route == "tc"))
    check("TP", route, tp, rt, bt, tag)
    # pad columns of the narrower blocks stay exactly zero
    for b, off, cout in p.blocks:
        assert (tp[:, off + cout:off + p.maxc] == 0).all(), f"{b}: TP pad columns written"
    return rt, bt


# ------------------------------------------------------------------------------------------------ cases
# (config, B, training plan, embed.0 scale)
FWD_CASES = [("tiny", 3, 1, 1.0), ("tiny", 64, 1, 1.0), ("small64", 3, 1, 1.0), ("small64", 64, 1, 1.0),
             ("cifar10", 1, 1, 1.0), ("cifar10", 3, 1, 1.0), ("cifar10", 63, 1, 1.0), ("cifar10", 64, 1, 1.0),
             ("cifar10", 128, 1, 1.0), ("cifar10", 256, 1, 1.0), ("cifar10", 3, 0, 1.0), ("cifar10", 64, 0, 1.0),
             ("cifar10", 256, 0, 1.0), ("cifar10", 3, 1, 100.0), ("cifar10", 128, 1, 100.0),
             ("celebahq", 3, 1, 1.0), ("celebahq", 64, 1, 1.0), ("celebahq", 64, 1, 100.0), ("wide", 3, 1, 1.0), ("wide", 64, 1, 1.0)]
TC_B = (64, 128, 256)


def _id(c):
    return f"{c[0]}-B{c[1]}-{'train' if c[2] else 'infer'}" + ("-x100" if c[3] != 1 else "")


@pytest.mark.parametrize("case", FWD_CASES, ids=_id)
def test_forward_and_backward_vs_fp64(case):
    name, B, train, scale0 = case
    p = Probe(name, B, train, seed=B, scale0=scale0)
    assert p.route == (1 if B in TC_B else 0), "the planner's route changed"
    t = t_rows(B, B)
    o = p.forward(t)
    tag = _id(case)
    check_forward(p, t, o, tag=tag)
    if scale0 != 1:
        assert o["e0"].abs().max().item() > 100, "the x100 case must drive SiLU past __expf overflow (|y| > 88.7)"
    # end to end: t -> TP from fp64 alone
    r = rel(o["tp"], p.tp_from_t(t))
    print(f"[e2e {p.rname} {tag}] t -> TP rel-L2 {r:.3e}")
    assert r <= (1e-2 if p.route == 1 else 1e-4)
    if not train:
        assert L().ddpm_unet_temb_backward(p.h, o["tp"].data_ptr(), None, None, None) != 0
        assert b"without training" in L().ddpm_last_error()
        return
    check_backward(p, t, o, tag)


def check_backward(p, t, o, tag):
    B, E, route = p.B, p.E, p.rname
    g = torch.Generator(device=DEV).manual_seed(7 + B)
    dtp = torch.randn(B, p.tp_ld, device=DEV, generator=g)
    for _, off, cout in p.blocks:
        dtp[:, off + cout:off + p.maxc] = 0           # the plan's dTP pads stay zero: nothing writes them
    out = p.backward(dtp)
    d_st, d_s0 = out["d_st"].double(), out["d_s0"].double()
    tc = p.route == 1
    e1 = o["e1"].double(); s1 = F.silu(e1); s1e = silu_err(e1)
    dT = dtp.double()
    # fc weight gradients: dW[o][e] = sum_b silu(e1[b][e]) dTP[b][off+o]    (K = B)
    for b, off, cout in p.blocks:
        dTb = dT[:, off:off + cout]
        ref = dTb.t() @ s1
        S = dTb.abs().t() @ s1.abs()
        bound = (B + 1) * F23 * S + (2 * U + U * U) * S * tc + dTb.abs().t() @ s1e + 1e-30
        check("dW_fc", route, p.grad(b + ".fc.weight"), ref, bound, f"{tag} {b}")
    # d_st[b][e] = sum_blocks sum_o dTP[b][off+o] W_fc[o][e]
    ref = torch.zeros(B, E, dtype=torch.float64, device=DEV); S = torch.zeros_like(ref)
    for b, off, cout in p.blocks:
        W = p.w(b + ".fc.weight")
        ref += dT[:, off:off + cout] @ W; S += dT[:, off:off + cout].abs() @ W.abs()
    n = (p.tp_ld + 32) if tc else (p.maxc + len(p.blocks))
    check("d_st", route, d_st, ref, n * F23 * S + (2 * U + U * U) * S * tc + 1e-30, tag)
    # embed.2 on the engine's d_st; embed.0 on the engine's d_s0
    e0 = o["e0"].double(); emb = o["emb"].double()
    W2 = p.w("embed.2.weight")
    for (lay, y, a, a_err, dy, nxt) in (("embed.2", e1, F.silu(e0), silu_err(e0), d_st, d_s0),
                                        ("embed.0", e0, emb, torch.zeros_like(emb), d_s0, None)):
        gq = silu_grad(y)
        d = dy * gq
        ed = dy.abs() * silu_grad_err(y) + F24 * d.abs()
        ref_w = d.t() @ a
        S = d.abs().t() @ a.abs()
        check("dW_" + lay, route, p.grad(lay + ".weight"), ref_w,
              (B + 1) * F23 * S + ed.t() @ a.abs() + d.abs().t() @ a_err + 1e-30, tag)
        check("db_" + lay, route, p.grad(lay + ".bias"), d.sum(0), (B + 1) * F23 * d.abs().sum(0) + ed.sum(0) + 1e-30, tag)
        if nxt is not None:
            check("d_s0", route, nxt, d @ W2, (E + 4) * F23 * (d.abs() @ W2.abs()) + ed @ W2.abs() + 1e-30, tag)
    # everything else in the flat gradient buffer is exactly zero (fc.bias included: it comes from the GroupNorm column sums)
    G = p.m._grads.clone()
    temb = [n for n, _, _ in p.m._meta if n.startswith("embed.") or n.endswith(".fc.weight")]
    for n in temb:
        gv = p.grad(n)
        assert torch.isfinite(gv).all(), n
        for nm, shape, off in p.m._meta:
            if nm == n:
                G[off:off + math.prod(shape)] = 0
    assert torch.equal(G, torch.zeros_like(G)), "the timestep backward wrote outside the timestep gradients"
    # end to end: dTP -> every timestep gradient against fp64 autograd from t
    ws = {n: p.w(n).clone().requires_grad_(True) for n in temb + [b + ".fc.bias" for b, _, _ in p.blocks]}
    e, _ = emb_ref(t, p.ch)
    x0 = e @ ws["embed.0.weight"].t() + ws["embed.0.bias"]
    x1 = F.silu(x0) @ ws["embed.2.weight"].t() + ws["embed.2.bias"]
    loss = sum((F.silu(x1) @ ws[b + ".fc.weight"].t() + ws[b + ".fc.bias"]).mul(dT[:, off:off + cout]).sum()
               for b, off, cout in p.blocks)
    loss.backward()
    worst = max(rel(p.grad(n), ws[n].grad) for n in temb)
    print(f"[e2e {route} {tag}] dTP -> timestep gradients worst per-tensor rel-L2 {worst:.3e}")
    assert worst <= (1e-2 if tc else 1e-4)


@pytest.mark.parametrize("B", [3, 256])
def test_uniform_route(B):
    p = Probe("cifar10", B, 0, seed=11)
    assert p.has_uni == 1 and p.route == (1 if B in TC_B else 0)
    ti = 999
    t = torch.full((B,), ti, dtype=torch.int64, device=DEV)
    u = p.forward(t, uniform=1)
    assert torch.equal(u["tp"], u["tp"][:1].expand_as(u["tp"])), "uniform: rows of TP differ from row 0"
    ru, bu = check_forward(p, t, u, rows=slice(0, 1), tag=f"B{B} t={ti}", route="uniform")
    # the per-row route of the same plan, same t: agreement within both bounds + the fp64 difference of their inputs
    o = p.forward(t)
    rr, br = check_forward(p, t, o, tag=f"B{B} t={ti} per-row")
    rr0, br0 = rr[:1], br[:1]
    check("uni~row", p.rname, u["tp"][:1], o["tp"][:1].double(), bu + br0 + (ru - rr0).abs() + 1e-30, f"B{B}")


def test_backward_needs_a_per_row_forward():
    """the backward reads every row of emb / e0 / e1: refused before any forward and after a uniform one"""
    p = Probe("tiny", 3, 1, seed=3)
    t = torch.full((3,), 5, dtype=torch.int64, device=DEV)
    dtp = torch.zeros(3, p.tp_ld, device=DEV)
    assert L().ddpm_unet_temb_backward(p.h, dtp.data_ptr(), None, None, None) != 0       # no forward yet
    p.forward(t, uniform=1)
    assert L().ddpm_unet_temb_backward(p.h, dtp.data_ptr(), None, None, None) != 0
    assert b"per-row" in L().ddpm_last_error()
    p.forward(t)
    with torch.no_grad():                    # any other forward of the plan rewrites the rows: refused again
        p.m._forward_nograd(torch.zeros(3, 3, 16, 16, device=DEV), t, training_plan=True)
    assert L().ddpm_unet_temb_backward(p.h, dtp.data_ptr(), None, None, None) != 0
    p.forward(t)
    p.backward(dtp)


def test_routes_agree_b64_vs_b63():
    a, b = Probe("cifar10", 64, 1, seed=5), Probe("cifar10", 63, 1, seed=5)
    assert (a.route, b.route) == (1, 0)
    t = t_rows(64, 5)
    oa, ob = a.forward(t), b.forward(t[:63].contiguous())
    ra, ba = a.tp_ref(oa["e1"][:63]); rb, bb = b.tp_ref(ob["e1"])
    check("tc~simt", "B64~B63", oa["tp"][:63], ob["tp"].double(), ba + bb + (ra - rb).abs() + 1e-30)


def test_repack_reaches_the_tensor_core_projections():
    p = Probe("cifar10", 64, 0, seed=9)
    assert p.route == 1
    t = t_rows(64, 9)
    p.forward(t)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for n, q in p.m.named_parameters():
            if n.startswith("embed.") or ".fc." in n:
                q.data.copy_(torch.randn(q.shape, generator=g).to(DEV) * (0.05 if n.endswith("weight") else 0.5))
    p.m.prepare(64, 32, 32, False, force_repack=True)
    o = p.forward(t)
    check_forward(p, t, o, tag="after repack")
    assert rel(o["tp"], p.tp_from_t(t)) <= 1e-2
