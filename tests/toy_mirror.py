"""Rounding-replicating mirror of the toy engine (csrc/toy_mlp.cuh), stage by stage, with a per-element error bound.

Every function below is written once over an arithmetic ``ar`` and runs in two modes:

* ``F64``: values are ``V(v, e)``.  ``v`` is the fp64 result of the kernel's operation sequence with bf16 rounding (RNE) applied
  exactly where the kernel rounds: the four [M][M] weights, the sinusoidal embedding, lrelu(t_proj), lrelu(LN1) and lrelu(LN2),
  the dh / du tiles of the backward and dE.  ``e`` bounds |kernel fp32 value - v| element by element.
* ``F32``: plain fp32 tensors, the same sequence evaluated on the CPU in fp32 (any summation order, no contraction).  It is one
  more fp32 evaluation of the sequence, so it must lie inside every ``e``; test_toy_stages_cpu.py checks that it does.

Error model (u = 2^-24, the fp32 unit roundoff; bounds are first order plus the second-order cross terms written out):

* RN operation on the CUDA cores (add, sub, mul, the division by D, the multiplication by 0.02f, fmad contractions included: a
  fused a*b + c has one rounding, which the two-rounding bound covers):  e_out = propagated e + u (|v| + propagated e).
* n-term fp32 sum in any order (LayerNorm row sums with quad shuffles, in_fc, out_fc, dx, the column sums):
  e = sum e_i + n u sum(|v_i| + e_i).
* wgmma with fp32 accumulation over n terms (the accumulator's initial value counts as a term):  n 2^-23 S,
  S = sum |a_k||w_k| + |c|.  Weight-gradient partials are summed over the tile's 64 rows by the wgmma, then added into the CTA's
  slot once per owned tile and application and summed over the slots by toy_reduce_kernel: n = 64 + L tiles-per-CTA + slots
  (``n_eff``), with 2^-23 per term for the column sums too.
* bf16 rounding of a value the kernel holds in fp32 with error e:  RNE is monotone, so the kernel's bf16 lies in
  [bf16(fp32(v - e)), bf16(fp32(v + e))] and so does the mirror's.  e_out = hi - lo: 0 unless the interval straddles a bf16
  rounding midpoint (a borderline operand), one bf16 ulp (|w| ulp_bf16 after the GEMM) when it does.
* rsqrtf (LayerNorm, two-pass statistics in fp32): 2 ulp, so relative 2^-22, plus the propagated relative error of var + eps,
  v ((1 - r)^-1/2 - 1) with r = e / (var + eps).
* LeakyReLU is 1-Lipschitz, so its input error passes through (times 0.02 on the negative side); the product by 0.02f rounds.
  Its derivative is 1 for v > 0 and 0.02 otherwise (torch's convention: 0 takes the slope).  Where |v| <= e (e > 0) the kernel may
  take either branch, which costs (1 - 0.02) |g| more.  An exactly-zero input (gamma = beta = 0) has e = 0 and is decided.
* Sinusoidal embedding: k = logf(10000) / (half - 1) (logf 1 ulp, the division u), the argument -(j k) (u), expf (2 ulp), t * that
  (u): relative error 2^-22 + |j k| (2^-23 + 2u) + u of the angle a, so |a| times that in sinf / cosf, plus their 2 ulp
  (2^-22 |value|).  At t = 10^4 this exceeds half a bf16 ulp and most embedding entries are borderline.

Stages (what each kernel computes, in the kernel's order):

* temb:  pre = bf(emb) bf(t_proj)^T (wgmma, n = M) + b; e = bf(lrelu(pre)); E = e bf(enc)^T (n = M) + b_enc.
* in_fc: h0 = x in_fc^T on CUDA cores (n = D + 1).
* LayerNorm: mean = sum(h) / M; a = h - mean; var = sum(a^2) / M; rstd = rsqrtf(var + eps); n = (a rstd) gamma + beta.
* layer: u = E + bf(lrelu(LN1(h))) bf(fc1)^T (wgmma, n = M + 1); h' = h + bf(lrelu(LN2(u))) bf(fc2)^T (n = M + 1).
* head: out = LN_out(h) out_fc^T + b (CUDA cores, n = M + 1); loss = sum_d (noise - out)^2 / D.
* backward (toy_bwd_kernel): seed d_out, or (g 2) (out - noise) / D; head gradients; LayerNorm backward
  dv = rstd (gy - mean(gy) - xh mean(gy xh)) with gy = dy gamma; per application l = L-1 .. 0: fc2 weight gradient
  bf(dh)^T bf(lrelu(LN2(u))), d = bf(dh) bf(fc2) (n = M), times lrelu'(LN2 pre), norm2 sums, LN2 backward -> du, dE += du,
  then the same through fc1 / LN1 from bf(du), and dh += the LN1 backward; in_fc weight gradient and dx on CUDA cores.
* temb backward (toy_temb_bwd_kernel): enc.bias = sum dE; enc.weight = bf(dE)^T e; de = bf(dE) bf(enc) (n = M) times lrelu'(pre);
  t_proj.bias = sum de; t_proj.weight = bf(de)^T bf(emb).
The whole backward chain is this running-error pass: the companion ``e`` is the same linearised backward on absolute values plus
each stage's new rounding terms.  It stays valid across layers, but on absolute values the LayerNorm backward's mean subtraction
cannot cancel, and rstd reaches 1/sqrt(eps) on rows with x = 0, so behind LN1's backward the bound is loose (test_toy_stages_gpu.py
adds a rel-L2 gate for those tensors).
"""
import math

import numpy as np
import torch

U = 2.0 ** -24
F23 = 2.0 ** -23
SLOPE = float(np.float32(0.02))
EPS = float(np.float32(1e-5))
KEYS = ["in_fc.weight", "temp_fc.0.norm1.weight", "temp_fc.0.norm1.bias", "temp_fc.0.fc1.weight", "temp_fc.0.norm2.weight",
        "temp_fc.0.norm2.bias", "temp_fc.0.fc2.weight", "temp_fc.0.enc.weight", "temp_fc.0.enc.bias", "out_norm.weight",
        "out_norm.bias", "out_fc.weight", "out_fc.bias", "t_proj.0.weight", "t_proj.0.bias"]
BF_KEYS = ("temp_fc.0.fc1.weight", "temp_fc.0.fc2.weight", "temp_fc.0.enc.weight", "t_proj.0.weight")
SLOTS_MAX = 132


def n_eff(B, L=1):
    """additions a weight-gradient term goes through: 64 rows in one wgmma or column sum, one slot add per owned tile and per
    application (every application adds into the same slot element), the slot reduce"""
    tiles = (B + 63) // 64
    slots = min(tiles, SLOTS_MAX)
    return 64 + L * ((tiles + slots - 1) // slots) + slots


def _bf(x):
    return x.float().to(torch.bfloat16).double()


class V:
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def __getitem__(self, k):
        return V(self.v[k], self.e[k])


class F64:
    """values with a per-element bound on the kernel's fp32 result"""

    @staticmethod
    def x(t):
        return V(t.double())

    @staticmethod
    def val(a):
        return a.v

    @staticmethod
    def add(a, b):
        v = a.v + b.v
        e = a.e + b.e
        return V(v, e + U * (v.abs() + e))

    @staticmethod
    def sub(a, b):
        v = a.v - b.v
        e = a.e + b.e
        return V(v, e + U * (v.abs() + e))

    @staticmethod
    def mul(a, b):
        v = a.v * b.v
        e = a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e
        return V(v, e + U * (v.abs() + e))

    @staticmethod
    def scale2(a, c):                          # by an exact power of two: no rounding
        return V(a.v * c, a.e * abs(c))

    @staticmethod
    def rowsum(a, n):
        return V(a.v.sum(-1, keepdim=True), a.e.sum(-1, keepdim=True) + n * U * (a.v.abs() + a.e).sum(-1, keepdim=True))

    @staticmethod
    def colsum(a, n):
        return V(a.v.sum(0), a.e.sum(0) + n * F23 * (a.v.abs() + a.e).sum(0))

    @staticmethod
    def rsqrt(a):
        r = a.e / a.v
        assert (r < 0.5).all(), "LayerNorm variance bound too loose"
        v = a.v.rsqrt()
        g = (1 - r) ** -0.5
        return V(v, v * (g - 1) + 2 * F23 * v * g)

    @staticmethod
    def lrelu(a):
        neg = a.v <= 0
        v = torch.where(neg, a.v * SLOPE, a.v)
        cross = a.v.abs() <= a.e
        e = torch.where(cross, a.e, torch.where(neg, SLOPE * a.e, a.e))
        return V(v, e + U * neg * (v.abs() + e))

    @staticmethod
    def lrelu_grad_mul(g, pre):
        neg = pre.v <= 0
        v = torch.where(neg, g.v * SLOPE, g.v)
        unsure = (pre.v.abs() <= pre.e) & (pre.e > 0)
        e = torch.where(unsure, g.e + (1 - SLOPE) * g.v.abs(), torch.where(neg, SLOPE * g.e, g.e))
        return V(v, e + U * (neg | unsure) * (v.abs() + e))

    @staticmethod
    def bf(a):
        lo, hi = _bf(a.v - a.e), _bf(a.v + a.e)
        return V(_bf(a.v), hi - lo)

    @staticmethod
    def mm(A, W, C=None, n=None, unit=F23):
        """A [R][K] @ W[N][K]^T (+ C): wgmma (unit 2^-23) or CUDA-core dot products (unit u)"""
        Aa, Wa = A.v.abs() + A.e, W.v.abs() + W.e
        v = A.v @ W.v.t()
        e = A.e @ W.v.abs().t() + A.v.abs() @ W.e.t() + A.e @ W.e.t()
        S = Aa @ Wa.t()
        if C is not None:
            v = v + C.v
            e = e + C.e
            S = S + C.v.abs() + C.e
        return V(v, e + n * unit * S)

    @staticmethod
    def wgrad(dY, A, n):
        """dY^T A summed over rows: the per-CTA wgmma partials and the slot reduce"""
        v = dY.v.t() @ A.v
        e = dY.e.t() @ A.v.abs() + dY.v.abs().t() @ A.e + dY.e.t() @ A.e
        S = (dY.v.abs() + dY.e).t() @ (A.v.abs() + A.e)
        return V(v, e + n * F23 * S)

    @staticmethod
    def emb(t, M):
        half = M // 2
        K = math.log(10000.0) / (half - 1)
        j = torch.arange(half, dtype=torch.float64, device=t.device)
        tv = t.reshape(-1).double()
        a = torch.outer(tv, torch.exp(-j * K))
        rel = 2 * F23 + (j * K) * (F23 + 2 * U) + U + 4 * U * U
        ea = a.abs() * rel[None]
        s, c = torch.sin(a), torch.cos(a)
        return V(torch.cat([s, c], 1), torch.cat([ea + 2 * F23 * (s.abs() + ea), ea + 2 * F23 * (c.abs() + ea)], 1))


class F32:
    """the same sequence in plain fp32 on whatever device the tensors are on"""

    @staticmethod
    def x(t):
        return t.float()

    @staticmethod
    def val(a):
        return a

    add = staticmethod(lambda a, b: a + b)
    sub = staticmethod(lambda a, b: a - b)
    mul = staticmethod(lambda a, b: a * b)
    scale2 = staticmethod(lambda a, c: a * c)
    rowsum = staticmethod(lambda a, n: a.sum(-1, keepdim=True))
    colsum = staticmethod(lambda a, n: a.sum(0))
    rsqrt = staticmethod(lambda a: a.rsqrt())
    lrelu = staticmethod(lambda a: torch.where(a > 0, a, a * np.float32(SLOPE)))
    lrelu_grad_mul = staticmethod(lambda g, pre: torch.where(pre > 0, g, g * np.float32(SLOPE)))
    bf = staticmethod(lambda a: a.to(torch.bfloat16).float())

    @staticmethod
    def mm(A, W, C=None, n=None, unit=None):
        y = A @ W.t()
        return y if C is None else y + C

    @staticmethod
    def wgrad(dY, A, n):
        return dY.t() @ A

    @staticmethod
    def emb(t, M):
        half = M // 2
        k = torch.log(torch.tensor(10000.0, device=t.device)) / (half - 1)
        j = torch.arange(half, dtype=torch.float32, device=t.device)
        a = t.reshape(-1).float()[:, None] * torch.exp(-(j * k))[None]
        return torch.cat([torch.sin(a), torch.cos(a)], 1)


def params(ar, p):
    """the 15 fp32 parameters as exact inputs; the [M][M] weights also rounded to bf16 (the kernel stages them RNE)"""
    q = {k: ar.x(p[k].detach()) for k in KEYS}
    for k in BF_KEYS:
        q[k + ".bf"] = ar.x(p[k].detach().to(torch.bfloat16).float())
    return q


# ------------------------------------------------------------------------------------------------ forward stages
def ln_xhat(ar, h, M):
    mean = ar.scale2(ar.rowsum(h, M), 1.0 / M)
    a = ar.sub(h, mean)
    var = ar.scale2(ar.rowsum(ar.mul(a, a), M), 1.0 / M)
    rstd = ar.rsqrt(ar.add(var, ar.x(torch.full_like(ar.val(var), EPS))))
    return ar.mul(a, rstd), rstd


def ln_pre(ar, h, g, b, M):
    """(xh, rstd, xh gamma + beta)"""
    xh, rstd = ln_xhat(ar, h, M)
    return xh, rstd, ar.add(ar.mul(xh, g), b)


def temb(ar, q, t, M):
    """(bf(emb), pre, bf(lrelu(pre)), E)"""
    emb = ar.bf(ar.emb(t, M))
    pre = ar.add(ar.mm(emb, q["t_proj.0.weight.bf"], n=M), q["t_proj.0.bias"])
    e = ar.bf(ar.lrelu(pre))
    E = ar.add(ar.mm(e, q["temp_fc.0.enc.weight.bf"], n=M), q["temp_fc.0.enc.bias"])
    return emb, pre, e, E


def in_fc(ar, q, x, D):
    return ar.mm(x, q["in_fc.weight"], n=D + 1, unit=U)


def layer_u(ar, q, h, E, M):
    _, _, pre = ln_pre(ar, h, q["temp_fc.0.norm1.weight"], q["temp_fc.0.norm1.bias"], M)
    return ar.mm(ar.bf(ar.lrelu(pre)), q["temp_fc.0.fc1.weight.bf"], C=E, n=M + 1)


def layer_h(ar, q, u, h, M):
    _, _, pre = ln_pre(ar, u, q["temp_fc.0.norm2.weight"], q["temp_fc.0.norm2.bias"], M)
    return ar.mm(ar.bf(ar.lrelu(pre)), q["temp_fc.0.fc2.weight.bf"], C=h, n=M + 1)


def head(ar, q, h, M):
    _, _, n = ln_pre(ar, h, q["out_norm.weight"], q["out_norm.bias"], M)
    return ar.add(ar.mm(n, q["out_fc.weight"], n=M + 1, unit=U), q["out_fc.bias"])


def loss(ar, out, noise, D):
    d = ar.sub(noise, out)
    s = ar.rowsum(ar.mul(d, d), D)
    return _div(ar, s, D)


def _div(ar, s, D):
    if ar is F32:
        return s / D
    v = s.v / D
    e = s.e / D
    return V(v, e + U * (v.abs() + e))


# ------------------------------------------------------------------------------------------------ backward
def seed_from_g(ar, g, out, noise, D):
    """d_out = (g 2) (out - noise) / D, per element"""
    return _div(ar, ar.mul(ar.scale2(g, 2.0), ar.sub(out, noise)), D)


def ln_bwd(ar, gy, xh, rstd, M):
    a = ar.scale2(ar.rowsum(gy, M), 1.0 / M)
    b = ar.scale2(ar.rowsum(ar.mul(gy, xh), M), 1.0 / M)
    return ar.mul(rstd, ar.sub(ar.sub(gy, a), ar.mul(xh, b)))


def backward(ar, q, sv, dout, M, D, L, B):
    """the whole toy_bwd_kernel teacher-forced on the saved forward: sv = {"h": [L+1] exact, "u": [L] exact, "x": exact}.
    Returns the gradients by KEYS name (without enc / t_proj), dx and dE."""
    n = n_eff(B, L)
    gr = {}
    xh, rstd, nrm = ln_pre(ar, sv["h"][L], q["out_norm.weight"], q["out_norm.bias"], M)
    gr["out_fc.weight"] = ar.wgrad(dout, nrm, n)
    gr["out_fc.bias"] = ar.colsum(dout, n)
    dn = ar.mm(dout, _t(ar, q["out_fc.weight"]), n=D + 1, unit=U)
    gr["out_norm.weight"] = ar.colsum(ar.mul(dn, xh), n)
    gr["out_norm.bias"] = ar.colsum(dn, n)
    dh = ln_bwd(ar, ar.mul(dn, q["out_norm.weight"]), xh, rstd, M)
    dE = None
    for k in ("temp_fc.0.fc1.weight", "temp_fc.0.fc2.weight", "temp_fc.0.norm1.weight", "temp_fc.0.norm1.bias",
              "temp_fc.0.norm2.weight", "temp_fc.0.norm2.bias"):
        gr[k] = None
    for l in range(L - 1, -1, -1):
        for (inp, gk, bk, wk) in (("u", "temp_fc.0.norm2.weight", "temp_fc.0.norm2.bias", "temp_fc.0.fc2.weight"),
                                  ("h", "temp_fc.0.norm1.weight", "temp_fc.0.norm1.bias", "temp_fc.0.fc1.weight")):
            xh, rstd, pre = ln_pre(ar, sv[inp][l], q[gk], q[bk], M)
            ta = ar.bf(dh if inp == "u" else du)
            gr[wk] = _acc(ar, gr[wk], ar.wgrad(ta, ar.bf(ar.lrelu(pre)), n))
            d = ar.lrelu_grad_mul(ar.mm(ta, _t(ar, q[wk + ".bf"]), n=M), pre)
            gr[gk] = _acc(ar, gr[gk], ar.colsum(ar.mul(d, xh), n))
            gr[bk] = _acc(ar, gr[bk], ar.colsum(d, n))
            d = ln_bwd(ar, ar.mul(d, q[gk]), xh, rstd, M)
            if inp == "u":
                du = d
                dE = du if dE is None else ar.add(dE, du)
            else:
                dh = ar.add(dh, d)
    x = sv["x"]
    gr["in_fc.weight"] = ar.wgrad(dh, x, n + 1)
    dx = ar.mm(dh, _t(ar, q["in_fc.weight"]), n=M + 1, unit=U)
    return gr, dx, dE


def temb_backward(ar, q, t, dE, M, B):
    """toy_temb_bwd_kernel on a given dE"""
    n = n_eff(B)
    emb, pre, e, _ = temb(ar, q, t, M)
    gr = {"temp_fc.0.enc.bias": ar.colsum(dE, n)}
    td = ar.bf(dE)
    gr["temp_fc.0.enc.weight"] = ar.wgrad(td, e, n)
    de = ar.lrelu_grad_mul(ar.mm(td, _t(ar, q["temp_fc.0.enc.weight.bf"]), n=M), pre)
    gr["t_proj.0.bias"] = ar.colsum(de, n)
    gr["t_proj.0.weight"] = ar.wgrad(ar.bf(de), emb, n)
    return gr


def _t(ar, w):
    return V(w.v.t(), w.e.t()) if isinstance(w, V) else w.t()


def _acc(ar, acc, x):
    """sum over the applications: the kernel adds every application's tile partial into the same slot element, and n_eff(B, L)
    already counts those adds, so the bounds add without a rounding term"""
    if acc is None:
        return x
    return acc + x if ar is F32 else V(acc.v + x.v, acc.e + x.e)


# ------------------------------------------------------------------------------------------------ test inputs
def case_params(M, D, wscale=1.0, seed=0, device="cpu"):
    """xavier-like weights (times wscale), LayerNorm affine and biases perturbed, and two columns of norm1 / norm2 with gamma =
    beta = 0, so those LeakyReLU inputs are exactly 0"""
    g = torch.Generator().manual_seed(seed)
    uni = lambda o, i: (torch.rand(o, i, generator=g) * 2 - 1) * math.sqrt(6.0 / (o + i)) * wscale
    rn = lambda *s: 0.1 * torch.randn(*s, generator=g)
    p = {"in_fc.weight": uni(M, D), "temp_fc.0.norm1.weight": 1 + rn(M), "temp_fc.0.norm1.bias": rn(M),
         "temp_fc.0.fc1.weight": uni(M, M), "temp_fc.0.norm2.weight": 1 + rn(M), "temp_fc.0.norm2.bias": rn(M),
         "temp_fc.0.fc2.weight": uni(M, M), "temp_fc.0.enc.weight": uni(M, M), "temp_fc.0.enc.bias": rn(M),
         "out_norm.weight": 1 + rn(M), "out_norm.bias": rn(M), "out_fc.weight": uni(D, M), "out_fc.bias": rn(D),
         "t_proj.0.weight": uni(M, M), "t_proj.0.bias": rn(M)}
    for k in ("temp_fc.0.norm1", "temp_fc.0.norm2"):
        for c in (3, M - 5):
            p[k + ".weight"][c] = 0.0
            p[k + ".bias"][c] = 0.0
    return {k: p[k].float().contiguous().to(device) for k in KEYS}


def case_rows(p, B, seed=0, device="cpu"):
    """x [B][D]: random rows, and (B >= 8) rows with x = 0, rows scaled so LayerNorm-1's variance of in_fc(x) is 1e-5, and rows with
    |x| ~ 10^3"""
    W = p["in_fc.weight"].double().cpu()
    D = W.shape[1]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, generator=g, dtype=torch.float64)
    if B >= 8:
        x[0] = 0.0
        x[B // 2] = 0.0
        for r in (1, B - 2, B // 3):
            x[r] *= math.sqrt(1e-5 / (x[r] @ W.t()).var(unbiased=False).item())
        for r in (2, B - 1):
            x[r] *= 1e3
    return x.float().to(device)
