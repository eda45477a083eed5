"""The toy engine (csrc/toy_mlp.cuh) stage by stage against the rounding-replicating fp64 mirror (tests/toy_mirror.py), each
kernel on the engine's own input to it, read from the workspace through ddpm_toy_ws_layout:

* forward (ddpm_toy_train_forward): x_t bit-identical to torch's fp32 q_sample; E from t; h0 from the saved x_t; u_l from the
  saved h_l and E, h_{l+1} from the saved u_l and h_l, for every application; out from the saved h_L; the per-row loss from the
  saved out.  ddpm_toy_forward's out is bit-identical at training 0 and 1 and to the saved out at the same x_t.
* backward (ddpm_toy_train_backward from g, ddpm_toy_backward from d_out with dx): every gradient, dx and dE against the mirror's
  backward teacher-forced on the saved forward, whose bound is the running-error companion pass (toy_mirror's docstring); enc.* and
  t_proj.* also from the engine's own dE; grad bit-identical to the fp32 sum of the partial slots in slot order.
* sampler (ddpm_toy_sample): with the row (0, -1, 1, 0, sigma, flag) a step returns eps (+ sigma z) exactly, so S = 1 and S = 5
  chains are bit-identical to chained forwards; one real step is bit-identical to the fp32 update on the forward's eps.

Every workspace and output is NaN-prefilled, so an unwritten element or a read of an unwritten save shows.  Cases cover
mid 64 / 128, in 1..4, 1..3 applications, B from 1 to 30 000 (8449 and up: backward CTAs owning two or more tiles, 16 897 and up:
forward CTAs owning two), t in {0, 1, T-1, random, up to 10^4}, rows with x = 0, with LayerNorm variance ~1e-5 and with |x| ~ 10^3,
gamma = beta = 0 columns (LeakyReLU inputs exactly 0) and weights x1 and x30."""
import ctypes as C

import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import toy as T
from ddpm_torch_b200.toy.model import ToyCfg, ToyParams

import toy_mirror as TM
from toy_mirror import F64, KEYS

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
WORST = {}
REL, BREL = {}, {}
# The running-error bound stays tight through the head and one LayerNorm backward (out_*, and at L = 1 fc2.weight, norm2.* and dE),
# but the absolute-value pass cannot cancel the LayerNorm backward's mean subtraction, and rows with x = 0 or variance ~1e-5 have
# rstd up to 1/sqrt(eps) = 316: behind LN1's backward, and behind LN2's at L >= 2, the element bound exceeds the values themselves.
# These tensors keep the element bound and also pass a per-tensor rel-L2 gate against the teacher-forced mirror.  The gate is the
# single-layer derivation: the element bounds of fc2.weight and dE at L = 1 are 3.2e-3 and 4.0e-3 in rel-L2 (mid 128, weights x1),
# rounded down to 2^-8.  enc.* and t_proj.* are held to their one-stage element bound from the engine's own dE instead.
FALLBACK = ("in_fc.weight", "temp_fc.0.norm1.weight", "temp_fc.0.norm1.bias", "temp_fc.0.fc1.weight", "temp_fc.0.norm2.weight",
            "temp_fc.0.norm2.bias", "temp_fc.0.fc2.weight", "dE", "dx")
GATE = 2.0 ** -8
T_SCHED = 10001


def _check(name, got, ref, gate=None):
    got = got.double().reshape(ref.v.shape)
    d = (got - ref.v).abs()
    assert torch.isfinite(got).all(), f"{name}: non-finite (unwritten?)"
    bad = d > ref.e
    assert not bad.any(), f"{name}: {int(bad.sum())} elements outside the bound, worst excess {(d - ref.e).max().item():.3e}"
    r = d / ref.e.clamp_min(1e-300)
    w = r[ref.e > 0].max().item() if (ref.e > 0).any() else 0.0
    assert torch.equal(d[ref.e == 0], torch.zeros_like(d[ref.e == 0])), name
    WORST[name] = max(WORST.get(name, 0.0), w)
    nv = ref.v.norm().clamp_min(1e-300)
    rl = (d.norm() / nv).item()
    REL[name] = max(REL.get(name, 0.0), rl)
    BREL[name] = max(BREL.get(name, 0.0), (ref.e.norm() / nv).item())
    if gate is not None:
        assert rl <= gate, f"{name}: rel-L2 {rl:.3e} against the teacher-forced mirror, gate {gate:.3e}"


def _layout(cfg, rows, training):
    off = (C.c_longlong * 8)()
    slots, P, Pp = C.c_int(), C.c_longlong(), C.c_longlong()
    _lib.check(_lib.lib().ddpm_toy_ws_layout(C.byref(cfg), rows, training, C.byref(off), C.byref(slots), C.byref(P), C.byref(Pp)),
               "toy_ws_layout")
    return [o // 4 for o in off], slots.value, P.value, Pp.value


def _nan(*shape):
    return torch.full(shape, NAN, dtype=torch.float32, device=DEV)


def _sched():
    b = torch.linspace(1e-4, 0.02, T_SCHED, dtype=torch.float64)
    ab = torch.cumprod(1 - b, 0)
    return ab.sqrt().float().to(DEV), (1 - ab).sqrt().float().to(DEV)


def _t(B, kind, g):
    if kind == "big":
        t = torch.randint(T_SCHED, (B,), generator=g)
        t[: min(B, 2)] = torch.tensor([10000, 9999])[: min(B, 2)]
        return t.to(DEV)
    if kind == "random":
        t = torch.randint(1000, (B,), generator=g)
        t[: min(B, 3)] = torch.tensor([0, 1, 999])[: min(B, 3)]
        return t.to(DEV)
    return torch.full((B,), {"0": 0, "1": 1, "T-1": 999}[kind], dtype=torch.int64, device=DEV)


class Toy:
    def __init__(self, M, D, L, p):
        self.M, self.D, self.L = M, D, L
        self.cfg = ToyCfg(D, M, L)
        self.p = p
        self.prm = ToyParams(*[p[k].data_ptr() for k in KEYS])
        self.lib = _lib.lib()

    def ws(self, rows, training):
        off, slots, P, Pp = _layout(self.cfg, rows, training)
        return _nan(off[7]), off, slots, P, Pp

    def views(self, ws, off, B, slots, Pp):
        M, D, L = self.M, self.D, self.L
        s = lambda i, n: ws[off[i]:off[i] + n]
        return {"E": s(0, B * M).view(B, M), "h": s(1, (L + 1) * B * M).view(L + 1, B, M), "u": s(2, L * B * M).view(L, B, M),
                "x": s(3, B * D).view(B, D), "out": s(4, B * D).view(B, D), "dE": s(5, B * M).view(B, M),
                "part": s(6, slots * Pp).view(slots, Pp)}

    def train_forward(self, x0, t, noise, sa, s1a, ws):
        B = x0.shape[0]
        losses = _nan(B)
        _lib.check(self.lib.ddpm_toy_train_forward(C.byref(self.cfg), C.byref(self.prm), x0.data_ptr(), t.data_ptr(), noise.data_ptr(),
                                                   sa.data_ptr(), s1a.data_ptr(), B, losses.data_ptr(), ws.data_ptr(), ws.numel() * 4,
                                                   None), "train_forward")
        return losses

    def forward(self, x, t, training):
        B = x.shape[0]
        ws = self.ws(B, training)[0]
        out = _nan(B, self.D)
        _lib.check(self.lib.ddpm_toy_forward(C.byref(self.cfg), C.byref(self.prm), x.data_ptr(), t.data_ptr(), B, out.data_ptr(),
                                             training, ws.data_ptr(), ws.numel() * 4, None), "forward")
        return out

    def train_backward(self, t, noise, g, ws, P):
        grad = _nan(P)
        _lib.check(self.lib.ddpm_toy_train_backward(C.byref(self.cfg), C.byref(self.prm), t.data_ptr(), noise.data_ptr(), g.data_ptr(),
                                                    t.numel(), grad.data_ptr(), ws.data_ptr(), ws.numel() * 4, None), "train_backward")
        return grad

    def backward(self, t, d_out, ws, P):
        grad, dx = _nan(P), _nan(*d_out.shape)
        _lib.check(self.lib.ddpm_toy_backward(C.byref(self.cfg), C.byref(self.prm), t.data_ptr(), d_out.data_ptr(), t.numel(),
                                              dx.data_ptr(), grad.data_ptr(), ws.data_ptr(), ws.numel() * 4, None), "backward")
        return grad, dx

    def split(self, grad):
        out, o = {}, 0
        for k in KEYS:
            n = self.p[k].numel()
            out[k] = grad[o:o + n].view_as(self.p[k])
            o += n
        return out


CASES = [  # M, D, L, B, weight scale, t
    (64, 1, 1, 1, 1.0, "0"), (128, 3, 2, 63, 1.0, "T-1"), (64, 3, 3, 64, 30.0, "random"), (128, 2, 1, 65, 1.0, "1"),
    (128, 4, 3, 1000, 1.0, "big"), (64, 2, 2, 8448, 1.0, "random"), (128, 3, 2, 8449, 1.0, "random"),
    (64, 4, 1, 16896, 30.0, "random"), (128, 1, 3, 16897, 1.0, "big"), (128, 3, 3, 30000, 1.0, "random"),
    (64, 3, 2, 30000, 30.0, "random"), (128, 2, 2, 8449, 30.0, "big")]


@pytest.mark.parametrize("M,D,L,B,ws_,tk", CASES)
def test_training_stages(M, D, L, B, ws_, tk):
    seed = M * 7 + D * 5 + L * 3 + B
    p = TM.case_params(M, D, ws_, seed, DEV)
    toy = Toy(M, D, L, p)
    q = TM.params(F64, p)
    g = torch.Generator().manual_seed(seed)
    x0 = TM.case_rows(p, B, seed, DEV)
    noise = torch.randn(B, D, generator=g).to(DEV)
    if B >= 8:                                 # the special rows keep their character through q_sample
        for r in (0, B // 2, 1, B - 2, B // 3, 2, B - 1):
            noise[r] = x0[r]
    t = _t(B, tk, g)
    sa, s1a = _sched()
    ws, off, slots, P, Pp = toy.ws(B, 1)
    losses = toy.train_forward(x0, t, noise, sa, s1a, ws)
    torch.cuda.synchronize()
    sv = {k: v.clone() for k, v in toy.views(ws, off, B, slots, Pp).items() if k in ("E", "h", "u", "x", "out")}

    # ---- forward, each stage on its saved input
    assert torch.equal(sv["x"], sa[t][:, None] * x0 + s1a[t][:, None] * noise)
    _check("E", sv["E"], TM.temb(F64, q, t, M)[3])
    _check("h0", sv["h"][0], TM.in_fc(F64, q, F64.x(sv["x"]), D))
    for l in range(L):
        _check("u", sv["u"][l], TM.layer_u(F64, q, F64.x(sv["h"][l]), F64.x(sv["E"]), M))
        _check("h", sv["h"][l + 1], TM.layer_h(F64, q, F64.x(sv["u"][l]), F64.x(sv["h"][l]), M))
    _check("out", sv["out"], TM.head(F64, q, F64.x(sv["h"][L]), M))
    _check("loss", losses, TM.loss(F64, F64.x(sv["out"]), F64.x(noise), D))
    out1 = toy.forward(sv["x"], t, 1)
    out0 = toy.forward(sv["x"], t, 0)
    assert torch.equal(out1, sv["out"]) and torch.equal(out0, sv["out"])

    # ---- backward from the loss gradient g: the seed 2 g (out - noise) / D, then the chain
    gl = torch.rand(B, generator=g).to(DEV) / B
    sv64 = {"h": [F64.x(v) for v in sv["h"]], "u": [F64.x(v) for v in sv["u"]], "x": F64.x(sv["x"])}
    seed64 = TM.seed_from_g(F64, F64.x(gl[:, None]), F64.x(sv["out"]), F64.x(noise), D)
    V = toy.views(ws, off, B, slots, Pp)
    grads = []
    for rep in range(2 if B >= 8449 else 1):
        V["dE"].fill_(NAN)
        V["part"].fill_(NAN)
        grads.append(toy.train_backward(t, noise, gl, ws, P))
    torch.cuda.synchronize()
    if len(grads) == 2:
        assert torch.equal(grads[0], grads[1])
        assert torch.equal(toy.train_forward(x0, t, noise, sa, s1a, toy.ws(B, 1)[0]), losses)
    _check_backward(toy, q, sv64, seed64, t, grads[0], V, slots, P, "g")

    # ---- backward from a given d_out, with dx
    d_out = torch.randn(B, D, generator=g).to(DEV)
    V["dE"].fill_(NAN)
    V["part"].fill_(NAN)
    grad, dx = toy.backward(t, d_out, ws, P)
    torch.cuda.synchronize()
    dx64 = _check_backward(toy, q, sv64, F64.x(d_out), t, grad, V, slots, P, "d_out")
    _check("dx", dx, dx64, GATE)


def _check_backward(toy, q, sv64, dout, t, grad, V, slots, P, tag):
    M, D, L, B = toy.M, toy.D, toy.L, t.numel()
    # toy_reduce_kernel and the slot accounting: grad is the fp32 sum of the slots in slot order
    part = V["part"].clone()
    s = torch.zeros(P, dtype=torch.float32, device=DEV)
    for k in range(slots):
        s = s + part[k, :P]
    assert torch.equal(grad, s), tag
    gr64, dx64, dE64 = TM.backward(F64, q, sv64, dout, M, D, L, B)
    got = toy.split(grad)
    for k, r in gr64.items():
        _check(k, got[k], r, GATE if k in FALLBACK else None)
    dE = V["dE"].clone()
    _check("dE", dE, dE64, GATE)
    tb = TM.temb_backward(F64, q, t, F64.x(dE), M, B)                 # one stage: from the engine's own dE
    for k, r in tb.items():
        _check(k + " (from dE)", got[k], r)
    tb = TM.temb_backward(F64, q, t, dE64, M, B)                      # the whole chain
    for k, r in tb.items():
        _check(k, got[k], r)
    return dx64


def test_zz_report_worst_ratios():
    if WORST:
        print("\n  worst kernel error / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))
        print("\n  worst rel-L2 kernel vs mirror / bound rel-L2: " + ", ".join(f"{k} {REL[k]:.2e}/{BREL[k]:.1e}" for k in sorted(REL)))


# ------------------------------------------------------------------------------------------------ sampler
def _sample(toy, x, coef, z):
    S = coef.shape[0]
    ws = toy.ws(S, 0)[0]
    _lib.check(toy.lib.ddpm_toy_sample(C.byref(toy.cfg), C.byref(toy.prm), x.data_ptr(), x.shape[0], S, coef.data_ptr(),
                                       z.data_ptr(), ws.data_ptr(), ws.numel() * 4, None), "sample")
    return x


@pytest.mark.parametrize("M,D,L,B", [(64, 1, 1, 65), (128, 3, 2, 1000), (128, 2, 3, 16897), (64, 4, 2, 30000)])
def test_sampler_eps_rows_chain_forwards(M, D, L, B):
    p = TM.case_params(M, D, 1.0, B, DEV)
    toy = Toy(M, D, L, p)
    g = torch.Generator().manual_seed(B)
    x = TM.case_rows(p, B, B, DEV)
    # S = 1: the row (0, -1, 1, 0, sigma, 0) returns eps = forward(x, t = 0)
    coef = torch.tensor([[0.0, -1.0, 1.0, 0.0, 0.7, 0.0]], device=DEV)
    got = _sample(toy, x.clone(), coef, torch.randn(1, B, D, generator=g).to(DEV))
    assert torch.equal(got, toy.forward(x, torch.zeros(B, dtype=torch.int64, device=DEV), 0))
    # S = 5 with the flag on: x <- forward(x, t) + sigma_t z[k] at t = 4 .. 0, so the per-step E row and z[k] are both pinned
    S = 5
    sig = torch.tensor([0.3, 0.55, 1.25, 0.01, 2.0], device=DEV)
    coef = torch.zeros(S, 6, device=DEV)
    coef[:, 1], coef[:, 2], coef[:, 4], coef[:, 5] = -1.0, 1.0, sig, 1.0
    z = torch.randn(S, B, D, generator=g).to(DEV)
    got = _sample(toy, x.clone(), coef, z)
    ref = x.clone()
    for k in range(S):
        ti = S - 1 - k
        ref = toy.forward(ref, torch.full((B,), ti, dtype=torch.int64, device=DEV), 0) + sig[ti] * z[k]
    assert torch.equal(got, ref)


@pytest.mark.parametrize("M,D,L,B", [(128, 2, 3, 30000), (64, 3, 1, 777)])
def test_sampler_real_step_exact(M, D, L, B):
    p = TM.case_params(M, D, 1.0, 5 + B, DEV)
    toy = Toy(M, D, L, p)
    d = T.GaussianDiffusion(T.get_beta_schedule("linear", 0.001, 0.2, 100), "eps", "fixed-large", "mse")
    coef = d._toy_coef_rows(DEV)
    g = torch.Generator().manual_seed(1)
    x = 2 * torch.randn(B, D, generator=g).to(DEV)
    for ti in (99, 50, 1, 0):
        # one real step at t = ti: a table of ti + 1 rows whose lower rows are the identity update (coef2 = 1, the rest 0)
        tab = torch.zeros(ti + 1, 6, device=DEV)
        tab[:, 3] = 1.0
        tab[ti] = coef[ti]
        z = torch.zeros(ti + 1, B, D, device=DEV)
        z[0] = torch.randn(B, D, generator=g).to(DEV)
        got = _sample(toy, x.clone(), tab, z)
        eps = toy.forward(x, torch.full((B,), ti, dtype=torch.int64, device=DEV), 0)
        ra, rb, c1, c2, sg, nz = coef[ti]
        x0 = ra * x - rb * eps
        mean = c1 * x0 + c2 * x
        ref = mean + (nz * sg) * z[0]
        assert torch.equal(got, ref), ti
