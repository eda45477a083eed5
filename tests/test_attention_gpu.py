"""The attention core softmax(Q K^T / sqrt(C)) V of AttentionBlock (unet.py:43-51) and its backward, route by route, against fp64
torch on the same bf16 q, k, v and dO, through the C ABI operators that run the launch steps the engine's plans run (same kernels,
same grids):
  1  fused     attn_kernel<false>; backward attn_kernel<true> + dV / dK products               T = 256, C = 256
  2  t16       k_attn16_fwd / k_attn16_bwd                                                   T = 16, C in {128, 256, 512}
  3  products  Q.K^T -> k_softmax_rows -> P.V; backward dP, dV, k_softmax_bwd, dQ, dK          any shape; the products run on the
               tensor cores for a power-of-two T % 128 == 0 with C % 64 == 0 ("products[tc]"), on CUDA cores otherwise ("[simt]")
Every case runs every route its shape is eligible for.  Outputs are filled with NaN before each call, so that an element that is
never written fails, and the device error flag is read after each call.  Each test prints its worst error-to-bound ratio under -s.

Error bounds (u = 2^-8, one bf16 rounding; all terms are worst-case, per element, computed in fp64 from the exact scores s):
  scores   a score is an fp32 sum of C bf16 products, in an order the kernel chooses and, on the tensor cores, without a guarantee of
           round-to-nearest: |ds_ij| <= E_ij = C 2^-23 scale sum_c |q_ic||k_jc|.  The stored / max-subtracted score and the exp
           argument add (|s_ij| + |m_i|) 2^-23, where m_i is the row maximum.
  exp      __expf(x) is within (2 + 1.16|x|) ulp of e^x (CUDA programming guide, fast intrinsics); ex2.approx.ftz is within 2 ulp:
           (4 + 1.16|s_ij - m_i|) 2^-24 relative covers both.
  softmax  with A_ij the sum of the two terms above (an absolute error of the exponent, i.e. a relative error of e^s), P_ij = e^s_ij /
           sum_k e^s_ik moves by at most A_ij + sum_k P_ik A_ik relative; the fp32 row sum of T terms, the reciprocal and the product
           add (T + 8) 2^-24.  kappa_ij = A_ij + sum_k P_ik A_ik + (T + 8) 2^-24.
  fused    the fused kernel rounds e to bf16 before it sums and multiplies (the P.V product sees exactly those values), so its P
           carries two more roundings: kappa + 2u(1 + u).
  P        |P^ - P| <= (u + (1 + u) kappa) P + 1e-37   (the absolute floor is the fp32 / bf16 flush-to-zero range of exp)
  out      |o^ - o| <= u|o| + (1 + u) sum_j (u + kappa_ij + T 2^-23) P_ij |v_jc|, the last term being the fp32 accumulation over T
  dS       with P the saved bf16 probabilities: dP = dO V^T (fp32 over C: C 2^-23 sum_c |dO_ic||v_jc| = e_ij), D_i = sum_j P_ij dP_ij
           (e_D = sum_j P_ij e_ij + T 2^-23 sum_j P_ij |dP_ij|), dS = P (dP - D) / sqrt(C):
           |dS^ - dS| <= u|dS| + (1 + u)(P scale (e_ij + e_D + 2^-23 (|dP| + |D|)) + 2^-22 |dS|) + 1e-36
  dQ/dK/dV |dQ^ - dQ| <= u|dQ| + (1 + u)(sum_j b(dS)_ij |k_jc| + T 2^-23 sum_j |dS_ij||k_jc|), dK alike over i with q;
           |dV^ - dV| <= u|dV| + (1 + u) T 2^-23 sum_i P_ij |dO_ic|   (dV reads exactly the saved P and dO)
Chains (forward route with probs -> backward route on those probs) are compared with fp64 autograd of exact softmax attention on
typical inputs: rel-L2 of out and of each third of d_qkv <= 1e-2 and per-token cosine >= 0.999 (stated bounds: the saved bf16 P
alone contributes ~u / sqrt(T) relative)."""
import ctypes as ct
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -8
F23 = 2.0 ** -23
F24 = 2.0 ** -24
P_FLOOR = 1e-37
FUSED, T16, PRODUCTS = 1, 2, 3
CHAIN_REL, CHAIN_COS = 1e-2, 0.999


def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _check(rc):
    from ddpm_torch_b200 import _lib
    _lib.check(rc, "attention operator")


def _stream():
    from ddpm_torch_b200 import _lib
    return _lib.stream_ptr()


def _p(t):
    return t.data_ptr() if t is not None else None


def _flag_ok():
    assert L().ddpm_device_error_flag() == 0


def routes(T, C):
    r = [PRODUCTS]
    if T == 16 and C in (128, 256, 512):
        r.insert(0, T16)
    if T == 256 and C == 256:
        r.insert(0, FUSED)
    return r


def route_name(route, T, C):
    if route == PRODUCTS:
        tc = T % 128 == 0 and C % 64 == 0 and (T & (T - 1)) == 0
        return "products[tc]" if tc else "products[simt]"
    return {FUSED: "fused", T16: "t16"}[route]


# ------------------------------------------------------------------------------------------------ operators
def _scratch(route, NB, T, C, backward):
    n = L().ddpm_attn_scratch_bytes(route, NB, T, C, backward)
    assert n >= 0, L().ddpm_last_error()
    return torch.full((n,), 0xFF, dtype=torch.uint8, device=DEV) if n else None


def attn_fwd(route, qkv, probs=True):
    from ddpm_torch_b200 import _lib
    NB, T, C3 = qkv.shape
    C = C3 // 3
    out = torch.full((NB, T, C), float("nan"), dtype=torch.bfloat16, device=DEV)
    P = torch.full((NB, T, T), float("nan"), dtype=torch.bfloat16, device=DEV) if probs or route == PRODUCTS else None
    scratch = _scratch(route, NB, T, C, 0)
    d = _lib.AttnDesc()
    d.route, d.NB, d.T, d.C = route, NB, T, C
    d.qkv, d.out, d.probs, d.scratch = _p(qkv), _p(out), _p(P), _p(scratch)
    _check(L().ddpm_attention_fwd_run(ct.byref(d), _stream()))
    torch.cuda.synchronize()
    _flag_ok()
    return out, P


def attn_bwd(route, qkv, dO, P):
    from ddpm_torch_b200 import _lib
    NB, T, C3 = qkv.shape
    C = C3 // 3
    dqkv = torch.full((NB, T, C3), float("nan"), dtype=torch.bfloat16, device=DEV)
    dS = torch.full((NB, T, T), float("nan"), dtype=torch.bfloat16, device=DEV) if route != T16 else None
    scratch = _scratch(route, NB, T, C, 1)
    d = _lib.AttnBwdDesc()
    d.route, d.NB, d.T, d.C = route, NB, T, C
    d.qkv, d.d_out, d.probs, d.d_qkv, d.d_scores, d.scratch = _p(qkv), _p(dO), _p(P), _p(dqkv), _p(dS), _p(scratch)
    _check(L().ddpm_attention_bwd_run(ct.byref(d), _stream()))
    torch.cuda.synchronize()
    _flag_ok()
    return dqkv, dS


# ------------------------------------------------------------------------------------------------ inputs
def make_qkv(NB, T, C, kind, seed):
    """bf16 [NB][T][3C].  typical: N(0, 1).  peaked: every row's scaled scores spread over 30-80 (nearly one-hot rows); every 4th
    query is a multiple of key 0, which key 1 duplicates, so its two largest scores tie.  flat: all keys identical (P = 1/T, out =
    the mean of v).  vbig / vsmall: v x 1e3 / x 1e-3."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q, k, v = (torch.randn(NB, T, C, device=DEV, generator=g, dtype=torch.float64) for _ in range(3))
    if kind == "peaked":
        s = torch.einsum("btc,bsc->bts", q, k) / math.sqrt(C)
        spread = s.amax(-1) - s.amin(-1)
        target = 30 + 50 * torch.rand(NB, T, device=DEV, generator=g, dtype=torch.float64)
        q = q * (target / spread)[..., None]
        if T >= 4:
            k[:, 1] = k[:, 0]
            beta = 50.0 / (math.sqrt(C) + 3.0)
            q[:, ::4] = beta * k[:, 0:1]
    elif kind == "flat":
        k[:] = k[:, :1]
    elif kind == "vbig":
        v = v * 1e3
    elif kind == "vsmall":
        v = v * 1e-3
    else:
        assert kind == "typical", kind
    return torch.cat([q, k, v], -1).to(torch.bfloat16).contiguous()


def offset_pair(NB, T, C, seed):
    """(qkv with a large constant added to every score of a row, its twin without): channel 0 of every key is A and channel 0 of
    query i is 0 (twin) or +-b (offset rows), so row i's scores move by +-A b / sqrt(C) = +-120 with the rest of each dot product
    unchanged.  The offset pushes e^s out of the fp32 range, so only a max-subtracted softmax gets it right."""
    base = make_qkv(NB, T, C, "typical", seed).double()
    A = 16.0
    b = float(torch.tensor(120.0 * math.sqrt(C) / A).to(torch.bfloat16))
    base[..., C] = A
    base[..., 0] = 0.0
    twin = base.clone()
    sign = torch.tensor([1.0, -1.0, 0.0], device=DEV, dtype=torch.float64).repeat(T // 3 + 1)[:T]
    base[..., 0] = b * sign
    return base.to(torch.bfloat16).contiguous(), twin.to(torch.bfloat16).contiguous()


def make_dO(NB, T, C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(NB, T, C, device=DEV, generator=g).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ fp64 reference and bounds
def ref_forward(qkv):
    q, k, v = qkv.double().chunk(3, -1)
    T, C = q.shape[1], q.shape[2]
    scale = 1.0 / math.sqrt(C)
    s = torch.einsum("btc,bsc->bts", q, k) * scale
    m = s.amax(-1, keepdim=True)
    P = torch.softmax(s, -1)
    o = P @ v
    E = C * F23 * scale * torch.einsum("btc,bsc->bts", q.abs(), k.abs())
    A = E + (s.abs() + m.abs()) * F23 + (4 + 1.16 * (s - m).abs()) * F24
    kappa = A + (P * A).sum(-1, keepdim=True) + (T + 8) * F24
    return dict(P=P, o=o, v=v, kappa=kappa, T=T)


def fwd_bounds(ref, route):
    kap = ref["kappa"] + (2 * U * (1 + U) if route == FUSED else 0.0)
    P, T = ref["P"], ref["T"]
    bP = (U + (1 + U) * kap) * P + P_FLOOR
    bo = U * ref["o"].abs() + (1 + U) * (((U + kap + T * F23 + F23) * P) @ ref["v"].abs()) + 1e-30
    return bP, bo


def ref_backward(qkv, dO, Pb):
    q, k, v = qkv.double().chunk(3, -1)
    T, C = q.shape[1], q.shape[2]
    scale = 1.0 / math.sqrt(C)
    g, P = dO.double(), Pb.double()
    dP = torch.einsum("btc,bsc->bts", g, v)
    D = (P * dP).sum(-1, keepdim=True)
    dS = P * (dP - D) * scale
    dQ = dS @ k
    dK = dS.transpose(1, 2) @ q
    dV = P.transpose(1, 2) @ g
    e = C * F23 * torch.einsum("btc,bsc->bts", g.abs(), v.abs())
    eD = (P * e).sum(-1, keepdim=True) + T * F23 * (P * dP.abs()).sum(-1, keepdim=True)
    bS = U * dS.abs() + (1 + U) * (P * scale * (e + eD + F23 * (dP.abs() + D.abs())) + 2 * F23 * dS.abs()) + 1e-36
    aS = dS.abs()
    bQ = U * dQ.abs() + (1 + U) * (bS @ k.abs() + T * F23 * (aS @ k.abs())) + 1e-30
    bK = U * dK.abs() + (1 + U) * (bS.transpose(1, 2) @ q.abs() + T * F23 * (aS.transpose(1, 2) @ q.abs())) + 1e-30
    bV = U * dV.abs() + (1 + U) * T * F23 * (P.transpose(1, 2) @ g.abs()) + 1e-30
    return dict(dS=dS, bS=bS, d=torch.cat([dQ, dK, dV], -1), b=torch.cat([bQ, bK, bV], -1))


def ratio(got, ref, bound):
    err = (got.double() - ref).abs()
    assert not torch.isnan(got).any(), "an element was never written (NaN)"
    return (err / bound).max().item()


def rel_l2(a, b):
    return ((a.double() - b).norm() / b.norm()).item()


def min_row_cos(a, b):
    return torch.nn.functional.cosine_similarity(a.double().flatten(0, -2), b.flatten(0, -2), dim=-1).min().item()


# ------------------------------------------------------------------------------------------------ cases
SHAPES = [(16, 64), (16, 96), (16, 128), (16, 256), (16, 512), (64, 64), (64, 256), (64, 512), (256, 128), (256, 256), (256, 512),
          (1024, 128)]
CASES = [(NB, T, C) for T, C in SHAPES for NB in ((1, 2) if T == 1024 else (1, 3))] + [(128, 16, 256), (128, 256, 256)]
IDS = [f"T{T}_C{C}_NB{NB}" for NB, T, C in CASES]
TWO_ROUTE = [c for c in CASES if len(routes(c[1], c[2])) > 1]
TWO_ROUTE_IDS = [f"T{T}_C{C}_NB{NB}" for NB, T, C in TWO_ROUTE]


def _seed(NB, T, C):
    return NB * 1000003 + T * 1009 + C


@pytest.mark.parametrize("NB,T,C", CASES, ids=IDS)
def test_forward(NB, T, C):
    """P element by element (a row normalised by the wrong sum, or a wrong scale, fails here) and the output element by element."""
    worst = {}
    for kind in ("typical", "peaked", "vbig", "vsmall"):
        qkv = make_qkv(NB, T, C, kind, _seed(NB, T, C))
        ref = ref_forward(qkv)
        for route in routes(T, C):
            out, P = attn_fwd(route, qkv)
            bP, bo = fwd_bounds(ref, route)
            rp, ro = ratio(P, ref["P"], bP), ratio(out, ref["o"], bo)
            nm = route_name(route, T, C)
            worst[nm] = max(worst.get(nm, (0, 0))[0], rp), max(worst.get(nm, (0, 0))[1], ro)
            assert rp <= 1.0, (kind, nm, "P", rp)
            assert ro <= 1.0, (kind, nm, "out", ro)
            if route != PRODUCTS:           # routes 1 and 2 write P only when asked; the product is the same either way
                out2, _ = attn_fwd(route, qkv, probs=False)
                assert torch.equal(out, out2), (kind, nm)
    print(f"\n[attention fwd T={T} C={C} NB={NB}] worst error/bound " +
          "  ".join(f"{k}: P {a:.3f} out {b:.3f}" for k, (a, b) in worst.items()))


@pytest.mark.parametrize("NB,T,C", CASES, ids=IDS)
def test_invariances(NB, T, C):
    """Offset rows (+-120 added to every scaled score of a row) give the P of their un-offset twin, and identical keys give exactly
    uniform P (1/T is a power of two: exact up to the one final rounding) and the mean of v."""
    worst = 0.0
    qoff, qtwin = offset_pair(NB, T, C, _seed(NB, T, C) + 1)
    ref_off, ref_twin = ref_forward(qoff), ref_forward(qtwin)
    assert torch.allclose(ref_off["P"], ref_twin["P"], rtol=1e-9, atol=1e-300)     # the offset is a row constant: same softmax
    flat = make_qkv(NB, T, C, "flat", _seed(NB, T, C) + 2)
    ref_flat = ref_forward(flat)
    for route in routes(T, C):
        nm = route_name(route, T, C)
        out_o, P_o = attn_fwd(route, qoff)
        out_t, P_t = attn_fwd(route, qtwin)
        bP_o, bo_o = fwd_bounds(ref_off, route)
        bP_t, _ = fwd_bounds(ref_twin, route)
        r = max(ratio(P_o, ref_off["P"], bP_o), ratio(out_o, ref_off["o"], bo_o),
                ((P_o.double() - P_t.double()).abs() / (bP_o + bP_t)).max().item())
        assert r <= 1.0, (nm, "offset", r)
        worst = max(worst, r)
        out_f, P_f = attn_fwd(route, flat)
        rf = ((P_f.double() - 1.0 / T).abs() / (U / T)).max().item()
        assert rf <= 1.0, (nm, "flat P", rf)
        _, bo_f = fwd_bounds(ref_flat, route)
        mean_v = flat.double()[..., 2 * C:].mean(1, keepdim=True).expand(-1, T, -1)
        assert torch.allclose(ref_flat["o"], mean_v, rtol=1e-12, atol=1e-12)
        rf = max(rf, ratio(out_f, mean_v, bo_f))
        assert rf <= 1.0, (nm, "flat out", rf)
        worst = max(worst, rf)
    print(f"\n[attention invariances T={T} C={C} NB={NB}] worst error/bound {worst:.3f}")


@pytest.mark.parametrize("NB,T,C", CASES, ids=IDS)
def test_backward(NB, T, C):
    """The backward kernels alone, from the saved bf16 P: dS (where the route writes it) and every third of d_qkv, element by
    element.  dO = 0 gives d_qkv = 0 exactly."""
    worst = {}
    dO = make_dO(NB, T, C, _seed(NB, T, C) + 3)
    for kind in ("typical", "peaked", "vbig"):
        qkv = make_qkv(NB, T, C, kind, _seed(NB, T, C) + 4)
        Pb = ref_forward(qkv)["P"].to(torch.bfloat16)
        ref = ref_backward(qkv, dO, Pb)
        for route in routes(T, C):
            nm = route_name(route, T, C)
            dqkv, dS = attn_bwd(route, qkv, dO, Pb)
            r = [ratio(dqkv[..., i * C:(i + 1) * C], ref["d"][..., i * C:(i + 1) * C], ref["b"][..., i * C:(i + 1) * C]) for i in range(3)]
            if dS is not None:
                r.append(ratio(dS, ref["dS"], ref["bS"]))
            old = worst.get(nm, [0.0] * len(r))
            worst[nm] = [max(a, b) for a, b in zip(old, r)]
            assert max(r) <= 1.0, (kind, nm, r)
    qkv = make_qkv(NB, T, C, "typical", _seed(NB, T, C) + 5)
    Pb = ref_forward(qkv)["P"].to(torch.bfloat16)
    for route in routes(T, C):
        dqkv, dS = attn_bwd(route, qkv, torch.zeros_like(dO), Pb)
        assert torch.count_nonzero(dqkv) == 0, route_name(route, T, C)
        assert dS is None or torch.count_nonzero(dS) == 0
    print(f"\n[attention bwd T={T} C={C} NB={NB}] worst error/bound " +
          "  ".join(f"{k}: dQ {v[0]:.3f} dK {v[1]:.3f} dV {v[2]:.3f}" + (f" dS {v[3]:.3f}" if len(v) > 3 else "") for k, v in worst.items()))


@pytest.mark.parametrize("NB,T,C", CASES, ids=IDS)
def test_chain(NB, T, C):
    """Each eligible forward route with probs, then each eligible backward route on those probs (fused forward -> products backward
    is the benchmarked training step; fused -> fused the opt-in one), against fp64 autograd of exact softmax attention."""
    qkv = make_qkv(NB, T, C, "typical", _seed(NB, T, C) + 6)
    dO = make_dO(NB, T, C, _seed(NB, T, C) + 7)
    x = qkv.double().requires_grad_(True)
    q, k, v = x.chunk(3, -1)
    o = torch.softmax(torch.einsum("btc,bsc->bts", q, k) / math.sqrt(C), -1) @ v
    (g,) = torch.autograd.grad(o, x, dO.double())
    o = o.detach()
    worst_rel, worst_cos = 0.0, 1.0
    for fr in routes(T, C):
        out, P = attn_fwd(fr, qkv)
        rel, cos = rel_l2(out, o), min_row_cos(out, o)
        for br in routes(T, C):
            dqkv, _ = attn_bwd(br, qkv, dO, P)
            for i in range(3):
                rel = max(rel, rel_l2(dqkv[..., i * C:(i + 1) * C], g[..., i * C:(i + 1) * C]))
                cos = min(cos, min_row_cos(dqkv[..., i * C:(i + 1) * C], g[..., i * C:(i + 1) * C]))
            assert rel <= CHAIN_REL and cos >= CHAIN_COS, (route_name(fr, T, C), route_name(br, T, C), rel, cos)
        worst_rel, worst_cos = max(worst_rel, rel), min(worst_cos, cos)
    print(f"\n[attention chain T={T} C={C} NB={NB}] worst rel-L2 {worst_rel:.3e} (bound {CHAIN_REL:.0e}, ratio "
          f"{worst_rel / CHAIN_REL:.3f})  worst per-token cosine {worst_cos:.6f} (bound {CHAIN_COS})")


@pytest.mark.parametrize("NB,T,C", TWO_ROUTE, ids=TWO_ROUTE_IDS)
def test_route_agreement(NB, T, C):
    """t16 vs products on CUDA cores at T = 16, fused vs products on the tensor cores at T = C = 256: P, out, dS and d_qkv agree
    within the sum of the two routes' bounds."""
    a, b = routes(T, C)
    worst = 0.0
    for kind in ("typical", "peaked"):
        qkv = make_qkv(NB, T, C, kind, _seed(NB, T, C) + 8)
        ref = ref_forward(qkv)
        (oa, Pa), (ob, Pb_) = attn_fwd(a, qkv), attn_fwd(b, qkv)
        (bPa, boa), (bPb, bob) = fwd_bounds(ref, a), fwd_bounds(ref, b)
        worst = max(worst, ((Pa.double() - Pb_.double()).abs() / (bPa + bPb)).max().item(),
                    ((oa.double() - ob.double()).abs() / (boa + bob)).max().item())
        dO = make_dO(NB, T, C, _seed(NB, T, C) + 9)
        P = ref["P"].to(torch.bfloat16)
        rb = ref_backward(qkv, dO, P)
        (ga, sa), (gb, sb) = attn_bwd(a, qkv, dO, P), attn_bwd(b, qkv, dO, P)
        for t in (Pa, oa, Pb_, ob, ga, gb, sa, sb):
            assert t is None or not torch.isnan(t).any(), (kind, "an element was never written (NaN)")
        worst = max(worst, ((ga.double() - gb.double()).abs() / (2 * rb["b"])).max().item())
        if sa is not None:
            worst = max(worst, ((sa.double() - sb.double()).abs() / (2 * rb["bS"])).max().item())
        assert worst <= 1.0, (kind, worst)
    print(f"\n[attention routes {route_name(a, T, C)} vs {route_name(b, T, C)} T={T} C={C} NB={NB}] worst difference / bound sum {worst:.3f}")
