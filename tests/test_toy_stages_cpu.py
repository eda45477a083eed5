"""The toy engine's stage mirror (tests/toy_mirror.py) on the CPU: its own fp32 evaluation of every stage, forward and the whole
backward chain, lies inside the per-element bound the GPU tests hold the kernels to; and the workspace-layout entry
ddpm_toy_ws_layout reports what the launches use and refuses what ddpm_toy_workspace_bytes refuses."""
import ctypes as C

import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200.toy.model import ToyCfg

import toy_mirror as TM
from toy_mirror import F32, F64

WORST = {}


def _inside(name, got, ref):
    """got: plain fp32 tensor; ref: V.  Returns the worst |got - v| / e over elements with e > 0; e = 0 must be exact."""
    d = (got.double() - ref.v).abs()
    assert torch.isfinite(d).all(), name
    e = ref.e
    assert (d <= e).all(), (name, (d - e).max().item())
    r = (d / e.clamp_min(1e-300))[e > 0]
    w = r.max().item() if r.numel() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), w)
    return w


def _run(M, D, L, B, wscale, seed, tmax):
    p = TM.case_params(M, D, wscale, seed)
    x = TM.case_rows(p, B, seed)
    g = torch.Generator().manual_seed(seed + 1)
    t = torch.randint(tmax, (B,), generator=g)
    t[0] = 0
    q64, q32 = TM.params(F64, p), TM.params(F32, p)
    # the forward in fp32: its values are the "saves" both modes then read as exact inputs, as the kernels' stages do
    _, _, _, E32 = TM.temb(F32, q32, t, M)
    _inside("E", E32, TM.temb(F64, q64, t, M)[3])
    h = [TM.in_fc(F32, q32, x, D)]
    _inside("h0", h[0], TM.in_fc(F64, q64, F64.x(x), D))
    u = []
    for l in range(L):
        u.append(TM.layer_u(F32, q32, h[l], E32, M))
        _inside("u", u[l], TM.layer_u(F64, q64, F64.x(h[l]), F64.x(E32), M))
        h.append(TM.layer_h(F32, q32, u[l], h[l], M))
        _inside("h", h[l + 1], TM.layer_h(F64, q64, F64.x(u[l]), F64.x(h[l]), M))
    out = TM.head(F32, q32, h[L], M)
    _inside("out", out, TM.head(F64, q64, F64.x(h[L]), M))
    noise = torch.randn(B, D, generator=g)
    _inside("loss", TM.loss(F32, out, noise, D), TM.loss(F64, F64.x(out), F64.x(noise), D))
    # backward from a given d_out and from the loss seed
    gl = torch.rand(B, generator=g)[:, None] / B
    seed32 = TM.seed_from_g(F32, gl, out, noise, D)
    _inside("seed", seed32, TM.seed_from_g(F64, F64.x(gl), F64.x(out), F64.x(noise), D))
    sv32 = {"h": h, "u": u, "x": x}
    sv64 = {"h": [F64.x(v) for v in h], "u": [F64.x(v) for v in u], "x": F64.x(x)}
    for dout in (seed32, torch.randn(B, D, generator=g)):
        g32, dx32, dE32 = TM.backward(F32, q32, sv32, dout, M, D, L, B)
        g64, dx64, dE64 = TM.backward(F64, q64, sv64, F64.x(dout), M, D, L, B)
        for k in g32:
            _inside(k, g32[k], g64[k])
        _inside("dx", dx32, dx64)
        _inside("dE", dE32, dE64)
        t32 = TM.temb_backward(F32, q32, t, dE32, M, B)
        t64 = TM.temb_backward(F64, q64, t, F64.x(dE32), M, B)
        for k in t32:
            _inside(k, t32[k], t64[k])


@pytest.mark.parametrize("M,D,L,B,wscale,tmax", [(64, 1, 1, 65, 1.0, 1000), (128, 3, 2, 200, 1.0, 1000), (64, 4, 3, 130, 30.0, 1000),
                                                 (128, 2, 3, 96, 1.0, 10001), (64, 3, 2, 300, 30.0, 10001)])
def test_mirror_fp32_inside_bounds(M, D, L, B, wscale, tmax):
    _run(M, D, L, B, wscale, seed=M + D + L + B, tmax=tmax)
    print("\n  worst fp32-mirror error / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))


def test_bf_interval_is_exact_without_error():
    """an exact fp32 value rounds to one bf16 value (no borderline), a value within its error of a midpoint spans two"""
    mid = torch.tensor([1.0 + 2.0 ** -8], dtype=torch.float64)            # halfway between two bf16 neighbours of 1
    assert F64.bf(TM.V(mid)).e.item() == 0.0
    assert F64.bf(TM.V(mid, torch.tensor([2.0 ** -20], dtype=torch.float64))).e.item() == 2.0 ** -7


def test_lrelu_grad_at_zero_takes_the_slope():
    z = TM.V(torch.zeros(3, dtype=torch.float64))
    g = TM.V(torch.ones(3, dtype=torch.float64))
    r = F64.lrelu_grad_mul(g, z)
    assert torch.equal(r.v, torch.full((3,), TM.SLOPE, dtype=torch.float64))
    assert torch.equal(F32.lrelu_grad_mul(torch.ones(3), torch.zeros(3)), torch.full((3,), TM.SLOPE, dtype=torch.float32))
    x = torch.zeros(3, requires_grad=True)                                # torch's own convention
    torch.nn.functional.leaky_relu(x, 0.02).sum().backward()
    assert torch.allclose(x.grad, torch.full((3,), 0.02))


def _layout(cfg, rows, training):
    L = _lib.lib()
    off = (C.c_longlong * 8)()
    slots, P, Pp = C.c_int(-1), C.c_longlong(-1), C.c_longlong(-1)
    rc = L.ddpm_toy_ws_layout(C.byref(ToyCfg(*cfg)), rows, training, C.byref(off), C.byref(slots), C.byref(P), C.byref(Pp))
    return rc, list(off), slots.value, P.value, Pp.value


@pytest.mark.parametrize("cfg", [(1, 64, 1), (3, 128, 2), (4, 64, 3), (2, 128, 3)])
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 8448, 8449, 30000])
def test_ws_layout(cfg, rows):
    L = _lib.lib()
    D, M, Ly = cfg
    for training in (0, 1):
        rc, off, slots, P, Pp = _layout(cfg, rows, training)
        assert rc == 0
        assert off[7] == L.ddpm_toy_workspace_bytes(C.byref(ToyCfg(*cfg)), rows, training)
        assert P == L.ddpm_toy_num_params(C.byref(ToyCfg(*cfg))) and Pp % 64 == 0 and P <= Pp < P + 64
        assert all(o % 256 == 0 for o in off)
        if not training:
            assert off[0] == 0 and slots == 0 and off[7] >= rows * M * 4
            continue
        tiles = (rows + 63) // 64
        assert slots == min(tiles, 132)
        sizes = [rows * M, (Ly + 1) * rows * M, Ly * rows * M, rows * D, rows * D, rows * M, slots * Pp]
        for i, n in enumerate(sizes):                                     # in order, disjoint, each large enough
            assert off[i + 1] - off[i] >= 4 * n, i


def test_ws_layout_refusals():
    L = _lib.lib()
    for cfg, rows, msg in [((2, 96, 3), 10, "mid_features"), ((5, 128, 3), 10, "in_features"), ((0, 128, 3), 10, "in_features"),
                           ((2, 128, 0), 10, "num_temporal_layers"), ((2, 128, 3), 0, "rows"), ((2, 128, 3), (1 << 24) + 1, "rows")]:
        assert _layout(cfg, rows, 1)[0] < 0
        assert msg in L.ddpm_last_error().decode()
        assert L.ddpm_toy_workspace_bytes(C.byref(ToyCfg(*cfg)), rows, 1) < 0
    off = (C.c_longlong * 8)()
    s, P, Pp = C.c_int(), C.c_longlong(), C.c_longlong()
    assert L.ddpm_toy_ws_layout(None, 10, 1, C.byref(off), C.byref(s), C.byref(P), C.byref(Pp)) < 0
    assert L.ddpm_toy_ws_layout(C.byref(ToyCfg(2, 64, 1)), 10, 1, None, C.byref(s), C.byref(P), C.byref(Pp)) < 0
