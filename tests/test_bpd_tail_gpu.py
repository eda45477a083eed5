"""The bits/dim terms of the engine against an fp64 reference, in both routes the planner takes, with eps pinned.

Kernels (csrc/kernels_simt.cuh): route 0 is ``k_bpd_tail<C>`` over a stored eps (C = 1..4; CUDA-core out_conv plans:
tiny, hid % 64 != 0, small64 at C = 4); route 1 is the bits/dim path of ``k_out_gather<C>`` (C = 1..3; tensor-core out_conv
plans), where eps never reaches memory.  Both call ``bpd_coef`` / ``bpd_elem`` / ``bpd_block_partial``, then
``k_bpd_finalize`` adds the B * ceil(HW / 256) block partials in a fixed order.  ``ddpm_bpd_terms_run`` launches exactly
these kernels, through the launch helpers ``ddpm_bpd_step`` uses, on caller buffers.

Bounds (u = 2^-24; every SIMT operation is round-to-nearest: explicit __fmul_rn / __fadd_rn, no --use_fast_math in
csrc/build.sh, IEEE division).  ``test_bpd_tail_cpu.ref_and_bound`` implements them, and the CPU test checks that the
mirror's own fp32 evaluation lies inside them.
  pred, mm, mt, dm, c, sq, x_t  the same RN fp32 operations as the mirror (diffusion.py / functions.py): bit-identical to it.
  KL (t > 0)   ref = fp64 of 0.5((-1 - d) + dm^2 e^-lvm + e^d) on the fp32 d, dm, lvm.  The only non-RN inputs are
               em = expf(-lvm) and ed = expf(d), 2 ulp each (CUDA Programming Guide); each RN op adds u of its result:
               |term - ref| <= 0.5 (dm^2 em (2u + e_e) + ed e_e + u(|a| + |s1| + |s2|)) to first order, e_e = 2^-22.
               Fixed-small has d = 0 exactly (ed = 1, a = -1).
  decoder (t = 0)   propagated through approx_std_normal_cdf: the RN ops of its argument c +- 1/255 (c = x0 - mm),
               inv_std = expf(-lvm / 2) (2 ulp), x^3, the 0.044715 and sqrt(2/pi) products, tanhf (2 ulp, times the largest
               tanh' over the argument's error interval) and 0.5(1 + .): an absolute error D_hi, D_lo on each side (none on a
               cutoff side: hi = 1 or lo = 0 exactly).  Then
               |term - ref| <= (D_hi + D_lo + u|hi - lo| + the RN of the tol steps) / max(v - e_v, 1e-12) + 1 ulp (logf),
               capped at -ln fp32(1e-12), the whole range of the term.  Elements with tiny hi - lo are ill-conditioned in any
               fp32 evaluation; the worst ratio is reported apart for hi - lo < 1e-3, and most of the sweep lies above.
  per image    loss = fl(fl(S / n) / ln2_f), S the kernel's fp32 sum: C adds per thread, 5 warp levels, 8 warp partials and
               nbi = ceil(HW / 256) block partials, so |S - sum term| <= g_k sum|term|, g_k = ku / (1 - ku), k = C + 13 + nbi;
               plus the sum of the element bounds, plus 3u of the result for the two divisions and fp32 ln 2.  mses the
               same without transcendentals (2u).  At H = W = 1 every other addend is an exact zero, so k = C - 1.

Tests
  a. element sweep at H = W = 1, both routes, every C they take, both variances, both clip settings, t in {0, 1, 2, 500,
     999} of T = 1000: 98 304 elements (every 8-bit level and the +-0.999f cutoff neighbours at model means from 0 to 20
     sigma, pred exactly on +-1 and one ulp past, a random bulk).  mses bit-identical to the mirror's (C = 1) or to its
     per-element squares added in channel order (C > 1); losses within the bound; the routes bit-identical.
  b. reductions: H x W in {7x5, 16x16, 17x15, 24x24, 28x28, 64x64, 256x256}, B in {1, 3, 257}, ~20 % of x0 at +-1; inputs
     are views into NaN-padded buffers (a read past the end poisons the result); outputs NaN-prefilled [B][T] with only
     column ti written (ti = 2^24 - 1 at T = 2^24 included); a second call bit-identical.
  c. calc_all_bpd end to end with out_conv.2.weight = 0 and bias = BETA (eps == BETA exactly on both routes), per-step
     noise given: every [B, T] entry within the per-image bound of fp64 from the mirror's fp32 x_t; tiny and small64
     bit-identical; graph replay, eager and given-noise runs bit-identical; total_bpd within both bounds of the mirror's
     generic loop.
  d. ddpm_device_error_flag() == 0 after every test."""
import math

import numpy as np
import pytest
import torch

from oracle import ddpm_ref as R
import test_bpd_tail_cpu as BC
import test_image_conv_cpu as IC

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32 = np.float32
BETA = torch.tensor([0.3, -0.7, 1.9, -0.2])
WORST = {}


def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k in sorted(WORST):
        print(f"[bpd worst error / bound] {' '.join(map(str, k))}: {WORST[k]:.3f}")


def flag_ok():
    assert L().ddpm_device_error_flag() == 0


def padded(a, pad, fill=float("nan")):
    """a (CPU) copied into the front of a device buffer with `pad` trailing `fill` elements; returns the view"""
    buf = torch.full((a.numel() + pad,), fill, dtype=torch.float32, device=DEV)
    buf[:a.numel()] = a.reshape(-1).to(DEV)
    return buf[:a.numel()].view(a.shape)


def terms_run(route, C, x0, xt, eps, row, ti, T, clip, taps=None, bias=None, out=None):
    """ddpm_bpd_terms_run on [B, C, H, W] fp32 CPU inputs; route 1 takes the tap sums (or, when taps is None, puts eps on the
    centre tap of a NaN tap tensor with zero bias, which is exact at H = W = 1).  Returns losses, mses [B][T] on the device."""
    from ddpm_torch_b200 import _lib
    B, _, H, W = x0.shape
    pad = 256 * C + 64
    dx0, dxt = padded(x0, pad), padded(xt, pad)
    if route == 0:
        src, bptr = padded(eps, pad), None
    else:
        if taps is None:
            assert H == W == 1
            taps = torch.full((B * H * W, 32), float("nan"))
            taps[:, 4 * C:5 * C] = eps.reshape(B, C)
            bias = torch.zeros(C)
        src = padded(taps, (256 + 4 * W) * 32)
        bptr = bias.to(DEV)
    r = torch.cat([row.float(), torch.tensor([float(ti)])])
    nb = L().ddpm_bpd_terms_scratch_bytes(B, H, W)
    assert nb > 0
    scratch = torch.full((nb // 4 + 4,), float("nan"), device=DEV)
    if out is None:
        out = (torch.full((B, T), float("nan"), device=DEV), torch.full((B, T), float("nan"), device=DEV))
    losses, mses = out
    rc = L().ddpm_bpd_terms_run(route, src.data_ptr(), None if bptr is None else bptr.data_ptr(), dx0.data_ptr(), dxt.data_ptr(),
                                r.data_ptr(), int(clip), B, C, H, W, T, scratch.data_ptr(), nb, losses.data_ptr(), mses.data_ptr(),
                                _lib.stream_ptr())
    assert rc == 0, L().ddpm_last_error()
    torch.cuda.synchronize()
    return losses, mses


# ------------------------------------------------------------------------------------------------ a. element sweep
ROUTES = [(0, c) for c in (1, 2, 3, 4)] + [(1, c) for c in (1, 2, 3)]


@pytest.mark.parametrize("var,clip,ti", BC.CASES)
def test_element_sweep(var, clip, ti):
    diff = BC.diffusion(var)
    T = BC.T_STEPS
    row = diff._bpd_rows()[ti]
    x0, xt, eps = BC.elements(diff, ti, clip)
    term, sq, pred = BC.mirror(diff, ti, x0, xt, eps, clip)
    ref, bnd, sq_ref, sq_bnd, width = BC.ref_and_bound(row.numpy(), x0, xt, eps, clip)
    N = len(x0)
    branch = "KL" if ti else "decoder"
    got = {}
    for route, C in ROUTES:
        shape = (N // C, C, 1, 1)
        t = lambda a: torch.from_numpy(a).view(shape)
        losses, mses = terms_run(route, C, t(x0), t(xt), t(eps), row, ti, T, clip)
        others = torch.ones(T, dtype=torch.bool)
        others[ti] = False
        assert torch.isnan(losses[:, others]).all() and torch.isnan(mses[:, others]).all()
        lo, ms = losses[:, ti].cpu().numpy(), mses[:, ti].cpu().numpy()
        got[(route, C)] = (lo, ms)
        # mses: the mirror's squares, added in channel order from 0 (the kernel's per-thread sum), / C
        s = np.zeros(N // C, F32)
        for c in range(C):
            s = (s + sq.reshape(-1, C)[:, c]).astype(F32)
        assert np.array_equal(ms, (s / F32(C)).astype(F32)), f"route {route} C={C}: mses differ from the mirror"
        want, b = BC.image_bound(ref, bnd, N // C, C, C - 1)
        r = np.abs(lo.astype(np.float64) - want) / b
        assert np.isfinite(r).all(), f"route {route} C={C}: non-finite loss"
        if ti == 0 and C == 1:
            wide = width >= 1e-3
            note((f"route{route}", branch, var, "hi-lo>=1e-3"), r[wide].max())
            note((f"route{route}", branch, var, "hi-lo<1e-3"), r[~wide].max())
        else:
            note((f"route{route}", branch, var), r.max())
        assert r.max() <= 1, f"route {route} C={C} {var} clip={clip} t={ti}: worst error / bound {r.max():.3f} at {int(r.argmax())}"
        wm, bm = BC.image_bound(sq_ref, sq_bnd, N // C, C, C - 1, ln2=False)
        assert (np.abs(ms.astype(np.float64) - wm) <= bm).all()
    for C in (1, 2, 3):
        for k in range(2):
            assert np.array_equal(got[(0, C)][k], got[(1, C)][k]), f"C={C}: routes differ"
    assert np.array_equal(got[(0, 1)][1], sq)
    flag_ok()


# ------------------------------------------------------------------------------------------------ b. reductions
def q(a, step=2.0 ** -12):
    return (a / step).round() * step


def reduction_inputs(B, C, H, W, diff, ti, seed):
    """x0 on the 8-bit grid (~20 % at +-1), x_t = the mirror's fp32 q_sample, and eps = a dyadic noise + perturbation spread
    over the in-bounds taps of T (bias + taps add up exactly, so both routes see the same eps)"""
    g = torch.Generator().manual_seed(seed)
    lev = torch.from_numpy(BC.grid_levels())
    x0 = lev[torch.randint(0, 256, (B, C, H, W), generator=g)]
    sat = torch.rand(B, C, H, W, generator=g) < 0.2
    x0 = torch.where(sat, torch.where(torch.rand(B, C, H, W, generator=g) < 0.5, -1.0, 1.0), x0)
    noise = torch.randn(B, C, H, W, generator=g)
    t = torch.full((B,), ti, dtype=torch.int64)
    xt = diff.q_sample(x0, t, noise)
    eps = q(noise + 0.05 * torch.randn(B, C, H, W, generator=g))
    bias = q(0.1 * torch.randn(C, generator=g))
    if 9 * C > 32:                                   # route 0 only: no tap layout holds 4 channels
        return x0, xt, eps, None, None
    taps = torch.full((B, H, W, 32), float("nan"))
    tv = q(torch.randn(B, H, W, 9, C, generator=g) / 3)
    other = torch.zeros(B, H, W, C)
    for tp in range(9):
        if tp == 4:
            continue
        dy, dx = tp // 3 - 1, tp % 3 - 1
        # pixel (y, x) adds tap tp of its neighbour (y + dy, x + dx) when that neighbour is in bounds
        ty, tx = slice(max(-dy, 0), H - max(dy, 0)), slice(max(-dx, 0), W - max(dx, 0))
        sy, sx = slice(max(dy, 0), H + min(dy, 0)), slice(max(dx, 0), W + min(dx, 0))
        other[:, ty, tx] += tv[:, sy, sx, tp]
        taps[..., tp * C:(tp + 1) * C] = tv[..., tp, :]
    centre = eps.permute(0, 2, 3, 1) - bias - other                                 # exact: everything on the 2^-12 grid
    taps[..., 4 * C:5 * C] = centre
    return x0, xt, eps, taps.view(B * H * W, 32), bias


RED = [(B, H, W) for (H, W) in ((7, 5), (16, 16), (17, 15), (24, 24), (28, 28)) for B in (1, 3, 257)] + \
      [(B, 64, 64) for B in (1, 3)] + [(B, 256, 256) for B in (1, 3)]


@pytest.mark.parametrize("B,H,W", RED)
def test_reductions(B, H, W):
    T = BC.T_STEPS
    k = RED.index((B, H, W))
    var, clip, ti = ("fixed-large", "fixed-small")[k % 2], bool(k % 3), (0, 999, 1, 500)[k % 4]
    C = 3
    diff = BC.diffusion(var)
    row = diff._bpd_rows()[ti]
    x0, xt, eps, taps, bias = reduction_inputs(B, C, H, W, diff, ti, seed=k)
    ref, bnd, sq_ref, sq_bnd, _ = BC.ref_and_bound(row.numpy(), x0.numpy().ravel(), xt.numpy().ravel(), eps.numpy().ravel(), clip)
    n = C * H * W
    nbi = -(-H * W // 256)
    want, b = BC.image_bound(ref, bnd, B, n, C + 13 + nbi)
    wm, bm = BC.image_bound(sq_ref, sq_bnd, B, n, C + 13 + nbi, ln2=False)
    res = []
    for route in (0, 1):
        lo, ms = terms_run(route, C, x0, xt, eps, row, ti, T, clip, taps=taps, bias=bias)
        others = torch.ones(T, dtype=torch.bool)
        others[ti] = False
        assert torch.isnan(lo[:, others]).all() and torch.isnan(ms[:, others]).all(), f"route {route}: a column other than {ti} written"
        l_, m_ = lo[:, ti].cpu().double().numpy(), ms[:, ti].cpu().double().numpy()
        r, rm = np.abs(l_ - want) / b, np.abs(m_ - wm) / bm
        assert np.isfinite(r).all() and np.isfinite(rm).all(), f"route {route}: non-finite result"
        note((f"route{route}", "per image", "losses"), r.max())
        note((f"route{route}", "per image", "mses"), rm.max())
        assert r.max() <= 1 and rm.max() <= 1, f"route {route} B={B} {H}x{W}: worst error / bound {r.max():.3f} / {rm.max():.3f}"
        again = terms_run(route, C, x0, xt, eps, row, ti, T, clip, taps=taps, bias=bias)
        assert all(torch.equal(torch.nan_to_num(a, 7.0), torch.nan_to_num(b_, 7.0)) for a, b_ in zip(again, (lo, ms)))
        res.append((lo[:, ti].cpu(), ms[:, ti].cpu()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), "routes differ"
    flag_ok()


@pytest.mark.parametrize("route,C", ROUTES)
def test_last_column_of_the_longest_chain(route, C):
    """ti = 2^24 - 1 at T = 2^24 (the index travels as a float): only that column of NaN-prefilled [2][2^24] outputs"""
    T = 1 << 24
    B, H, W = 2, 17, 15
    diff = BC.diffusion("fixed-large")
    row = diff._bpd_rows()[500]
    x0, xt, eps, taps, bias = reduction_inputs(B, C, H, W, diff, 500, seed=C)
    lo, ms = terms_run(route, C, x0, xt, eps, row, T - 1, T, True, taps=taps, bias=bias)
    assert torch.isfinite(lo[:, T - 1]).all() and torch.isfinite(ms[:, T - 1]).all()
    assert torch.isnan(lo[:, :T - 1]).all() and torch.isnan(ms[:, :T - 1]).all()
    ref = terms_run(route, C, x0, xt, eps, row, 3, 4, True, taps=taps, bias=bias)
    assert torch.equal(ref[0][:, 3], lo[:, T - 1]) and torch.equal(ref[1][:, 3], ms[:, T - 1])
    flag_ok()


# ------------------------------------------------------------------------------------------------ c. end to end, eps pinned
E2E = {
    "tiny": (R.TINY_CFG, 2, 32, 0),
    "small64": (R.SMALL64_CFG, 2, 32, 1),
    "small64_c1": (dict(R.SMALL64_CFG, in_channels=1, out_channels=1), 2, 32, 1),
    "small64_c2": (dict(R.SMALL64_CFG, in_channels=2, out_channels=2), 2, 32, 1),
    "small64_c4": (dict(R.SMALL64_CFG, in_channels=4, out_channels=4), 2, 32, 0),
    "hid96": (IC._cfg(96), 2, 32, 0),
}


def pinned_model(cfg, C):
    import ddpm_torch_b200 as D
    c = R.normalize_cfg(cfg)
    m = D.UNet(c["in_channels"], c["hid_channels"], c["out_channels"], c["ch_multipliers"], c["num_res_blocks"],
               c["apply_attn"], drop_rate=0.0)
    m.load_state_dict(R.make_state_dict(cfg, 3))
    P = dict(m.named_parameters())
    with torch.no_grad():
        P["out_conv.2.weight"].zero_()
        P["out_conv.2.bias"].copy_(BETA[:C])
    return m.to(DEV).eval()


def e2e_reference(diff, x0, noise, clip, C):
    """per-entry fp64 reference and bound of losses / mses [B, T] from the mirror's fp32 x_t and eps = BETA"""
    B, T = x0.shape[0], diff.timesteps
    n = x0[0].numel()
    nbi = -(-x0[0, 0].numel() // 256)
    rows = diff._bpd_rows()
    out = [np.zeros((B, T)) for _ in range(5)]
    beta = BETA[:C].view(1, C, 1, 1).expand_as(x0).contiguous()
    for ti in range(T):
        xt = diff.q_sample(x0, torch.full((B,), ti, dtype=torch.int64), noise[ti])
        ref, bnd, sq_ref, sq_bnd, _ = BC.ref_and_bound(rows[ti].numpy(), x0.numpy().ravel(), xt.numpy().ravel(), beta.numpy().ravel(), clip)
        out[0][:, ti], out[1][:, ti] = BC.image_bound(ref, bnd, B, n, C + 13 + nbi)
        out[2][:, ti], out[3][:, ti] = BC.image_bound(sq_ref, sq_bnd, B, n, C + 13 + nbi, ln2=False)
        out[4][:, ti] = BC.image_bound(ref, bnd, B, n, n)[1]          # the mirror's: torch's flat_mean, at most n - 1 adds deep
    return out


def check_e2e(name, got, refs):
    (lo, ms), (wl, bl, wm, bm) = got, refs[:4]
    r = np.abs(lo.double().numpy() - wl) / bl
    rm = np.abs(ms.double().numpy() - wm) / bm
    note(("e2e", name.split()[0], "losses"), r.max())
    note(("e2e", name.split()[0], "mses"), rm.max())
    assert np.isfinite(r).all() and r.max() <= 1, f"{name}: losses worst error / bound {r.max():.3f}"
    assert np.isfinite(rm).all() and rm.max() <= 1, f"{name}: mses worst error / bound {rm.max():.3f}"


def data(B, C, HW, seed):
    g = torch.Generator().manual_seed(seed)
    lev = torch.from_numpy(BC.grid_levels())
    x0 = lev[torch.randint(0, 256, (B, C, HW, HW), generator=g)]
    sat = torch.rand(B, C, HW, HW, generator=g) < 0.2
    return torch.where(sat, torch.where(torch.rand(B, C, HW, HW, generator=g) < 0.5, -1.0, 1.0), x0)


def routed(name):
    cfg, B, HW, want = E2E[name]
    C = cfg["in_channels"]
    m = pinned_model(cfg, C)
    h = m.prepare(B, HW, HW, False)
    assert IC.layout(L(), h)[2] == want, f"{name}: out_conv route {IC.layout(L(), h)[2]}, expected {want}"
    return m, cfg, B, HW, C


@pytest.mark.parametrize("name", sorted(E2E))
def test_calc_all_bpd_eps_pinned(name):
    m, cfg, B, HW, C = routed(name)
    x0 = data(B, C, HW, 11)
    for var in ("fixed-large", "fixed-small"):
        diff = BC.diffusion(var, T=20)
        noise = torch.randn((20, B, C, HW, HW), generator=torch.Generator().manual_seed(5))
        for clip in (False, True):
            total, losses, prior, mses = diff.calc_all_bpd(m, x0.to(DEV), clip_denoised=clip, noise=noise)
            refs = e2e_reference(diff, x0, noise, clip, C)
            check_e2e(f"{name} {var} clip={clip}", (losses, mses), refs)
            # the mirror's generic loop on the CPU with the same noise: total_bpd within both bounds + the two T-term sums
            pinned = lambda x, t: BETA[:C].view(1, C, 1, 1).expand_as(x).contiguous()
            g_total, g_losses, g_prior, _ = diff.calc_all_bpd(pinned, x0, clip_denoised=clip, noise=noise)
            bt = (refs[1] + refs[4]).sum(1) + 2 * 20 * BC.U * losses.abs().double().sum(1).numpy() \
                + (prior.double() - g_prior.double()).abs().numpy() + 2 * BC.U * total.abs().double().numpy()
            rt = (total.double() - g_total.double()).abs().numpy() / bt
            note(("e2e", "total vs mirror loop"), rt.max())
            assert rt.max() <= 1, f"{name} {var} clip={clip}: total_bpd off the mirror's generic loop by {rt.max():.3f} of the bound"
    flag_ok()


def test_tail_and_gather_bit_identical():
    """tiny (k_bpd_tail) and small64 (fused gather) at the same shape and inputs: pinned eps makes their arithmetic identical"""
    x0 = data(2, 3, 32, 12).to(DEV)
    noise = torch.randn((20, 2, 3, 32, 32), generator=torch.Generator().manual_seed(6))
    outs = {}
    for name in ("tiny", "small64"):
        m = routed(name)[0]
        for var in ("fixed-large", "fixed-small"):
            diff = BC.diffusion(var, T=20)
            for clip in (False, True):
                outs[(name, var, clip)] = diff.calc_all_bpd(m, x0, clip_denoised=clip, noise=noise)
    for var in ("fixed-large", "fixed-small"):
        for clip in (False, True):
            a, b = outs[("tiny", var, clip)], outs[("small64", var, clip)]
            assert torch.equal(a[1], b[1]) and torch.equal(a[3], b[3]) and torch.equal(a[0], b[0]), (var, clip)
    flag_ok()


@pytest.mark.parametrize("name", ["tiny", "small64"])
def test_graph_replay_eager_and_given_noise_bit_identical(name):
    m, cfg, B, HW, C = routed(name)
    x0 = data(B, C, HW, 13).to(DEV)
    diff = BC.diffusion("fixed-large", T=20)
    runs = []
    for use_graph in (True, True, False):
        torch.manual_seed(77)
        runs.append(diff.calc_all_bpd(m, x0, use_graph=use_graph))
    torch.manual_seed(77)
    draws = [torch.randn_like(x0) for _ in range(20)]                      # step k of the loop draws for ti = T - 1 - k
    noise = torch.stack(draws[::-1]).cpu()
    runs.append(diff.calc_all_bpd(m, x0, noise=noise))
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))
    check_e2e(f"{name} graph", (runs[0][1], runs[0][3]), e2e_reference(diff, x0.cpu(), noise, True, C))
    flag_ok()


def test_cifar10_t1000():
    m = pinned_model(R.CIFAR10_CFG, 3)
    h = m.prepare(4, 32, 32, False)
    assert IC.layout(L(), h)[2] == 1
    x0 = data(4, 3, 32, 14)
    diff = BC.diffusion("fixed-large", T=1000)
    noise = torch.randn((1000, 4, 3, 32, 32), generator=torch.Generator().manual_seed(8))
    _, losses, _, mses = diff.calc_all_bpd(m, x0.to(DEV), clip_denoised=True, noise=noise)
    check_e2e("cifar10 T=1000", (losses, mses), e2e_reference(diff, x0, noise, True, 3))
    flag_ok()
