"""The error model of the bits/dim terms, checked without a GPU, and the argument checks of ``ddpm_bpd_terms_run``.

``bpd_elem`` (csrc/kernels_simt.cuh) repeats, for each element, the fp32 operations of the mirror (``diffusion.py``
``q_posterior_mean_var`` / ``p_mean_var``, ``functions.py`` ``normal_kl`` / ``approx_std_normal_cdf`` /
``discretized_gaussian_loglik``) in the same operand order, each rounded to nearest.  ``ref_and_bound`` below gives the fp64
value of the same formulas and a bound on how far any such fp32 evaluation can lie from it; ``test_bpd_tail_gpu.py``
derives its bounds from it (its docstring has the derivation).  Here the mirror's own CPU evaluation must lie inside that
bound over the adversarial element set the GPU test uses: a bound too tight for the mirror would be wrong before any GPU
run.  Torch's CPU exp / tanh / log are within the 2 / 2 / 1 ulp the bound allows."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24                 # unit roundoff of fp32
EXP_REL = 2.0 ** -22           # 2 ulp of expf / tanhf (CUDA Programming Guide), relative to the result
LOG_REL = 2.0 ** -23           # 1 ulp of logf
TINY = 2.0 ** -149             # absolute error of a product that lands among the subnormals
F32 = np.float32
K1, K2 = float(F32(0.044715)), float(F32(math.sqrt(2.0 / math.pi)))
PREC, TOL, CUT = float(F32(1.0 / 255)), float(F32(1e-12)), float(F32(0.999))
LN2_32 = float(F32(math.log(2.0)))
CAP = -math.log(TOL) * (1 + 2 * LOG_REL)      # |term - ref| can never exceed the range of -log over [tol, 1]
T_STEPS = 1000


def diffusion(var, T=T_STEPS):
    import ddpm_torch_b200 as D
    return D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, T), "eps", var, "mse")


# ------------------------------------------------------------------------------------------------ error propagation
# (value, bound) pairs: value is the exact fp64 result of the operation on exact operands, bound >= |fp32 result - value|
def _mul(a, ea, b, eb):
    v = a * b
    prop = np.abs(a) * eb + np.abs(b) * ea + ea * eb
    return v, prop + U * (np.abs(v) + prop) + TINY


def _add(a, ea, b, eb):
    v = a + b
    prop = ea + eb
    return v, prop + U * (np.abs(v) + prop)


def _exp_err(v):
    """2 ulp of a correctly signed result near v > 0"""
    return EXP_REL * v * (1 + 2.0 ** -20)


def _cdf(z, ez):
    """approx_std_normal_cdf: 0.5 (1 + tanh(K2 (z + K1 z^3))), each op rounded, tanhf within 2 ulp"""
    z2, e2 = _mul(z, ez, z, ez)
    x3, e3 = _mul(z2, e2, z, ez)
    k3, ek3 = _mul(K1, 0.0, x3, e3)
    s, es = _add(z, ez, k3, ek3)
    w, ew = _mul(K2, 0.0, s, es)
    th = np.tanh(w)
    slope = 1.0 / np.cosh(np.clip(np.abs(w) - ew, 0.0, 40.0)) ** 2       # max of tanh' over [w - ew, w + ew]
    eth = slope * ew
    eth = eth + EXP_REL * (np.abs(th) + eth)
    one, eone = _add(1.0, 0.0, th, eth)
    return 0.5 * one, 0.5 * eone


def fp32_chain(row, x0, xt, eps, clip):
    """pred, mm, mt, dm, c and sq as bpd_elem forms them (numpy fp32: one rounding per operation, no contraction)"""
    r = row.astype(F32)
    pred = (r[2] * xt - r[3] * eps).astype(F32)
    if clip:
        pred = np.clip(pred, F32(-1), F32(1))
    mm = (r[4] * pred + r[5] * xt).astype(F32)
    mt = (r[4] * x0 + r[5] * xt).astype(F32)
    e = (pred - x0).astype(F32)
    return dict(pred=pred, mm=mm, dm=(mt - mm).astype(F32), c=(x0 - mm).astype(F32), sq=(e * e).astype(F32))


def ref_and_bound(row, x0, xt, eps, clip):
    """Per element: (term_ref, term_bound, sq_ref, sq_bound, hi - lo) in fp64.
    term_ref is the exact value of the bits/dim term on the fp32 operands bpd_elem shares bit for bit with the mirror
    (d = fp32(true_logvar - model_logvar), dm, lvm for the KL; x0 and mm for the decoder), with the formulas' constants as
    fp32 evaluates them; term_bound bounds |fp32 evaluation - term_ref| for any evaluation with RN operations, expf / tanhf
    within 2 ulp and logf within 1 ulp.  sq_ref = (pred - x0)^2 exactly."""
    x0, xt, eps = (np.asarray(a, dtype=F32) for a in (x0, xt, eps))
    ch = fp32_chain(row, x0, xt, eps, clip)
    r = row.astype(F32).astype(np.float64)
    lvm = r[6]
    e64 = ch["pred"].astype(np.float64) - x0.astype(np.float64)
    sq_ref = e64 * e64
    _, sq_bound = _mul(e64, U * np.abs(e64), e64, U * np.abs(e64))
    if r[8] != 0:                                                  # KL branch, t > 0
        d = float(F32(F32(r[7]) - F32(lvm)))
        dm = ch["dm"].astype(np.float64)
        a, ea = _add(-1.0, 0.0, -d, 0.0)
        sq, esq = _mul(dm, 0.0, dm, 0.0)
        em = math.exp(-lvm)
        p, ep = _mul(sq, esq, em, _exp_err(em))
        s1, es1 = _add(a, ea, p, ep)
        ed = math.exp(d)
        s2, es2 = _add(s1, es1, ed, _exp_err(ed))
        ones = np.ones_like(dm)
        return 0.5 * s2, 0.5 * es2, sq_ref, sq_bound, np.nan * ones
    inv = math.exp(-0.5 * lvm)                                     # fl(0.5 lvm) is exact
    einv = _exp_err(inv)
    xd, mmd = x0.astype(np.float64), ch["mm"].astype(np.float64)
    c, ec = _add(xd, 0.0, -mmd, 0.0)
    cdfs = []
    for s in (1.0, -1.0):
        a, ea = _add(c, ec, s * PREC, 0.0)
        z, ez = _mul(inv, einv, a, ea)
        cdfs.append(_cdf(z, ez))
    (hi, ehi), (lo, elo) = cdfs
    top, bot = x0 > F32(CUT), x0 < F32(-CUT)
    hi, ehi = np.where(top, 1.0, hi), np.where(top, 0.0, ehi)
    lo, elo = np.where(bot, 0.0, lo), np.where(bot, 0.0, elo)
    D, eD = _add(hi, ehi, -lo, elo)
    D2, eD2 = _add(D, eD, -TOL, 0.0)
    v, ev = _add(np.maximum(D2, 0.0), eD2, TOL, 0.0)
    term = -np.log(v)
    et = ev / np.maximum(v - ev, TOL)
    et = et + LOG_REL * (np.abs(term) + et)
    return term, np.minimum(et, CAP), sq_ref, sq_bound, hi - lo


def image_bound(ref, bnd, n_img, n, k, ln2=True):
    """Per image of n elements (groups of n consecutive entries): the reference mean (/ ln 2) and the bound on the kernel's
    fl(fl(S / n) / ln2_f), S its fp32 sum of the n terms with at most k rounded additions on any path."""
    ref, bnd = ref.reshape(n_img, n), bnd.reshape(n_img, n)
    sref = ref.sum(1)
    gam = k * U / (1 - k * U)
    eS = bnd.sum(1) + gam * (np.abs(ref) + bnd).sum(1)
    div = math.log(2.0) if ln2 else 1.0
    q = 3 if ln2 else 2
    out = sref / n / div
    return out, eS / n / div * (1 + (q + 1) * U) + q * U * np.abs(out) * (1 + q * U)


# ------------------------------------------------------------------------------------------------ the element set
def _nearest(v, toward):
    return np.nextafter(F32(v), F32(toward)).astype(F32)


def grid_levels():
    """the 256 levels of 8-bit data as the data pipeline forms them in fp32: (k / 255 - 0.5) / 0.5, +-1 included"""
    return torch.arange(256, dtype=torch.float32).div(255).sub(0.5).div(0.5).numpy()


def elements(diff, ti, clip, n=98304, seed=0):
    """x0, xt, eps (fp32, n elements) for step ti: every 8-bit level and the cutoff neighbours at mean distances that take
    hi - lo from ~0.4 through 1e-3, 1e-8 and the 1e-12 floor to exactly 0 (or dm over the same scale for the KL), pred
    landing exactly on +-1 and one ulp past, and a random bulk (20 % of x0 saturated at +-1, eps = noise + a perturbation)."""
    g = np.random.default_rng(seed + 7919 * ti + 31 * clip)
    row = diff._bpd_rows()[ti].numpy().astype(np.float64)
    sa, s1m, ra, rm1, c1, c2, lvm = (float(row[i]) for i in range(7))
    sig = math.exp(0.5 * lvm)
    lev = grid_levels()
    cut = [F32(CUT), -F32(CUT)]
    edge = np.array(cut + [_nearest(v, w) for v in cut for w in (2.0, -2.0)], dtype=F32)
    ks = np.concatenate([np.linspace(0, 4, 17), [5, 6, 6.5, 7, 7.5, 8, 9, 10, 12, 20]])
    ks = np.concatenate([ks, -ks[1:]])
    xs, ts, es = [], [], []

    def structured(x0):
        """x0 against model means at k sigma from the true mean mt (mt = x0 at t = 0), k over ks"""
        X = np.repeat(x0, len(ks)).astype(F32)
        K = np.tile(ks, len(x0))
        xt = (F32(sa) * X + F32(s1m) * g.standard_normal(len(X)).astype(F32)).astype(F32)
        mt = (F32(c1) * X + F32(c2) * xt).astype(F32).astype(np.float64)
        pred = (mt - K * sig - c2 * xt.astype(np.float64)) / c1
        xs.append(X); ts.append(xt); es.append(((ra * xt.astype(np.float64) - pred) / rm1).astype(F32))

    structured(lev)
    structured(edge)
    # pred exactly on +-1 and one ulp past / inside, walked by ulps of x_t as the sampler-tail test walks them
    for v in (1.0, -1.0, float(_nearest(1, 2)), float(_nearest(-1, -2)), float(_nearest(1, 0)), float(_nearest(-1, 0))):
        for x0 in (1.0, -1.0, 0.0, 0.5, -0.5):
            e = F32(g.standard_normal())
            x = F32((v + F32(rm1) * e) / F32(ra))
            for _ in range(64):
                got = F32(F32(F32(ra) * x) - F32(F32(rm1) * e))
                if got == F32(v):
                    break
                x = np.nextafter(x, F32(np.inf if got < F32(v) else -np.inf))
            xs.append(np.array([x0], F32)); ts.append(np.array([x], F32)); es.append(np.array([e], F32))
    # the random bulk
    m = n - sum(len(a) for a in xs)
    assert m >= n // 4
    X = lev[g.integers(0, 256, m)].astype(np.float64)
    sat = g.random(m) < 0.2
    X[sat] = np.where(g.random(sat.sum()) < 0.5, -1.0, 1.0)
    noise = g.standard_normal(m)
    xt = (F32(sa) * X.astype(F32) + F32(s1m) * noise.astype(F32)).astype(F32)
    pert = np.exp(g.uniform(np.log(1e-4), np.log(3.0), m)) * g.standard_normal(m)
    xs.append(X.astype(F32)); ts.append(xt); es.append((noise + pert).astype(F32))
    out = [np.concatenate(a).astype(F32) for a in (xs, ts, es)]
    for a in out:
        assert a.shape == (n,) and np.isfinite(a).all()
    return out


def mirror(diff, ti, x0, xt, eps, clip):
    """the mirror's fp32 CPU evaluation, per element: (term, sq, pred) through diffusion.py / functions.py"""
    from ddpm_torch_b200.functions import discretized_gaussian_loglik, normal_kl
    x0, xt, eps = (torch.from_numpy(np.ascontiguousarray(a)).view(-1, 1, 1, 1) for a in (x0, xt, eps))
    t = torch.full((x0.shape[0],), ti, dtype=torch.int64)
    true_mean, _, true_logvar = diff.q_posterior_mean_var(x_0=x0, x_t=xt, t=t)
    model_mean, _, model_logvar, pred = diff.p_mean_var(lambda x, t_: eps, xt, t, clip, True)
    if ti > 0:
        term = normal_kl(true_mean, true_logvar, model_mean, model_logvar)
    else:
        term = -discretized_gaussian_loglik(x0, model_mean, log_scale=0.5 * model_logvar)
    return term.flatten().numpy(), (pred - x0).pow(2).flatten().numpy(), pred.flatten().numpy()


STEPS = (0, 1, 2, T_STEPS // 2, T_STEPS - 1)
CASES = [(v, c, t) for v in ("fixed-large", "fixed-small") for c in (False, True) for t in STEPS]


@pytest.mark.parametrize("var,clip,ti", CASES)
def test_mirror_lies_within_the_element_bound(var, clip, ti):
    diff = diffusion(var)
    x0, xt, eps = elements(diff, ti, clip)
    term, sq, pred = mirror(diff, ti, x0, xt, eps, clip)
    row = diff._bpd_rows()[ti].numpy()
    ch = fp32_chain(row, x0, xt, eps, clip)
    assert np.array_equal(pred, ch["pred"]) and np.array_equal(sq, ch["sq"])       # the RN chain is the mirror's, bit for bit
    ref, bnd, sq_ref, sq_bnd, width = ref_and_bound(row, x0, xt, eps, clip)
    r = np.abs(term.astype(np.float64) - ref) / bnd
    assert np.isfinite(r).all() and r.max() <= 1, (var, clip, ti, r.max(), int(r.argmax()))
    assert (np.abs(sq.astype(np.float64) - sq_ref) <= sq_bnd).all()
    if ti == 0:
        wide = width >= 1e-3
        assert wide.mean() > 0.5 and (width < 1e-10).any() and (width == 0).any() and (width > 0.3).any()
        assert (x0 == 1).any() and (x0 == -1).any() and (x0 == F32(CUT)).any()
        print(f"[mirror {var} clip={clip} t=0] worst error / bound: hi - lo >= 1e-3 {r[wide].max():.3f}, "
              f"below {r[~wide].max():.3f}")
    else:
        print(f"[mirror {var} clip={clip} t={ti}] worst error / bound {r.max():.3f}")
    if clip:
        assert (pred == 1).any() and (pred == -1).any()


def test_per_image_bound_covers_the_mirror_means():
    """the mirror's flat_mean over an image (torch's CPU sum, then / n, / ln 2) lies within image_bound's fp64 reference +
    bound when k is the recursive-summation depth n"""
    diff = diffusion("fixed-large")
    for ti in (0, 500):
        x0, xt, eps = elements(diff, ti, True, n=3 * 32 * 32 * 8)
        term, sq, _ = mirror(diff, ti, x0, xt, eps, True)
        ref, bnd, sq_ref, sq_bnd, _ = ref_and_bound(diff._bpd_rows()[ti].numpy(), x0, xt, eps, True)
        n = 3 * 32 * 32
        got = torch.from_numpy(term).view(8, n).mean(1) / math.log(2.0)
        want, b = image_bound(ref, bnd, 8, n, n)
        assert (np.abs(got.double().numpy() - want) <= b).all()
        gm = torch.from_numpy(sq).view(8, n).mean(1)
        want, b = image_bound(sq_ref, sq_bnd, 8, n, n, ln2=False)
        assert (np.abs(gm.double().numpy() - want) <= b).all()


# ------------------------------------------------------------------------------------------------ the C ABI operator
def test_bpd_terms_run_validates_arguments_before_touching_the_device():
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    buf = (C.c_float * 64)()
    a = C.addressof(buf)
    a16 = (a + 15) & ~15
    row = (C.c_float * 10)(*([0.5] * 9 + [3.0]))
    err = lambda: L.ddpm_last_error()

    def run(route=0, src=a16, bias=a16, x0=a16, xt=a16, r=row, B=2, Cc=3, H=4, W=5, T=10, scr=a16, nb=1 << 20, lo=a16, ms=a16):
        return L.ddpm_bpd_terms_run(route, src, bias, x0, xt, r, 1, B, Cc, H, W, T, scr, nb, lo, ms, None)

    assert L.ddpm_bpd_terms_scratch_bytes(2, 4, 5) == 64 + 2 * 1 * 8
    assert L.ddpm_bpd_terms_scratch_bytes(3, 17, 16) == 64 + 3 * 2 * 8
    assert L.ddpm_bpd_terms_scratch_bytes(1, 256, 256) == 64 + 256 * 8
    assert L.ddpm_bpd_terms_scratch_bytes(0, 4, 5) < 0 and b"B, H, W" in err()
    assert L.ddpm_bpd_terms_scratch_bytes(1, 1 << 16, 1 << 16) < 0 and b"too large" in err()
    for route in (-1, 2):
        assert run(route=route) != 0 and b"route must be" in err()
    for route, cc in ((0, 0), (0, 5), (1, 0), (1, 4)):
        assert run(route=route, Cc=cc) != 0 and b"C must be" in err()
    for dims in ((0, 4, 5), (2, 0, 5), (2, 4, 0), (-1, 4, 5)):
        B, H, W = dims
        assert run(B=B, H=H, W=W) != 0 and b"B, H, W" in err()
    assert run(B=1 << 20, H=1 << 12, W=1 << 12) != 0 and b"too large" in err()
    for kw in ("src", "x0", "xt", "r", "scr", "lo", "ms"):
        assert run(**{kw: None}) != 0 and b"null" in err(), kw
    assert run(route=1, bias=None) != 0 and b"null" in err()
    # calls valid up to the scratch size must fail there, on it alone (nothing here is a device buffer)
    assert run(route=0, bias=None, nb=0) != 0 and b"scratch of" in err()  # route 0 reads no bias
    for T in (0, -1, (1 << 24) + 1):
        assert run(T=T) != 0 and b"T must be" in err()
    for ti in (-1.0, 10.0, 2.5, float("nan"), float("inf"), 1e9):
        bad = (C.c_float * 10)(*([0.5] * 9 + [ti]))
        assert run(r=bad) != 0 and b"step index" in err(), ti
    assert run(scr=a16 + 4) != 0 and b"aligned" in err()
    assert run(nb=64 + 2 * 8 - 1) != 0 and b"scratch of" in err()
    big = (C.c_float * 10)(*([0.5] * 9 + [float((1 << 24) - 1)]))           # ti = 2^24 - 1 is a valid index at T = 2^24
    assert run(r=big, T=1 << 24, nb=0) != 0 and b"scratch of" in err()
