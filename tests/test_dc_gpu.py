"""Density and coverage on the engine (ddpm_knn_count and ddpm_knn_kth with kk = 1, csrc/knn.cuh; ``calc_dc``) against the recipe
they implement, on an H100.

Recipe (on the fp16 features as stored; X real [N], Y generated [M], r the real radii):
  d2[j, i] = max(0, |Y_j|^2 + |X_i|^2 - 2 <Y_j, X_i>);  d = fp16_rn(sqrt_rn(d2));
  count[j] = #{i : d(Y_j, X_i) < r_i};  nearest[i] = min_j d(X_i, Y_j);  covered[i] = nearest[i] < r_i;
  density = sum_j count[j] / (k M);  coverage = #covered / N.

Exact mode: integer features in [-3, 3], so every d2 is an integer below 2^21 and fp32 accumulation in any order is exact; the
engine must reproduce the recipe (fp64, then fp32 sqrt and fp16 on the CPU, which is correctly rounded) bit for bit.

Random mode: VGG-like fp16 features at D = 4096.  With the accumulation model of tests/test_pr_gpu.py (u = 2^-24), every engine
d2 of a pair lies within E = (3 D + 3) u (|a|^2 + |b|^2) of the exact one, whichever set is the rows.  A pair's decision is forced
where it survives that perturbation: inside if fp16(sqrt(d2 + E)) < r, outside if fp16(sqrt(max(0, d2 - E))) >= r (each with a
2^-10 margin for the double rounding of the fp64 bound).  So count[j] lies in [lo_j, hi_j] = [#forced inside, #not forced
outside], coverage is forced on a real row where some pair is forced inside or every pair is forced outside, and density and
coverage lie in the intervals those imply.
"""
import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
U = 2.0 ** -24
SENTINEL = -12345


def d2_exact(a, b):
    a, b = a.to(DEV, torch.float64), b.to(DEV, torch.float64)
    return ((a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2.0 * (a @ b.T)).clamp_min(0.0)


def fp16_sqrt(d2):
    return d2.float().cpu().sqrt().half()


def abi_count(p, s, r):
    """ddpm_knn_count on DEV: counts start as a sentinel and the scratch as 0xAB, so anything left unwritten shows."""
    L = _lib.lib()
    n, m, D = p.shape[0], s.shape[0], p.shape[1]
    A, B = M._device_rows(p, DEV), M._device_rows(s, DEV)
    nbytes = L.ddpm_knn_count_scratch_bytes(n, m, D)
    _lib.check(nbytes if nbytes < 0 else 0, "count_scratch_bytes")
    scratch = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device=DEV)
    out = torch.full((n,), SENTINEL, dtype=torch.int32, device=DEV)
    rr = r.to(DEV, torch.float16).contiguous()
    _lib.check(L.ddpm_knn_count(A.data_ptr(), n, A.stride(0), B.data_ptr(), m, B.stride(0), D, rr.data_ptr(), out.data_ptr(),
                                scratch.data_ptr(), nbytes, _lib.stream_ptr(DEV)), "knn_count")
    torch.cuda.synchronize()
    assert L.ddpm_device_error_flag() == 0
    out = out.cpu()
    assert ((out >= 0) & (out <= m)).all()
    return out


def abi_nearest(a, b):
    """ddpm_knn_kth with kk = 1: the fp16 distance from each row of a to its nearest row of b; outputs start as NaN."""
    L = _lib.lib()
    n, m, D = a.shape[0], b.shape[0], a.shape[1]
    A, B = M._device_rows(a, DEV), M._device_rows(b, DEV)
    nbytes = L.ddpm_knn_scratch_bytes(n, m, D, 1)
    scratch = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device=DEV)
    out = torch.full((n,), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(L.ddpm_knn_kth(A.data_ptr(), n, A.stride(0), B.data_ptr(), m, B.stride(0), D, 1, out.data_ptr(),
                              scratch.data_ptr(), nbytes, _lib.stream_ptr(DEV)), "knn_kth")
    torch.cuda.synchronize()
    assert L.ddpm_device_error_flag() == 0
    out = out.cpu()
    assert not torch.isnan(out).any()
    return out


def recipe(y, x, r, block=1024):
    """(counts [M], nearest [N]) of the recipe, fp64 d2 on DEV, then fp32 sqrt and fp16 on the CPU."""
    rf = r.float()
    counts, near = [], torch.full((x.shape[0],), float("inf"), dtype=torch.float64, device=DEV)
    for i in range(0, y.shape[0], block):
        d2 = d2_exact(y[i:i + block], x)
        counts.append((fp16_sqrt(d2).float() < rf[None, :]).sum(1).int())
        near = torch.minimum(near, d2.min(0).values)
    return torch.cat(counts), fp16_sqrt(near)


def int_features(n, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-3, 4, (n, D), generator=g).half()


def bits(t):
    return t.view(torch.int16)


def exact_radii(x, y, seed):
    """Real radii: the k-th neighbour within x (many ties at exactly r), some placed exactly on an achieved real-to-generated
    distance, and 0, negative, +inf and NaN ones."""
    n = x.shape[0]
    r = recipe_kth(x, min(4, n))
    g = torch.Generator().manual_seed(seed)
    sel = torch.rand(n, generator=g)
    pick = y[torch.randint(0, y.shape[0], (n,), generator=g)]
    on = fp16_sqrt(((x.double() - pick.double()) ** 2).sum(1))          # exact for integer features
    r = torch.where(sel < 0.3, on, r)
    r[(sel >= 0.3) & (sel < 0.38)] = 0.0
    r[(sel >= 0.38) & (sel < 0.43)] = -1.0
    r[(sel >= 0.43) & (sel < 0.46)] = float("inf")
    r[(sel >= 0.46) & (sel < 0.49)] = float("nan")
    return r


def recipe_kth(x, kk, block=2048):
    return torch.cat([fp16_sqrt(d2_exact(x[i:i + block], x).kthvalue(kk, dim=1).values) for i in range(0, x.shape[0], block)])


# (M generated, N real, D)
EXACT = [
    (1, 1, 3), (1, 4099, 8), (4099, 1, 64), (127, 127, 100), (128, 129, 520), (129, 128, 4096), (1000, 1000, 64),
    (127, 4099, 3), (4099, 127, 520), (1000, 129, 4096), (129, 1000, 8), (4099, 4099, 100), (128, 1, 3), (1, 128, 4096),
    (200, 60000, 64),         # few row tiles, many columns: the column split of the count pass
    (60000, 200, 64),         # ... and of the kk = 1 pass
]


@pytest.mark.parametrize("m,n,D", EXACT)
def test_exact(m, n, D):
    x = int_features(n, D, 1000 + n + D)
    y = int_features(m, D, 2000 + m + D)
    y[: min(n, m) // 3] = x[: min(n, m) // 3]                          # generated points sitting on real ones
    r = exact_radii(x, y, n + m)
    want_c, want_n = recipe(y, x, r)
    got_c = abi_count(y, x, r)
    got_n = abi_nearest(x, y)
    assert torch.equal(got_c, want_c)
    assert torch.equal(bits(got_n), bits(want_n))
    assert torch.equal(abi_count(y, x, r), got_c) and torch.equal(bits(abi_nearest(x, y)), bits(got_n))   # repeatable
    k = 3
    dens, cov = M.calc_dc(y, (x, r), k, DEV)
    assert dens == int(want_c.long().sum()) / (k * m)
    assert cov == int((want_n.float() < r.float()).sum()) / n
    assert (dens, cov) == M.calc_dc(y, (x, r), k, "cpu")


def test_counts_on_all_edges_of_the_strict_compare():
    x = int_features(1, 100, 5).repeat(300, 1)                         # 300 identical real points: radius 0
    r0 = recipe_kth(x, 4)
    assert (r0 == 0).all()
    assert (abi_count(x, x, r0) == 0).all()
    y = x.clone(); y[:, 0] += 1                                         # every generated point at distance exactly 1
    assert (abi_count(y, x, torch.ones(300)) == 0).all()              # on the radius: not inside
    assert (abi_count(y, x, torch.full((300,), 1.0009765625)) == 300).all()     # the next fp16 above 1
    assert (abi_count(y, x, torch.full((300,), float("inf"))) == 300).all()
    assert (abi_count(y, x, torch.full((300,), float("nan"))) == 0).all()
    assert M.calc_dc(y, (x, torch.ones(300)), 1, DEV) == (0.0, 0.0)
    assert M.calc_dc(y, (x, torch.full((300,), 2.0)), 2, DEV) == (150.0, 1.0)   # density far above 1


def vgg_like(n, W, shift, g):
    z = torch.randn(n, W.shape[0], generator=g, device=DEV) * (1 + shift) + shift
    return torch.relu(z @ W / 4).half()


def forced(y, x, r, block=1024):
    """Per generated row (lo, hi) counts and per real row (must_cover, must_not_cover), from fp64 distances moved by -+E."""
    D = x.shape[1]
    ny = (y.to(DEV, torch.float64) ** 2).sum(1)
    nx = (x.to(DEV, torch.float64) ** 2).sum(1)
    rf = r.to(DEV).float()
    lo, hi = [], []
    some_in = torch.zeros(x.shape[0], dtype=torch.bool, device=DEV)
    not_all_out = torch.zeros(x.shape[0], dtype=torch.bool, device=DEV)
    for i in range(0, y.shape[0], block):
        d2 = d2_exact(y[i:i + block], x)
        e = (3 * D + 3) * U * (ny[i:i + block, None] + nx[None, :])
        up = (d2 + e).sqrt().float().half().float() * (1 + 2.0 ** -10)
        dn = (d2 - e).clamp_min(0).sqrt().float().half().float() * (1 - 2.0 ** -10)
        inside = up < rf[None]
        maybe = dn < rf[None]
        lo.append(inside.sum(1).cpu()); hi.append(maybe.sum(1).cpu())
        some_in |= inside.any(0)
        not_all_out |= maybe.any(0)
    return torch.cat(lo), torch.cat(hi), some_in.cpu(), (~not_all_out).cpu()


def check_random(m, n, seed, nhood=3):
    D = 4096
    g = torch.Generator(DEV).manual_seed(seed)
    W = torch.randn(16, D, generator=g, device=DEV)
    x, y = vgg_like(n, W, 0.0, g), vgg_like(m, W, 0.15, g)
    r = M.ManifoldBuilder(features=x, nhood_size=nhood, device=DEV).kth
    counts = abi_count(y, x, r)
    near = abi_nearest(x, y)
    covered = near.float() < r.float()
    lo, hi, must, must_not = forced(y, x, r)
    assert ((counts >= lo) & (counts <= hi)).all(), f"count outside [lo, hi] on {int(((counts < lo) | (counts > hi)).sum())} rows"
    assert covered[must].all() and not covered[must_not].any()
    d64 = torch.cat([d2_exact(x[i:i + 2048], y).min(1).values.sqrt() for i in range(0, n, 2048)]).cpu()
    fp64_cov = d64 < r.double()
    border = ~must & ~must_not
    assert torch.equal(covered[~border], fp64_cov[~border])              # fp64's coverage on every non-borderline row
    dens, cov = M.calc_dc(y.cpu(), (x.cpu(), r), nhood, DEV)
    assert dens == int(counts.long().sum()) / (nhood * m) and cov == int(covered.sum()) / n
    assert int(lo.sum()) / (nhood * m) <= dens <= int(hi.sum()) / (nhood * m)
    assert int(must.sum()) / n <= cov <= 1 - int(must_not.sum()) / n
    pairs_border = int((hi - lo).sum())
    return dens, cov, pairs_border / (m * n), int(border.sum())


@pytest.mark.parametrize("m,n", [(5000, 5000), (3000, 20000)])
def test_random_mode_within_bound(m, n, capsys):
    dens, cov, fb, rb = check_random(m, n, m + n)
    with capsys.disabled():
        print(f"\n  random {m}x{n}x4096: density {dens:.5f}, coverage {cov:.5f}; borderline pairs {fb:.2e}, rows {rb}")


def test_random_mode_full_size(capsys):
    dens, cov, fb, rb = check_random(50000, 50000, 11)
    with capsys.disabled():
        print(f"\n  random 50000^2 x 4096: density {dens:.5f}, coverage {cov:.5f}; borderline pairs {fb:.2e}, rows {rb}")


def test_calc_dc_cuda_matches_cpu_device_lists_and_current_stream():
    x = int_features(700, 200, 21)
    y = int_features(600, 200, 22)
    y[:50] = x[:50]
    r = exact_radii(x, y, 3)
    want = M.calc_dc(y, (x, r), 3, "cpu")
    mx = M.Manifold(x, r)
    assert M.calc_dc(y, mx, 3, DEV) == want
    assert M.calc_dc((y, None), mx, 3, [DEV]) == want
    assert M.calc_dc(M.Manifold(y.to(DEV), torch.zeros(600)), M.Manifold(x.to(DEV), r.to(DEV)), 3, "cuda") == want
    if torch.cuda.device_count() >= 2:
        with torch.cuda.device(0):
            assert M.calc_dc(y, mx, 3, torch.device("cuda", 1)) == want
    # the passes are ordered on the current stream: features written there just before the call are the ones they read
    s = torch.cuda.Stream(DEV)
    yd, xd = torch.zeros_like(y, device=DEV), torch.zeros_like(x, device=DEV)
    ys, xs = y.to(DEV), x.to(DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        yd.copy_(ys); xd.copy_(xs)
        got = M.calc_dc(yd, (xd, r), 3, DEV)
    assert got == want
