"""The k-NN half of precision/recall on the engine (ddpm_knn_kth / ddpm_knn_cover, csrc/knn.cuh) against the recipe it
implements, on an H100.

Recipe (the numerical contract, on the fp16 features as stored):
  na[i] = sum_d a[i,d]^2;  d2[i,j] = max(0, na[i] + nb[j] - 2 <a_i, b_j>);
  kth[i] = fp16_rn(sqrt_rn(kk-th smallest d2[i, .]));  probe i covered iff exists j: fp16_rn(sqrt_rn(d2[i,j])) <= r[j].

Exact mode: integer features in [-3, 3].  Every product, partial sum, norm and d2 is an integer below 9 * 4096 < 2^21 (the
bound tests/test_conv_gpu.py relies on), so fp32 accumulation in any order is exact and the engine must reproduce the recipe
(evaluated in fp64, then sqrt in fp32 on the CPU, which is correctly rounded) bit for bit.

Random mode: VGG-like fp16 features (relu of a rank-16 projection).  Accumulation model of the engine, with u = 2^-24:
  * the fp32 norm of a row, a sum of D non-negative terms:       |dna| <= D u na
  * the wgmma inner product, fp32 accumulation of D products:    |ddot| <= D 2u sum_d |a_d||b_d| <= D u (na + nb)
    (Cauchy-Schwarz: sum |a||b| <= sqrt(na nb) <= (na + nb) / 2)
  * the rounding of na + nb and of the final fma:                <= 2u (na + nb) + u d2 <= 3u (na + nb)
so with E_i = (3 D + 3) u (na_i + max_j nb_j), every engine d2[i, j] lies within E_i of the exact one.  The kk-th smallest of
values each moved by at most E_i moves by at most E_i, and sqrt is monotone, so
  fp16_down(sqrt(max(0, d2k - E_i))) <= kth[i] <= fp16_up(sqrt(d2k + E_i))   (fp16 rounding: a factor 1 -+ 2^-11).
A probe's flag is forced where the exact decision survives that perturbation: covered if some j has
fp16(sqrt(d2 + E_i)) <= r_j, not covered if no j has fp16(sqrt(max(0, d2 - E_i))) <= r_j; the rest are reported as borderline.
"""
import os

import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
U = 2.0 ** -24


def d2_exact(a, b):
    """fp64 squared distances of fp16 features (exact for the exact-mode integers)."""
    a, b = a.to(DEV, torch.float64), b.to(DEV, torch.float64)
    na, nb = (a * a).sum(1), (b * b).sum(1)
    return (na[:, None] + nb[None, :] - 2.0 * (a @ b.T)).clamp_min(0.0)


def fp16_sqrt(d2):
    """fp16_rn(sqrt_rn(d2)) for d2 exactly representable in fp32 (CPU fp32 sqrt is correctly rounded)."""
    return d2.float().cpu().sqrt().half()


def abi_kth(a, b, kk, prefill=True):
    """ddpm_knn_kth on features already on DEV (any D: padded rows as the mirror makes them); outputs start as NaN and the
    scratch as 0xAB, so anything the engine leaves unwritten shows."""
    L = _lib.lib()
    n, m, D = a.shape[0], b.shape[0], a.shape[1]
    A, B = M._device_rows(a, DEV), M._device_rows(b, DEV)
    nbytes = L.ddpm_knn_scratch_bytes(n, m, D, kk)
    _lib.check(nbytes if nbytes < 0 else 0, "scratch_bytes")
    scratch = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device=DEV)
    out = torch.full((n,), float("nan"), dtype=torch.float16, device=DEV)
    _lib.check(L.ddpm_knn_kth(A.data_ptr(), n, A.stride(0), B.data_ptr(), m, B.stride(0), D, kk, out.data_ptr(),
                              scratch.data_ptr(), nbytes, _lib.stream_ptr(DEV)), "knn_kth")
    torch.cuda.synchronize()
    assert L.ddpm_device_error_flag() == 0
    return out.cpu()


def abi_cover(p, s, r):
    L = _lib.lib()
    n, m, D = p.shape[0], s.shape[0], p.shape[1]
    A, B = M._device_rows(p, DEV), M._device_rows(s, DEV)
    nbytes = L.ddpm_knn_scratch_bytes(n, m, D, 0)
    scratch = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device=DEV)
    out = torch.full((n,), 0xFF, dtype=torch.uint8, device=DEV)
    rr = r.to(DEV, torch.float16).contiguous()
    _lib.check(L.ddpm_knn_cover(A.data_ptr(), n, A.stride(0), B.data_ptr(), m, B.stride(0), D, rr.data_ptr(), out.data_ptr(),
                                scratch.data_ptr(), nbytes, _lib.stream_ptr(DEV)), "knn_cover")
    torch.cuda.synchronize()
    assert L.ddpm_device_error_flag() == 0
    out = out.cpu()
    assert ((out == 0) | (out == 1)).all()
    return out.bool()


def recipe_kth(a, b, kk, block=2048):
    return torch.cat([fp16_sqrt(d2_exact(a[i:i + block], b).kthvalue(kk, dim=1).values) for i in range(0, a.shape[0], block)])


def recipe_cover(p, s, r, block=512):
    return torch.cat([(fp16_sqrt(d2_exact(p[i:i + block], s)).float() <= r.float()[None, :]).any(1)
                      for i in range(0, p.shape[0], block)])


def int_features(n, D, seed, dup=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-3, 4, (n, D), generator=g).half()
    if dup and n > 3:
        x[1::3] = x[0::3][: len(x[1::3])]
    return x


def bits(t):
    return t.view(torch.int16)


# (n_rows, n_cols, D, kk, self): self = the kth of a set against itself (compute_kth); otherwise two sets
EXACT_KTH = [
    (1, 16, 3, 16, False), (127, 127, 8, 4, True), (128, 128, 64, 2, True), (129, 129, 100, 8, True),
    (1000, 1000, 520, 4, True), (4099, 4099, 64, 16, True), (129, 1, 8, 1, False), (1000, 129, 4096, 8, False),
    (127, 4099, 100, 4, False), (4099, 128, 3, 2, False), (128, 16, 520, 16, False), (1, 1, 3, 1, True),
    (129, 8, 4096, 8, False), (1000, 1000, 3, 16, True),
    (200, 60000, 64, 4, False),          # few row tiles, many columns: the column split
]


@pytest.mark.parametrize("n,m,D,kk,self_", EXACT_KTH)
def test_kth_exact(n, m, D, kk, self_):
    a = int_features(n, D, 1000 + n + D, dup=True)
    b = a if self_ else int_features(m, D, 2000 + m + D, dup=True)
    got = abi_kth(a, b, kk)
    want = recipe_kth(a, b, kk)
    assert not torch.isnan(got).any()
    assert torch.equal(bits(got), bits(want))
    assert torch.equal(bits(abi_kth(a, b, kk)), bits(got))          # a second call: identical bits


@pytest.mark.parametrize("n,m,D", [(1, 16, 3), (127, 4099, 100), (4099, 128, 520), (1000, 1000, 4096), (129, 129, 8),
                                   (200, 60000, 64), (128, 1, 64)])
def test_cover_exact(n, m, D):
    p = int_features(n, D, 3000 + n + D, dup=True)
    s = int_features(m, D, 4000 + m + D, dup=True)
    p[: min(n, m) // 2] = s[: min(n, m) // 2]                     # some probes sit exactly on a support point
    kk = min(4, m)
    r = recipe_kth(s, s, kk)                                       # the radii calc_pr uses: many ties at exactly r
    g = torch.Generator().manual_seed(n + m)
    r2 = r.clone()
    sel = torch.rand(m, generator=g)
    r2[sel < 0.1] = 0.0
    r2[(sel >= 0.1) & (sel < 0.15)] = -1.0
    r2[(sel >= 0.15) & (sel < 0.17)] = float("inf")
    for radii in (r, r2):
        got = abi_cover(p, s, radii)
        assert torch.equal(got, recipe_cover(p, s, radii))
        assert torch.equal(abi_cover(p, s, radii), got)


def test_identical_sets_have_zero_radii_and_full_coverage():
    x = int_features(1, 100, 5).repeat(300, 1)
    k = abi_kth(x, x, 16)
    assert (k == 0).all() and not torch.signbit(k).any()
    assert abi_cover(x, x, k).all()
    y = x.clone(); y[:, 0] += 1
    assert not abi_cover(y, x, k).any()


def vgg_like(n, W, shift, g):
    z = torch.randn(n, W.shape[0], generator=g, device=DEV) * (1 + shift) + shift
    return torch.relu(z @ W / 4).half()


def bound_E(a, b):
    """E_i of the module docstring, fp64 on DEV."""
    D = a.shape[1]
    na = (a.to(DEV, torch.float64) ** 2).sum(1)
    nb = (b.to(DEV, torch.float64) ** 2).sum(1)
    return (3 * D + 3) * U * (na + nb.max())


def kth_bounds(a, b, kk, block=4096):
    lo, hi = [], []
    E = bound_E(a, b)
    for i in range(0, a.shape[0], block):
        d2 = d2_exact(a[i:i + block], b)
        dk = d2.kthvalue(kk, dim=1).values
        e = E[i:i + block]
        lo.append(((dk - e).clamp_min(0).sqrt() * (1 - 2.0 ** -11)).cpu())
        hi.append(((dk + e).sqrt() * (1 + 2.0 ** -11)).cpu())
    return torch.cat(lo), torch.cat(hi)


def forced_flags(p, s, r, block=2048):
    """(must_cover, must_not_cover) per probe, from fp64 distances moved by -+E_i."""
    E = bound_E(p, s)
    rf = r.to(DEV).float()
    cov, unc = [], []
    for i in range(0, p.shape[0], block):
        d2 = d2_exact(p[i:i + block], s)
        e = E[i:i + block, None]
        up = (d2 + e).sqrt().float().half().float()        # fp16 of an upper bound: any rounding of it is fine here
        dn = (d2 - e).clamp_min(0).sqrt().float().half().float()
        cov.append(((up * (1 + 2.0 ** -10)) <= rf[None]).any(1).cpu())
        unc.append(~((dn * (1 - 2.0 ** -10)) <= rf[None]).any(1).cpu())
    return torch.cat(cov), torch.cat(unc)


@pytest.mark.parametrize("n,m,D", [(5000, 5000, 4096), (3000, 20000, 4096)])
def test_random_mode_within_bound(n, m, D, capsys):
    g = torch.Generator(DEV).manual_seed(n + m)
    W = torch.randn(16, D, generator=g, device=DEV)
    s = vgg_like(m, W, 0.0, g)
    p = vgg_like(n, W, 0.15, g)
    kth = abi_kth(s, s, 4)
    lo, hi = kth_bounds(s, s, 4)
    k = kth.double()
    assert ((k >= lo) & (k <= hi)).all(), f"kth outside the bound at {int(((k < lo) | (k > hi)).sum())} rows"
    flags = abi_cover(p, s, kth)
    must, must_not = forced_flags(p, s, kth)
    assert (flags[must]).all() and not (flags[must_not]).any()
    border = int((~must & ~must_not).sum())
    with capsys.disabled():
        print(f"\n  random {n}x{m}x{D}: kth within bound on all rows, {border} borderline probes of {n}")


def test_full_size_manifolds_and_calc_pr(capsys):
    n = 50000
    D = 4096
    g = torch.Generator(DEV).manual_seed(11)
    W = torch.randn(16, D, generator=g, device=DEV)
    real, fake = vgg_like(n, W, 0.0, g).cpu(), vgg_like(n, W, 0.15, g).cpu()
    mr = M.ManifoldBuilder(features=real, nhood_size=3, device=DEV)
    mf = M.ManifoldBuilder(features=fake, nhood_size=3, device=DEV)
    precision, recall = M.calc_pr(mf.manifold, mr.manifold, 10000, 10000, device=DEV)
    lines = []
    for feats, kth in ((real, mr.kth), (fake, mf.kth)):
        lo, hi = kth_bounds(feats.to(DEV), feats.to(DEV), 4)
        assert ((kth.double() >= lo) & (kth.double() <= hi)).all()
    for probes, support, kth, got in ((fake, real, mr.kth, precision), (real, fake, mf.kth, recall)):
        flags = abi_cover(probes, support, kth)
        assert torch.equal(flags.to(torch.float32).mean(), got)
        must, must_not = forced_flags(probes.to(DEV), support.to(DEV), kth)
        assert flags[must].all() and not flags[must_not].any()
        border = int((~must & ~must_not).sum())
        lo_f, hi_f = must.float().mean().item(), 1 - must_not.float().mean().item()
        assert lo_f <= got.item() <= hi_f
        lines.append(f"{got.item():.5f} (fp64 in [{lo_f:.5f}, {hi_f:.5f}], {border} borderline)")
    with capsys.disabled():
        print(f"\n  50000^2 x 4096: precision {lines[0]}, recall {lines[1]}")


def margin_fraction(probes, support, kth64, rel=2e-3):
    """Fraction of probes whose fp64 decision flips when every distance / radius moves by `rel` relative."""
    d = d2_exact(probes, support).sqrt()
    ratio = (d / kth64[None, :].clamp_min(1e-30)).min(1).values
    return ((ratio - 1).abs() <= rel).double().mean().item()


def kth64(x, kk):
    return d2_exact(x, x).kthvalue(kk, dim=1).values.sqrt()


def _check_against_reference(real, fake, nhood, p_ref, r_ref):
    mr = M.ManifoldBuilder(features=real, nhood_size=nhood, device=DEV)
    mf = M.ManifoldBuilder(features=fake, nhood_size=nhood, device=DEV)
    p, r = M.calc_pr(mf.manifold, mr.manifold, 10000, 10000, device=DEV)
    n = real.shape[0]
    mp = margin_fraction(fake, real, kth64(real, nhood + 1))
    mrr = margin_fraction(real, fake, kth64(fake, nhood + 1))
    assert abs(p.item() - float(p_ref)) <= mp + 1.0 / n + 1e-7, (p, p_ref, mp)
    assert abs(r.item() - float(r_ref)) <= mrr + 1.0 / n + 1e-7, (r, r_ref, mrr)
    return p.item(), r.item()


@pytest.mark.parametrize("case", [0, 1, 2])
@pytest.mark.parametrize("nhood", [1, 3, 7])
def test_against_reference_goldens(golden, case, nhood):
    c = golden("pr.pt")["cases"][case]
    res = c["results"][nhood]
    real, fake = c["real_q"].half() * c["scale"], c["fake_q"].half() * c["scale"]
    _check_against_reference(real, fake, nhood, res["precision"], res["recall"])


def test_against_reference_at_1500x4096(capsys):
    import importlib.util
    from oracle import ref_loader
    r = ref_loader.root()
    if r is None:
        pytest.skip("the reference is not staged (oracle/_ref)")
    spec = importlib.util.spec_from_file_location("ref_pr", os.path.join(r, "ddpm_torch", "metrics", "precision_recall.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    ref.ManifoldBuilder.op_device = DEV          # upstream sets it only when extracting (see metrics.ManifoldBuilder)
    g = torch.Generator(DEV).manual_seed(1500)
    W = torch.randn(16, 4096, generator=g, device=DEV)
    real, fake = vgg_like(1500, W, 0.0, g).cpu(), vgg_like(1500, W, 0.15, g).cpu()
    mr = ref.ManifoldBuilder(features=real, nhood_size=3, device=DEV)
    mf = ref.ManifoldBuilder(features=fake, nhood_size=3, device=DEV)
    p_ref, r_ref = ref.calc_pr(mf.manifold, mr.manifold, 10000, 10000, device=DEV)
    p, r = _check_against_reference(real, fake, 3, p_ref, r_ref)
    with capsys.disabled():
        print(f"\n  1500x4096: native {p:.5f}/{r:.5f}, reference {float(p_ref):.5f}/{float(r_ref):.5f}")


def test_device_list_other_device_and_current_stream():
    g = torch.Generator().manual_seed(3)
    x = torch.relu(torch.randn(700, 256, generator=g)).half()
    y = torch.relu(torch.randn(600, 256, generator=g) + 0.1).half()
    base = M.ManifoldBuilder(features=x, nhood_size=3, device=DEV)
    lst = M.ManifoldBuilder(features=x, nhood_size=3, device=[DEV])
    assert torch.equal(bits(base.kth), bits(lst.kth))
    pr0 = M.calc_pr((y, base.kth), base.manifold, 100, 100, device=[DEV])
    if torch.cuda.device_count() >= 2:
        other = torch.device("cuda", 1)
        with torch.cuda.device(0):
            m1 = M.ManifoldBuilder(features=x, nhood_size=3, device=other)
            assert torch.equal(bits(m1.kth), bits(base.kth))
            pr1 = M.calc_pr((y, base.kth), base.manifold, 100, 100, device=other)
            assert torch.equal(pr1[0], pr0[0]) and torch.equal(pr1[1], pr0[1])
    # the call is ordered on the current stream: features written there just before it are the ones it reads
    s = torch.cuda.Stream(DEV)
    xd = torch.zeros_like(x, device=DEV)
    src = x.to(DEV)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        xd.copy_(src)
        k = M._native("test", xd, xd, 4, None, DEV)
    assert torch.equal(bits(k), bits(base.kth))


def test_padded_copy_for_odd_dimensions_and_strided_views():
    g = torch.Generator().manual_seed(4)
    x = torch.randint(-3, 4, (300, 77), generator=g).half()
    wide = torch.randint(-3, 4, (300, 96), generator=g).half()
    wide[:, :77] = x
    k1 = M.ManifoldBuilder(features=x, nhood_size=5, device=DEV).kth
    v = wide.to(DEV)[:, :77]                                       # pitch 96, D = 77: read in place, no copy
    assert M._device_rows(v, DEV).data_ptr() == v.data_ptr()
    k2 = M._native("test", v, v, 6, None, DEV)
    assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(k1), bits(recipe_kth(x, x, 6)))
