"""Density and coverage (Naeem et al., 2020) without a GPU: the CPU ``calc_dc`` against an independent restatement of the paper's
formulas on fp64 distances (sklearn), hand-built cases at the edges of the strict comparison, the ``nhood_size`` scaling of
density, the manifold formats, the refusals in Python and through the C ABI, the public names and the SASS of the counting
kernel."""
import collections
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from sklearn.metrics import pairwise_distances

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "ddpm_torch_b200", "libddpm_b200.so")
NAMES = ("ddpm_knn_count_scratch_bytes", "ddpm_knn_count")
INF, NAN = float("inf"), float("nan")


def paper_dc(real, fake, radii, k):
    """The paper's formulas on fp64 Euclidean distances (sklearn), written out independently of calc_dc."""
    d = pairwise_distances(real.double().numpy(), fake.double().numpy())          # [N, M]
    r = radii.double().numpy()[:, None]
    density = (d < r).sum() / (k * fake.shape[0])
    coverage = (d.min(axis=1) < r[:, 0]).mean()
    return density, coverage


def separated_radii(real, fake, g, margin=1e-3):
    """fp16 radii that sit in a gap of each real point's distances to the generated set, at least `margin` (relative) from every
    one of them, so no decision is borderline under fp16 rounding (2^-11 relative).  The gap is picked near a random rank, so counts vary."""
    d = np.sort(pairwise_distances(real.double().numpy(), fake.double().numpy()), axis=1)
    M_ = d.shape[1]
    ext = np.concatenate([np.zeros((d.shape[0], 1)), d, 2 * d[:, -1:] + 1], axis=1)
    out = []
    for i in range(d.shape[0]):
        t0 = int(torch.randint(0, M_ + 1, (1,), generator=g))
        cand = range(max(0, t0 - 20), min(M_ + 1, t0 + 21))
        t = max(cand, key=lambda t: (ext[i, t + 1] - ext[i, t]) / ext[i, t + 1])
        out.append((ext[i, t] + ext[i, t + 1]) / 2)
    r = torch.tensor(out).half()
    rel = np.abs(d - r.double().numpy()[:, None]) / r.double().numpy()[:, None]
    assert rel.min() > margin, rel.min()
    return r


@pytest.mark.parametrize("n,m,D,seed", [(150, 150, 16, 0), (120, 200, 32, 1), (300, 90, 8, 2), (64, 257, 24, 3)])
def test_cpu_matches_the_paper_formulas(n, m, D, seed):
    g = torch.Generator().manual_seed(seed)
    real = torch.randn(n, D, generator=g).half()
    fake = (torch.randn(m, D, generator=g) * 1.1 + 0.1).half()
    r = separated_radii(real, fake, g)
    for k in (1, 3, 5):
        dens, cov = M.calc_dc(fake, (real, r), k, "cpu")
        assert isinstance(dens, float) and isinstance(cov, float)
        want = paper_dc(real, fake, r, k)
        assert dens == want[0] and cov == want[1], (dens, cov, want)
    assert 0 < cov < 1 and dens > 0


def test_radii_from_the_builder_match_the_paper():
    """With the real manifold's own radii (ManifoldBuilder on the CPU), on data whose decisions are not borderline."""
    g = torch.Generator().manual_seed(0)
    real = torch.randn(60, 6, generator=g).half()
    fake = (torch.randn(50, 6, generator=g) + 0.2).half()
    mr = M.ManifoldBuilder(features=real, nhood_size=3)
    d = pairwise_distances(real.double().numpy(), fake.double().numpy())
    r = mr.kth.double().numpy()[:, None]
    assert (np.abs(d - r) / r).min() > 1e-3                          # no pair within fp16 rounding of its radius
    assert M.calc_dc(fake, mr.manifold, 3, "cpu") == paper_dc(real, fake, mr.kth, 3)


def test_ties_on_the_radius_do_not_count():
    real = torch.tensor([[0.0, 0.0], [10.0, 0.0]]).half()
    fake = torch.tensor([[1.0, 0.0], [10.0, 2.0], [10.0, 1.5]]).half()
    r = torch.tensor([1.0, 2.0]).half()                                # each real ball has a generated point exactly on it
    dens, cov = M.calc_dc(fake, (real, r), 1, "cpu")
    assert dens == 1 / 3 and cov == 0.5                                 # only (10, 1.5) is inside; real 0 is not covered
    counts, nearest = M._dc_host(fake, real, r)
    assert counts.tolist() == [0, 0, 1] and nearest.tolist() == [1.0, 1.5]


def test_zero_negative_inf_and_nan_radii():
    real = torch.tensor([[0.0, 0.0], [0.0, 0.0], [5.0, 5.0], [5.0, 5.0], [9.0, 9.0]]).half()
    fake = torch.tensor([[0.0, 0.0], [5.0, 5.0], [100.0, 100.0]]).half()
    for r, dens, cov in (([0.0, 0.0, 0.0, 0.0, 0.0], 0, 0),            # duplicated real points: radius 0 holds nothing
                         ([-1.0, -0.0, 0.0, -3.0, -1.0], 0, 0),
                         ([NAN, NAN, NAN, NAN, NAN], 0, 0),
                         ([INF, 0.0, NAN, -1.0, 0.0], 3, 1),            # +inf holds every generated point
                         ([INF, INF, INF, INF, INF], 15, 5)):
        got = M.calc_dc(fake, (real, torch.tensor(r).half()), 1, "cpu")
        assert got == (dens / 3, cov / 5), (r, got)


def test_generated_point_on_a_real_point_density_above_one_and_m_ne_n():
    real = torch.tensor([[0.0, 0.0], [0.5, 0.0], [0.0, 0.5], [0.25, 0.25], [30.0, 30.0]]).half()
    fake = torch.tensor([[0.0, 0.0], [0.1, 0.1]]).half()             # the first sits on a real point
    r = torch.tensor([1.0, 1.0, 1.0, 1.0, 0.5]).half()
    dens, cov = M.calc_dc(fake, (real, r), 1, "cpu")
    assert dens == 8 / 2 and dens > 1                                  # each generated point is in the four near balls
    assert cov == 4 / 5
    counts, nearest = M._dc_host(fake, real, r)
    assert counts.tolist() == [4, 4] and nearest[0] == 0


def test_density_scales_with_nhood_size():
    g = torch.Generator().manual_seed(5)
    real, fake = torch.randn(90, 12, generator=g).half(), torch.randn(70, 12, generator=g).half()
    mr = M.ManifoldBuilder(features=real, nhood_size=4)
    total = int(M._dc_host(fake, real, mr.kth)[0].sum())
    assert total > 0
    for k in (1, 2, 4, 7, 15, 100):
        dens, cov = M.calc_dc(fake, mr.manifold, k, "cpu")
        assert dens == total / (k * 70)
        assert cov == M.calc_dc(fake, mr.manifold, 1, "cpu")[1]


def test_all_manifold_formats():
    g = torch.Generator().manual_seed(6)
    real, fake = torch.randn(60, 8, generator=g).half(), torch.randn(50, 8, generator=g).half()
    mr = M.ManifoldBuilder(features=real, nhood_size=3)
    mf = M.ManifoldBuilder(features=fake, nhood_size=3)
    RefManifold = collections.namedtuple("Manifold", ["features", "kth"])   # the reference's type, from another module
    want = M.calc_dc(mf.manifold, mr.manifold, 3, "cpu")
    for gen in (mf.manifold, (fake, mf.kth), RefManifold(fake, mf.kth), fake, fake.float(), (fake, None)):
        for rl in (mr.manifold, (real, mr.kth), RefManifold(real, mr.kth), (real.float(), mr.kth.float())):
            assert M.calc_dc(gen, rl, 3, "cpu") == want
            assert M.calc_dc(gen, rl, 3, ["cpu"]) == want


def test_refusals():
    real, fake = torch.rand(10, 4).half(), torch.rand(6, 4).half()
    r = torch.ones(10).half()
    for args, match in (((fake[0], (real, r)), "features must be"), ((fake[None], (real, r)), "features must be"),
                        ((fake, (real[0], r)), "features must be"), ((fake[:, :3], (real, r)), "dimensions differ"),
                        ((fake[:0], (real, r)), "non-empty"), ((fake, (real[:0], r[:0])), "non-empty"),
                        ((fake[:, :0], (real[:, :0], r)), "non-empty"),
                        ((fake, (real, r[:9])), "one radius per real"), ((fake, (real, r[:, None])), "one radius per real"),
                        ((fake, (real, None)), "needs its radii")):
        with pytest.raises(ValueError, match=match):
            M.calc_dc(*args, 3, "cpu")
    for k in (0, -1, 1.5):
        with pytest.raises(ValueError, match="nhood_size"):
            M.calc_dc(fake, (real, r), k, "cpu")


def test_refusals_precede_any_device_work():
    """On a CUDA device the same refusals are raised before the engine (or even a device) is touched."""
    real, fake = torch.rand(10, 4).half(), torch.rand(6, 4).half()
    with pytest.raises(ValueError, match="one radius per real"):
        M.calc_dc(fake, (real, torch.ones(9)), 3, torch.device("cuda", 0))
    with pytest.raises(ValueError, match="nhood_size"):
        M.calc_dc(fake, (real, torch.ones(10)), 0, [torch.device("cuda", 0)])


def test_exports_and_header():
    assert "calc_dc" in M.__all__ and hasattr(M, "calc_dc")
    hdr = open(os.path.join(ROOT, "include", "ddpm_b200.h")).read()
    for name in NAMES:
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)
        assert re.search(r"\b" + name + r"\(", hdr)
    assert re.search(r"long long ddpm_knn_count_scratch_bytes\(int n_probes, int n_support, int D\);", hdr)
    assert re.search(r"int ddpm_knn_count\(const void\* probes, int n_probes, long long ld_p, const void\* support, int n_support, "
                     r"long long ld_s, int D,\s+const void\* radii, int32_t\* counts, void\* scratch, long long bytes, void\* stream\);", hdr)


def test_scratch_sizes():
    L = _lib.lib()
    al = lambda b: -(-b // 256) * 256                                   # noqa: E731
    for n, m, D in ((100, 100, 64), (1, 1, 1), (4099, 60000, 4096), (50000, 50000, 4096)):
        head = al(n * 4) + al(m * 4)                                     # the row and column norms
        assert L.ddpm_knn_count_scratch_bytes(n, m, D) == head + al(_splits(n, m) * n * 4)
        assert L.ddpm_knn_scratch_bytes(n, m, D, 0) == head + al(_splits(n, m) * n)      # the cover pass: the same plan
    for n, m, D in ((0, 10, 8), (10, 0, 8), (10, 10, 0), ((1 << 30) + 1, 10, 8)):
        assert L.ddpm_knn_count_scratch_bytes(n, m, D) < 0
        assert b"ddpm_knn_count_scratch_bytes" in L.ddpm_last_error()


def _splits(n, m, sms=132):
    """The column splits of csrc/knn.cuh's knn_plan, restated."""
    mt, nt = -(-n // 128), -(-m // 256)
    cap = min(nt, max(16, -(-sms // mt)))
    best, s_best = -1, 1
    for s in range(1, cap + 1):
        per = -(-nt // s)
        cost = -(-(mt * -(-nt // per)) // sms) * per
        if best < 0 or cost <= best:
            best, s_best = cost, s
    per = -(-nt // s_best)
    return -(-nt // per)


def test_abi_refusals_without_a_device():
    L = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = C.addressof(buf) + (-C.addressof(buf)) % 16                     # aligned, never dereferenced: every call is refused
    nb = L.ddpm_knn_count_scratch_bytes(4, 4, 12)
    good = dict(a=p, n=4, lda=16, b=p, m=4, ldb=16, D=12, r=p, out=p, s=p, bytes=nb)
    bad = [dict(a=None), dict(b=None), dict(a=p + 2), dict(b=p + 8), dict(lda=12), dict(ldb=8), dict(lda=20), dict(D=0),
           dict(n=0), dict(m=0), dict(n=-1), dict(r=None), dict(out=None), dict(r=p + 1), dict(out=p + 2), dict(s=None),
           dict(s=p + 4), dict(bytes=nb - 1), dict(bytes=0)]
    for b in bad:
        a = {**good, **b}
        rc = L.ddpm_knn_count(a["a"], a["n"], a["lda"], a["b"], a["m"], a["ldb"], a["D"], a["r"], a["out"], a["s"], a["bytes"], None)
        assert rc < 0 and b"ddpm_knn_count" in L.ddpm_last_error(), b


def test_count_kernel_sass_and_spills():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    per, cur = {}, None
    for ln in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1); per[cur] = set(); continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", ln)
        if m and cur:
            per[cur].add(m.group(1))
    main = [ops for fn, ops in per.items() if "knn_count_kernel" in fn]
    assert len(main) == 1
    ops = main[0]
    assert any(o.startswith("HGMMA") for o in ops) and any(o.startswith("UTMALDG") for o in ops)
    assert any(o.startswith("USETMAXREG") for o in ops)
    assert not any(o.startswith("HMMA") for o in ops)
    final = [ops for fn, ops in per.items() if "k_knn_count_final" in fn]
    assert len(final) == 1 and not any(o.startswith(("HGMMA", "HMMA")) for o in final[0])
    res = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True, check=True).stdout
    lines = res.splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        if re.search(r"Function (\S*knn_count_kernel|\S*k_knn_count_final)", ln):
            seen += 1
            assert re.search(r"STACK:0\b", lines[i + 1]) and re.search(r"LOCAL:0\b", lines[i + 1]), (ln, lines[i + 1])
    assert seen == 2
    log = os.path.join(ROOT, "ddpm_torch_b200", "csrc", "build.log")
    if not os.path.exists(log):
        pytest.skip("no build log (-Xptxas -v) next to the sources")
    lines = open(log).read().splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and re.search(r"knn_count_kernel|k_knn_count_final", ln):
            seen += 1
            spill = next(x for x in lines[i + 1:i + 5] if "bytes spill stores" in x)
            assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", spill), (ln, spill)
    assert seen == 2
