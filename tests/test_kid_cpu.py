"""The Kernel Inception Distance without a GPU: the numpy formula against a per-pair loop and the degree-1 closed form, the subset
index stream, the refusals of ``calc_kid``, the C ABI's sizes and refusals, the kernels' SASS and spills, a CPU
``KernelInceptionDistance`` end to end with seeded weights, and the public names.  Nothing reaches the network."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import inception as I
from ddpm_torch_b200 import metrics as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "ddpm_torch_b200", "libddpm_b200.so")
NAMES = ("ddpm_kid_scratch_bytes", "ddpm_kid")


@pytest.fixture
def offline(monkeypatch, tmp_path):
    def refuse(*a, **k):
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    os.makedirs(os.path.dirname(I.weights_path()))
    torch.save(I.seeded_state_dict(0), I.weights_path())


def loop_mmd2(x, y, ix, iy, degree, gamma, coef0):
    """The unbiased MMD^2 of one subset, pair by pair in Python floats."""
    k = lambda a, b: (gamma * float(np.dot(a, b)) + coef0) ** degree      # noqa: E731
    m = len(ix)
    xx = sum(k(x[i], x[j]) for i in ix for j in ix if i != j)
    yy = sum(k(y[i], y[j]) for i in iy for j in iy if i != j)
    xy = sum(k(x[i], y[j]) for i in ix for j in iy)
    return (xx + yy) / (m * (m - 1)) - 2 * xy / (m * m)


def features(n1, n2, d, seed, shift=0.3):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((n1, d)).astype(np.float32),
            (rng.standard_normal((n2, d)) + shift).astype(np.float32))


@pytest.mark.parametrize("degree,gamma,coef0", [(3, None, 1.0), (1, 0.5, 0.0), (2, 0.1, -0.5), (5, None, 2.0)])
def test_numpy_formula_is_the_pair_loop(degree, gamma, coef0):
    x, y = features(13, 11, 5, degree)
    S, m = 4, 7
    idx = M._kid_indices(13, 11, S, m, 9)
    g = 1 / 5 if gamma is None else gamma
    want = [loop_mmd2(x.astype(np.float64), y.astype(np.float64), idx[s, 0], idx[s, 1], degree, g, coef0) for s in range(S)]
    got = M._kid_numpy(x, y, idx, degree, g, coef0)
    np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-13)
    mean, std = M.calc_kid(x, y, S, m, degree, gamma, coef0, seed=9, device="cpu")
    assert isinstance(mean, float) and isinstance(std, float)
    np.testing.assert_allclose([mean, std], [np.mean(want), np.std(want)], rtol=1e-11, atol=1e-13)
    assert M.calc_kid(torch.from_numpy(x), torch.from_numpy(y), S, m, degree, gamma, coef0, seed=9, device="cpu") == (mean, std)


@pytest.mark.parametrize("coef0", [0.0, 1.0, -3.0])
def test_degree_one_closed_form(coef0):
    x, y = features(40, 30, 6, 2)
    S, m, gamma = 3, 20, 0.25
    idx = M._kid_indices(40, 30, S, m, 5)
    want = []
    for s in range(S):
        a, b = x[idx[s, 0]].astype(np.float64), y[idx[s, 1]].astype(np.float64)
        sa, sb = a.sum(0), b.sum(0)
        want.append(gamma * ((sa @ sa - (a * a).sum()) / (m * (m - 1)) + (sb @ sb - (b * b).sum()) / (m * (m - 1))
                             - 2 * (sa @ sb) / (m * m)))
    np.testing.assert_allclose(M._kid_numpy(x, y, idx, 1, gamma, coef0), want, rtol=1e-10, atol=1e-13)


def test_subset_index_stream():
    idx = M._kid_indices(50, 40, 3, 10, 1234)
    assert idx.dtype == np.int32 and idx.shape == (3, 2, 10)
    rng = np.random.RandomState(1234)
    for s in range(3):                                  # ix, then iy, subset by subset, from one stream
        assert np.array_equal(idx[s, 0], rng.choice(50, 10, replace=False))
        assert np.array_equal(idx[s, 1], rng.choice(40, 10, replace=False))
    assert np.array_equal(idx, M._kid_indices(50, 40, 3, 10, 1234))
    assert not np.array_equal(idx, M._kid_indices(50, 40, 3, 10, 1235))
    for s in range(3):
        assert len(set(idx[s, 0])) == 10 and len(set(idx[s, 1])) == 10


def test_calc_kid_refusals():
    x, y = features(10, 8, 4, 0)
    with pytest.raises(ValueError, match="subset_size"):
        M.calc_kid(x, y, 2, 9, device="cpu")            # m > min(n1, n2)
    with pytest.raises(ValueError, match="subset_size"):
        M.calc_kid(x, y, 2, 1, device="cpu")
    with pytest.raises(ValueError, match="dimensions differ"):
        M.calc_kid(x, y[:, :3], 2, 5, device="cpu")
    with pytest.raises(ValueError, match=r"\[n, d\]"):
        M.calc_kid(x[0], y, 2, 5, device="cpu")
    with pytest.raises(ValueError, match=r"\[n, d\]"):
        M.calc_kid(x[None], y, 2, 5, device="cpu")
    with pytest.raises(ValueError, match="degree"):
        M.calc_kid(x, y, 2, 5, degree=9, device="cpu")
    with pytest.raises(ValueError, match="num_subsets"):
        M.calc_kid(x, y, 0, 5, device="cpu")
    bad = x.copy()
    bad[:, 2] = np.nan                                  # every row, so every subset draws one
    with pytest.raises(ValueError, match="non-finite"):
        M.calc_kid(bad, y, 2, 5, device="cpu")
    bad[:, 2] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        M.calc_kid(bad, y, 2, 5, device="cpu")


def test_exports_and_sizes():
    hdr = open(os.path.join(ROOT, "include", "ddpm_b200.h")).read()
    for name in NAMES:
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)
        assert re.search(r"\b" + name + r"\(", hdr)
    L = _lib.lib()
    al = lambda b: -(-b // 256) * 256                     # noqa: E731
    for S, m in ((100, 1000), (1, 2), (10, 777), (7, 64), (3, 65)):
        T = -(-m // 64)
        assert L.ddpm_kid_scratch_bytes(S, m) == al(S * 2 * m * 4) + al(S * (T * (T + 1) + T * T) * 8)
    for S, m in ((0, 10), (-1, 10), (10, 1), (10, 0), (1 << 20, 50000)):
        assert L.ddpm_kid_scratch_bytes(S, m) < 0


def test_refusals_without_a_device():
    L = _lib.lib()
    p = 1 << 20                                         # a well-aligned non-null address that is never dereferenced
    S, m, n1, n2 = 3, 5, 8, 6
    idx = M._kid_indices(n1, n2, S, m, 0)
    nb = L.ddpm_kid_scratch_bytes(S, m)
    good = dict(x=p, ldx=16, n1=n1, y=p, ldy=16, n2=n2, d=16, idx=idx, S=S, m=m, degree=3, out=p, scratch=p, bytes=nb)

    def with_idx(s, h, i, v):
        j = idx.copy()
        j[s, h, i] = v
        return j
    bad = [dict(x=None), dict(x=p + 2), dict(y=None), dict(y=p + 1), dict(ldx=15), dict(ldy=15), dict(d=0), dict(d=4097, ldx=4097, ldy=4097),
           dict(m=1), dict(m=7), dict(n2=4), dict(S=0), dict(degree=0), dict(degree=9), dict(idx=None), dict(out=None), dict(out=p + 4),
           dict(scratch=None), dict(scratch=p + 8), dict(bytes=nb - 1),
           dict(idx=with_idx(1, 0, 2, n1)), dict(idx=with_idx(2, 1, 4, n2)), dict(idx=with_idx(0, 0, 0, -1)),
           dict(idx=with_idx(2, 0, 3, idx[2, 0, 1])), dict(idx=with_idx(1, 1, 0, idx[1, 1, 4]))]
    for b in bad:
        a = {**good, **b}
        ip = None if a["idx"] is None else np.ascontiguousarray(a["idx"], dtype=np.int32).ctypes.data
        rc = L.ddpm_kid(a["x"], a["ldx"], a["n1"], a["y"], a["ldy"], a["n2"], a["d"], ip, a["S"], a["m"], a["degree"], 1 / 16, 1.0,
                        a["out"], a["scratch"], a["bytes"], None)
        assert rc < 0 and b"ddpm_kid" in L.ddpm_last_error(), b


def test_kernels_sass_and_spills():
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
    tiles = [ops for fn, ops in per.items() if "k_kid_tiles" in fn]
    assert len(tiles) == 1 and any(o.startswith("DMMA") for o in tiles[0])
    finish = [ops for fn, ops in per.items() if "k_kid_finish" in fn]
    assert len(finish) == 1 and not any(o.startswith("DMMA") for o in finish[0])
    log = os.path.join(ROOT, "ddpm_torch_b200", "csrc", "build.log")
    if not os.path.exists(log):
        pytest.skip("no build log (-Xptxas -v) next to the sources")
    lines = open(log).read().splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and re.search(r"k_kid_(tiles|finish)", ln):
            seen += 1
            spill = next(x for x in lines[i + 1:i + 5] if "bytes spill stores" in x)
            assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", spill), (ln, spill)
    assert seen == 2


def test_cpu_kernel_inception_distance_end_to_end(offline):
    g = torch.Generator().manual_seed(5)
    x = torch.rand(5, 3, 40, 40, generator=g) * 2 - 1
    kid = M.KernelInceptionDistance(num_subsets=3, subset_size=4, degree=2, seed=7)
    kid(x[:2])
    kid(x[2:])
    assert kid.count == 5
    f = kid.features
    assert f.shape == (5, 2048) and f.dtype == torch.float32 and f.device.type == "cpu"
    net = I.InceptionV3([3]).eval()
    with torch.inference_mode():                        # batch by batch, as kid saw them: CPU kernels may differ with the batch
        want = torch.cat([net(b)[0].flatten(1) for b in (x[:2], x[2:])])
    assert torch.equal(f, want)
    other = torch.randn(6, 2048, generator=g).abs()
    got = kid.get_kid(other)
    assert got == M.calc_kid(f, other, 3, 4, degree=2, seed=7, device="cpu")
    assert kid.get_kid(other.numpy()) == got
    twin = M.KernelInceptionDistance(num_subsets=3, subset_size=4)
    twin._feats = [other]
    assert kid.get_kid(twin) == got
    kid.reset()
    assert kid.count == 0 and kid.features.shape == (0, 2048)
    with pytest.raises(ValueError):
        kid.get_kid(other)
    with pytest.raises(TypeError):
        M.KernelInceptionDistance(splits=3)


def test_public_names():
    for name in ("KernelInceptionDistance", "calc_kid"):
        assert name in M.__all__ and hasattr(M, name)
    assert M.calc_kid.__defaults__ == (100, 1000, 3, None, 1., 1234, None)
