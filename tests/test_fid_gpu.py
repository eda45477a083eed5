"""FID on the engine (csrc/fid.cuh): streaming statistics and the Fréchet distance against fp64 numpy.

Statistics bound (random mode).  Every product of two fp32 features is exact in fp64; what differs from the reference's recipe
(per-batch np.cov, Chan merge) is the order of O(n) fp64 additions of terms bounded by (|x_i| + |c_i|)(|x_j| + |c_j|), so
|cov_ij - ref_ij| <= 4 n u max|x_i - c_i| max|x_j - c_j| / (n - 1) + (the reference's own error, of the same form), with u = 2^-53.
The test uses that per-element bound with both error terms, B_ij = 8 n u a_i a_j / (n - 1), a_i = max_r |x_ri| + |mean_i|.

Distance bounds.  Full-rank inputs: both routes are backward stable in fp64, so |fd - ref| <= 1e-10 (tr S1 + tr S2).  Rank-deficient
inputs: the zero eigenvalues of S1 S2 come out as rounding noise of size ~ u lam_max(S1) lam_max(S2) in any fp64 route, and
their square roots, up to D of them, enter tr sqrt: floor = D sqrt(u lam_max(S1) lam_max(S2)) (fp64 numpy prototypes of this
route differ from scipy's sqrtm by 0.25-0.4 of that floor at D = 64 and 200)."""
import numpy as np
import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


def native_stats(batches, D, ddof=1, stream=None):
    L = _lib.lib()
    dev = torch.device("cuda", torch.cuda.current_device())
    state = torch.zeros(L.ddpm_fid_stats_bytes(D), dtype=torch.uint8, device=dev)
    st = _lib.stream_ptr() if stream is None else torch.cuda.current_stream().cuda_stream
    n = 0
    for x in batches:
        x = torch.as_tensor(x, dtype=torch.float32, device=dev).contiguous()
        _lib.check(L.ddpm_fid_stats_update(state.data_ptr(), D, x.data_ptr(), x.shape[0], D, st), "update")
        n += x.shape[0]
    mean = torch.full((D,), float("nan"), dtype=torch.float64, device=dev)
    cov = torch.full((D, D), float("nan"), dtype=torch.float64, device=dev)
    _lib.check(L.ddpm_fid_stats_finalize(state.data_ptr(), D, n, ddof, mean.data_ptr(), cov.data_ptr(), st), "finalize")
    return mean.cpu().numpy(), cov.cpu().numpy()


def chan_recipe(batches):
    """fid_score.py:116-142 in numpy: per-batch np.cov (ddof 0) merged, then rescaled to ddof 1."""
    m = v = None
    cnt = 0
    for x in batches:
        x = np.asarray(x, dtype=np.float32)
        mean = np.mean(x, axis=0, dtype=np.float64)
        var = np.cov(x, rowvar=False, ddof=0, dtype=np.float64).reshape(x.shape[1], x.shape[1])
        k = x.shape[0]
        a = k / (cnt + k)
        if cnt == 0:
            m, v = mean.copy(), var.copy()
        else:
            d = mean - m
            m += a * d
            v += a * (var - v)
            v += a * (1 - a) * np.outer(d, d)
        cnt += k
    return m, v * cnt / (cnt - 1)


def inception_like(n, D, seed):
    """Non-negative features with a low-rank structure and a wide range, like pool3 activations."""
    g = np.random.default_rng(seed)
    r = min(D, 64)
    W = g.standard_normal((r, D)).astype(np.float32) / np.sqrt(r)
    return np.maximum(g.standard_normal((n, r)).astype(np.float32) @ W + 0.2, 0).astype(np.float32) * 3


SEQUENCES = {"single": [512], "ones": [1, 1, 1, 5], "unequal": [7, 300, 33, 1000, 2], "ragged": [512] * 3 + [100]}


@pytest.mark.parametrize("D", [1, 3, 64, 100, 192, 768, 2048, 4096])
@pytest.mark.parametrize("seq", list(SEQUENCES))
def test_stats_random_within_bound(D, seq):
    sizes = SEQUENCES[seq]
    if D == 4096 and seq != "ragged":
        pytest.skip("D = 4096 runs the ragged sequence only")
    x = inception_like(sum(sizes), D, D + len(sizes))
    batches = np.split(x, np.cumsum(sizes)[:-1])
    m, c = native_stats(batches, D)
    m2, c2 = native_stats(batches, D)
    assert np.array_equal(m, m2) and np.array_equal(c, c2), "not bit-identical from run to run"
    rm, rc = chan_recipe(batches)
    n = x.shape[0]
    a = np.abs(x).max(0).astype(np.float64) + np.abs(rm)
    B = 8 * n * U * np.outer(a, a) / (n - 1)
    assert np.all(np.abs(c - rc) <= B), f"cov err/bound {np.max(np.abs(c - rc) / B):.3f}"
    assert np.all(np.abs(m - rm) <= 4 * n * U * a)
    assert np.array_equal(c, c.T)


def test_stats_full_size_50000x2048():
    x = inception_like(50000, 2048, 5)
    batches = np.split(x, np.arange(512, 50000, 512))
    m, c = native_stats(batches, 2048)
    rm, rc = chan_recipe(batches)
    a = np.abs(x).max(0).astype(np.float64) + np.abs(rm)
    B = 8 * 50000 * U * np.outer(a, a) / 49999
    ratio = np.max(np.abs(c - rc) / B)
    print(f"stats 50000x2048: err/bound {ratio:.3e}")
    assert ratio <= 1


@pytest.mark.parametrize("D", [1, 5, 64, 130])
def test_stats_exact_mode(D):
    """Integer features and a power-of-two first batch: the shift is a dyadic rational and every product and sum is exact."""
    g = np.random.default_rng(D)
    sizes = [64, 3, 17, 1]
    x = g.integers(0, 16, size=(sum(sizes), D)).astype(np.float32)
    batches = np.split(x, np.cumsum(sizes)[:-1])
    n = x.shape[0]
    c = x[:64].astype(np.float64).mean(0)
    s = (x - c).sum(0)
    Cm = (x - c).T @ (x - c)
    m, cov = native_stats(batches, D)
    assert np.array_equal(m, c + s / n)
    assert np.array_equal(cov, (Cm - np.outer(s, s) / n) / (n - 1))
    m0, cov0 = native_stats(batches, D, ddof=0)
    assert np.array_equal(cov0, (Cm - np.outer(s, s) / n) / n)


def test_stats_zero_row_batch_is_a_noop_and_current_stream():
    x = inception_like(300, 64, 1)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = native_stats([x[:100], x[:0], x[100:]], 64, stream=True)
    s.synchronize()
    b = native_stats([x[:100], x[100:]], 64)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def eig_route(mu1, s1, mu2, s2):
    """The same formula in fp64 numpy: tr sqrt(S1 S2) from eigh of S1 and of L^T S2 L."""
    s1, s2 = (s1 + s1.T) / 2, (s2 + s2.T) / 2
    lam, Q = np.linalg.eigh(s1)
    Lm = Q * np.sqrt(np.maximum(lam, 0))
    Mm = Lm.T @ s2 @ Lm
    nu = np.linalg.eigvalsh((Mm + Mm.T) / 2)
    d = mu1 - mu2
    return d @ d + np.trace(s1) + np.trace(s2) - 2 * np.sqrt(np.maximum(nu, 0)).sum()


def gauss_stats(D, n, seed, shift=0.0):
    g = np.random.default_rng(seed)
    W = g.standard_normal((D, D)) / np.sqrt(D)
    x = np.maximum((g.standard_normal((n, D)) * (1 + shift) + shift) @ W, 0)
    return x.mean(0), np.cov(x, rowvar=False).reshape(D, D)


def floor(s1, s2):
    D = s1.shape[0]
    return D * np.sqrt(U * np.linalg.eigvalsh(s1).max() * np.linalg.eigvalsh(s2).max())


@pytest.mark.parametrize("D,n", [(1, 50), (2, 50), (3, 50), (64, 5000), (100, 3000), (2048, 6000), (64, 40), (100, 60), (300, 200)])
def test_distance_against_fp64(D, n, capsys):
    mu1, s1 = gauss_stats(D, n, D)
    mu2, s2 = gauss_stats(D, n, D + 1, shift=0.2)
    fd, info = M.frechet_distance_native(mu1, s1, mu2, s2, "cuda")
    fd2, _ = M.frechet_distance_native(mu1, s1, mu2, s2, "cuda")
    assert fd == fd2
    ref = eig_route(mu1, s1, mu2, s2)
    full = n > D
    tol = 1e-10 * (np.trace(s1) + np.trace(s2)) + (0 if full else floor(s1, s2))
    with capsys.disabled():
        print(f"\nD={D} n={n}: fd {fd:.12g} eig {ref:.12g} err/tol {abs(fd - ref) / tol:.3e} sweeps {info['sweeps']}")
    assert abs(fd - ref) <= tol
    if D <= 300:
        sref = M.calculate_frechet_distance(mu1, s1, mu2, s2)
        assert abs(fd - sref) <= tol + floor(s1, s2)
    assert max(info["sweeps"]) < 60


def test_distance_4096():
    mu1, s1 = gauss_stats(4096, 9000, 1)
    mu2, s2 = gauss_stats(4096, 9000, 2, shift=0.2)
    fd, info = M.frechet_distance_native(mu1, s1, mu2, s2, "cuda")
    ref = eig_route(mu1, s1, mu2, s2)
    print(f"D=4096 err {abs(fd - ref):.3e} sweeps {info['sweeps']}")
    assert abs(fd - ref) <= 1e-10 * (np.trace(s1) + np.trace(s2))


def test_analytic_cases():
    g = np.random.default_rng(3)
    for D in (1, 2, 3, 64, 100):
        a, b = g.uniform(0.1, 3, D), g.uniform(0, 2, D)
        mu1, mu2 = g.standard_normal(D), g.standard_normal(D)
        fd = M.calc_fd(mu1, np.diag(a), mu2, np.diag(b), device="cuda")
        want = ((mu1 - mu2) ** 2).sum() + a.sum() + b.sum() - 2 * np.sqrt(a * b).sum()
        assert abs(fd - want) <= 1e-12 * (a.sum() + b.sum())
        Q, _ = np.linalg.qr(g.standard_normal((D, D)))        # commuting pair: same eigenvectors
        fd = M.calc_fd(mu1, (Q * a) @ Q.T, mu2, (Q * b) @ Q.T, device="cuda")
        assert abs(fd - want) <= 1e-10 * (a.sum() + b.sum())
    mu, s = gauss_stats(64, 30, 9)
    assert abs(M.calc_fd(mu, s, mu, s, device="cuda")) <= floor(s, s) + 1e-10 * 2 * np.trace(s)


def test_rounding_asymmetry_is_accepted_and_non_psd_refused():
    mu1, s1 = gauss_stats(64, 500, 4)
    mu2, s2 = gauss_stats(64, 500, 5)
    e = np.random.default_rng(0).standard_normal(s1.shape) * 1e-15 * np.abs(s1).max()
    fd = M.calc_fd(mu1, s1 + e, mu2, s2, device="cuda")
    assert abs(fd - eig_route(mu1, s1 + e, mu2, s2)) <= 1e-10 * (np.trace(s1) + np.trace(s2))
    bad = s1 - 0.5 * np.linalg.eigvalsh(s1).max() * np.eye(64)
    with pytest.raises(ValueError, match="sigma1"):
        M.calc_fd(mu1, bad, mu2, s2, device="cuda")
    with pytest.raises(ValueError, match="sigma2"):
        M.calc_fd(mu1, s1, mu2, bad, device="cuda")
    for arr in (mu1.copy(), s1.copy()):
        arr.flat[3] = np.nan
        args = (arr, s1, mu2, s2) if arr.ndim == 1 else (mu1, arr, mu2, s2)
        with pytest.raises(ValueError, match="non-finite"):
            M.calc_fd(*args, device="cuda")


class Fixed(torch.nn.Module):
    """Returns the given features as [B, D, 1, 1] maps, whatever the input."""
    def __init__(self, f):
        super().__init__()
        self.f = f

    def forward(self, x):
        return self.f[:, :, None, None]


def test_end_to_end_statistics_and_evaluator(monkeypatch, tmp_path):
    from ddpm_torch_b200.inception import seeded_state_dict, weights_path

    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))

    def refuse(*a, **k):
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    import requests
    monkeypatch.setattr(requests, "get", refuse)
    import os
    os.makedirs(os.path.dirname(weights_path()), exist_ok=True)
    torch.save(seeded_state_dict(0), weights_path())
    g = torch.Generator().manual_seed(0)
    imgs = torch.rand(24, 3, 32, 32, generator=g) * 2 - 1
    gpu = M.InceptionStatistics(device=torch.device("cuda"))
    cpu = M.InceptionStatistics(device=torch.device("cpu"))
    feats = []
    for b in imgs.split([10, 10, 4]):
        gpu(b.cuda())
        with torch.inference_mode():
            f = gpu.model(b.cuda()).flatten(1).cpu()
        feats.append(f)
        cpu.model = Fixed(f)
        cpu(b)
    mg, cg = gpu.get_statistics()
    mc, cc = cpu.get_statistics()
    x = torch.cat(feats).double().numpy()
    a = np.abs(x).max(0) + np.abs(mc)
    assert np.all(np.abs(cg - cc) <= 8 * 24 * U * np.outer(a, a) / 23)
    assert np.all(np.abs(gpu.running_var - cpu.running_var) <= 8 * 24 * U * np.outer(a, a) / 24)
    np.savez(tmp_path / "fid_stats_toy.npz", mu=mc + 0.01, sigma=cc)
    monkeypatch.chdir(tmp_path)
    os.makedirs("precomputed", exist_ok=True)
    os.replace(tmp_path / "fid_stats_toy.npz", os.path.join("precomputed", "fid_stats_toy.npz"))
    ev = M.Evaluator("toy", eval_batch_size=8, eval_total_size=24, device=torch.device("cuda"))
    pos = [0]

    def sample_fn(sample_size, diffusion):
        out = imgs[pos[0]: pos[0] + sample_size]
        pos[0] += sample_size
        return out
    fid = ev.eval(sample_fn)["fid"]
    assert pos[0] == 24 and ev.istats.count == 24
    me, ce = ev.istats.get_statistics()          # Inception saw batches of 8 here: its own features, not feats above
    want = eig_route(me, ce, mc + 0.01, cc)
    assert np.isfinite(fid) and abs(fid - want) <= 1e-10 * (np.trace(ce) + np.trace(cc)) + floor(ce, cc)
