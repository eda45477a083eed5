"""FID mirror (ddpm_torch_b200.metrics, ddpm_torch_b200.inception) without a GPU: the CPU routes against tests/golden/fid.pt (the
unmodified reference, tools/gen_golden_fid.py), the three upstream fixes, local precomputed statistics, the Evaluator, exports,
ABI refusals and the SASS of the FID kernels.  Nothing here reaches the network."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M
from ddpm_torch_b200.inception import seeded_state_dict, weights_path

SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ddpm_torch_b200", "libddpm_b200.so")


@pytest.fixture
def offline(monkeypatch, tmp_path):
    """Seeded FID weights in a temporary hub directory; every download path raises and is recorded."""
    reached = []

    def refuse(*a, **k):
        reached.append(a)
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    import requests
    monkeypatch.setattr(requests, "get", refuse)
    os.makedirs(os.path.dirname(weights_path()))
    torch.save(seeded_state_dict(0), weights_path())
    yield reached
    assert not reached, "a download was attempted"


class AsMaps(torch.nn.Module):
    def forward(self, t):
        return t[:, :, None, None]


def test_inception_reproduces_reference_features(golden, offline):
    g = golden("fid.pt")
    net = M.InceptionV3([0, 1, 2, 3]).eval()
    with torch.inference_mode():
        feats = net(g["images"])
    assert torch.equal(feats[3], g["block3"])
    for b in range(3):
        assert torch.equal(feats[b].flatten()[g[f"idx{b}"].long()], g[f"val{b}"])
    assert set(net.state_dict()) == set(net.state_dict().keys())
    assert all(k.startswith("blocks.") for k in net.state_dict())


def test_weights_load_strict_and_missing_file_goes_to_download(offline, monkeypatch):
    from ddpm_torch_b200 import inception
    net = inception.fid_inception_v3()
    assert set(net.state_dict()) == set(seeded_state_dict(0))
    os.remove(weights_path())
    with pytest.raises(AssertionError, match="network"):
        inception.fid_inception_v3()
    offline.clear()


def test_statistics_cpu_route_bit_for_bit(golden, offline):
    s = golden("fid.pt")["stats"]
    ist = M.InceptionStatistics(activation_dim=64)
    ist.model = AsMaps()
    for b in s["features"].split(s["sizes"]):
        ist(b)
    assert ist.count == sum(s["sizes"])
    assert np.array_equal(ist.running_mean, s["running_mean"]) and np.array_equal(ist.running_var, s["running_var"])
    m, v = ist.get_statistics()
    assert np.array_equal(m, s["mean"]) and np.array_equal(v, s["cov"])
    with pytest.raises(ValueError):
        ist.running_mean[0] = 1.0
    ist.reset()
    assert ist.count == 0 and not ist.running_var.any()
    with pytest.raises(AssertionError, match="Count must be greater than 1"):
        ist.get_statistics()


def test_calc_fd_cpu_route_bit_for_bit(golden):
    for c in golden("fid.pt")["fd"]:
        args = (c["mu1"], c["sigma1"], c["mu2"], c["sigma2"])
        if c["fd"] is None:
            with pytest.raises(ValueError, match="Imaginary component"):
                M.calc_fd(*args, device="cpu")
        else:
            assert float(M.calc_fd(*args, device="cpu")) == c["fd"]
            assert float(M.calculate_frechet_distance(*args)) == c["fd"]


def test_fix_sqrtm_without_disp():
    """Upstream's sqrtm(..., disp=False) raises TypeError on SciPy >= 1.18; the mirror's CPU formula runs."""
    import scipy
    from scipy import linalg
    a = np.diag([4.0, 9.0])
    if tuple(int(v) for v in scipy.__version__.split(".")[:2]) >= (1, 18):
        with pytest.raises(TypeError):
            linalg.sqrtm(a, disp=False)
    assert M.calculate_frechet_distance(np.zeros(2), a, np.zeros(2), np.eye(2)) == pytest.approx(13 + 2 - 2 * 5)


def test_fix_pooled_features_for_small_activation_dims(offline):
    """Upstream pools a numpy array with adaptive_avg_pool2d (TypeError) for activation_dim 64 / 192 / 768."""
    x = torch.rand(5, 3, 32, 32, generator=torch.Generator().manual_seed(3)) * 2 - 1
    ist = M.InceptionStatistics(activation_dim=64)
    ist(x)
    with torch.inference_mode():
        f = torch.nn.functional.adaptive_avg_pool2d(ist.model(x), (1, 1)).flatten(1).numpy()
    assert ist.count == 5
    assert np.array_equal(ist.running_mean, np.mean(f, axis=0, dtype=np.float64))


def _precomputed(tmp_path, monkeypatch, mu, sigma):
    monkeypatch.chdir(tmp_path)
    os.makedirs("precomputed", exist_ok=True)
    np.savez(os.path.join("precomputed", "fid_stats_cifar10_train.npz"), mu=mu, sigma=sigma)


def test_get_precomputed_reads_local_file(tmp_path, monkeypatch, offline):
    mu, sigma = np.arange(3.0), np.eye(3)
    _precomputed(tmp_path, monkeypatch, mu, sigma)
    m, s = M.get_precomputed("cifar10")
    assert np.array_equal(m, mu) and np.array_equal(s, sigma)
    with pytest.raises(AssertionError, match="network"):
        M.get_precomputed("cifar10", download_dir=str(tmp_path / "elsewhere"))
    offline.clear()


@pytest.mark.parametrize("total,batch", [(24, 8), (20, 8)])
def test_fix_evaluator_last_batch(tmp_path, monkeypatch, offline, total, batch):
    """Upstream's last batch is total % batch: 0 when batch divides total, and the empty batch made the FID NaN."""
    g = torch.Generator().manual_seed(0)
    imgs = torch.rand(total, 3, 32, 32, generator=g) * 2 - 1
    ref = M.InceptionStatistics(activation_dim=2048)
    ref(imgs)
    mu, sigma = ref.get_statistics()
    _precomputed(tmp_path, monkeypatch, mu + 0.01, sigma)
    ev = M.Evaluator("cifar10", eval_batch_size=batch, eval_total_size=total)
    sizes = []

    def sample_fn(sample_size, diffusion):
        sizes.append(sample_size)
        return imgs[sum(sizes) - sample_size: sum(sizes)]
    fid = ev.eval(sample_fn)["fid"]
    assert sum(sizes) == total and min(sizes) > 0
    assert np.isfinite(fid) and ev.istats.count == total


def test_exports():
    for name in ("InceptionV3", "InceptionStatistics", "get_precomputed", "calc_fd", "calculate_frechet_distance", "Evaluator",
                 "ManifoldBuilder", "calc_pr"):
        assert name in M.__all__ and hasattr(M, name)
    assert M.InceptionV3.BLOCK_INDEX_BY_DIM == {64: 0, 192: 1, 768: 2, 2048: 3}
    names = ("ddpm_fid_stats_bytes", "ddpm_fid_stats_update", "ddpm_fid_stats_finalize", "ddpm_fid_distance_scratch_bytes",
             "ddpm_fid_distance")
    hdr = open(os.path.join(os.path.dirname(SO), "..", "include", "ddpm_b200.h")).read()
    for name in names:
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)
        assert re.search(r"\b" + name + r"\(", hdr)


def test_abi_refusals_without_a_device():
    L = _lib.lib()
    assert L.ddpm_fid_stats_bytes(2048) > 2048 * 2048 * 8
    assert L.ddpm_fid_distance_scratch_bytes(4096) > 4 * 4096 * 4096 * 8
    for D in (0, 4097, -1):
        assert L.ddpm_fid_stats_bytes(D) < 0 and L.ddpm_fid_distance_scratch_bytes(D) < 0
    assert b"1..4096" in L.ddpm_last_error()
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf) + (-C.addressof(buf)) % 16
    assert L.ddpm_fid_stats_update(p, 8, p, 4, 4, None) < 0            # ld < D
    assert L.ddpm_fid_stats_update(None, 8, p, 4, 8, None) < 0         # null state
    assert L.ddpm_fid_stats_update(p + 8, 8, p, 4, 8, None) < 0        # misaligned state
    assert L.ddpm_fid_stats_update(p, 8, p + 2, 4, 8, None) < 0        # misaligned features
    assert L.ddpm_fid_stats_update(p, 8, None, 0, 8, None) == 0        # zero rows: a no-op
    assert L.ddpm_fid_stats_finalize(p, 8, 1, 1, p, p, None) < 0       # n <= ddof
    assert L.ddpm_fid_stats_finalize(p, 8, 5, 2, p, p, None) < 0       # ddof
    assert L.ddpm_fid_distance(p, p, p, p, 8, p, p, 16, None) < 0      # scratch too small
    assert L.ddpm_fid_distance(p, None, p, p, 8, p, p, 1 << 30, None) < 0
    assert L.ddpm_fid_distance(p, p, p, p, 8, p, p + 8, 1 << 30, None) < 0


def test_fid_kernel_sass_is_dmma_only():
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
    fid = {fn: ops for fn, ops in per.items() if "k_fid_" in fn}
    gemms = [ops for fn, ops in fid.items() if "k_fid_gemm" in fn]
    assert len(gemms) == 2 and all(any(o.startswith("DMMA") for o in ops) for ops in gemms)
    for ops in fid.values():
        assert not any(o.startswith(("HMMA", "IMMA")) for o in ops)
