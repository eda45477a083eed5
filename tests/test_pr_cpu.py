"""Precision / recall mirror (ddpm_torch_b200.metrics) without a GPU: the CPU path against tests/golden/pr.pt (the unmodified
reference, tools/gen_golden_pr.py), the data paths of the extraction branch, manifold formats, refusals, the ABI surface and
the SASS of the k-NN kernel."""
import collections
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import ddpm_torch_b200 as D
from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M

SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ddpm_torch_b200", "libddpm_b200.so")


class Identity(torch.nn.Module):
    """The identity feature extractor the golden was generated with."""
    def forward(self, x):
        return x.flatten(1).float()


class Images(torch.utils.data.Dataset):
    def __init__(self, x):
        self.x = x

    def __getitem__(self, i):
        return self.x[i], 0

    def __len__(self):
        return len(self.x)


class Sampler:
    def __init__(self):
        self.g = torch.Generator().manual_seed(7)

    def sample_x(self, n):
        return torch.rand(n, 3, 4, 4, generator=self.g) * 2.4 - 1.2


@pytest.fixture
def no_download(monkeypatch, tmp_path):
    """Any attempt to fetch the VGG16 weights fails the test."""
    def refuse(*a, **k):
        raise AssertionError("download_url_to_file reached")
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))


def features(c):
    """The golden's (real, fake) fp16 features from their uint8 codes (exact)."""
    return c["real_q"].half() * c["scale"], c["fake_q"].half() * c["scale"]


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


@pytest.mark.parametrize("case", [0, 1, 2])
@pytest.mark.parametrize("nhood", [1, 3, 7])
def test_cpu_path_matches_reference_bit_for_bit(golden, no_download, case, nhood):
    g = golden("pr.pt")
    c = g["cases"][case]
    res = c["results"][nhood]
    kw = dict(nhood_size=nhood, row_batch_size=c["row_batch_size"], col_batch_size=c["col_batch_size"])
    real, fake = features(c)
    mr = M.ManifoldBuilder(features=real, **kw)
    mf = M.ManifoldBuilder(features=fake, **kw)
    assert mr.op_device == torch.device("cpu")
    assert torch.equal(bits(mr.kth), bits(res["kth_real"])) and torch.equal(bits(mf.kth), bits(res["kth_fake"]))
    p, r = M.calc_pr(mf.manifold, mr.manifold, row_batch_size=c["row_batch_size"], col_batch_size=c["col_batch_size"], device="cpu")
    assert p.dtype == torch.float32 and p.dim() == 0 and p.device.type == "cpu"
    assert torch.equal(bits(p), bits(res["precision"])) and torch.equal(bits(r), bits(res["recall"]))
    assert f"{p:.5f}" == f"{res['precision']:.5f}"


def test_features_only_builder_sets_op_device(no_download):
    """Upstream's ManifoldBuilder(features=...) raises AttributeError (op_device); the mirror uses the device given."""
    f = torch.rand(40, 8)
    m = M.ManifoldBuilder(features=f, nhood_size=2)
    assert m.op_device == torch.device("cpu") and m.features.dtype == torch.float16 and m.kth.shape == (40,)
    m = M.ManifoldBuilder(features=f, nhood_size=2, device=["cpu"])
    assert m.op_device == "cpu"


def _data_builder(monkeypatch, g, **src):
    monkeypatch.setattr(M, "VGGFeatureExtractor", Identity)
    return M.ManifoldBuilder(**g["data"]["kwargs"], **src)


@pytest.mark.parametrize("source", ["tensor", "ndarray", "npy", "pt", "dataset", "model"])
def test_data_paths_match_reference(golden, monkeypatch, no_download, tmp_path, source):
    g = golden("pr.pt")
    imgs = g["data"]["images"]
    want = g["data"]["results"]["dataset" if source == "dataset" else "model" if source == "model" else "tensor"]
    if source == "tensor":
        src = dict(data=imgs)
    elif source == "ndarray":
        src = dict(data=imgs.numpy())
    elif source == "npy":
        np.save(tmp_path / "x.npy", imgs.numpy())
        src = dict(data=str(tmp_path / "x.npy"))
    elif source == "pt":
        torch.save(imgs, tmp_path / "x.pt")
        src = dict(data=str(tmp_path / "x.pt"))
    elif source == "dataset":
        src = dict(data=Images(imgs))
    else:
        src = dict(model=Sampler())
    m = _data_builder(monkeypatch, g, **src)
    assert torch.equal(bits(m.features), bits(want["features"]))
    assert torch.equal(bits(m.kth), bits(want["kth"]))
    if "inds" in want:
        assert torch.equal(m.features, imgs.flatten(1).half()[want["inds"]])


def test_subset_indices_are_upstreams_draw(golden):
    g = golden("pr.pt")
    np.random.seed(g["data"]["kwargs"]["random_state"])
    inds = torch.as_tensor(np.random.choice(300, size=g["data"]["kwargs"]["max_sample_size"], replace=False))
    assert torch.equal(inds, g["data"]["results"]["tensor"]["inds"])
    assert torch.equal(inds, g["data"]["results"]["dataset"]["inds"])


def test_to_uint8_matches_reference(golden):
    t = golden("pr.pt")["to_uint8"]
    assert torch.equal(M.to_uint8(t["x"]), t["y"])


def test_only_the_real_extractor_reaches_the_download(no_download):
    with pytest.raises(AssertionError, match="download_url_to_file reached"):
        M.VGGFeatureExtractor()


def test_reference_manifold_formats_are_accepted(golden, no_download):
    c = golden("pr.pt")["cases"][0]
    res = c["results"][3]
    RefManifold = collections.namedtuple("Manifold", ["features", "kth"])   # the reference's type, from another module
    kw = dict(row_batch_size=c["row_batch_size"], col_batch_size=c["col_batch_size"], device="cpu")
    for make in (RefManifold, lambda f, k: (f, k), M.Manifold):
        p, r = M.calc_pr(make(features(c)[1], res["kth_fake"]), make(features(c)[0], res["kth_real"]), **kw)
        assert torch.equal(p, res["precision"]) and torch.equal(r, res["recall"])


def test_manifold_roundtrips_through_torch_save(tmp_path, no_download):
    m = M.ManifoldBuilder(features=torch.rand(30, 16), nhood_size=3)
    m.save(str(tmp_path / "sub" / "m.pt"))
    back = torch.load(tmp_path / "sub" / "m.pt", weights_only=False)
    assert torch.equal(back.features, m.features) and torch.equal(back.kth, m.kth)


def test_refusals(no_download):
    f = torch.rand(5, 8)
    with pytest.raises(RuntimeError, match="nhood_size"):
        M.ManifoldBuilder(features=f, nhood_size=5)          # kk = 6 > 5 columns
    with pytest.raises(ValueError, match="nhood_size <= 15"):
        M._check_nhood(16, 100, native=True)
    M._check_nhood(16, 100, native=False)                     # the CPU path has no limit
    M._check_nhood(15, 100, native=True)


def test_cuda_refusal_of_large_nhood_precedes_any_launch(no_download):
    """nhood_size > 15 on a CUDA device is refused before the engine (or even a device) is touched."""
    with pytest.raises(ValueError, match="nhood_size <= 15"):
        M.ManifoldBuilder(features=torch.rand(40, 8), nhood_size=16, device=torch.device("cuda", 0))


def test_exports():
    assert D.metrics is M
    for name in ("Manifold", "ManifoldBuilder", "calc_pr", "compute_distance", "to_uint8", "VGGFeatureExtractor"):
        assert hasattr(M, name)
    for name in ("ddpm_knn_scratch_bytes", "ddpm_knn_kth", "ddpm_knn_cover"):
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)
    hdr = open(os.path.join(os.path.dirname(SO), "..", "include", "ddpm_b200.h")).read()
    for name in ("ddpm_knn_scratch_bytes", "ddpm_knn_kth", "ddpm_knn_cover"):
        assert re.search(r"\b" + name + r"\(", hdr)


def test_abi_refusals_without_a_device():
    L = _lib.lib()
    assert L.ddpm_knn_scratch_bytes(100, 100, 64, 4) > 0
    assert L.ddpm_knn_scratch_bytes(100, 100, 64, 0) > 0
    assert L.ddpm_knn_scratch_bytes(100, 100, 64, 17) < 0
    assert b"1..16" in L.ddpm_last_error()
    assert L.ddpm_knn_scratch_bytes(100, 3, 64, 4) < 0          # kk > n_cols
    assert L.ddpm_knn_scratch_bytes(0, 3, 64, 1) < 0
    buf = (C.c_uint8 * 4096)()
    p = C.addressof(buf) + (-C.addressof(buf)) % 16
    # pitch not a multiple of 8, pitch < D, null scratch: refused before any device work
    assert L.ddpm_knn_kth(p, 4, 12, p, 4, 16, 12, 2, p, p, 4096, None) < 0
    assert L.ddpm_knn_kth(p, 4, 8, p, 4, 16, 12, 2, p, p, 4096, None) < 0
    assert L.ddpm_knn_kth(p, 4, 16, p, 4, 16, 12, 2, p, None, 4096, None) < 0
    assert L.ddpm_knn_cover(p, 4, 16, p, 4, 16, 12, None, p, p, 4096, None) < 0


def test_knn_kernel_sass_is_hopper_native():
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
    hits = [ops for fn, ops in per.items() if "knn_wgmma_kernel" in fn]
    assert len(hits) == 2
    for ops in hits:
        assert any(o.startswith("HGMMA") for o in ops) and any(o.startswith("UTMALDG") for o in ops)
        assert any(o.startswith("USETMAXREG") for o in ops)
        assert not any(o.startswith("HMMA") for o in ops)
