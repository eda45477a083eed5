"""Improved precision and recall (Kynkäänniemi et al., 2019) of ``ddpm_torch/metrics/precision_recall.py``, with its k-NN
half on the engine.

Public names, signatures and defaults are the reference's: ``Manifold``, ``ManifoldBuilder``, ``calc_pr``,
``compute_distance``, ``to_uint8`` and ``VGGFeatureExtractor``.

* CUDA ``device`` (a device, or a list whose first entry is used): ``ManifoldBuilder.compute_kth`` and ``calc_pr`` run
  ``ddpm_knn_kth`` / ``ddpm_knn_cover`` (one fp16 wgmma GEMM with a selection epilogue, ``csrc/knn.cuh``) on that device's
  current stream.  Only the [N] radii and coverage flags come back to the host; no distance matrix is formed.  The radii are
  ``fp16(sqrt(kk-th smallest d2))`` from exact fp16 features and fp32 accumulation, where the reference uses fp16
  ``torch.cdist`` (whose self-distances alone reach ~2 at D = 4096).  The two agree statistically, not bit for bit.
  ``row_batch_size`` / ``col_batch_size`` do not change any result there and are ignored.  ``nhood_size`` is limited to 15.
* CPU ``device``: the reference's own ``cdist`` formulas, batch by batch, as upstream.

The VGG16 extractor stays the reference's TorchScript model run by torch; it is only built when features are extracted.
"""
import math
import os
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn
from torch.utils.data import DataLoader, Subset

from . import _lib

# precision_recall.py:19.  calc_pr also takes the reference's own namedtuple (eval.py:114-122 reloads torch.save'd
# manifolds) or any (features, kth) pair.
Manifold = namedtuple("Manifold", ["features", "kth"])

MAX_NHOOD_SIZE = 15          # kk = nhood_size + 1 <= 16: the register lists of the native kth pass


class VGGFeatureExtractor(nn.Module):
    """VGG16 feature embedding of the StyleGAN2-ADA metrics (precision_recall.py:22-41): the TorchScript model
    ``vgg16.pt`` from the torch hub directory, fetched into it only when it is not there yet.  Constructed only by
    ``ManifoldBuilder`` when it has to extract features, so passing ``features=`` never reaches the network."""
    WEIGHTS_URL = "https://nvlabs-fi-cdn.nvidia.com/stylegan2-ada-pytorch/pretrained/metrics/vgg16.pt"

    def __init__(self):
        super().__init__()
        path = os.path.join(torch.hub.get_dir(), self.WEIGHTS_URL.rsplit("/", 1)[-1])
        if not os.path.isfile(path):
            torch.hub.download_url_to_file(self.WEIGHTS_URL, path)
        self.model = torch.jit.load(path).eval()
        self.model.requires_grad_(False)

    def forward(self, x):
        return self.model(x, return_features=True)


def compute_distance(row_features, col_features, row_batch_size, col_batch_size, device):
    """precision_recall.py:43-55: the full distance matrix on the host, assembled from ``torch.cdist`` blocks computed on
    ``device``.  Kept for callers of the reference function; the metric itself does not go through it on CUDA."""
    rows = []
    for rb in row_features.split(row_batch_size, dim=0):
        blocks = [torch.cdist(rb.to(device)[None], cb.to(device)[None])[0].cpu() for cb in col_features.split(col_batch_size, dim=0)]
        rows.append(torch.cat(blocks, dim=1))
    return torch.cat(rows, dim=0)


def to_uint8(x):
    """precision_recall.py:58-59: samples in [-1, 1] -> uint8 images."""
    return (x * 127.5 + 128).clamp(0, 255).to(torch.uint8)


def _op_device(device):
    return device[0] if isinstance(device, (list, tuple)) else device


def _cuda_device(device):
    """torch.device of a CUDA ``device`` (index filled in), or None for any other device."""
    d = torch.device(device)
    if d.type != "cuda":
        return None
    return d if d.index is not None else torch.device("cuda", torch.cuda.current_device())


def _fields(manifold):
    if hasattr(manifold, "features") and hasattr(manifold, "kth"):
        return manifold.features, manifold.kth
    features, kth = manifold
    return features, kth


def _check_nhood(nhood_size, n_cols, native):
    kk = nhood_size + 1
    if kk < 1 or kk > n_cols:
        # upstream: kthvalue(nhood_size + 1) raises a RuntimeError; here it is raised before any distance is computed
        raise RuntimeError(f"nhood_size + 1 = {kk} must be in 1..{n_cols} (the number of columns)")
    if native and nhood_size > MAX_NHOOD_SIZE:
        raise ValueError(f"nhood_size = {nhood_size}: the native k-NN pass supports nhood_size <= {MAX_NHOOD_SIZE} "
                         "(kk = nhood_size + 1 <= 16); use a CPU device for larger neighbourhoods")
    return kk


def _device_rows(x, dev):
    """fp16 features on ``dev`` as the engine reads them: unit column stride, 16-byte aligned rows whose pitch is a multiple
    of 8 elements.  Otherwise (e.g. D % 8 != 0) a zero-padded copy; zero columns change no distance."""
    x = x.to(device=dev, dtype=torch.float16)
    D = x.shape[1]
    if x.stride(1) != 1 or x.stride(0) % 8 or x.stride(0) < D or x.data_ptr() % 16:
        y = torch.zeros(x.shape[0], -(-D // 8) * 8, dtype=torch.float16, device=dev)
        y[:, :D] = x
        x = y
    return x


def _native(fn_name, rows, cols, kk, radii, dev):
    """One engine pass on ``dev``'s current stream.  kk >= 1: kth radii of ``rows`` against ``cols`` (fp16 [n]);
    kk = 0: coverage of ``rows`` by the balls (``cols``, ``radii``) (bool [n]).  Returns a CPU tensor."""
    L = _lib.lib()
    n, m, D = rows.shape[0], cols.shape[0], rows.shape[1]
    if cols.shape[1] != D:
        raise ValueError(f"feature dimensions differ: {D} and {cols.shape[1]}")
    with torch.cuda.device(dev):
        a = _device_rows(rows, dev)
        b = a if cols is rows else _device_rows(cols, dev)
        nbytes = L.ddpm_knn_scratch_bytes(n, m, D, kk)
        if nbytes < 0:
            _lib.check(nbytes, "knn_scratch_bytes")
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        st = _lib.stream_ptr(dev)
        if kk > 0:
            out = torch.empty(n, dtype=torch.float16, device=dev)
            _lib.check(L.ddpm_knn_kth(a.data_ptr(), n, a.stride(0), b.data_ptr(), m, b.stride(0), D, kk,
                                      out.data_ptr(), scratch.data_ptr(), nbytes, st), fn_name)
            return out.cpu()
        r = radii.to(device=dev, dtype=torch.float16).contiguous()
        out = torch.empty(n, dtype=torch.uint8, device=dev)
        _lib.check(L.ddpm_knn_cover(a.data_ptr(), n, a.stride(0), b.data_ptr(), m, b.stride(0), D, r.data_ptr(),
                                    out.data_ptr(), scratch.data_ptr(), nbytes, st), fn_name)
        return out.cpu().bool()


class ManifoldBuilder:
    """precision_recall.py:62-174.  Features come from ``features`` (any tensor, cast to fp16 as upstream, :141) or are
    extracted with VGG16 from a map-style dataset, a uint8 array / tensor / ``.npy`` / ``.pt`` path, or
    ``to_uint8(model.sample_x(n))``; a subset of ``max_sample_size`` rows is drawn with
    ``np.random.seed(random_state); np.random.choice(...)`` as upstream.  ``kth`` holds the fp16 radii of the
    ``nhood_size``-th neighbour (the point itself counted as its own nearest)."""

    def __init__(
            self,
            data=None,
            model=None,
            features=None,
            extr_batch_size=128,
            max_sample_size=50000,
            nhood_size=3,
            row_batch_size=10000,
            col_batch_size=10000,
            random_state=1234,
            num_workers=0,
            device=torch.device("cpu")
    ):
        # Upstream sets op_device only on the extraction branch (:126), so ManifoldBuilder(features=...) raises
        # AttributeError in compute_distance.  The evident intent, kept here: the (first) device of ``device``.
        self.op_device = _op_device(device)
        if features is None:
            features = self._extract(data, model, extr_batch_size, max_sample_size, random_state, num_workers, device)
        else:
            assert isinstance(features, torch.Tensor) and features.grad_fn is None
        features = features.to(torch.float16)

        self.nhood_size = nhood_size
        self.row_batch_size = row_batch_size
        self.col_batch_size = col_batch_size
        self.device = device

        self.features = features
        self.kth = self.compute_kth(features)

    @staticmethod
    def _batches(data, model, extr_batch_size, max_sample_size, random_state, num_workers):
        n_batches = math.ceil(max_sample_size / extr_batch_size)
        if model is not None:                                   # :110-116
            for i in range(n_batches):
                n = max_sample_size - extr_batch_size * i if i == n_batches - 1 else extr_batch_size
                yield to_uint8(model.sample_x(n))
            return
        # Upstream tests for a map-style dataset first (:78), which a str also passes: a .npy / .pt path then reaches the
        # DataLoader as a sequence of characters and fails.  The evident intent, kept here: paths take the array branch.
        # (Arrays and tensors take the dataset branch upstream; both branches draw the same rows in the same order.)
        if not isinstance(data, str) and hasattr(data, "__getitem__") and hasattr(data, "__len__"):   # :78-94
            if len(data) > max_sample_size:
                np.random.seed(random_state)
                data = Subset(data, indices=torch.as_tensor(np.random.choice(len(data), size=max_sample_size, replace=False)))
            loader = DataLoader(data, batch_size=extr_batch_size, shuffle=False, num_workers=num_workers,
                                drop_last=False, pin_memory=True)
            for x in loader:
                yield x[0] if isinstance(x, (list, tuple)) else x
            return
        assert isinstance(data, (np.ndarray, torch.Tensor, str))      # :95-109
        if isinstance(data, str) and os.path.exists(data):
            ext = data.rsplit(".", 1)[-1]
            if ext == "npy":
                data = np.load(data)
            elif ext == "pt":
                data = torch.load(data)
        data = torch.as_tensor(data)
        assert data.dtype == torch.uint8
        if data.shape[0] > max_sample_size:
            np.random.seed(random_state)
            data = data[torch.as_tensor(np.random.choice(data.shape[0], size=max_sample_size, replace=False))]
        for i in range(n_batches):
            yield data[i * extr_batch_size: max_sample_size if i == n_batches - 1 else (i + 1) * extr_batch_size]

    def _extract(self, data, model, extr_batch_size, max_sample_size, random_state, num_workers, device):
        batches = self._batches(data, model, extr_batch_size, max_sample_size, random_state, num_workers)
        if isinstance(device, (list, tuple)):                  # :127-132: DataParallel over the listed devices
            extractor = nn.DataParallel(VGGFeatureExtractor().to(device[0]), device_ids=list(device))
            input_device = "cpu"
        else:
            extractor = VGGFeatureExtractor().to(device)
            input_device = device
        out = []
        with torch.inference_mode():
            for x in batches:
                out.append(extractor(x.to(input_device)).cpu())
        return torch.cat(out, dim=0)

    def compute_distance(self, row_features, col_features):
        return compute_distance(row_features, col_features, row_batch_size=self.row_batch_size,
                                col_batch_size=self.col_batch_size, device=self.op_device)

    def compute_kth(self, row_features: torch.Tensor, col_features: torch.Tensor = None):
        """:156-164: for each row, the (nhood_size + 1)-th smallest distance to all columns (its own row included when
        ``col_features`` is None), fp16 on the CPU."""
        if col_features is None:
            col_features = row_features
        dev = _cuda_device(self.op_device)
        kk = _check_nhood(self.nhood_size, col_features.shape[0], dev is not None)
        if dev is not None:
            return _native("ManifoldBuilder.compute_kth", row_features, col_features, kk, None, dev)
        kth = []
        for rb in row_features.split(self.row_batch_size, dim=0):
            d = self.compute_distance(row_features=rb, col_features=col_features)
            kth.append(d.to(torch.float32).kthvalue(kk, dim=1).values.to(torch.float16))
        return torch.cat(kth)

    def save(self, fpath):
        save_dir = os.path.dirname(fpath)
        if not os.path.exists(save_dir):
            os.makedirs(save_dir)
        torch.save(self.manifold, fpath)

    @property
    def manifold(self):
        return Manifold(features=self.features, kth=self.kth)


def calc_pr(manifold_1: Manifold, manifold_2: Manifold, row_batch_size: int, col_batch_size: int, device):
    """precision_recall.py:177-206.  manifold_1: generated (features, kth); manifold_2: real.  Precision = fraction of
    generated points inside some real point's k-NN ball, recall the converse; each a 0-dim fp32 CPU tensor computed as
    upstream, ``torch.cat(pred).to(torch.float32).mean()``."""
    f1, k1 = _fields(manifold_1)
    f2, k2 = _fields(manifold_2)
    op_device = _op_device(device)
    dev = _cuda_device(op_device)
    if dev is not None:
        precision = _native("calc_pr", f1, f2, 0, k2, dev).to(torch.float32).mean()
        recall = _native("calc_pr", f2, f1, 0, k1, dev).to(torch.float32).mean()
        return precision, recall

    def coverage(probes, support, radii):
        pred = []
        for pb in probes.split(row_batch_size):
            d = compute_distance(pb, support, row_batch_size=row_batch_size, col_batch_size=col_batch_size, device=op_device)
            pred.append((d <= radii.unsqueeze(0)).any(dim=1))
        return torch.cat(pred).to(torch.float32).mean()

    return coverage(f1, f2, k2), coverage(f2, f1, k1)
