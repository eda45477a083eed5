"""The evaluation metrics of ``ddpm_torch/metrics``: improved precision and recall (Kynkäänniemi et al., 2019) of
``precision_recall.py`` with its k-NN half on the engine, density and coverage (Naeem et al., 2020; ``calc_dc``, see its
section) on the same real manifold, FID (``fid_score.py``, ``__init__.py``'s ``Evaluator``) with its
statistics and Fréchet distance on the engine (see the FID section below; sFID's spatial statistics come from the same pass with
``InceptionStatistics(spatial=True)``), and the Inception Score (``InceptionScore``, ``calc_is``)
and the Kernel Inception Distance (``KernelInceptionDistance``, ``calc_kid``; see their sections), which the reference does not have.

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
import torch.nn.functional as F
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


# ================================================================================================ density and coverage
# Naeem et al. (2020), "Reliable Fidelity and Diversity Metrics for Generative Models": with X the N real features, Y the M
# generated ones, r_i the real manifold's fp16 radius (the k-th neighbour of X_i within X, X_i itself excluded:
# ManifoldBuilder(nhood_size=k).kth) and d = fp16_rn(sqrt_rn(d2)) on the fp16 features as stored (the convention of calc_pr),
#   density  = 1 / (k M) * sum_j #{i : d(Y_j, X_i) < r_i}      (may exceed 1)
#   coverage = 1 / N * #{i : min_j d(X_i, Y_j) < r_i}.
# Both comparisons are strict, unlike calc_pr's `<=`: a radius of 0 (duplicated real points), a negative radius or NaN holds
# nothing; +inf holds every point whose fp16 distance is finite.  fp16 o sqrt is monotone, so coverage is decided by the nearest
# generated point alone.
# * CUDA ``device``: ``ddpm_knn_count`` (the k-NN GEMM with a counting epilogue, csrc/knn.cuh) gives the [M] counts and
#   ``ddpm_knn_kth`` with kk = 1 (rows real, columns generated) the [N] nearest distances; only those come back to the host.
# * CPU ``device``: the same recipe blockwise in torch, d2 in fp64 from the fp16 features, rounded to fp32, then fp32 sqrt and fp16,
#   with no M x N matrix held.

def _native_count(probes, support, radii, dev):
    """``ddpm_knn_count`` on ``dev``'s current stream: int32 [n] counts of the balls (``support``, ``radii``) holding each probe,
    as a CPU tensor."""
    L = _lib.lib()
    n, m, D = probes.shape[0], support.shape[0], probes.shape[1]
    with torch.cuda.device(dev):
        a, b = _device_rows(probes, dev), _device_rows(support, dev)
        nbytes = L.ddpm_knn_count_scratch_bytes(n, m, D)
        if nbytes < 0:
            _lib.check(int(nbytes), "knn_count_scratch_bytes")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        r = radii.to(device=dev, dtype=torch.float16).contiguous()
        out = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(L.ddpm_knn_count(a.data_ptr(), n, a.stride(0), b.data_ptr(), m, b.stride(0), D, r.data_ptr(), out.data_ptr(),
                                    scratch.data_ptr(), nbytes, _lib.stream_ptr(dev)), "calc_dc")
        return out.cpu()


def _dc_host(y, x, radii, max_elems=1 << 22):
    """The CPU recipe: (int64 [M] counts of the balls (x, radii) holding each row of y, fp16 [N] distance from each row of x to
    its nearest row of y), one block of y rows against all of x at a time."""
    x64 = x.detach().cpu().to(torch.float16).double()
    nx = (x64 * x64).sum(1)
    rf = radii.cpu().float()
    counts = []
    min_d2 = torch.full((x.shape[0],), float("inf"), dtype=torch.float64)
    for yb in y.detach().cpu().to(torch.float16).split(max(1, max_elems // x.shape[0])):
        y64 = yb.double()
        d2 = ((y64 * y64).sum(1)[:, None] + nx[None, :] - 2.0 * (y64 @ x64.T)).clamp_min(0.0)
        d = d2.float().sqrt().half().float()
        counts.append((d < rf[None, :]).sum(1))
        min_d2 = torch.minimum(min_d2, d2.min(0).values)
    return torch.cat(counts), min_d2.float().sqrt().half()


def calc_dc(manifold_1, manifold_2, nhood_size, device):
    """Density and coverage ``(density, coverage)`` as Python floats, as defined in the section comment above.

    ``manifold_1``: the generated set, a Manifold, a (features, kth) pair or a bare [M, D] tensor (its kth is not used).
    ``manifold_2``: the real manifold, in any format calc_pr takes (a Manifold, the reference's namedtuple, a (features, kth)
    pair).  ``nhood_size``: the k the real radii were built with; it divides the density, so it has no default.  ``device``: a
    CUDA device (or a list, whose first entry is used) runs the native passes on its current stream; a CPU device the torch
    recipe on the host.  ValueError for features that are not 2-D, a feature-dimension mismatch, an empty set,
    ``nhood_size`` < 1 and radii whose length is not N."""
    f1 = manifold_1 if isinstance(manifold_1, torch.Tensor) else _fields(manifold_1)[0]
    f2, radii = _fields(manifold_2)
    if radii is None:
        raise ValueError("the real manifold needs its radii (kth); build it with ManifoldBuilder")
    f1, f2, radii = torch.as_tensor(f1), torch.as_tensor(f2), torch.as_tensor(radii)
    if f1.dim() != 2 or f2.dim() != 2:
        raise ValueError(f"features must be [n, D], got {tuple(f1.shape)} and {tuple(f2.shape)}")
    (m, D), n = f1.shape, f2.shape[0]
    if f2.shape[1] != D:
        raise ValueError(f"feature dimensions differ: {D} and {f2.shape[1]}")
    if m == 0 or n == 0 or D == 0:
        raise ValueError(f"density and coverage need non-empty sets (M = {m}, N = {n}, D = {D})")
    if int(nhood_size) != nhood_size or nhood_size < 1:
        raise ValueError(f"nhood_size must be an integer >= 1, got {nhood_size}")
    if tuple(radii.shape) != (n,):
        raise ValueError(f"the real manifold needs one radius per real feature: {tuple(radii.shape)} radii for N = {n}")
    radii = radii.to(torch.float16)
    dev = _cuda_device(_op_device(device))
    if dev is None:
        counts, nearest = _dc_host(f1, f2, radii)
    else:
        with torch.cuda.device(dev):
            y, x = _device_rows(f1, dev)[:, :D], _device_rows(f2, dev)[:, :D]     # copied once, read by both passes
            counts = _native_count(y, x, radii, dev)
            nearest = _native("calc_dc", x, y, 1, None, dev)
    total = int(counts.to(torch.int64).sum())
    covered = int((nearest.float() < radii.cpu().float()).sum())
    return total / (int(nhood_size) * m), covered / n


# ================================================================================================ FID (fid_score.py)
# * CUDA ``device``: InceptionStatistics keeps fp64 shift / sum / co-moment state on the device and folds each batch of features in
#   with ``ddpm_fid_stats_update`` (a DMMA GEMM, csrc/fid.cuh) on that device's current stream; calc_fd runs ``ddpm_fid_distance``
#   (two one-sided Jacobi eigen-solves and two DMMA GEMMs), with no scipy.linalg.sqrtm.  Only the final statistics and the distance
#   come back to the host.
# * Inception itself runs on the engine whenever ``InceptionV3.native_eligible`` holds (one sm_90 device, eval mode, no gradient;
#   csrc/inception.cuh), and InceptionStatistics then folds the engine's [N, D] global averages in directly.  A device list keeps
#   DataParallel over the torch modules, as upstream.
# * CPU ``device``: the reference's numpy formulas.
# Three upstream bugs are fixed, each next to its code: sqrtm's removed ``disp`` keyword (calculate_frechet_distance), numpy
# features handed to adaptive_avg_pool2d for activation_dim != 2048 (InceptionStatistics.forward), and the empty last batch of
# Evaluator.eval when the batch size divides the total.

from .inception import InceptionV3, FID_WEIGHTS_URL, SPATIAL_CHANNELS  # noqa: E402

IMAGE_RES = 299
SPATIAL_DIM = 17 * 17 * SPATIAL_CHANNELS      # sFID's features per image: Mixed_6d is 17 x 17 at 299 x 299
FID_STATUS = {1: "a non-finite input", 2: "sigma1 (mean1's covariance) is not positive semi-definite",
              3: "sigma2 (mean2's covariance) is not positive semi-definite",
              4: "the eigen-solve of sigma1 did not converge", 5: "the eigen-solve of L^T sigma2 L did not converge"}
FID_NEG_TOL = 1e-6            # csrc/fid.cuh: lam_min < -1e-6 lam_max is not rounding


class InceptionStatistics(nn.Module):
    """fid_score.py:79-147: mean and covariance of the Inception features of every batch passed to ``forward``.

    On a CUDA ``device`` (or the first device of a list, where Inception runs under ``DataParallel`` as upstream) the statistics
    live in the native fp64 state on that device; on the CPU they follow the reference's per-batch ``np.cov`` and merge.
    ``get_statistics()`` returns numpy fp64 ``(mean, cov)`` with cov divided by ``count - 1``; ``running_mean`` /
    ``running_var`` are the population values (read-only).

    With ``spatial=True`` every ``forward`` also folds sFID's 2023 spatial features (``inception.spatial_features``: channels
    0..6 of Mixed_6d's output at 17 x 17, NHWC order) into a second set of statistics, from the same Inception pass, and
    ``get_spatial_statistics()`` returns them like ``get_statistics()``.  sFID is then
    ``calc_fd(*gen.get_spatial_statistics(), *real.get_spatial_statistics())``.  The features follow the guided-diffusion
    evaluator's ``mixed_6/conv:0[..., :7]``; that TensorFlow tensor is assumed to be this one, which has not been verified, so
    the values are meant to be comparable to ADM's sFID but have not been checked against it.  ``activation_dim`` 64 and 192
    stop before Mixed_6d and refuse ``spatial=True``."""

    def __init__(self, input_transform=lambda x: x, activation_dim=2048, device=torch.device("cpu"), spatial=False):
        super().__init__()
        if spatial and InceptionV3.BLOCK_INDEX_BY_DIM.get(activation_dim, 3) < 2:
            raise ValueError(f"spatial=True needs Mixed_6d, which activation_dim {activation_dim} stops before (use 768 or 2048)")
        self.input_transform = input_transform
        self.activation_dim = activation_dim
        self.device = device
        self.spatial = bool(spatial)
        self.model = self.load_model()
        self._dev = _cuda_device(_op_device(device))
        self.count = 0
        self._dims = (activation_dim, SPATIAL_DIM) if self.spatial else (activation_dim,)
        if self._dev is not None:
            self._states = []
            for D in self._dims:
                nbytes = _lib.lib().ddpm_fid_stats_bytes(D)
                _lib.check(0 if nbytes > 0 else int(nbytes), "fid_stats_bytes")
                self._states.append(torch.zeros(nbytes, dtype=torch.uint8, device=self._dev))
        else:
            self._moments = [(np.zeros((D,), dtype=np.float64), np.zeros((D, D), dtype=np.float64)) for D in self._dims]
            self._mean, self._var = self._moments[0]

    def load_model(self):
        model = InceptionV3([InceptionV3.BLOCK_INDEX_BY_DIM[self.activation_dim]])
        model.eval()
        model.requires_grad_(False)
        extractor = _FirstOutput(model, spatial=self.spatial)
        if isinstance(self.device, (list, tuple)):
            model.use_engine = False                           # under DataParallel, on torch, as upstream
            model.to(self.device[0])
            return nn.DataParallel(extractor, device_ids=list(self.device))
        return extractor.to(self.device)

    def forward(self, x):
        x = self.input_transform(x)
        with torch.inference_mode():
            net = self.model._module if isinstance(self.model, _FirstOutput) else None
            if self._dev is not None and net is not None and net.native_eligible(x):
                # the engine's global average of the last block, [N, D] rows fed to the statistics as they are (and with
                # spatial, the engine's [N, 2023] spatial features of the same pass)
                out = net.forward_native(x, pooled=True, spatial=self.spatial)
                self._fold(*(out if self.spatial else (out,)))
                return
            act = self.model(x)
            if self.spatial:
                act, sp = act
            # Upstream pools after .cpu().numpy(), and adaptive_avg_pool2d refuses a numpy array: activation_dim 64 / 192 / 768
            # raised TypeError.  Pooled here, on the features' own device, before they leave it.
            if act.shape[2] != 1 or act.shape[3] != 1:
                act = F.adaptive_avg_pool2d(act, (1, 1))
            act = act.flatten(1)
        n = act.shape[0]
        if n == 0:
            return
        feats = (act, sp) if self.spatial else (act,)
        if self._dev is not None:
            self._fold(*feats)
            return
        for (m, v), f in zip(self._moments, feats):
            self._merge(m, v, f.cpu().numpy())
        self.count += n

    def _merge(self, m, v, act):
        """fid_score.py:116-135: the batch's np.cov (ddof 0) merged into the running mean m and population covariance v."""
        n = act.shape[0]
        mean = np.mean(act, axis=0, dtype=np.float64)
        var = np.cov(act, rowvar=False, ddof=0, dtype=np.float64)
        alpha = n / (self.count + n)
        if self.count == 0:
            m += mean
            v += var
        else:
            diff = mean - m
            m += alpha * diff
            v += alpha * (var - v)
            v += alpha * (1 - alpha) * np.outer(diff, diff)

    def _fold(self, *feats):
        """Each [n, D] batch into its native state (pool3, then the spatial features)."""
        n = feats[0].shape[0]
        with torch.cuda.device(self._dev):
            for state, D, act in zip(self._states, self._dims, feats):
                f = act.to(device=self._dev, dtype=torch.float32).contiguous()
                _lib.check(_lib.lib().ddpm_fid_stats_update(state.data_ptr(), D, f.data_ptr(), n, f.stride(0),
                                                            _lib.stream_ptr(self._dev)), "InceptionStatistics")
        self.count += n

    def _native_stats(self, ddof, which=0):
        D = self._dims[which]
        with torch.cuda.device(self._dev):
            mean = torch.empty(D, dtype=torch.float64, device=self._dev)
            cov = torch.empty(D, D, dtype=torch.float64, device=self._dev)
            _lib.check(_lib.lib().ddpm_fid_stats_finalize(self._states[which].data_ptr(), D, self.count, ddof, mean.data_ptr(),
                                                          cov.data_ptr(), _lib.stream_ptr(self._dev)), "InceptionStatistics")
            return mean.cpu().numpy(), cov.cpu().numpy()

    @property
    def running_mean(self):
        if self._dev is None:
            return _readonly(self._mean)
        if self.count == 0:
            return _readonly(np.zeros(self.activation_dim))
        return _readonly(self._native_stats(0)[0])

    @property
    def running_var(self):
        if self._dev is None:
            return _readonly(self._var)
        if self.count == 0:
            return _readonly(np.zeros((self.activation_dim, self.activation_dim)))
        return _readonly(self._native_stats(0)[1])

    def get_statistics(self):
        assert self.count > 1, "Count must be greater than 1!"
        if self._dev is not None:
            return self._native_stats(1)
        return self._mean.copy(), self._var.copy() * self.count / (self.count - 1)

    def get_spatial_statistics(self):
        """sFID's statistics (``spatial=True``): numpy fp64 ``(mean [2023], cov [2023, 2023])``, cov divided by ``count - 1``."""
        if not self.spatial:
            raise RuntimeError("get_spatial_statistics needs InceptionStatistics(spatial=True)")
        assert self.count > 1, "Count must be greater than 1!"
        if self._dev is not None:
            return self._native_stats(1, which=1)
        m, v = self._moments[1]
        return m.copy(), v.copy() * self.count / (self.count - 1)

    def reset(self):
        if self._dev is not None:
            for s in self._states:
                s.zero_()
        else:
            for m, v in self._moments:
                m.fill(0)
                v.fill(0)
        self.count = 0


class _FirstOutput(nn.Module):
    """The module's first output; with ``spatial`` the pair (first output, sFID's spatial features)."""
    def __init__(self, module, spatial=False):
        super().__init__()
        self._module = module
        self.spatial = spatial

    def forward(self, x):
        if self.spatial:
            out, sp = self._module(x, spatial=True)
            return out[0], sp
        return self._module(x)[0]


def _readonly(a):
    a = a.view()
    a.flags.writeable = False
    return a


# fid_score.py:150-158
PRE_COMPUTED_LIST = {
    "celeba": "https://github.com/tqch/VAEGAN/releases/download/precomputed_statistics_celeba/fid_stats_celeba_148x148.npz",
    "lsun_bedroom": "http://bioinf.jku.at/research/ttur/ttur_stats/fid_stats_lsun_train.npz",
    "cifar10": "http://bioinf.jku.at/research/ttur/ttur_stats/fid_stats_cifar10_train.npz",
    "svhn": "http://bioinf.jku.at/research/ttur/ttur_stats/fid_stats_svhn_train.npz",
    "imagenet_train": "http://bioinf.jku.at/research/ttur/ttur_stats/fid_stats_imagenet_train.npz",
    "imagenet_valid": "http://bioinf.jku.at/research/ttur/ttur_stats/fid_stats_imagenet_valid.npz",
}


def get_precomputed(dataset, download_dir="precomputed"):
    """fid_score.py:161-183: ``(mu, sigma)`` of the dataset's precomputed statistics, read from ``download_dir`` and fetched
    into it only when the file is absent (``download_dir=None``: fetched into memory)."""
    url = PRE_COMPUTED_LIST.get(dataset, f"fid_stats_{dataset}.npz")
    name = os.path.basename(url)
    if download_dir is None:
        import io
        import requests
        src = io.BytesIO(requests.get(url).content)
    else:
        src = os.path.join(download_dir, name)
        if not os.path.exists(src):
            import requests
            os.makedirs(download_dir, exist_ok=True)
            r = requests.get(url, timeout=120)
            assert r.status_code == 200
            with open(src, "wb") as f:
                f.write(r.content)
    data = np.load(src)
    return data["mu"], data["sigma"]


def _sqrtm(a):
    """scipy.linalg.sqrtm(a) as a matrix.  Upstream calls ``sqrtm(..., disp=False)``, a keyword SciPy has removed (1.18 raises
    TypeError), so calc_fd did not run at all; with that keyword gone the matrix is the whole return value."""
    from scipy import linalg
    try:
        return linalg.sqrtm(a, disp=False)[0]
    except TypeError:
        return linalg.sqrtm(a)


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """fid_score.py:269-323 on the CPU: ||mu1 - mu2||^2 + tr(sigma1 + sigma2 - 2 sqrtm(sigma1 sigma2)), with ``eps`` added to both
    diagonals when the product's square root is not finite, and a ValueError when it has a significant imaginary part."""
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    assert mu1.shape == mu2.shape, "Training and test mean vectors have different lengths"
    assert sigma1.shape == sigma2.shape, "Training and test covariances have different dimensions"
    diff = mu1 - mu2
    covmean = _sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        print(f"fid calculation produces singular product; adding {eps} to diagonal of cov estimates")
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = _sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(covmean.imag))))
        covmean = covmean.real
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean)


def _fd_device(args, device):
    if device is not None:
        return _cuda_device(_op_device(device))
    for a in args:
        if isinstance(a, torch.Tensor) and a.is_cuda:
            return a.device
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None


def frechet_distance_native(mean1, var1, mean2, var2, device):
    """``ddpm_fid_distance`` on ``device``'s current stream.  Returns ``(fd, info)``: ``info`` holds the status, the sweep counts of
    both eigen-solves, the most negative eigenvalue of sigma1 and of M = L^T sigma2 L relative to their largest, and
    tr sqrt(sigma1 sigma2).  Raises ValueError for non-finite or non-PSD input, RuntimeError when an eigen-solve did not converge."""
    dev = _cuda_device(device)
    L = _lib.lib()
    with torch.cuda.device(dev):
        t = [torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to(device=dev, dtype=torch.float64)
             for a in (mean1, var1, mean2, var2)]
        mu1, s1, mu2, s2 = (t[0].reshape(-1).contiguous(), t[1].reshape(t[1].shape[0] if t[1].dim() else 1, -1).contiguous(),
                            t[2].reshape(-1).contiguous(), t[3].reshape(t[3].shape[0] if t[3].dim() else 1, -1).contiguous())
        assert mu1.shape == mu2.shape, "Training and test mean vectors have different lengths"
        assert s1.shape == s2.shape, "Training and test covariances have different dimensions"
        D = mu1.shape[0]
        if s1.shape != (D, D):
            raise ValueError(f"covariances must be {D} x {D} to match the means, got {tuple(s1.shape)}")
        nbytes = L.ddpm_fid_distance_scratch_bytes(D)
        if nbytes < 0:
            _lib.check(int(nbytes), "fid_distance_scratch_bytes")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.full((8,), float("nan"), dtype=torch.float64, device=dev)
        _lib.check(L.ddpm_fid_distance(mu1.data_ptr(), s1.data_ptr(), mu2.data_ptr(), s2.data_ptr(), D, out.data_ptr(),
                                       scratch.data_ptr(), nbytes, _lib.stream_ptr(dev)), "calc_fd")
        o = out.cpu().numpy()
    status = int(o[1])
    info = {"status": status, "sweeps": (int(o[2]), int(o[3])), "min_ratio": (float(o[4]), float(o[5])), "tr_sqrt": float(o[6])}
    if status in (1, 2, 3):
        ratio = f" (lam_min / lam_max = {o[3 + status]:.3e}, below -{FID_NEG_TOL:g})" if status > 1 else ""
        raise ValueError(f"calc_fd: {FID_STATUS[status]}{ratio}")
    if status:
        raise RuntimeError(f"calc_fd: {FID_STATUS[status]}")
    return np.float64(o[0]), info


def calc_fd(mean1, var1, mean2, var2, eps=1e-6, device=None):
    """fid_score.py:186-187.  On the device of a CUDA tensor argument, on ``device``, or else on the current CUDA device when one
    is present: the native eigenvalue route (``frechet_distance_native``).  ``eps`` is accepted for the reference's signature and
    never needed there: the route takes no square root of a possibly singular product, so there is no diagonal offset to
    retry with.  Non-PSD input raises ValueError, the counterpart of upstream's "Imaginary component" error.  Otherwise (a CPU
    ``device``, or no CUDA device): the reference formula, ``calculate_frechet_distance``.  Returns a numpy float64."""
    dev = _fd_device((mean1, var1, mean2, var2), device)
    if dev is None:
        args = [a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a for a in (mean1, var1, mean2, var2)]
        return calculate_frechet_distance(*args, eps)
    return frechet_distance_native(mean1, var1, mean2, var2, dev)[0]


class Evaluator:
    """metrics/__init__.py:18-53: FID of ``eval_total_size`` samples drawn ``eval_batch_size`` at a time, against the dataset's
    precomputed statistics."""

    def __init__(self, dataset, diffusion=None, eval_batch_size=256, eval_total_size=50000, device=torch.device("cpu")):
        self.diffusion = diffusion
        self.istats = InceptionStatistics(device=device)
        self.eval_batch_size = eval_batch_size
        self.eval_total_size = eval_total_size
        self.device = device
        self.target_mean, self.target_var = get_precomputed(dataset)

    def eval(self, sample_fn, is_leader=True):
        try:
            from tqdm import trange
        except ImportError:
            def trange(n, **kw):
                return range(n)
        if is_leader:
            self.istats.reset()
        fid = None
        num_batches = math.ceil(self.eval_total_size / self.eval_batch_size)
        with trange(num_batches, desc="Evaluating FID", disable=not is_leader) as t:
            for i in t:
                batch_size = self.eval_batch_size
                if i == num_batches - 1:
                    # Upstream takes eval_total_size % eval_batch_size, which is 0 when the batch size divides the total: the
                    # empty batch's NaN mean then turned the running statistics, and the FID, into NaN.
                    batch_size = self.eval_total_size - self.eval_batch_size * (num_batches - 1)
                x = sample_fn(sample_size=batch_size, diffusion=self.diffusion)
                if is_leader:
                    op = _op_device(self.device)
                    self.istats(x.to(op))
                    if i == num_batches - 1:
                        gen_mean, gen_var = self.istats.get_statistics()
                        fid = calc_fd(gen_mean, gen_var, self.target_mean, self.target_var, device=op)
                        t.set_postfix({"fid": fid})
        return {"fid": fid}


# ================================================================================================ Inception Score
# Salimans et al. (2016) as the TensorFlow improved-gan/inception_score.py computes it, which is what papers report: p = softmax over
# all 1008 classes of pool3 . W^T (W the checkpoint's fc.weight, no bias), the N images cut in order into ``splits`` parts, part i
# being rows [i N // splits, (i + 1) N // splits), IS_i = exp(mean_x sum_y p(y|x) (log p(y|x) - log pbar_i(y))), and the mean and
# population std of the IS_i.
# * CUDA ``device``: the logits are a 3xTF32 GEMM (``ddpm_is_logits``, csrc/inception_score.cuh) that stays on the device, and the
#   score is ``ddpm_is_score`` in fp64 with fixed-order reductions, so it is bit-identical however the images were batched.
#   Inception runs on the engine when ``InceptionV3.native_eligible`` holds; a device list runs DataParallel over the torch modules,
#   then the logits and the score on the first device.
# * CPU ``device``: the torch modules, fp32 ``x @ W.T`` and the same formula in numpy fp64.
# Both take log p as z - logsumexp(z) in fp64, where the TF code takes np.log of an fp32 softmax: on well-conditioned logits the two
# agree to rounding, and a saturated row (a p that underflows in fp32) stays finite here.

IS_CLASSES = 1008
IS_FEATURES = 2048
IS_STATUS = {1: "a non-finite logit"}


def _is_pack(fc_weight, dev):
    """fc.weight [1008, 2048] packed on ``dev`` for ``_is_logits`` (``ddpm_is_fc_pack``)."""
    L = _lib.lib()
    with torch.cuda.device(dev):
        w = torch.as_tensor(fc_weight).to(device=dev, dtype=torch.float32).contiguous()
        if tuple(w.shape) != (IS_CLASSES, IS_FEATURES):
            raise ValueError(f"fc weight must be [{IS_CLASSES}, {IS_FEATURES}], got {tuple(w.shape)}")
        packed = torch.empty(L.ddpm_is_fc_packed_bytes(), dtype=torch.uint8, device=dev)
        _lib.check(L.ddpm_is_fc_pack(w.data_ptr(), packed.data_ptr(), _lib.stream_ptr(dev)), "InceptionScore")
    return packed


def _is_logits(packed, feats, dev, ws=None):
    """fp32 [N, 1008] logits on ``dev`` of [N, 2048] features (``ddpm_is_logits``).  ``ws``: a uint8 workspace to reuse when it is
    large enough.  Returns ``(logits, ws)``."""
    L = _lib.lib()
    with torch.cuda.device(dev):
        f = feats.to(device=dev, dtype=torch.float32)
        if f.dim() != 2 or f.shape[1] != IS_FEATURES:
            raise ValueError(f"features must be [N, {IS_FEATURES}], got {tuple(f.shape)}")
        if f.stride(1) != 1 or f.stride(0) < IS_FEATURES:
            f = f.contiguous()
        n = f.shape[0]
        need = L.ddpm_is_logits_workspace_bytes(n)
        if need < 0:
            _lib.check(int(need), "is_logits_workspace_bytes")
        if ws is None or ws.device != dev or ws.numel() < need:
            ws = None
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
        out = torch.empty(n, IS_CLASSES, dtype=torch.float32, device=dev)
        _lib.check(L.ddpm_is_logits(packed.data_ptr(), f.data_ptr(), n, f.stride(0), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                    _lib.stream_ptr(dev)), "InceptionScore")
    return out, ws


def _is_check(n, splits):
    if splits < 1 or n < splits:
        raise ValueError(f"the Inception Score needs 1 <= splits <= N (N = {n}, splits = {splits})")


def _is_numpy(logits, splits):
    z = np.asarray(logits, dtype=np.float64)
    if not np.isfinite(z).all():
        raise ValueError(f"calc_is: {IS_STATUS[1]}")
    m = z.max(axis=1, keepdims=True)
    logp = z - (m + np.log(np.exp(z - m).sum(axis=1, keepdims=True)))
    p = np.exp(logp)
    n = z.shape[0]
    scores = []
    for i in range(splits):
        b, e = i * n // splits, (i + 1) * n // splits
        pbar = p[b:e].mean(axis=0)
        nz = pbar > 0                                     # 0 log 0 = 0
        kl = np.sum(p[b:e] * logp[b:e]) / (e - b) - np.sum(pbar[nz] * np.log(pbar[nz]))
        scores.append(np.exp(kl))
    return scores


def _is_native(logits, splits, dev):
    L = _lib.lib()
    with torch.cuda.device(dev):
        z = torch.as_tensor(logits).to(device=dev, dtype=torch.float32)
        if z.stride(1) != 1 or z.stride(0) < z.shape[1]:
            z = z.contiguous()
        n, c = z.shape
        nbytes = L.ddpm_is_score_scratch_bytes(n, c, splits)
        if nbytes < 0:
            _lib.check(int(nbytes), "is_score_scratch_bytes")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty(splits + 1, dtype=torch.float64, device=dev)
        _lib.check(L.ddpm_is_score(z.data_ptr(), n, c, z.stride(0), splits, out.data_ptr(), scratch.data_ptr(), nbytes,
                                   _lib.stream_ptr(dev)), "calc_is")
        o = out.cpu().numpy()
    status = int(o[splits])
    if status:
        raise ValueError(f"calc_is: {IS_STATUS[status]}")
    return list(o[:splits])


def calc_is(logits, splits=10, device=None):
    """Inception Score ``(mean, std)`` (Python floats) of [N, C] logits (a tensor or an array; C = 1008 for the Inception network),
    cut in order into ``splits`` parts.  On the device of a CUDA tensor, on a CUDA ``device``, or else on the current CUDA device
    when one is present: ``ddpm_is_score``.  Otherwise (a CPU ``device``, or no CUDA device): the same formula in numpy fp64.
    ValueError for N < splits or a non-finite logit."""
    shape = tuple(logits.shape)
    if len(shape) != 2 or shape[1] < 1:
        raise ValueError(f"logits must be [N, C], got {shape}")
    _is_check(shape[0], splits)
    dev = _fd_device((logits,), device)
    if dev is None:
        z = logits.detach().cpu().numpy() if isinstance(logits, torch.Tensor) else logits
        scores = _is_numpy(z, splits)
    else:
        scores = _is_native(logits, splits, dev)
    return float(np.mean(scores)), float(np.std(scores))


class InceptionScore(nn.Module):
    """Inception Score of every batch passed to ``forward`` (see the section comment above), shaped like InceptionStatistics.

    ``forward(x)`` takes images in [-1, 1] after ``input_transform``, of any size (resized to 299 x 299 as for FID), and keeps their
    1008-way logits: on a CUDA ``device`` (or the first device of a list, where Inception runs under ``DataParallel``) fp32 on that
    device, 4 KB per image; on the CPU in host memory.  ``get_score()`` returns ``(mean, std)`` as Python floats; ``reset()`` drops
    the logits.  The fc weights are the checkpoint's (``weights_path()``), read with the network."""

    def __init__(self, splits=10, input_transform=lambda x: x, device=torch.device("cpu")):
        super().__init__()
        self.splits = splits
        self.input_transform = input_transform
        self.device = device
        self.model = self.load_model()
        self._dev = _cuda_device(_op_device(device))
        net = self.model.module._module if isinstance(self.model, nn.DataParallel) else self.model._module
        if self._dev is not None:
            self._packed = _is_pack(net.fc_weight, self._dev)
        else:
            self._fc = net.fc_weight.to(torch.float32)
        self._ws = None
        self._logits = []
        self.count = 0

    def load_model(self):
        model = InceptionV3([3])
        model.eval()
        model.requires_grad_(False)
        extractor = _FirstOutput(model)
        if isinstance(self.device, (list, tuple)):
            model.use_engine = False                           # under DataParallel, on torch, as InceptionStatistics
            model.to(self.device[0])
            return nn.DataParallel(extractor, device_ids=list(self.device))
        return extractor.to(self.device)

    def forward(self, x):
        x = self.input_transform(x)
        with torch.inference_mode():
            net = self.model._module if isinstance(self.model, _FirstOutput) else None
            if self._dev is not None and net is not None and net.native_eligible(x):
                feats = net.forward_native(x, pooled=True)
            else:
                feats = self.model(x).flatten(1)
            n = feats.shape[0]
            if n == 0:
                return
            if self._dev is not None:
                logits, self._ws = _is_logits(self._packed, feats, self._dev, self._ws)
            else:
                logits = feats.to(device="cpu", dtype=torch.float32) @ self._fc.T
            self._logits.append(logits)
        self.count += n

    def get_score(self):
        _is_check(self.count, self.splits)
        if len(self._logits) > 1:
            self._logits = [torch.cat(self._logits)]
        return calc_is(self._logits[0], self.splits, device=self._dev if self._dev is not None else "cpu")

    def reset(self):
        self._logits = []
        self.count = 0


# ================================================================================================ Kernel Inception Distance
# Bińkowski et al. (2018), "Demystifying MMD GANs": the unbiased estimator of the squared MMD with the polynomial kernel
# k(x, y) = (gamma x . y + coef0)^degree (gamma = 1 / d by default), averaged over ``num_subsets`` subsets of ``subset_size`` = m rows
# of each feature set:
#   mmd2_s = (sum_{i != j} k(x_i, x_j) + sum_{i != j} k(y_i, y_j)) / (m (m - 1)) - 2 sum_{i, j} k(x_i, y_j) / m^2,
# and the mean and population std (ddof = 0) of the mmd2_s.  Unlike FID its expectation does not depend on the sample count, so it
# is the metric to compare runs evaluated on a few thousand samples.  Subset s takes ix = rng.choice(n1, m, replace=False), then
# iy = rng.choice(n2, m, replace=False), from one ``np.random.RandomState(seed)``; the indices are drawn on the host, so both paths
# see the same subsets.
# * CUDA ``device``: ``ddpm_kid`` (csrc/kid.cuh), fp64 Gram tiles on the DMMA tensor cores with the kernel and the sums fused in, no
#   m x m matrix in memory, every sum in a fixed order: bit-identical from run to run and however the features were batched.
# * CPU ``device``: the same formula in numpy fp64, the reference the tests compare against.

KID_STATUS = {1: "a non-finite feature or kernel value"}
KID_MAX_DEGREE = 8                                        # csrc/kid.cuh
KID_KERNEL_ARGS = ("degree", "gamma", "coef0", "seed")


def _kid_indices(n1, n2, num_subsets, subset_size, seed):
    """int32 [num_subsets, 2, subset_size]: per subset ix (rows of the first set) then iy (rows of the second), drawn in that order."""
    rng = np.random.RandomState(seed)
    idx = np.empty((num_subsets, 2, subset_size), dtype=np.int32)
    for s in range(num_subsets):
        idx[s, 0] = rng.choice(n1, subset_size, replace=False)
        idx[s, 1] = rng.choice(n2, subset_size, replace=False)
    return idx


def _kid_numpy(x, y, idx, degree, gamma, coef0):
    """mmd2_s per subset in numpy fp64 (features cast to fp64 first)."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    m = idx.shape[2]
    out = np.empty(idx.shape[0])
    with np.errstate(invalid="ignore", over="ignore"):          # a non-finite value is reported by the caller
        for s in range(idx.shape[0]):
            a, b = x[idx[s, 0]], y[idx[s, 1]]
            kxx = (gamma * (a @ a.T) + coef0) ** degree
            kyy = (gamma * (b @ b.T) + coef0) ** degree
            kxy = (gamma * (a @ b.T) + coef0) ** degree
            out[s] = (kxx.sum() - np.trace(kxx) + kyy.sum() - np.trace(kyy)) / (m * (m - 1)) - 2 * kxy.sum() / (m * m)
    return out


def _kid_rows(f, dev):
    f = torch.as_tensor(f).to(device=dev, dtype=torch.float32)
    return f if f.stride(1) == 1 and f.stride(0) >= f.shape[1] else f.contiguous()


def _kid_native(x, y, idx, degree, gamma, coef0, dev):
    """``ddpm_kid`` on ``dev``'s current stream: the numpy array of mmd2_s per subset and the status."""
    L = _lib.lib()
    S, _, m = idx.shape
    idx = np.ascontiguousarray(idx, dtype=np.int32)
    with torch.cuda.device(dev):
        a, b = _kid_rows(x, dev), _kid_rows(y, dev)
        nbytes = L.ddpm_kid_scratch_bytes(S, m)
        if nbytes < 0:
            _lib.check(int(nbytes), "kid_scratch_bytes")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty(S + 3, dtype=torch.float64, device=dev)
        _lib.check(L.ddpm_kid(a.data_ptr(), a.stride(0), a.shape[0], b.data_ptr(), b.stride(0), b.shape[0], a.shape[1],
                              idx.ctypes.data, S, m, degree, gamma, coef0, out.data_ptr(), scratch.data_ptr(), nbytes,
                              _lib.stream_ptr(dev)), "calc_kid")
        o = out.cpu().numpy()
    return o[:S], int(o[S + 2])


def calc_kid(features1, features2, num_subsets=100, subset_size=1000, degree=3, gamma=None, coef0=1., seed=1234, device=None):
    """Kernel Inception Distance ``(mean, std)`` (Python floats) between [n1, d] and [n2, d] features (tensors or arrays), as defined
    in the section comment above.  This follows the unbiased estimator as torch-fidelity and clean-fid compute it (subset MMD^2
    with the cubic polynomial kernel, mean and population std); it has not been checked against either, which are not
    dependencies of this project.  On the device of a CUDA tensor, on a CUDA ``device``, or else on the current CUDA device when one
    is present: ``ddpm_kid``.  Otherwise (a CPU ``device``, or no CUDA device): numpy fp64.  ValueError for inputs that are not 2-D,
    a feature-dimension mismatch or d outside 1..4096, ``subset_size`` outside 2..min(n1, n2), ``num_subsets`` < 1, ``degree``
    outside 1..8, and a non-finite feature in a drawn row or a non-finite kernel value."""
    s1, s2 = tuple(features1.shape), tuple(features2.shape)
    if len(s1) != 2 or len(s2) != 2:
        raise ValueError(f"features must be [n, d], got {s1} and {s2}")
    (n1, d), n2 = s1, s2[0]
    if s2[1] != d:
        raise ValueError(f"feature dimensions differ: {d} and {s2[1]}")
    if not 1 <= d <= 4096:
        raise ValueError(f"the feature dimension must be in 1..4096, got {d}")
    if not 2 <= subset_size <= min(n1, n2):
        raise ValueError(f"the KID needs 2 <= subset_size <= min(n1, n2) (subset_size = {subset_size}, n1 = {n1}, n2 = {n2})")
    if num_subsets < 1:
        raise ValueError(f"num_subsets must be >= 1, got {num_subsets}")
    if int(degree) != degree or not 1 <= degree <= KID_MAX_DEGREE:
        raise ValueError(f"degree must be an integer in 1..{KID_MAX_DEGREE}, got {degree}")
    degree = int(degree)
    gamma = 1.0 / d if gamma is None else float(gamma)
    idx = _kid_indices(n1, n2, num_subsets, subset_size, seed)
    dev = _fd_device((features1, features2), device)
    if dev is None:
        host = [f.detach().cpu().numpy() if isinstance(f, torch.Tensor) else f for f in (features1, features2)]
        mmd = _kid_numpy(host[0], host[1], idx, degree, gamma, float(coef0))
        status = 0 if np.isfinite(mmd).all() else 1
    else:
        mmd, status = _kid_native(features1, features2, idx, degree, gamma, float(coef0), dev)
    if status:
        raise ValueError(f"calc_kid: {KID_STATUS[status]}")
    return float(np.mean(mmd)), float(np.std(mmd))


class KernelInceptionDistance(nn.Module):
    """Kernel Inception Distance of every batch passed to ``forward`` against another feature set (see the section comment above),
    shaped like InceptionScore.

    ``forward(x)`` takes images in [-1, 1] after ``input_transform``, of any size (resized to 299 x 299 as for FID), and keeps their
    2048 pool3 features: on a CUDA ``device`` (or the first device of a list, where Inception runs under ``DataParallel``) fp32 on
    that device, 8 KB per image; on the CPU in host memory.  ``features`` is the [N, 2048] tensor of all of them; ``get_kid(other)``
    returns ``(mean, std)`` against ``other``'s features -- a tensor, an array, or another KernelInceptionDistance (for example real
    images' features computed once and kept with ``torch.save``) -- with the subsets' ix drawn from this set and iy from ``other``;
    ``reset()`` drops the features.  ``kernel_kwargs``: ``degree``, ``gamma``, ``coef0`` and ``seed`` of ``calc_kid``."""

    def __init__(self, num_subsets=100, subset_size=1000, input_transform=lambda x: x, device=torch.device("cpu"), **kernel_kwargs):
        super().__init__()
        unknown = set(kernel_kwargs) - set(KID_KERNEL_ARGS)
        if unknown:
            raise TypeError(f"unexpected keyword arguments {sorted(unknown)}; the kernel takes {', '.join(KID_KERNEL_ARGS)}")
        self.num_subsets = num_subsets
        self.subset_size = subset_size
        self.kernel_kwargs = kernel_kwargs
        self.input_transform = input_transform
        self.device = device
        self.model = self.load_model()
        self._dev = _cuda_device(_op_device(device))
        self._feats = []
        self.count = 0

    def load_model(self):
        model = InceptionV3([3])
        model.eval()
        model.requires_grad_(False)
        extractor = _FirstOutput(model)
        if isinstance(self.device, (list, tuple)):
            model.use_engine = False                           # under DataParallel, on torch, as InceptionStatistics
            model.to(self.device[0])
            return nn.DataParallel(extractor, device_ids=list(self.device))
        return extractor.to(self.device)

    def forward(self, x):
        x = self.input_transform(x)
        with torch.inference_mode():
            net = self.model._module if isinstance(self.model, _FirstOutput) else None
            if self._dev is not None and net is not None and net.native_eligible(x):
                feats = net.forward_native(x, pooled=True)
            else:
                feats = self.model(x).flatten(1)
            n = feats.shape[0]
            if n == 0:
                return
            self._feats.append(feats.to(device=self._dev if self._dev is not None else "cpu", dtype=torch.float32))
        self.count += n

    @property
    def features(self):
        if len(self._feats) > 1:
            self._feats = [torch.cat(self._feats)]
        if not self._feats:
            return torch.empty(0, IS_FEATURES, dtype=torch.float32, device=self._dev if self._dev is not None else "cpu")
        return self._feats[0]

    def get_kid(self, other):
        other = other.features if isinstance(other, KernelInceptionDistance) else other
        return calc_kid(self.features, other, self.num_subsets, self.subset_size,
                        device=self._dev if self._dev is not None else "cpu", **self.kernel_kwargs)

    def reset(self):
        self._feats = []
        self.count = 0


__all__ = ["Manifold", "ManifoldBuilder", "calc_pr", "calc_dc", "compute_distance", "to_uint8", "VGGFeatureExtractor",
           "InceptionV3", "InceptionStatistics", "get_precomputed", "calc_fd", "calculate_frechet_distance", "Evaluator",
           "InceptionScore", "calc_is", "KernelInceptionDistance", "calc_kid"]
