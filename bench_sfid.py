"""sFID on one H100: FID and sFID from one native Inception pass, against FID alone and against the route a user has without it.

    python bench_sfid.py [--rows 50176] [--batch 512] [--out-dir DIR]

Prints one JSON line per measurement, each with the card name, power limit and max SM clock (nvidia-smi query), over ``rows``
seeded CIFAR-sized images (32 x 32, resized to 299) with seeded Inception weights, ``batch`` images per call, images already on
the device, every time taken to a device synchronise:
  * ``fid_native``: ``InceptionStatistics(spatial=False)`` on the engine, through ``get_statistics()``;
  * ``fid_sfid_native``: ``InceptionStatistics(spatial=True)``, the same pass also folding the 2023 spatial features, through
    both ``get_statistics()`` and ``get_spatial_statistics()``; its overhead over ``fid_native``;
  * ``torch_route``: what a user runs without the spatial tap: the cuDNN forward with the spatial features read out of Mixed_6d,
    fp64 sums and X^T X of both feature sets with torch on the GPU, the covariances on the host, then ``scipy.linalg.sqrtm`` for
    the sFID at D = 2023 (timed separately, then added);
  * ``calc_fd``: the distance at D = 2023 on those statistics, native (``ddpm_fid_distance``) against scipy's sqrtm formula;
    ``sfid_*`` are the values of both routes and their difference.
Seeded inputs only; nothing is read or written outside ``--out-dir`` (default: a temporary directory).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "sm_max_clock": None}


def timed(fn, sync=True):
    if sync:
        torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    if sync:
        torch.cuda.synchronize()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50176)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_sfid"))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sfid.py measures on a CUDA device"

    def offline(*args, **kw):
        raise RuntimeError("bench_sfid.py runs on seeded weights and never downloads")
    import requests
    torch.hub.download_url_to_file = torch.hub.load_state_dict_from_url = requests.get = offline
    os.makedirs(a.out_dir, exist_ok=True)
    from ddpm_torch_b200 import _lib, metrics as M
    from ddpm_torch_b200.inception import seeded_state_dict, weights_path
    _lib.runtime_check()
    info = card()
    lines = []

    def emit(d):
        d.update(card=info)
        lines.append(d)
        print(json.dumps(d), flush=True)

    hub = tempfile.TemporaryDirectory()              # the seeded weights (100 MB) are not a result
    torch.hub.set_dir(hub.name)
    os.makedirs(os.path.dirname(weights_path()), exist_ok=True)
    torch.save(seeded_state_dict(0), weights_path())
    n_b = -(-a.rows // a.batch)
    g = torch.Generator(device="cuda").manual_seed(0)
    imgs = [torch.rand(a.batch, 3, 32, 32, device="cuda", generator=g) * 2 - 1 for _ in range(n_b)]
    dev = torch.device("cuda")

    def native(spatial):
        ist = M.InceptionStatistics(device=dev, spatial=spatial)
        ist(imgs[0])                                 # warm-up: pack the weights, size the workspace, load the kernels
        ist.reset()

        def run():
            for x in imgs:
                ist(x)
            return ist.get_statistics(), ist.get_spatial_statistics() if spatial else None
        return timed(run)
    (fid_a, _), t_a = native(False)
    (fid_b, sp_b), t_b = native(True)
    (_, _), t_a2 = native(False)                     # again after (b): the spread of (a)
    t_a = min(t_a, t_a2)
    emit({"metric": "fid_native", "rows": n_b * a.batch, "batch": a.batch, "seconds": t_a, "seconds_repeat": t_a2})
    emit({"metric": "fid_sfid_native", "rows": n_b * a.batch, "batch": a.batch, "seconds": t_b,
          "overhead_over_fid_native": t_b / t_a - 1,
          "pool3_stats_identical_to_fid_native": bool(np.array_equal(fid_a[0], fid_b[0]) and np.array_equal(fid_a[1], fid_b[1]))})

    # (c) the torch route: cuDNN forward with the features read out of Mixed_6d, fp64 moments on the GPU, covariance on the host
    ist = M.InceptionStatistics(device=dev, spatial=True)
    net = ist.model._module
    net.use_engine = False
    with torch.inference_mode():
        net(imgs[0], spatial=True)

    def torch_route():
        sums = [torch.zeros(d, dtype=torch.float64, device=dev) for d in (2048, M.SPATIAL_DIM)]
        grams = [torch.zeros(d, d, dtype=torch.float64, device=dev) for d in (2048, M.SPATIAL_DIM)]
        n = 0
        with torch.inference_mode():
            for x in imgs:
                out, sp = net(x, spatial=True)
                for s, G, f in zip(sums, grams, (out[0].flatten(1), sp)):
                    f = f.double()
                    s += f.sum(0)
                    G.addmm_(f.T, f)
                n += x.shape[0]
        stats = []
        for s, G in zip(sums, grams):
            mean = s / n
            cov = (G - n * torch.outer(mean, mean)) / (n - 1)
            stats.append((mean.cpu().numpy(), cov.cpu().numpy()))
        return stats
    stats_c, t_c = timed(torch_route)
    del ist, net
    torch.cuda.empty_cache()

    # calc_fd at D = 2023: the native spatial statistics against the torch route's with the mean moved, a non-zero sFID
    mu1, s1 = sp_b
    mu2, s2 = stats_c[1]
    mu2 = mu2 * 1.05 + 0.01
    M.frechet_distance_native(mu1, s1, mu2, s2, "cuda")
    (fd, fi), t_fd = timed(lambda: M.frechet_distance_native(mu1, s1, mu2, s2, "cuda"))
    (fd2, _), t_fd2 = timed(lambda: M.frechet_distance_native(mu1, s1, mu2, s2, "cuda"))
    ref_fd, t_sqrtm = timed(lambda: M.calculate_frechet_distance(mu1, s1, mu2, s2), sync=False)
    emit({"metric": "torch_route", "rows": n_b * a.batch, "batch": a.batch, "forward_and_moments_s": t_c, "sqrtm_fd_s": t_sqrtm,
          "seconds": t_c + t_sqrtm, "torch_cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
          "speedup_of_fid_sfid_native": (t_c + t_sqrtm) / (t_b + min(t_fd, t_fd2)),
          "max_abs_spatial_cov_diff_vs_native": float(np.abs(stats_c[1][1] - s1).max()),
          "max_abs_spatial_cov": float(np.abs(s1).max())})
    emit({"metric": "calc_fd", "dim": M.SPATIAL_DIM, "native_s": min(t_fd, t_fd2), "scipy_sqrtm_s": t_sqrtm,
          "sfid_native": float(fd), "sfid_scipy": float(ref_fd), "abs_diff": abs(float(fd) - float(ref_fd)),
          "sweeps": fi["sweeps"]})
    hub.cleanup()
    with open(os.path.join(a.out_dir, "bench_sfid.json"), "w") as f:
        json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
