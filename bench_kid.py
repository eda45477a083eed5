"""Kernel Inception Distance on one H100: native ``ddpm_kid`` against numpy fp64 on the CPU (the torch-fidelity route) and torch fp64
on the same GPU, on the same features and subsets.

    python bench_kid.py [--rows 50000] [--dim 2048] [--subsets 100] [--subset-size 1000] [--reps 3] [--out-dir DIR]

Two seeded Gaussian feature sets of ``rows`` x ``dim`` fp32 (the second with a mean shift of 0.05), the default kernel (degree 3,
gamma = 1 / dim, coef0 = 1) and the subsets ``calc_kid`` draws (seed 1234).  The three routes run alternately ``reps`` times and
each reports its median; every route ends with its result on the host, so each time is wall-clock to a finished result.  Nothing is
written outside ``--out-dir`` (default: a temporary directory).  Prints one JSON line per measurement, each with the card name,
power limit and max SM clock (nvidia-smi query):
  * ``kid_native``: ``_kid_native`` (the index check, its copy to the device, the tile and finish kernels, the result's copy back),
    with the work counted as 2 m^2 dim 2 subsets FLOP (the XX and YY upper triangles and all of XY: 2 m^2 kernel entries per
    subset, a multiply-add per feature) and the rate that gives;
  * ``kid_numpy``: ``_kid_numpy`` on fp64 host copies of the features (made before timing);
  * ``kid_torch``: per subset three ``torch.mm`` in fp64 on the gathered rows, the kernel and the sums on the device;
  * ``kid_draw``: drawing the subset indices on the host, which every route needs once and ``calc_kid`` does first;
  * ``kid_diff``: the largest per-subset difference of each route from the native one, against the per-subset bound that
    ``tests/test_kid_gpu.py`` derives (the check fails the run when it is exceeded).
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
sys.path.insert(1, os.path.join(ROOT, "tests"))          # the bound of test_kid_gpu.py


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "sm_max_clock": None}


def torch_route(x, y, idx, degree, gamma, coef0):
    """Per subset: fp64 rows gathered on the device, three torch.mm, the kernel and the sums; mmd2_s to the host at the end."""
    m = idx.shape[2]
    ix = torch.as_tensor(idx[:, 0]).to(x.device).long()
    iy = torch.as_tensor(idx[:, 1]).to(x.device).long()
    out = []
    for s in range(idx.shape[0]):
        a, b = x[ix[s]].double(), y[iy[s]].double()
        kxx = (gamma * torch.mm(a, a.T) + coef0) ** degree
        kyy = (gamma * torch.mm(b, b.T) + coef0) ** degree
        kxy = (gamma * torch.mm(a, b.T) + coef0) ** degree
        out.append((kxx.sum() - kxx.trace() + kyy.sum() - kyy.trace()) / (m * (m - 1)) - 2 * kxy.sum() / (m * m))
    return torch.stack(out).cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50000)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--subsets", type=int, default=100)
    ap.add_argument("--subset-size", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_kid"))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_kid.py measures on a CUDA device"
    os.makedirs(a.out_dir, exist_ok=True)
    from ddpm_torch_b200 import _lib, metrics as M
    from test_kid_gpu import bound
    _lib.runtime_check()
    info = card()
    lines = []

    def emit(d):
        d.update(card=info)
        lines.append(d)
        print(json.dumps(d), flush=True)

    dev = torch.device("cuda", 0)
    n, d, S, m = a.rows, a.dim, a.subsets, a.subset_size
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, d, device="cuda", generator=g)
    y = torch.randn(n, d, device="cuda", generator=g) + 0.05
    xh, yh = x.double().cpu().numpy(), y.double().cpu().numpy()
    degree, gamma, coef0 = 3, 1.0 / d, 1.0
    t = time.perf_counter()
    idx = M._kid_indices(n, n, S, m, 1234)
    t_draw = time.perf_counter() - t

    def native():
        mmd, status = M._kid_native(x, y, idx, degree, gamma, coef0, dev)
        assert status == 0
        return mmd
    routes = {"native": native, "numpy": lambda: M._kid_numpy(xh, yh, idx, degree, gamma, coef0),
              "torch": lambda: torch_route(x, y, idx, degree, gamma, coef0)}
    native()                                            # warm-up: module load, cuBLAS handles
    torch_route(x, y, idx[:1], degree, gamma, coef0)
    times = {k: [] for k in routes}
    res = {}
    for _ in range(a.reps):
        for k, fn in routes.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            res[k] = fn()
            times[k].append(time.perf_counter() - t)
    med = {k: float(np.median(v)) for k, v in times.items()}
    flop = 2.0 * m * m * d * 2 * S
    emit({"metric": "kid_native", "rows": n, "dim": d, "subsets": S, "subset_size": m, "seconds": med["native"],
          "all_seconds": times["native"], "flop": flop, "fp64_tflops": flop / med["native"] / 1e12,
          "mean": float(np.mean(res["native"])), "std": float(np.std(res["native"]))})
    for k in ("numpy", "torch"):
        emit({"metric": f"kid_{k}", "rows": n, "dim": d, "subsets": S, "subset_size": m, "seconds": med[k], "all_seconds": times[k],
              "native_speedup": med[k] / med["native"], "mean": float(np.mean(res[k])), "std": float(np.std(res[k]))})
    emit({"metric": "kid_draw", "rows": n, "subsets": S, "subset_size": m, "seconds": t_draw})
    bd = bound(x, y, idx, degree, gamma, coef0)
    diff = {k: float(np.max(np.abs(res[k] - res["native"]))) for k in ("numpy", "torch")}
    ratio = {k: float(np.max(np.abs(res[k] - res["native"]) / bd)) for k in ("numpy", "torch")}
    emit({"metric": "kid_diff", "max_abs_diff": diff, "max_ratio_to_bound": ratio, "bound_max": float(bd.max()),
          "mmd2_range": [float(res["native"].min()), float(res["native"].max())]})
    with open(os.path.join(a.out_dir, "bench_kid.json"), "w") as f:
        json.dump(lines, f, indent=1)
    assert max(ratio.values()) <= 1.0, ratio


if __name__ == "__main__":
    main()
