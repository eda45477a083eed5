"""Density and coverage benchmark (Naeem et al., 2020; ``metrics.calc_dc``) on one GPU.

In one process:
  * the card name, power limit and max SM clock (nvidia-smi query);
  * the native count pass (``ddpm_knn_count``, m generated probes against n real balls) and nearest pass (``ddpm_knn_kth`` with
    kk = 1, n real rows against m generated), each timed alone with CUDA events after warm-up, with TFLOP/s from the GEMM's
    2 M N D against the 989 TFLOP/s fp16 data-sheet rate;
  * ``calc_dc`` end to end from CPU fp16 features, host-to-device copies included;
  * a torch baseline on the same card: blockwise fp32 ``torch.cdist``, rounded to fp16, the strict compare against the radii, the
    per-row count and the per-column min, all kept on the device;
  * density and coverage of both routes, and the fraction of pair decisions and of coverage rows that the accumulation bound of
    tests/test_dc_gpu.py leaves borderline (fp64 distances).
The real radii are the native ``ManifoldBuilder(nhood_size=k).kth``.  Features are those of bench_pr.py: seeded, VGG-like (relu of
a rank-16 projection of N(0, 1) latents), the generated set's latents shifted and widened by 15 %.  Writes
<out-dir>/bench_dc.json (default: a directory under the system temp dir) and prints it as one line.

    python bench_dc.py --n 50000 --m 50000 --dim 4096 --nhood 3 [--out-dir DIR]
"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_pr import PEAK_TFLOPS, card, event_ms, features, wall  # noqa: E402


def torch_dc(real, fake, radii, k, block=4096):
    """The baseline: fp32 cdist blocks of generated rows against all real rows, on the device."""
    x = real.float()
    r = radii.float()
    total = torch.zeros((), dtype=torch.int64, device=x.device)
    near = torch.full((x.shape[0],), float("inf"), device=x.device)
    for yb in fake.float().split(block):
        d = torch.cdist(yb, x).half().float()
        total += (d < r[None]).sum()
        near = torch.minimum(near, d.min(0).values)
    return total, (near < r).sum()


def borderline(real, fake, radii, block=2048):
    """Fractions of (pair decisions, coverage rows) that the bound E = (3 D + 3) u (|a|^2 + |b|^2) can flip."""
    U, D = 2.0 ** -24, real.shape[1]
    x = real.double()
    nx = (x * x).sum(1)
    rf = radii.float()
    pairs = 0
    some_in = torch.zeros(x.shape[0], dtype=torch.bool, device=x.device)
    maybe_any = torch.zeros_like(some_in)
    for yb in fake.split(block):
        y = yb.double()
        ny = (y * y).sum(1)
        d2 = (ny[:, None] + nx[None] - 2 * y @ x.T).clamp_min(0)
        e = (3 * D + 3) * U * (ny[:, None] + nx[None])
        inside = ((d2 + e).sqrt().float().half().float() * (1 + 2.0 ** -10)) < rf[None]
        maybe = ((d2 - e).clamp_min(0).sqrt().float().half().float() * (1 - 2.0 ** -10)) < rf[None]
        pairs += int((maybe & ~inside).sum())
        some_in |= inside.any(0)
        maybe_any |= maybe.any(0)
    return pairs / (fake.shape[0] * real.shape[0]), float((maybe_any & ~some_in).double().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000, help="real features")
    ap.add_argument("--m", type=int, default=50000, help="generated features")
    ap.add_argument("--dim", type=int, default=4096)
    ap.add_argument("--nhood", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-check", action="store_true", help="skip the fp64 borderline count")
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_dc"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dc.py measures on a CUDA device; none is present")
    from ddpm_torch_b200 import _lib
    from ddpm_torch_b200 import metrics as M
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, m, D, k = a.n, a.m, a.dim, a.nhood
    real, fake = features(n, m, D)
    res = {"card": card(), "n": n, "m": m, "dim": D, "nhood": k}
    kth = M.ManifoldBuilder(features=real, nhood_size=k, device=dev).kth

    # the two passes alone, on device-resident features
    L = _lib.lib()
    R, F, rad = real.to(dev), fake.to(dev), kth.to(dev)
    st = _lib.stream_ptr(dev)
    cb = L.ddpm_knn_count_scratch_bytes(m, n, D)
    nb = L.ddpm_knn_scratch_bytes(n, m, D, 1)
    scratch = torch.empty(max(cb, nb), dtype=torch.uint8, device=dev)
    counts = torch.empty(m, dtype=torch.int32, device=dev)
    near = torch.empty(n, dtype=torch.float16, device=dev)
    run_count = lambda: _lib.check(L.ddpm_knn_count(F.data_ptr(), m, D, R.data_ptr(), n, D, D, rad.data_ptr(), counts.data_ptr(),
                                                    scratch.data_ptr(), cb, st), "knn_count")
    run_near = lambda: _lib.check(L.ddpm_knn_kth(R.data_ptr(), n, D, F.data_ptr(), m, D, D, 1, near.data_ptr(),
                                                 scratch.data_ptr(), nb, st), "knn_kth")
    flop = 2.0 * m * n * D
    for name, fn in (("count", run_count), ("nearest", run_near)):
        ms = event_ms(fn, a.reps)
        res[f"{name}_pass_ms"] = ms
        res[f"{name}_pass_tflops"] = flop / ms / 1e9
        res[f"{name}_pass_vs_datasheet"] = flop / ms / 1e9 / PEAK_TFLOPS
    del scratch

    # end to end through the public API, CPU fp16 features in, Python floats out
    run_e2e = lambda: M.calc_dc(fake, (real, kth), k, dev)
    run_e2e()
    el, (dens, cov) = wall(run_e2e)
    res["native_e2e_s"] = el
    res["native_density"], res["native_coverage"] = dens, cov

    # the torch baseline on the same card, features already on the device
    run_torch = lambda: torch_dc(R, F, rad, k)
    res["torch_ms"] = event_ms(run_torch, max(1, a.reps // 5))
    total, covered = run_torch()
    res["torch_density"], res["torch_coverage"] = int(total) / (k * m), int(covered) / n
    res["speedup_vs_torch"] = res["torch_ms"] / (res["count_pass_ms"] + res["nearest_pass_ms"])

    if not a.no_check:
        res["borderline_pair_fraction"], res["borderline_coverage_row_fraction"] = borderline(R, F, rad)
    res["device_error_flag"] = L.ddpm_device_error_flag()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bench_dc.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
