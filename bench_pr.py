"""Precision/recall benchmark (the k-NN half of ``ddpm_torch/metrics/precision_recall.py``) on one GPU.

In one process:
  * the card name, power limit and max SM clock (nvidia-smi query);
  * the native kth pass (``ddpm_knn_kth``, n rows against themselves) and cover pass (``ddpm_knn_cover``, n probes against m
    supports), each timed alone with CUDA events after warm-up, with TFLOP/s from the GEMM's 2 N M D against the 989 TFLOP/s
    fp16 data-sheet rate;
  * end to end through the public API: two ``ManifoldBuilder(features=<CPU fp16>)`` + ``calc_pr``, host-to-device copies
    included;
  * with ``--reference``: the same end-to-end workflow with the staged reference (``oracle/_ref``) on the same card;
  * precision / recall of both, and the native radii and flags against the fp64 recipe at the bench size (radii within the
    accumulation bound of tests/test_pr_gpu.py, flags equal on every probe whose decision that bound cannot flip).
Features are seeded and VGG-like: relu of a rank-16 projection of N(0, 1) latents; the generated set's latents are shifted
and widened by 15 %.  Writes <out-dir>/bench_pr.json (default: a directory under the system temp dir) and prints it as one line.

    python bench_pr.py --n 50000 --m 50000 --dim 4096 --nhood 3 [--reference] [--out-dir DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0       # H100 SXM dense fp16, data sheet (700 W)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:             # the measurement stands without it, but say so
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "sm_max_clock": None}


def features(n, m, dim, seed=0):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(16, dim, generator=g)
    real = torch.relu(torch.randn(n, 16, generator=g) @ W / 4).half()
    fake = torch.relu((torch.randn(m, 16, generator=g) * 1.15 + 0.15) @ W / 4).half()
    return real, fake


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def check_fp64(probes, support, kth_s, flags, kk, dev, block=2048):
    """Native radii of ``support`` and flags of ``probes`` against fp64 distances (the bound E_i of tests/test_pr_gpu.py)."""
    U = 2.0 ** -24
    D = support.shape[1]
    s64 = support.to(dev, torch.float64)
    ns = (s64 * s64).sum(1)
    rf = kth_s.to(dev).float()
    out = dict(kth_outside_bound=0, flags_forced_wrong=0, flags_borderline=0)
    for i in range(0, support.shape[0], block):
        a = s64[i:i + block]
        na = (a * a).sum(1)
        d2 = (na[:, None] + ns[None] - 2 * a @ s64.T).clamp_min(0)
        dk = d2.kthvalue(kk, dim=1).values
        e = (3 * D + 3) * U * (na + ns.max())
        k = kth_s[i:i + block].to(dev).double()
        lo, hi = (dk - e).clamp_min(0).sqrt() * (1 - 2.0 ** -11), (dk + e).sqrt() * (1 + 2.0 ** -11)
        out["kth_outside_bound"] += int(((k < lo) | (k > hi)).sum())
    for i in range(0, probes.shape[0], block):
        a = probes[i:i + block].to(dev, torch.float64)
        na = (a * a).sum(1)
        d2 = (na[:, None] + ns[None] - 2 * a @ s64.T).clamp_min(0)
        e = ((3 * D + 3) * U * (na + ns.max()))[:, None]
        must = (((d2 + e).sqrt().float().half().float() * (1 + 2.0 ** -10)) <= rf[None]).any(1).cpu()
        must_not = ~(((d2 - e).clamp_min(0).sqrt().float().half().float() * (1 - 2.0 ** -10)) <= rf[None]).any(1).cpu()
        f = flags[i:i + block]
        out["flags_forced_wrong"] += int((f & must_not).sum() + (~f & must).sum())
        out["flags_borderline"] += int((~must & ~must_not).sum())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000, help="real (support) features")
    ap.add_argument("--m", type=int, default=50000, help="generated (probe) features")
    ap.add_argument("--dim", type=int, default=4096)
    ap.add_argument("--nhood", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--reference", action="store_true", help="also run the staged reference end to end on the same card")
    ap.add_argument("--no-check", action="store_true", help="skip the fp64 check")
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_pr"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pr.py measures on a CUDA device; none is present")
    from ddpm_torch_b200 import _lib
    from ddpm_torch_b200 import metrics as M
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, m, D, kk = a.n, a.m, a.dim, a.nhood + 1
    real, fake = features(n, m, D)
    res = {"card": card(), "n": n, "m": m, "dim": D, "nhood": a.nhood}

    # the two passes alone, on device-resident features
    L = _lib.lib()
    R, F = real.to(dev), fake.to(dev)
    st = _lib.stream_ptr(dev)
    kb = L.ddpm_knn_scratch_bytes(n, n, D, kk)
    cb = L.ddpm_knn_scratch_bytes(m, n, D, 0)
    scratch = torch.empty(max(kb, cb), dtype=torch.uint8, device=dev)
    kth = torch.empty(n, dtype=torch.float16, device=dev)
    cov = torch.empty(m, dtype=torch.uint8, device=dev)
    run_kth = lambda: _lib.check(L.ddpm_knn_kth(R.data_ptr(), n, D, R.data_ptr(), n, D, D, kk, kth.data_ptr(),
                                                scratch.data_ptr(), kb, st), "knn_kth")
    run_cov = lambda: _lib.check(L.ddpm_knn_cover(F.data_ptr(), m, D, R.data_ptr(), n, D, D, kth.data_ptr(), cov.data_ptr(),
                                                  scratch.data_ptr(), cb, st), "knn_cover")
    for name, fn, flop in (("kth", run_kth, 2.0 * n * n * D), ("cover", run_cov, 2.0 * m * n * D)):
        ms = event_ms(fn, a.reps)
        res[f"{name}_pass_ms"] = ms
        res[f"{name}_pass_tflops"] = flop / ms / 1e9
        res[f"{name}_pass_vs_datasheet"] = flop / ms / 1e9 / PEAK_TFLOPS
    del R, F, scratch

    # end to end through the public API, CPU fp16 features in, CPU results out
    def native_e2e():
        mr = M.ManifoldBuilder(features=real, nhood_size=a.nhood, device=dev)
        mf = M.ManifoldBuilder(features=fake, nhood_size=a.nhood, device=dev)
        return mr, mf, M.calc_pr(mf.manifold, mr.manifold, 10000, 10000, device=dev)
    native_e2e()
    el, (mr, mf, (p, r)) = wall(native_e2e)
    res["native_e2e_s"] = el
    res["native_precision"], res["native_recall"] = p.item(), r.item()
    res["native_pr_str"] = f"{p:.5f}/{r:.5f}"

    if a.reference:
        import importlib.util
        from oracle import ref_loader
        root = ref_loader.root()
        if root is None:
            raise SystemExit("--reference needs the staged reference (oracle/_ref, made by build())")
        spec = importlib.util.spec_from_file_location("ref_pr", os.path.join(root, "ddpm_torch", "metrics", "precision_recall.py"))
        ref = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ref)
        ref.ManifoldBuilder.op_device = dev       # upstream sets op_device only when it extracts features

        def ref_e2e():
            rr = ref.ManifoldBuilder(features=real, nhood_size=a.nhood, device=dev)
            rf = ref.ManifoldBuilder(features=fake, nhood_size=a.nhood, device=dev)
            return ref.calc_pr(rf.manifold, rr.manifold, 10000, 10000, device=dev)
        el_ref, (pr_, rr_) = wall(ref_e2e)
        res["reference_e2e_s"] = el_ref
        res["reference_precision"], res["reference_recall"] = float(pr_), float(rr_)
        res["speedup_vs_reference"] = el_ref / el

    if not a.no_check:
        flags = M._native("bench", fake, real, 0, mr.kth, dev)
        res["fp64_check"] = check_fp64(fake, real, mr.kth, flags, kk, dev)
    res["device_error_flag"] = L.ddpm_device_error_flag()
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bench_pr.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
