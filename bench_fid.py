"""FID on one H100: the native statistics and Fréchet distance against the reference recipes on the same host.

    python bench_fid.py [--rows 50000] [--batch 512] [--dim 2048] [--inception] [--reference] [--out-dir DIR]

Prints one JSON line per measurement, each with the card name, power limit and max SM clock (nvidia-smi query):
  * ``stats``: folding ``rows`` seeded fp32 features into the statistics, ``batch`` rows at a time (eval.py's eval_batch_size 512,
    D = 2048), native (features already on the device, timed to a device synchronise) against the reference's numpy recipe
    (``.cpu().numpy()``, per-batch np.cov, merge);
  * ``calc_fd``: the distance at D = 2048 on full-rank statistics, native against the CPU formula (scipy sqrtm), and their
    difference;
  * ``--inception``: the Inception forward over ``rows`` images (32 x 32, resized to 299) with seeded weights, batch ``batch``:
    the native leg (``ddpm_inception_forward``) and the torch leg (cuDNN) in the same call, the TF32 rate of the native leg from
    the conv FLOP count of the layer shapes, the largest per-image relative L2 difference between the legs, and the shares of a
    FID evaluation after sampling that the statistics and the distance take next to the native forward;
  * ``--reference``: the same statistics and distance through the staged reference (oracle/_ref), SciPy's removed ``disp`` keyword
    shimmed by patching scipy.linalg in this process.
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


def features(rows, dim, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = torch.randn(64, dim, device="cuda", generator=g) / 8
    return (torch.relu(torch.randn(rows, 64, device="cuda", generator=g) @ W + 0.2) * 3).contiguous()


def numpy_recipe(batches):
    m = v = None
    cnt = 0
    for b in batches:
        x = b.cpu().numpy()
        mean = np.mean(x, axis=0, dtype=np.float64)
        var = np.cov(x, rowvar=False, ddof=0, dtype=np.float64)
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
    ap.add_argument("--rows", type=int, default=50000)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--inception", action="store_true")
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_fid"))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fid.py measures on a CUDA device"

    def offline(*args, **kw):
        raise RuntimeError("bench_fid.py runs on seeded weights and never downloads")
    import requests
    torch.hub.download_url_to_file = torch.hub.load_state_dict_from_url = requests.get = offline
    os.makedirs(a.out_dir, exist_ok=True)
    from ddpm_torch_b200 import _lib, metrics as M
    _lib.runtime_check()
    info = card()
    lines = []

    def emit(d):
        d.update(card=info)
        lines.append(d)
        print(json.dumps(d), flush=True)

    x = features(a.rows, a.dim, 0)
    batches = list(x.split(a.batch))
    L = _lib.lib()
    state = torch.zeros(L.ddpm_fid_stats_bytes(a.dim), dtype=torch.uint8, device="cuda")

    def native_stats():
        state.zero_()
        for b in batches:
            _lib.check(L.ddpm_fid_stats_update(state.data_ptr(), a.dim, b.data_ptr(), b.shape[0], a.dim, _lib.stream_ptr()))
        mean = torch.empty(a.dim, dtype=torch.float64, device="cuda")
        cov = torch.empty(a.dim, a.dim, dtype=torch.float64, device="cuda")
        _lib.check(L.ddpm_fid_stats_finalize(state.data_ptr(), a.dim, a.rows, 1, mean.data_ptr(), cov.data_ptr(), _lib.stream_ptr()))
        return mean, cov
    native_stats()
    (mn, cn), t_nat = timed(native_stats)
    (mn2, cn2), t_nat2 = timed(native_stats)
    (mr, cr), t_np = timed(lambda: numpy_recipe(batches))
    cn = cn.cpu().numpy()
    emit({"metric": "stats", "rows": a.rows, "batch": a.batch, "dim": a.dim, "native_s": min(t_nat, t_nat2), "numpy_s": t_np,
          "max_abs_cov_diff": float(np.abs(cn - cr).max()), "max_abs_cov": float(np.abs(cr).max())})

    mu1, s1 = mr, cr
    y = features(a.rows, a.dim, 1) * 1.1 + 0.05
    mu2, s2 = numpy_recipe(list(y.split(a.batch)))
    M.frechet_distance_native(mu1, s1, mu2, s2, "cuda")
    (fd, fi), t_fd = timed(lambda: M.frechet_distance_native(mu1, s1, mu2, s2, "cuda"))
    ref_fd, t_cpu = timed(lambda: M.calculate_frechet_distance(mu1, s1, mu2, s2), sync=False)
    emit({"metric": "calc_fd", "dim": a.dim, "native_s": t_fd, "cpu_formula_s": t_cpu, "fd_native": float(fd),
          "fd_cpu_formula": float(ref_fd), "abs_diff": abs(float(fd) - float(ref_fd)), "sweeps": fi["sweeps"]})

    if a.reference:
        import importlib
        import scipy.linalg
        orig = scipy.linalg.sqrtm

        def sqrtm(A, disp=None, **kw):
            r = orig(A, **kw)
            return (r, None) if disp is False else r
        scipy.linalg.sqrtm = sqrtm
        from oracle import ref_loader
        ref_loader.load()
        fs = importlib.import_module("ddpm_torch.metrics.fid_score")
        ist = fs.InceptionStatistics.__new__(fs.InceptionStatistics)
        torch.nn.Module.__init__(ist)
        ist.input_transform = lambda t: t
        ist.model = torch.nn.Identity()
        ist.running_mean = np.zeros(a.dim)
        ist.running_var = np.zeros((a.dim, a.dim))
        ist.count = 0

        def ref_stats():
            for b in batches:
                ist(b[:, :, None, None])
            return ist.get_statistics()
        (rm, rc), t_ref = timed(ref_stats)
        rfd, t_rfd = timed(lambda: fs.calc_fd(mu1, s1, mu2, s2), sync=False)
        emit({"metric": "reference", "stats_s": t_ref, "calc_fd_s": t_rfd, "fd_reference": float(rfd),
              "fd_native_minus_reference": float(fd) - float(rfd), "max_abs_cov_diff": float(np.abs(cn - rc).max())})

    if a.inception:
        from ddpm_torch_b200.inception import InceptionV3, seeded_state_dict, weights_path
        hub = tempfile.TemporaryDirectory()          # the seeded weights (100 MB) are not a result
        torch.hub.set_dir(hub.name)
        os.makedirs(os.path.dirname(weights_path()), exist_ok=True)
        torch.save(seeded_state_dict(0), weights_path())
        net = InceptionV3([3]).cuda().eval()
        g = torch.Generator(device="cuda").manual_seed(2)
        imgs = torch.rand(a.batch, 3, 32, 32, device="cuda", generator=g) * 2 - 1
        n_b = -(-a.rows // a.batch)
        # multiply-adds of every conv at the resized 299 x 299 input, from the shapes the torch module produces
        shapes = []
        hooks = [m.register_forward_hook(lambda m, i, o: shapes.append((m, o.shape))) for m in net.modules()
                 if isinstance(m, torch.nn.Conv2d)]
        net.use_engine = False
        with torch.inference_mode():
            net(imgs[:1])
        for h in hooks:
            h.remove()
        flops = sum(2 * o[1] * o[2] * o[3] * m.in_channels * m.kernel_size[0] * m.kernel_size[1] for m, o in shapes) * n_b * a.batch
        legs = {}
        for leg in ("torch", "native"):                # same images, same call, torch first
            net.use_engine = leg == "native"
            with torch.inference_mode():
                ref = net(imgs)[0]
                _, legs[leg] = timed(lambda: [net(imgs) for _ in range(n_b)])
                legs[leg + "_out"] = ref
        t_inc = legs["native"]
        diff = (legs["native_out"] - legs["torch_out"]).flatten(1).double()
        rel = (diff.norm(dim=1) / legs["torch_out"].flatten(1).double().norm(dim=1)).max().item()
        emit({"metric": "inception", "rows": n_b * a.batch, "batch": a.batch, "native_forward_s": legs["native"],
              "torch_forward_s": legs["torch"], "torch_cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
              "speedup": legs["torch"] / legs["native"], "conv_flop": flops, "native_tf32_tflops": flops / legs["native"] / 1e12,
              "max_rel_l2_native_vs_torch": rel,
              "stats_share": min(t_nat, t_nat2) / (t_inc + min(t_nat, t_nat2) + t_fd),
              "calc_fd_share": t_fd / (t_inc + min(t_nat, t_nat2) + t_fd)})
        hub.cleanup()

    with open(os.path.join(a.out_dir, "bench_fid.json"), "w") as f:
        json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
