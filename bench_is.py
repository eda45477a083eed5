"""Inception Score on one H100: the native ``InceptionScore`` against the torch route on the same images.

    python bench_is.py [--rows 50176] [--batch 512] [--splits 10] [--out-dir DIR]

Seeded weights (``seeded_state_dict``) and seeded CIFAR-sized images (32 x 32, resized to 299 x 299); nothing is downloaded and
nothing is written outside ``--out-dir`` (default: a temporary directory).  Prints one JSON line per measurement, each with the
card name, power limit and max SM clock (nvidia-smi query):
  * ``is_native``: ``InceptionScore`` on the CUDA device end to end (engine forward, 3xTF32 logits, fp64 score), timed from the
    first batch to ``get_score()`` returning, which ends in a device synchronise;
  * ``is_torch``: the torch leg over the same images: the cuDNN forward (``use_engine = False``), a torch fp32 matmul with
    fc.weight, and the numpy fp64 formula;
  * ``is_tail``: the IS-specific work alone in CUDA events: the logits GEMM over all rows (in ``batch``-row calls, as
    ``InceptionScore`` issues it), and the score kernels on the logits that GEMM produced (status checked), with the GEMM's
    achieved TFLOP/s counted as 2 x rows x 1008 x 2048 x 3 (three TF32 products per multiply-add);
  * ``is_diff``: the two legs' (mean, std) and their differences.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50176)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--splits", type=int, default=10)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_is"))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_is.py measures on a CUDA device"

    def offline(*args, **kw):
        raise RuntimeError("bench_is.py runs on seeded weights and never downloads")
    torch.hub.download_url_to_file = torch.hub.load_state_dict_from_url = offline
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

    hub = tempfile.TemporaryDirectory()                 # the seeded weights (100 MB) are not a result
    torch.hub.set_dir(hub.name)
    os.makedirs(os.path.dirname(weights_path()), exist_ok=True)
    torch.save(seeded_state_dict(0), weights_path())
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cuda").manual_seed(2)
    n_b = -(-a.rows // a.batch)
    rows = n_b * a.batch
    imgs = torch.rand(rows, 3, 32, 32, device="cuda", generator=g) * 2 - 1
    batches = list(imgs.split(a.batch))

    ist = M.InceptionScore(splits=a.splits, device=dev)
    net = ist.model._module
    ist(batches[0])                                     # warm-up: module load, packing, workspaces
    ist.get_score()

    def native():
        ist.reset()
        for b in batches:
            ist(b)
        return ist.get_score()
    torch.cuda.synchronize()
    t = time.perf_counter()
    s_nat = native()
    t_nat = time.perf_counter() - t
    emit({"metric": "is_native", "rows": rows, "batch": a.batch, "splits": a.splits, "seconds": t_nat, "mean": s_nat[0],
          "std": s_nat[1]})

    w = net.fc_weight.to(dev)
    net.use_engine = False
    with torch.inference_mode():
        net(batches[0])                                 # warm-up: cuDNN algorithm choice
        torch.cuda.synchronize()
        t = time.perf_counter()
        logits = torch.cat([(net(b)[0].flatten(1) @ w.T).cpu() for b in batches])
        s_torch = M.calc_is(logits.numpy(), a.splits, device="cpu")
        t_torch = time.perf_counter() - t
    net.use_engine = True
    emit({"metric": "is_torch", "rows": rows, "batch": a.batch, "splits": a.splits, "seconds": t_torch, "mean": s_torch[0],
          "std": s_torch[1], "torch_cudnn_allow_tf32": torch.backends.cudnn.allow_tf32,
          "torch_matmul_allow_tf32": torch.backends.cuda.matmul.allow_tf32, "speedup": t_torch / t_nat})

    # the tail alone: logits from features already on the device, then the score
    feats = [torch.relu(torch.randn(a.batch, 2048, device="cuda", generator=g)) * 0.5 for _ in range(n_b)]
    packed, ws = ist._packed, ist._ws
    out = [None] * n_b
    L = M._lib.lib()
    nbytes = L.ddpm_is_score_scratch_bytes(rows, 1008, a.splits)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    res = torch.empty(a.splits + 1, dtype=torch.float64, device="cuda")

    def gemm():
        for i, f in enumerate(feats):
            out[i], _ = M._is_logits(packed, f, dev, ws)

    def score():
        _lib.check(L.ddpm_is_score(z.data_ptr(), rows, 1008, 1008, a.splits, res.data_ptr(), scratch.data_ptr(), nbytes,
                                   _lib.stream_ptr(dev)), "bench score")
    gemm()
    z = torch.cat(out)                                  # the score is timed on the logits the GEMM produced
    score()
    r = res.cpu().numpy()
    assert r[a.splits] == 0 and np.isfinite(r[:a.splits]).all(), r
    reps = 10
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    for _ in range(reps):
        gemm()
    ev[1].record()
    for _ in range(reps):
        score()
    ev[2].record()
    torch.cuda.synchronize()
    t_gemm = ev[0].elapsed_time(ev[1]) / reps / 1e3
    t_score = ev[1].elapsed_time(ev[2]) / reps / 1e3
    flop = 2.0 * rows * 1008 * 2048 * 3
    emit({"metric": "is_tail", "rows": rows, "batch": a.batch, "splits": a.splits, "logits_s": t_gemm, "score_s": t_score,
          "logits_flop": flop, "logits_tf32_tflops": flop / t_gemm / 1e12, "tail_share_of_native": (t_gemm + t_score) / t_nat})

    emit({"metric": "is_diff", "native": list(s_nat), "torch": list(s_torch), "mean_diff": s_nat[0] - s_torch[0],
          "std_diff": s_nat[1] - s_torch[1], "mean_rel_diff": (s_nat[0] - s_torch[0]) / s_torch[0]})
    hub.cleanup()
    with open(os.path.join(a.out_dir, "bench_is.json"), "w") as f:
        json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
