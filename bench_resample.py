"""Cost of ``resample_with_conv=False`` against the default conv resampling, on the CIFAR-10 config (one GPU):

    python bench_resample.py [--steps K] [--warmup W] [--rounds R]

* the bs = 128 training step (repack + ddpm_train_forward + ddpm_train_backward through the C ABI, as bench.py drives it);
* the bs = 256 ancestral sampler step (ddpm_sampler_step, built-in Philox noise);
  both models are built in one process and timed in alternating rounds (median per side);
* the pool / upsample kernels and their adjoints alone (k_upsample2x_bwd / k_upsample2x at the plan's shapes, statistics
  modes and accumulate flags), over rotating buffers four times the L2 size, against the HBM bound: bytes from the shapes over
  3.35 TB/s (H100 SXM data sheet).  The kernels are compiled from ddpm_torch_b200/csrc into a temporary directory.

Prints ONE JSON line with the card's name and power limit, read in the same run, and ddpm_device_error_flag()."""
import argparse
import ctypes as C
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
CIFAR = dict(in_channels=3, hid_channels=128, out_channels=3, ch_multipliers=(1, 2, 2, 2), num_res_blocks=2,
             apply_attn=(False, True, False, False), drop_rate=0.1)
HBM_BPS = 3.35e12

HARNESS = r"""
#include "ptx.cuh"
#include "gn_epilogue.cuh"
#include "kernels_simt.cuh"
using namespace ddpm;
static int grid(long long n) { long long g = (n + 255) / 256; if (g > 132 * 16) g = 132 * 16; return (int)(g < 1 ? 1 : g); }
// kind 0: pool forward, 1: pool backward, 2: upsample forward, 3: upsample backward; (H, W) = low-res map.
// qs: per-buffer statistics (null = off); qs_in: upsample forward's input statistics (null = reduce the output).
extern "C" int run(int kind, void** a, void** b, void** qs, const void* qs_in, int nbuf, int B, int H, int W, int C, int acc, int iters, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < iters; ++i) {
        const int k = i % nbuf;
        const bf16* src = (const bf16*)a[k]; bf16* dst = (bf16*)b[k]; double* q = qs ? (double*)qs[k] : nullptr;
        const long long lo = (long long)B * H * W, hi = 4 * lo;
        switch (kind) {
            case 0: launch_k(k_upsample2x_bwd, q ? grid(lo * (C / 32)) : grid(lo * (C / 8)), 256, 0, st, src, dst, B, H, W, C, acc, 0.25f, q); break;
            case 1: launch_k(k_upsample2x, grid(hi * (C / 8)), 256, 0, st, src, dst, B, H, W, C, 0.25f, acc, (const double*)nullptr, (double*)nullptr); break;
            case 2: launch_k(k_upsample2x, (q && !qs_in) ? grid(hi * (C / 32)) : grid(hi * (C / 8)), 256, 0, st, src, dst, B, H, W, C, 1.f, acc, (const double*)qs_in, q); break;
            default: launch_k(k_upsample2x_bwd, grid(lo * (C / 8)), 256, 0, st, src, dst, B, H, W, C, acc, 1.f, (double*)nullptr); break;
        }
    }
    return (int)cudaGetLastError();
}
"""


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception as e:      # the card name still comes from torch
        return torch.cuda.get_device_name(0), f"unknown ({type(e).__name__})"


def build_model(D, flag, dev):
    m = D.UNet(**CIFAR, resample_with_conv=flag).to(dev).train()
    with torch.no_grad():
        gi = torch.Generator(device=dev).manual_seed(7)
        for p in m.parameters():
            if p.ndim >= 2:
                fan_in = p[0].numel()
                p.copy_((torch.rand(p.shape, device=dev, generator=gi) * 2 - 1) * (3.0 / fan_in) ** 0.5)
    return m


def train_stepper(D, _lib, m, dev, B=128):
    L = _lib.lib()
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    g = torch.Generator(device=dev).manual_seed(100)
    nb = 4
    x0s = [torch.rand(B, 3, 32, 32, device=dev, generator=g) * 2 - 1 for _ in range(nb)]
    ts = [torch.randint(1000, (B,), device=dev, generator=g) for _ in range(nb)]
    nzs = [torch.randn(B, 3, 32, 32, device=dev, generator=g) for _ in range(nb)]
    ta, tsb = diff._dev_tables(dev)
    losses = torch.empty(B, device=dev)
    gscale = torch.full((B,), 1.0 / B, device=dev)

    def step(i):
        h = m.prepare(B, 32, 32, training=True)
        sp = _lib.stream_ptr()
        _lib.check(L.ddpm_unet_repack(h, sp))
        k = i % nb
        _lib.check(L.ddpm_train_forward(h, x0s[k].data_ptr(), ts[k].data_ptr(), nzs[k].data_ptr(), ta.data_ptr(), tsb.data_ptr(),
                                        losses.data_ptr(), 1000 + i, sp))
        _lib.check(L.ddpm_train_backward(h, gscale.data_ptr(), sp))
    return step, losses


def sampler_stepper(D, _lib, m, dev, B=256):
    L = _lib.lib()
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    coef, tmod = d._coef_rows(), d._model_timesteps().contiguous()
    x = torch.randn(B, 3, 32, 32, device=dev, generator=torch.Generator(device=dev).manual_seed(5))

    def arm():
        h = m.prepare(B, 32, 32, training=False, force_repack=True)
        _lib.check(L.ddpm_sampler_setup(h, coef.shape[0], tmod.data_ptr(), coef.data_ptr()))
        _lib.check(L.ddpm_sampler_reset(h, coef.shape[0] - 1, _lib.stream_ptr()))
        return h

    def step(h, i):
        _lib.check(L.ddpm_sampler_step(h, x.data_ptr(), None, 99 + i, _lib.stream_ptr()))
    return arm, step, x


def timed(fn, n):
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def bench_kernels(dev, iters=200):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    csrc = os.path.join(ROOT, "ddpm_torch_b200", "csrc")
    with tempfile.TemporaryDirectory() as td:
        src, so = os.path.join(td, "h.cu"), os.path.join(td, "h.so")
        open(src, "w").write(HARNESS)
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-shared", "-Xcompiler", "-fPIC",
                        "-I", csrc, "-o", so, src, "-lcudart", "-lcuda"], check=True, capture_output=True)
        H = C.CDLL(so)
        H.run.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int] * 7 + [C.c_void_p]
        H.run.restype = C.c_int
        l2 = torch.cuda.get_device_properties(dev).L2_cache_size
        B = 128
        # (name, kind, low-res H = W, C, statistics: 0 off / 1 reduced / 2 = 4 x input statistics, accumulate) as the bs = 128 plan runs them
        cases = [("pool 32->16 C128 +stats", 0, 16, 128, 1, 0), ("pool 16->8 C256 +stats", 0, 8, 256, 1, 0), ("pool 8->4 C256", 0, 4, 256, 0, 0),
                 ("pool_bwd 16->32 C128 acc", 1, 16, 128, 0, 1), ("pool_bwd 8->16 C256 acc", 1, 8, 256, 0, 1), ("pool_bwd 4->8 C256 acc", 1, 4, 256, 0, 1),
                 ("upsample 4->8 C256 +stats", 2, 4, 256, 1, 0), ("upsample 8->16 C256 stats x4", 2, 8, 256, 2, 0),
                 ("upsample 16->32 C256 stats x4", 2, 16, 256, 2, 0),
                 ("upsample_bwd 8->4 C256", 3, 4, 256, 0, 0), ("upsample_bwd 16->8 C256", 3, 8, 256, 0, 0), ("upsample_bwd 32->16 C256", 3, 16, 256, 0, 0)]
        out = []
        st = torch.cuda.current_stream().cuda_stream
        for name, kind, h, Cc, stats, acc in cases:
            lo, hi = B * h * h * Cc * 2, 4 * B * h * h * Cc * 2
            ia, ib = (hi, lo) if kind in (0, 3) else (lo, hi)       # bytes of the tensor read / written
            moved = ia + ib + (ib if acc else 0)
            nbuf = max(2, -(-4 * l2 // (ia + ib)))
            a = [torch.randn(ia // 2, device=dev).to(torch.bfloat16) for _ in range(nbuf)]
            b = [torch.randn(ib // 2, device=dev).to(torch.bfloat16) for _ in range(nbuf)]
            qs = [torch.zeros(B * Cc // 4 * 2, dtype=torch.float64, device=dev) for _ in range(nbuf)] if stats else None
            qin = torch.ones(B * Cc // 4 * 2, dtype=torch.float64, device=dev) if stats == 2 else None
            pa = (C.c_void_p * nbuf)(*[t.data_ptr() for t in a]); pb = (C.c_void_p * nbuf)(*[t.data_ptr() for t in b])
            pq = (C.c_void_p * nbuf)(*[t.data_ptr() for t in qs]) if qs else None

            def go(n):
                rc = H.run(kind, pa, pb, pq, qin.data_ptr() if qin is not None else None, nbuf, B, h, h, Cc, acc, n, st)
                assert rc == 0, rc
            go(2 * nbuf)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
            e0.record(); go(iters); e1.record(); torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / iters * 1e3
            out.append({"kernel": name, "us": round(us, 2), "bytes": moved, "hbm_bound_us": round(moved / HBM_BPS * 1e6, 2),
                        "frac_of_hbm_bound": round(moved / HBM_BPS * 1e6 / us, 3), "buffers": nbuf})
            del a, b, qs, qin
            torch.cuda.empty_cache()
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sampler-steps", type=int, default=50)
    args = ap.parse_args()
    sys.stdout.flush()
    real = os.dup(1); os.dup2(2, 1)           # stdout carries only the JSON line
    import ddpm_torch_b200 as D
    from ddpm_torch_b200 import _lib
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    _lib.runtime_check()
    name, plimit = card_info()
    res = {"card": name, "power_limit": plimit, "config": "cifar10", "train_bs": 128, "sampler_bs": 256}
    models = {flag: build_model(D, flag, dev) for flag in (True, False)}
    tr = {flag: train_stepper(D, _lib, models[flag], dev) for flag in models}
    for flag in models:
        for i in range(args.warmup):
            tr[flag][0](i)
    torch.cuda.synchronize()
    times = {True: [], False: []}
    for r in range(args.rounds):
        for flag in ((True, False) if r % 2 == 0 else (False, True)):
            times[flag].append(timed(tr[flag][0], args.steps))
    res["train_step_ms"] = {"resample_with_conv": [round(v, 3) for v in times[True]], "pool_upsample": [round(v, 3) for v in times[False]],
                            "median_conv": round(statistics.median(times[True]), 3), "median_pool": round(statistics.median(times[False]), 3)}
    for m in models.values():
        m.eval()
    sm = {flag: sampler_stepper(D, _lib, models[flag], dev) for flag in models}
    stimes = {True: [], False: []}
    for r in range(args.rounds + 1):
        for flag in ((True, False) if r % 2 == 0 else (False, True)):
            arm, step, _ = sm[flag]
            h = arm()
            if r == 0:
                timed(lambda i: step(h, i), 5)          # warm-up round (plans, modules)
                continue
            stimes[flag].append(timed(lambda i: step(h, i), args.sampler_steps))
    res["sampler_step_ms"] = {"resample_with_conv": [round(v, 3) for v in stimes[True]], "pool_upsample": [round(v, 3) for v in stimes[False]],
                              "median_conv": round(statistics.median(stimes[True]), 3), "median_pool": round(statistics.median(stimes[False]), 3)}
    ok = all(torch.isfinite(tr[f][1]).all().item() and torch.isfinite(sm[f][2]).all().item() for f in models)
    res["kernels_bs128"] = bench_kernels(dev)
    res["finite"] = bool(ok)
    res["device_error_flag"] = int(_lib.lib().ddpm_device_error_flag())
    sys.stdout.flush(); os.dup2(real, 1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
