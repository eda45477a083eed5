"""Bits-per-dim evaluation benchmark (GaussianDiffusion.calc_all_bpd) on one GPU, CIFAR-10 config.

In one process:
  * the card name, power limit and max SM clock (nvidia-smi query);
  * the native bits/dim step (ddpm_bpd_step replayed from a CUDA graph): ms per step, and images/s of a full T-step evaluation;
  * the generic torch loop (diffusion.py:252-268 over ``lambda x, t: m(x, t)``) on the same native UNet: ms per step;
  * the ancestral sampler step (p_sample, CUDA graph) at the same batch, for reference;
  * the native and generic [B, k] terms of the first k steps on the same seeded noise.
Writes <out-dir>/bench_bpd.json (default: a directory under the system temp dir) and prints it as one line.  Model weights are ``oracle.ddpm_ref.make_state_dict`` (seeded).

    python bench_bpd.py --batch 256 --timesteps 1000 --out-dir /tmp/bench_bpd
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clk = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:             # the measurement stands without it, but say so
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})", "sm_max_clock": None}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--timesteps", type=int, default=1000)
    ap.add_argument("--step-chain", type=int, default=200, help="chain length of the per-step timings")
    ap.add_argument("--reps", type=int, default=3, help="alternating repetitions of the native / sampler per-step timings")
    ap.add_argument("--compare-steps", type=int, default=20, help="k: steps of the generic loop timed and compared")
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "bench_bpd"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bpd.py measures on a CUDA device; none is present")
    import ddpm_torch_b200 as D
    from oracle import ddpm_ref as R
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    c = R.normalize_cfg(R.CIFAR10_CFG)
    m = D.UNet(3, c["hid_channels"], 3, c["ch_multipliers"], c["num_res_blocks"], c["apply_attn"], drop_rate=c["drop_rate"])
    m.load_state_dict(R.make_state_dict(R.CIFAR10_CFG, 0))
    m = m.to(dev).eval()
    B, T, S = a.batch, a.timesteps, a.step_chain
    sched = lambda n: D.get_beta_schedule("linear", 1e-4, 0.02, n)
    g = torch.Generator().manual_seed(0)
    x0 = (torch.rand(B, 3, 32, 32, generator=g) * 2 - 1).mul(127.5).round().div(127.5).to(dev)
    res = {"card": card(), "config": "cifar10", "batch": B, "timesteps": T, "step_chain": S}

    # per-step timings: native bits/dim step and sampler step, alternated; each call is warmed up once (plan, graph capture)
    dS = D.GaussianDiffusion(sched(S), "eps", "fixed-large", "mse")
    dS.calc_all_bpd(m, x0)
    dS.p_sample(m, shape=(B, 3, 32, 32), device=dev)
    bpd_ms, samp_ms = [], []
    for _ in range(a.reps):
        bpd_ms.append(timed(lambda: dS.calc_all_bpd(m, x0))[0] * 1e3 / S)
        samp_ms.append(timed(lambda: dS.p_sample(m, shape=(B, 3, 32, 32), device=dev))[0] * 1e3 / S)
    res["native_ms_per_step"] = sorted(bpd_ms)[len(bpd_ms) // 2]
    res["sampler_ms_per_step"] = sorted(samp_ms)[len(samp_ms) // 2]
    res["native_ms_per_step_all"], res["sampler_ms_per_step_all"] = bpd_ms, samp_ms
    res["native_over_sampler"] = res["native_ms_per_step"] / res["sampler_ms_per_step"]

    # full T-step evaluation (warm call, then timed) on the seeded default generator
    d = D.GaussianDiffusion(sched(T), "eps", "fixed-large", "mse")
    d.calc_all_bpd(m, x0)
    torch.manual_seed(1234)
    el, (total, losses, prior, mses) = timed(lambda: d.calc_all_bpd(m, x0))
    res["native_full_eval_s"] = el
    res["native_images_per_s"] = B / el
    res["mean_total_bpd"] = total.mean().item()

    # generic loop over the same UNet: its first k steps on the same seeded noise (the draws come in the same order)
    k = a.compare_steps
    torch.manual_seed(1234)
    fn = lambda x, t: m(x, t)
    t = torch.empty(B, dtype=torch.int64, device=dev)
    g_losses, g_mses = torch.zeros(B, k, device=dev), torch.zeros(B, k, device=dev)

    def generic():
        with torch.no_grad():
            for j, ti in enumerate(range(T - 1, T - 1 - k, -1)):
                t.fill_(ti)
                x_t = d.q_sample(x0, t=t)
                term, pred = d._loss_term_bpd(fn, x0, x_t=x_t, t=t, clip_denoised=True, return_pred=True)
                g_losses[:, k - 1 - j] = term
                g_mses[:, k - 1 - j] = (pred - x0).pow(2).mean(dim=(1, 2, 3))
    el_g, _ = timed(generic)
    res["generic_ms_per_step"] = el_g * 1e3 / k
    res["speedup_vs_generic"] = res["generic_ms_per_step"] / res["native_ms_per_step"]
    nl, nm = losses[:, T - k:], mses[:, T - k:]
    gl, gm = g_losses.cpu(), g_mses.cpu()
    res["compare_steps"] = k
    res["terms_max_abs_diff_bits"] = (nl - gl).abs().max().item()
    res["terms_max_err_over_bound"] = ((nl - gl).abs() / (1e-5 + 1e-3 * gl.abs())).max().item()
    res["terms_within_rtol1e-3_atol1e-5"] = bool(torch.allclose(nl, gl, rtol=1e-3, atol=1e-5))
    # pred-x_0 at t near T is x_t / sqrt(ab) - sqrt(1/ab - 1) * eps: eps differences are amplified ~157x in these mses
    res["mses_max_rel_diff"] = ((nm - gm).abs() / gm.abs()).max().item()
    from ddpm_torch_b200 import _lib
    res["device_error_flag"] = _lib.lib().ddpm_device_error_flag()

    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bench_bpd.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
