"""Cost of the input gradient (ddpm_unet_backward_ex) on the CIFAR-10 config with a training plan (one GPU):

    python bench_input_grad.py [--steps K] [--rounds R]

* at bs = 128 and at the guidance-typical bs = 16, through the C ABI, alternating in every round (median over rounds):
    full      forward + full backward                       (ddpm_unet_backward: flat gradients, no dx)
    full+dx   forward + full backward + dx                  (param_grads = 1, dx)
    dx-only   forward + input-only backward + dx            (param_grads = 0, dx): what a frozen model's guidance step runs
* the dx op alone: the plan's in_conv.dx ops timed by CUDA events around each op inside the input-only backward
  (DDPM_OP_TIMING, a separate process so that the per-op events stay out of the timings above), against its HBM bound:
  the weight pack + dh0 bf16 read + the 32-column fp32 tap scratch written and read back + dx fp32 written, over 3.35 TB/s
  (H100 SXM data sheet);
* one guided ancestral step at bs = 16 (forward, input-only backward through autograd, the ancestral update), against the
  same step over the reference's fp32 torch UNet when the reference is staged under oracle/_ref/.

Prints ONE JSON line with the card's name and power limit, read in the same run, and ddpm_device_error_flag()."""
import argparse
import json
import os
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


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception as e:
        return torch.cuda.get_device_name(0), f"unknown ({type(e).__name__})"


def build_model(D, dev):
    m = D.UNet(**CIFAR).to(dev).eval()
    with torch.no_grad():
        gi = torch.Generator(device=dev).manual_seed(7)
        for p in m.parameters():
            if p.ndim >= 2:
                fan_in = p[0].numel()
                p.copy_((torch.rand(p.shape, device=dev, generator=gi) * 2 - 1) * (3.0 / fan_in) ** 0.5)
    return m


def variants(_lib, m, dev, B):
    """Closures running forward + one backward variant through the C ABI on a training plan of batch B."""
    L = _lib.lib()
    g = torch.Generator(device=dev).manual_seed(100 + B)
    nb = 4
    xs = [torch.randn(B, 3, 32, 32, device=dev, generator=g) for _ in range(nb)]
    ts = [torch.randint(1000, (B,), device=dev, generator=g) for _ in range(nb)]
    gs = [torch.randn(B, 3, 32, 32, device=dev, generator=g) for _ in range(nb)]
    dxs = [torch.empty(B, 3, 32, 32, device=dev) for _ in range(nb)]
    eps = torch.empty(B, 3, 32, 32, device=dev)

    def make(want_dx, params):
        def step(i):
            h = m.prepare(B, 32, 32, training=True)
            sp = _lib.stream_ptr()
            k = i % nb
            _lib.check(L.ddpm_unet_forward(h, xs[k].data_ptr(), ts[k].data_ptr(), eps.data_ptr(), 0, sp))
            _lib.check(L.ddpm_unet_backward_ex(h, gs[k].data_ptr(), dxs[k].data_ptr() if want_dx else None, params, sp))
        return step
    return {"full": make(0, 1), "full+dx": make(1, 1), "dx-only": make(1, 0)}


def timed(fn, n):
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def op_timing(args):
    """Child process: per-op CUDA-event times of the input-only backward (DDPM_OP_TIMING is set by the parent)."""
    import ddpm_torch_b200 as D
    from ddpm_torch_b200 import _lib
    dev = torch.device("cuda", 0)
    m = build_model(D, dev)
    B = args.op_timing
    step = variants(_lib, m, dev, B)["dx-only"]
    for i in range(args.steps):
        step(i)
    torch.cuda.synchronize()


def dx_times(path):
    """Median in_conv.dx time (ms, its pack + GEMM + gather ops summed per backward) over the second half of a DDPM_OP_TIMING log."""
    per, cur = [], 0.0
    with open(path) as f:
        for line in f:
            name, ms = line.rsplit(" ", 1)
            if name.startswith("in_conv.dx"):
                cur += float(ms)
            elif cur:
                per.append(cur)
                cur = 0.0
    if cur:
        per.append(cur)
    return statistics.median(per[len(per) // 2:]) if per else float("nan")


def dx_bytes(B, H=32, W=32, ch=128, cin=3, tc=True):
    P = B * H * W
    b = P * ch * 2 + P * cin * 4                         # dh0 read, dx written
    b += ch * cin * 9 * 4 + 32 * ch * 2                  # weight pack: fp32 masters read, bf16 operand written
    if tc:
        b += 2 * P * 32 * 4                              # tap scratch written by the GEMM and read by the gather
    return b


def guided_step_ms(D, m_fn, B, dev, n):
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    g = torch.Generator(device=dev).manual_seed(9)
    x = torch.randn(B, 3, 32, 32, device=dev, generator=g)
    y = torch.rand(B, 3, 32, 32, device=dev, generator=g) * 2 - 1
    mask = torch.zeros_like(x); mask[..., :16] = 1
    t = torch.full((B,), 500, dtype=torch.int64, device=dev)
    z = torch.randn_like(x)

    def step(_):
        xg = x.detach().requires_grad_(True)
        mean, _, logvar, pred = d.p_mean_var(m_fn, xg, t, clip_denoised=False, return_pred=True)
        (gx,) = torch.autograd.grad((mask * (pred - y)).pow(2).sum(), xg)
        with torch.no_grad():
            return mean + torch.exp(0.5 * logvar) * z - 0.1 * gx
    for i in range(3):
        step(i)
    return timed(step, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--op-timing", type=int, default=0, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.op_timing:
        return op_timing(args)
    import ddpm_torch_b200 as D
    from ddpm_torch_b200 import _lib
    assert torch.cuda.is_available(), "bench_input_grad.py measures on the GPU; there is no CPU path"
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    name, power = card_info()
    m = build_model(D, dev)
    L = _lib.lib()
    res = {"card": name, "power_limit": power}
    for B in (128, 16):
        vs = variants(_lib, m, dev, B)
        for fn in vs.values():
            for i in range(3):
                fn(i)
        times = {k: [] for k in vs}
        for _ in range(args.rounds):
            for k, fn in vs.items():
                times[k].append(timed(fn, args.steps))
        h = m.prepare(B, 32, 32, training=True)
        res[f"bs{B}"] = {
            "ms_median": {k: round(statistics.median(v), 4) for k, v in times.items()},
            "ms_rounds": {k: [round(x, 4) for x in v] for k, v in times.items()},
            "launches": {"full": L.ddpm_unet_backward_launches(h, 0, 1), "full+dx": L.ddpm_unet_backward_launches(h, 1, 1),
                         "dx-only": L.ddpm_unet_backward_launches(h, 1, 0)},
        }
        # the dx op alone, per-op CUDA events in a child process
        with tempfile.TemporaryDirectory() as td:
            log = os.path.join(td, "ops.txt")
            env = dict(os.environ, DDPM_OP_TIMING=log)
            subprocess.run([sys.executable, os.path.abspath(__file__), "--op-timing", str(B), "--steps", "40"], env=env, check=True)
            ms = dx_times(log)
        nbytes = dx_bytes(B)
        res[f"bs{B}"]["dx_op"] = {"ms": round(ms, 5), "bytes": nbytes, "hbm_bound_ms": round(nbytes / HBM_BPS * 1e3, 5),
                                  "share_of_hbm_bound": round(nbytes / HBM_BPS * 1e3 / ms, 3) if ms == ms and ms > 0 else None}
    # guided ancestral step at bs = 16: engine (frozen) vs the reference's fp32 torch UNet
    m.requires_grad_(False)
    gs = {"engine_ms": round(guided_step_ms(D, m, 16, dev, args.steps), 4)}
    try:
        from oracle import ref_loader
        if ref_loader.available():
            ddpm_torch, _ = ref_loader.load()
            c = dict(CIFAR)
            ref = ddpm_torch.UNet(in_channels=3, hid_channels=128, out_channels=3, ch_multipliers=c["ch_multipliers"],
                                  num_res_blocks=2, apply_attn=c["apply_attn"], drop_rate=0.1)
            ref.load_state_dict(m.state_dict())
            ref = ref.to(dev).eval().requires_grad_(False)
            gs["reference_fp32_ms"] = round(guided_step_ms(D, ref, 16, dev, args.steps), 4)
        else:
            gs["reference_fp32_ms"] = "not staged"
    except Exception as e:      # the engine number stands on its own
        gs["reference_fp32_ms"] = f"failed: {type(e).__name__}: {e}"
    res["guided_step_bs16"] = gs
    res["device_error_flag"] = L.ddpm_device_error_flag()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
