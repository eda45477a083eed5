"""Generate tests/golden/bpd_unet.pt by running the UNMODIFIED reference on CPU fp32 (build container only, where the
reference checkout exists; it is imported through oracle/ref_loader.py exactly as oracle/gen_golden.py does):

    python tools/gen_golden_bpd_unet.py [OUT_DIR]          # default OUT_DIR: tests/golden

Bits-per-dim terms with the real ``ddpm_torch.UNet`` (``oracle.ddpm_ref.make_state_dict`` weights): tiny at 16x16 (the
engine's tail-kernel path) and small64 at 32x32 (the fused tensor-core gather), T = 20 linear 1e-4..0.02, 8-bit data in
[-1, 1], per-step noise stored.  For both fixed variances and clip_denoised in {True, False}: losses[B, T] (the
_loss_term_bpd term of every step) and mses[B, T] (pred-x_0 MSE).  The reference's own calc_all_bpd / _prior_bpd raise
(see oracle/gen_golden.py::gen_bpd), so its loop (diffusion.py:252-268) runs here over the pinned _loss_term_bpd.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ddpm_ref as R  # noqa: E402
from oracle.gen_golden import build_ref_unet, import_reference  # noqa: E402


def gen_bpd_unet(out_dir):
    ddpm_torch, _ = import_reference()
    from ddpm_torch.functions import flat_mean
    T = 20
    betas = ddpm_torch.get_beta_schedule("linear", 1e-4, 0.02, T)
    fx = dict(T=T, models={})
    for name, cfg, B, HW, seed in (("tiny", R.TINY_CFG, 2, 16, 41), ("small64", R.SMALL64_CFG, 2, 32, 42)):
        m, _ = build_ref_unet(ddpm_torch, cfg, seed)
        g = torch.Generator().manual_seed(seed)
        x0 = (torch.rand(B, 3, HW, HW, generator=g) * 2 - 1).mul(127.5).round().div(127.5)
        noise = torch.randn(T, B, 3, HW, HW, generator=g)
        cases = {}
        with torch.no_grad():
            for vt in ("fixed-small", "fixed-large"):
                d = ddpm_torch.GaussianDiffusion(betas=betas, model_mean_type="eps", model_var_type=vt, loss_type="mse")
                for clip in (True, False):
                    losses, mses = torch.zeros(B, T), torch.zeros(B, T)
                    t = torch.empty(B, dtype=torch.int64)
                    for ti in range(T - 1, -1, -1):
                        t.fill_(ti)
                        x_t = d.q_sample(x0, t, noise=noise[ti])
                        term, pred = d._loss_term_bpd(m, x0, x_t=x_t, t=t, clip_denoised=clip, return_pred=True)
                        losses[:, ti] = term
                        mses[:, ti] = flat_mean((pred - x0).pow(2))
                    cases[(vt, clip)] = dict(losses=losses, mses=mses)
        fx["models"][name] = dict(cfg=dict(cfg), seed=seed, x0=x0, noise=noise, cases=cases)
        print(f"bpd_unet {name}:", {k: round(float(c["losses"].sum(1).mean()), 4) for k, c in cases.items()})
    os.makedirs(out_dir, exist_ok=True)
    torch.save(fx, os.path.join(out_dir, "bpd_unet.pt"))
    print("bpd_unet.pt written to", out_dir)


if __name__ == "__main__":
    gen_bpd_unet(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
