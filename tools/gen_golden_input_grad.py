"""Generate tests/golden/unet_input_grad.pt by running the UNMODIFIED reference on CPU fp32 (build container only, where the
reference checkout exists; it is imported through oracle/ref_loader.py exactly as oracle/gen_golden.py does):

    python tools/gen_golden_input_grad.py [OUT_DIR]          # default OUT_DIR: tests/golden

Gradients of the UNet with respect to its INPUT x (autograd of unet.py:205-233 through x), for the uses that need them:
guided sampling and inverse problems, saliency, Hutchinson divergence estimates.  Weights: ``oracle.ddpm_ref.make_state_dict``
(``tests/noresample_ref.make_state_dict`` for the resample_with_conv=False model), loaded with ``strict=True``; models in eval
mode (no dropout).

Per case (CASES below): cfg, seed, resample_with_conv, x f32[B,Cin,H,W], t i64[B] (first 0, last 999), a seeded cotangent
g f32[B,Cout,H,W], dx = d(sum(m(x, t) * g))/dx and its per-image L2 norm dx_norm f32[B].

The CIFAR-10 case also carries ``guide``: the x_t-gradient of the guidance loss  sum(mask * (x0_hat(x_t) - y)^2)  with
x0_hat from eps (GaussianDiffusion.p_mean_var(..., clip_denoised=False, return_pred=True), fixed-large, linear 1e-4..0.02,
T = 1000) for a stored target y and a 0/1 mask (the left half of every image), at mid-chain timesteps GUIDE_T, where the
eps term of x0_hat weighs about as much as the x_t term: t, y, mask, loss, grad.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ddpm_ref as R  # noqa: E402
from oracle.gen_golden import build_ref_unet, import_reference  # noqa: E402
import noresample_ref as N  # noqa: E402

# (name, cfg, B, H/W, seed, resample_with_conv)
CASES = [(f"tiny_c{C}", dict(R.TINY_CFG, in_channels=C, out_channels=C), 2, 16, 100 + C, True) for C in (1, 3, 4)] + \
        [(f"small64_c{C}", dict(R.SMALL64_CFG, in_channels=C, out_channels=C), 2, 32, 110 + C, True) for C in (1, 2, 3)] + \
        [("cifar10", R.CIFAR10_CFG, 4, 32, 120, True),
         ("small64_c1to2", dict(R.SMALL64_CFG, in_channels=1, out_channels=2), 2, 32, 121, True),
         ("small64_noresample", N.SMALL64_CFG, 2, 32, 122, False)]
GUIDE_CASE = "cifar10"
GUIDE_T = (200, 400, 600, 800)


def case_inputs(cfg, B, HW, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cfg["in_channels"], HW, HW, generator=g)
    t = torch.randint(1000, (B,), generator=g)
    t[0] = 0; t[-1] = 999
    cot = torch.randn(B, cfg["out_channels"], HW, HW, generator=g)
    return x, t, cot


def guide_inputs(x, seed):
    g = torch.Generator().manual_seed(seed + 7)
    y = torch.rand(x.shape, generator=g) * 2 - 1
    mask = torch.zeros_like(x)
    mask[..., : x.shape[-1] // 2] = 1.0
    return y, mask


def build(ddpm_torch, cfg, seed, resample):
    if resample:
        return build_ref_unet(ddpm_torch, cfg, seed)[0]
    c = N.normalize_cfg(cfg)
    m = ddpm_torch.UNet(in_channels=c["in_channels"], hid_channels=c["hid_channels"], out_channels=c["out_channels"],
                        ch_multipliers=c["ch_multipliers"], num_res_blocks=c["num_res_blocks"], apply_attn=c["apply_attn"],
                        drop_rate=c["drop_rate"], resample_with_conv=False)
    m.load_state_dict(N.make_state_dict(cfg, seed), strict=True)
    return m.eval()


def gen_input_grad(out_dir):
    ddpm_torch, _ = import_reference()
    fx = dict(models={})
    for name, cfg, B, HW, seed, resample in CASES:
        m = build(ddpm_torch, cfg, seed, resample)
        m.requires_grad_(False)
        x, t, cot = case_inputs(cfg, B, HW, seed)
        xg = x.clone().requires_grad_(True)
        (dx,) = torch.autograd.grad((m(xg, t) * cot).sum(), xg)
        e = dict(cfg=dict(cfg), seed=seed, resample_with_conv=resample, B=B, H=HW, W=HW, x=x, t=t, g=cot, dx=dx,
                 dx_norm=dx.flatten(1).norm(dim=1))
        if name == GUIDE_CASE:
            diff = ddpm_torch.GaussianDiffusion(ddpm_torch.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
            y, mask = guide_inputs(x, seed)
            tg = torch.tensor(GUIDE_T[:B], dtype=torch.int64)
            xg = x.clone().requires_grad_(True)
            pred = diff.p_mean_var(m, xg, tg, clip_denoised=False, return_pred=True)[-1]
            loss = (mask * (pred - y)).pow(2).sum()
            (gx,) = torch.autograd.grad(loss, xg)
            e["guide"] = dict(t=tg, y=y, mask=mask, loss=loss.item(), grad=gx)
        fx["models"][name] = e
        print(f"{name}: |dx| per image {[round(v, 4) for v in e['dx_norm'].tolist()]}" +
              (f"  guidance loss {e['guide']['loss']:.3f} |grad| {e['guide']['grad'].norm():.3f}" if "guide" in e else ""))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "unet_input_grad.pt")
    torch.save(fx, path)
    print("unet_input_grad.pt written to", out_dir, f"({os.path.getsize(path) / 1e6:.3f} MB)")


if __name__ == "__main__":
    gen_input_grad(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
