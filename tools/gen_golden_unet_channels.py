"""Generate tests/golden/unet_channels.pt by running the UNMODIFIED reference on CPU fp32 (build container only, where the
reference checkout exists; it is imported through oracle/ref_loader.py exactly as oracle/gen_golden.py does):

    python tools/gen_golden_unet_channels.py [OUT_DIR]          # default OUT_DIR: tests/golden

Models whose image side is not 3 channels (the engine accepts 1..4; the reference trains MNIST with in_channels = 1,
datasets.py / train.py).  ``oracle.ddpm_ref.make_state_dict`` weights, linear 1e-4..0.02 schedule.

* models[f"{tiny|small64}_c{C}"], C in {1, 2, 4}, in_channels = out_channels = C: tiny at 16x16 (the engine's CUDA-core
  image convs) and small64 at 32x32 (tensor-core in_conv; tensor-core out_conv for C <= 3).  B = 2, t = [0, 999] on the
  T = 1000 chain: x0, t, noise, x_t, eps = m(x_t, t), the train_losses per-sample losses (fixed-large, mse) and the
  per-parameter gradient norms of losses.mean().
  For C in {1, 4} also ``bpd``: T = 20 bits/dim terms exactly as tools/gen_golden_bpd_unet.py writes them (losses[B, T],
  mses[B, T] for both fixed variances and both clip settings, per-step noise stored), over 8-bit data with a band of
  pixels at exactly +1 and -1 (the decoder's edge-bin branches).  C = 4 uses B = 1 to keep the fixture near 1 MB.
* models["small64_c1to2"]: in_channels = 1, out_channels = 2 (what train.py builds for a 1-channel dataset with a learned
  variance; upstream's GaussianDiffusion cannot construct one, so the model alone): eps and the gradient norms of
  (m(x_t, t) * g).sum() for a stored g.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ddpm_ref as R  # noqa: E402
from oracle.gen_golden import build_ref_unet, import_reference, inputs  # noqa: E402

# (name, base cfg, C, B, HW, seed, bpd batch or 0)
CASES = [(f"tiny_c{C}", R.TINY_CFG, C, 2, 16, 60 + C, {1: 2, 4: 1}.get(C, 0)) for C in (1, 2, 4)] + \
        [(f"small64_c{C}", R.SMALL64_CFG, C, 2, 32, 70 + C, {1: 2, 4: 1}.get(C, 0)) for C in (1, 2, 4)]
BPD_T = 20


def bpd_data(B, C, HW, g):
    """8-bit data in [-1, 1]; row 0 of every image is exactly +1 and row 1 exactly -1."""
    x0 = (torch.rand(B, C, HW, HW, generator=g) * 2 - 1).mul(127.5).round().div(127.5)
    x0[:, :, 0, :] = 1.0
    x0[:, :, 1, :] = -1.0
    return x0


def gen_bpd(ddpm_torch, m, B, C, HW, seed):
    from ddpm_torch.functions import flat_mean
    T = BPD_T
    betas = ddpm_torch.get_beta_schedule("linear", 1e-4, 0.02, T)
    g = torch.Generator().manual_seed(seed + 1000)
    x0 = bpd_data(B, C, HW, g)
    noise = torch.randn(T, B, C, HW, HW, generator=g)
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
    return dict(T=T, x0=x0, noise=noise, cases=cases)


def gen_unet_channels(out_dir):
    ddpm_torch, _ = import_reference()
    betas = ddpm_torch.get_beta_schedule("linear", 1e-4, 0.02, 1000)
    diff = ddpm_torch.GaussianDiffusion(betas, "eps", "fixed-large", "mse")
    fx = dict(models={})
    for name, base, C, B, HW, seed, bpd_B in CASES:
        cfg = dict(base, in_channels=C, out_channels=C)
        m, _ = build_ref_unet(ddpm_torch, cfg, seed)
        x0, t, noise = inputs(cfg, B, HW, HW, seed)
        t[0] = 0; t[-1] = 999
        x_t = diff.q_sample(x0, t, noise)
        for p in m.parameters():
            p.requires_grad_(True)
        with torch.no_grad():
            eps = m(x_t, t)
        losses = diff.train_losses(m, x0, t, noise)
        losses.mean().backward()
        e = dict(cfg=cfg, seed=seed, B=B, H=HW, W=HW, x0=x0, t=t, noise=noise, x_t=x_t, eps=eps.clone(),
                 losses=losses.detach().clone(), grad_norm={k: p.grad.norm().item() for k, p in m.named_parameters()})
        if bpd_B:
            m.zero_grad(set_to_none=True)
            e["bpd"] = gen_bpd(ddpm_torch, m, bpd_B, C, HW, seed)
        fx["models"][name] = e
        print(f"{name}: |eps|max {eps.abs().max():.4f} loss {losses.mean():.5f}" +
              (f" bpd {[round(float(c['losses'].sum(1).mean()), 4) for c in e['bpd']['cases'].values()]}" if bpd_B else ""))
    # asymmetric model: 1 image channel in, 2 out
    cfg = dict(R.SMALL64_CFG, in_channels=1, out_channels=2)
    seed, B, HW = 81, 2, 32
    m, _ = build_ref_unet(ddpm_torch, cfg, seed)
    x_t, t, _ = inputs(cfg, B, HW, HW, seed)
    t[0] = 0; t[-1] = 999
    g = torch.randn(B, 2, HW, HW, generator=torch.Generator().manual_seed(seed + 1))
    for p in m.parameters():
        p.requires_grad_(True)
    out = m(x_t, t)
    (out * g).sum().backward()
    fx["models"]["small64_c1to2"] = dict(cfg=cfg, seed=seed, B=B, H=HW, W=HW, x_t=x_t, t=t, g=g, eps=out.detach().clone(),
                                         grad_norm={k: p.grad.norm().item() for k, p in m.named_parameters()})
    print(f"small64_c1to2: |eps|max {out.abs().max():.4f}")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "unet_channels.pt")
    torch.save(fx, path)
    print("unet_channels.pt written to", out_dir, f"({os.path.getsize(path) / 1e6:.3f} MB)")


if __name__ == "__main__":
    gen_unet_channels(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
