"""Generate tests/golden/unet_noresample.pt by running the UNMODIFIED reference on CPU fp32 (build container only, where the
reference checkout exists; it is imported through oracle/ref_loader.py exactly as oracle/gen_golden.py does):

    python tools/gen_golden_noresample.py [OUT_DIR]          # default OUT_DIR: tests/golden

UNets built with ``resample_with_conv=False`` (unet.py:106,164-170,199-202: AvgPool2d(2) down, bare nearest x2 up, no resample
convs), constructed directly as ``ddpm_torch.UNet(..., resample_with_conv=False)``.  Weights: ``oracle.ddpm_ref.fill_params``
over the reference module's own state_dict inventory, loaded with ``strict=True``; linear 1e-4..0.02 schedule, T = 1000.

Cases (tests/noresample_ref.py::CASES): tiny at 16x16, small64 at 32x32 and the CIFAR-10 config at 32x32, B = 2, t = [0, 999].
Per case: the reference's state_dict key / shape list, x0, t, noise, x_t, eps = m(x_t, t), the train_losses per-sample losses
(fixed-large, mse) and the per-parameter gradient norms of losses.mean().  For small64 also ``bpd``: T = 20 bits/dim terms as
tools/gen_golden_bpd_unet.py writes them (losses[B, T], mses[B, T] for both fixed variances and both clip settings, per-step
noise stored) over 8-bit data.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ddpm_ref as R  # noqa: E402
from oracle.gen_golden import import_reference, inputs  # noqa: E402
from noresample_ref import BPD_CASE, BPD_T, CASES  # noqa: E402


def build_ref_unet_noresample(ddpm_torch, cfg, seed):
    c = R.normalize_cfg(dict(cfg, resample_with_conv=True))
    m = ddpm_torch.UNet(in_channels=c["in_channels"], hid_channels=c["hid_channels"], out_channels=c["out_channels"],
                        ch_multipliers=c["ch_multipliers"], num_res_blocks=c["num_res_blocks"], apply_attn=c["apply_attn"],
                        drop_rate=c["drop_rate"], resample_with_conv=False)
    keys = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    sd = R.fill_params(dict(keys), seed)
    m.load_state_dict(sd, strict=True)
    return m.eval(), keys


def gen_bpd(ddpm_torch, m, B, HW, seed):
    from ddpm_torch.functions import flat_mean
    T = BPD_T
    betas = ddpm_torch.get_beta_schedule("linear", 1e-4, 0.02, T)
    g = torch.Generator().manual_seed(seed + 1000)
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
    return dict(T=T, x0=x0, noise=noise, cases=cases)


def gen_noresample(out_dir):
    ddpm_torch, _ = import_reference()
    betas = ddpm_torch.get_beta_schedule("linear", 1e-4, 0.02, 1000)
    diff = ddpm_torch.GaussianDiffusion(betas, "eps", "fixed-large", "mse")
    fx = dict(models={})
    for name, cfg, B, HW, seed in CASES:
        m, keys = build_ref_unet_noresample(ddpm_torch, cfg, seed)
        x0, t, noise = inputs(cfg, B, HW, HW, seed)
        t[0] = 0; t[-1] = 999
        x_t = diff.q_sample(x0, t, noise)
        for p in m.parameters():
            p.requires_grad_(True)
        with torch.no_grad():
            eps = m(x_t, t)
        losses = diff.train_losses(m, x0, t, noise)
        losses.mean().backward()
        e = dict(cfg=dict(cfg), seed=seed, B=B, H=HW, W=HW, keys=keys, x0=x0, t=t, noise=noise, x_t=x_t, eps=eps.clone(),
                 losses=losses.detach().clone(), grad_norm={k: p.grad.norm().item() for k, p in m.named_parameters()})
        if name == BPD_CASE:
            m.zero_grad(set_to_none=True)
            e["bpd"] = gen_bpd(ddpm_torch, m, B, HW, seed)
        fx["models"][name] = e
        print(f"{name}: {len(keys)} tensors, |eps|max {eps.abs().max():.4f} loss {losses.mean():.5f}" +
              (f" bpd {[round(float(c['losses'].sum(1).mean()), 4) for c in e['bpd']['cases'].values()]}" if "bpd" in e else ""))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "unet_noresample.pt")
    torch.save(fx, path)
    print("unet_noresample.pt written to", out_dir, f"({os.path.getsize(path) / 1e6:.3f} MB)")


if __name__ == "__main__":
    gen_noresample(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
