"""Write tests/golden/toy.pt from the UNMODIFIED reference toy package on the CPU (oracle/ref_loader.py).

``ddpm_torch/toy/__init__.py`` imports ``toy_data.py``, which needs scikit-learn at import time; the two modules used here
(``toy_model.py``, ``diffusion.py``) do not, so they are loaded as submodules of an empty ``ddpm_torch.toy`` package object.
Nothing of the reference is edited.

Contents, for seeded Decoder(2, 128, 3) and Decoder(1, 64, 1) (T = 100, the train_toy.py default schedule):
state dicts; forward outputs over edge and random t; train_losses with given noise and the per-parameter gradients of
loss.mean(); single p_sample_step results given z; _loss_term_bpd at t = 0 (continuous decoder NLL) and t > 0 (KL)."""
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load_toy():
    from oracle import ref_loader
    ddpm_torch, _ = ref_loader.load()
    pkg_dir = os.path.join(os.path.dirname(ddpm_torch.__file__), "toy")
    if "ddpm_torch.toy" not in sys.modules or not hasattr(sys.modules["ddpm_torch.toy"], "Decoder"):
        pkg = types.ModuleType("ddpm_torch.toy"); pkg.__path__ = [pkg_dir]
        sys.modules["ddpm_torch.toy"] = pkg
    out = {}
    for name in ("toy_model", "diffusion"):
        full = "ddpm_torch.toy." + name
        if full not in sys.modules:
            spec = importlib.util.spec_from_file_location(full, os.path.join(pkg_dir, name + ".py"))
            mod = importlib.util.module_from_spec(spec)
            sys.modules[full] = mod
            spec.loader.exec_module(mod)
        out[name] = sys.modules[full]
    return ddpm_torch, out["toy_model"], out["diffusion"]


CASES = [("default", 2, 128, 3, 1234), ("small", 1, 64, 1, 7)]


def main(path=os.path.join(ROOT, "tests", "golden", "toy.pt")):
    ddpm_torch, tm, td = load_toy()
    T = 100
    betas = ddpm_torch.diffusion.get_beta_schedule("linear", 0.001, 0.2, T)
    diff = td.GaussianDiffusion(betas=betas, model_mean_type="eps", model_var_type="fixed-large", loss_type="mse")
    res = {"T": T}
    for name, D, M, L, seed in CASES:
        torch.manual_seed(seed)
        m = tm.Decoder(D, M, L)
        g = torch.Generator().manual_seed(seed + 1)
        B = 37
        x = torch.randn(B, D, generator=g)
        t = torch.cat([torch.tensor([0, 1, T - 1]), torch.randint(T, (B - 3,), generator=g)])
        noise = torch.randn(B, D, generator=g)
        z = torch.randn(B, D, generator=g)
        with torch.no_grad():
            out = m(x, t)
        m.zero_grad()
        loss = diff.train_losses(m, x_0=x, t=t, noise=noise)
        loss.mean().backward()
        grads = [p.grad.clone() for p in m.parameters()]
        with torch.no_grad():
            mean, _, logvar, pred = diff.p_mean_var(m, x, t, clip_denoised=True, return_pred=True)
            step = mean + (t > 0).float().reshape(-1, 1) * torch.exp(0.5 * logvar) * z
            x_t = diff.q_sample(x, t, noise=noise)
            bpd = diff._loss_term_bpd(m, x_0=x, x_t=x_t, t=t, clip_denoised=True, return_pred=False)
        res[name] = {"cfg": (D, M, L, seed), "state_dict": m.state_dict(),
                     "x": x, "t": t, "noise": noise, "z": z, "out": out, "losses": loss.detach(), "grads": grads,
                     "step": step, "pred_x_0": pred, "bpd": bpd}
    torch.save(res, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
