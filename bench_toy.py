"""Toy-model benchmark (train_toy.py's default configuration: Decoder(2, 128, 3), T = 100, eps / fixed-large / mse):
the toy engine (ddpm_torch_b200.toy) against the unmodified reference (ddpm_torch.toy, staged under oracle/_ref) on the same GPU,
in one process with alternating rounds timed by CUDA events.

* train: one training step at B = 1000 (train_losses, backward, torch.optim.Adam step);
* sample: the 100-step p_sample chain at B = 30 000 (Evaluator's batch);
* agreement: loss and flat-gradient rel-L2 on the same weights and batch, and the reference discrete_klv2d between the two
  sample histograms (and between two reference runs, for scale).

Prints the card name and power limit read in the same run, and one JSON line (also written to --out when given)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                               # noqa: BLE001 - the number is reported as unknown, not guessed
        pl = "unknown"
    return name, pl


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train-reps", type=int, default=50)
    ap.add_argument("--sample-reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_toy.py measures on a GPU"
    from ddpm_torch_b200 import toy as N
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from gen_golden_toy import load_toy
    ref_pkg, RM, RD = load_toy()
    dev = "cuda"
    T = 100
    betas = N.get_beta_schedule("linear", 0.001, 0.2, T)
    torch.manual_seed(1234)
    ref_model = RM.Decoder(2, 128, 3).to(dev)
    nat_model = N.Decoder(2, 128, 3).to(dev)
    nat_model.load_state_dict(ref_model.state_dict())
    rdiff = RD.GaussianDiffusion(betas=ref_pkg.diffusion.get_beta_schedule("linear", 0.001, 0.2, T), model_mean_type="eps",
                                 model_var_type="fixed-large", loss_type="mse")
    ndiff = N.GaussianDiffusion(betas, "eps", "fixed-large", "mse")

    g = torch.Generator(dev).manual_seed(0)
    x0 = torch.randn(1000, 2, device=dev, generator=g)
    t = torch.randint(T, (1000,), device=dev, generator=g)
    noise = torch.randn(1000, 2, device=dev, generator=g)
    # agreement on identical weights and batch (before any optimiser step)
    lr_ = rdiff.train_losses(ref_model, x_0=x0, t=t, noise=noise); lr_.mean().backward()
    ln_ = ndiff.train_losses(nat_model, x0, t, noise); ln_.mean().backward()
    gr = torch.cat([p.grad.flatten() for p in ref_model.parameters()]).double()
    gn = torch.cat([p.grad.flatten() for p in nat_model.parameters()]).double()
    agree = {"loss_ref": lr_.mean().item(), "loss_native": ln_.mean().item(),
             "loss_rel_err": abs(ln_.mean().item() - lr_.mean().item()) / abs(lr_.mean().item()),
             "grad_rel_l2": ((gn - gr).norm() / gr.norm()).item()}

    def step_fn(model, diff, opt):
        def f():
            opt.zero_grad(set_to_none=True)
            diff.train_losses(model, x_0=x0, t=t, noise=noise).mean().backward()
            opt.step()
        return f

    ropt = torch.optim.Adam(ref_model.parameters(), lr=1e-3)
    nopt = torch.optim.Adam(nat_model.parameters(), lr=1e-3)
    fr, fn = step_fn(ref_model, rdiff, ropt), step_fn(nat_model, ndiff, nopt)
    sr = lambda: rdiff.p_sample(ref_model, shape=(30000, 2), device=torch.device(dev), noise=None)
    sn = lambda: ndiff.p_sample(nat_model, shape=(30000, 2), device=torch.device(dev))
    for f in (fr, fn):
        for _ in range(5):
            f()
    sr(); sn(); torch.cuda.synchronize()
    tr, tn, smr, smn = [], [], [], []
    for _ in range(a.rounds):
        tr.append(timed(fr, a.train_reps)); tn.append(timed(fn, a.train_reps))
        smr.append(timed(sr, a.sample_reps)); smn.append(timed(sn, a.sample_reps))

    # sample agreement on identical weights
    nat_model.load_state_dict(ref_model.state_dict())
    F = ref_pkg.functions
    h = lambda s: F.hist2d(s, bins=64, value_range=4)
    torch.manual_seed(5); s_ref = sr().cpu().numpy()
    torch.manual_seed(6); s_ref2 = sr().cpu().numpy()
    torch.manual_seed(5); s_nat = sn().cpu().numpy()
    agree["sample_kl_native_vs_ref"] = float(F.discrete_klv2d(h(s_ref), h(s_nat)))
    agree["sample_kl_ref_vs_ref"] = float(F.discrete_klv2d(h(s_ref), h(s_ref2)))
    name, pl = card()
    med = lambda v: float(np.median(v))
    res = {"workload": "toy Decoder(2,128,3) T=100", "gpu": name, "power_limit": pl,
           "train_step_ms": {"reference": med(tr), "native": med(tn), "speedup": med(tr) / med(tn), "B": 1000},
           "sample_chain_ms": {"reference": med(smr), "native": med(smn), "speedup": med(smr) / med(smn), "B": 30000, "steps": T},
           "agreement": agree, "rounds": a.rounds}
    print(f"{name}, power limit {pl}")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
