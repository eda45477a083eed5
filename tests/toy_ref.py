"""Restatement of ddpm_torch/toy/toy_model.py's Decoder as plain tensor ops, pinned to tests/golden/toy.pt
(test_toy_cpu.py).  In fp64 it is the reference the toy engine is measured against; it is differentiable, so autograd over
its tied weights gives the reference gradients."""
import math

import torch
import torch.nn.functional as F

KEYS = ["in_fc.weight", "temp_fc.0.norm1.weight", "temp_fc.0.norm1.bias", "temp_fc.0.fc1.weight", "temp_fc.0.norm2.weight",
        "temp_fc.0.norm2.bias", "temp_fc.0.fc2.weight", "temp_fc.0.enc.weight", "temp_fc.0.enc.bias", "out_norm.weight",
        "out_norm.bias", "out_fc.weight", "out_fc.bias", "t_proj.0.weight", "t_proj.0.bias"]


def timestep_embedding(t, dim, dtype):
    half = dim // 2
    k = math.log(10000) / (half - 1)
    f = torch.exp(-torch.arange(half, dtype=dtype, device=t.device) * k)
    a = torch.outer(t.reshape(-1).to(dtype), f)
    return torch.cat([torch.sin(a), torch.cos(a)], dim=1)


def decoder_forward(p, L, x, t):
    """p: the 15 unique parameters by KEYS name; one TemporalLayer applied L times."""
    M = p["in_fc.weight"].shape[0]
    lr = lambda v: F.leaky_relu(v, 0.02)
    ln = lambda v, g, b: F.layer_norm(v, (M,), g, b, 1e-5)
    e = lr(F.linear(timestep_embedding(t, M, x.dtype), p["t_proj.0.weight"], p["t_proj.0.bias"]))
    E = F.linear(e, p["temp_fc.0.enc.weight"], p["temp_fc.0.enc.bias"])
    h = F.linear(x, p["in_fc.weight"])
    for _ in range(L):
        u = F.linear(lr(ln(h, p["temp_fc.0.norm1.weight"], p["temp_fc.0.norm1.bias"])), p["temp_fc.0.fc1.weight"]) + E
        h = F.linear(lr(ln(u, p["temp_fc.0.norm2.weight"], p["temp_fc.0.norm2.bias"])), p["temp_fc.0.fc2.weight"]) + h
    return F.linear(ln(h, p["out_norm.weight"], p["out_norm.bias"]), p["out_fc.weight"], p["out_fc.bias"])


def params_of(module_or_sd, dtype=torch.float64, device=None, grad=False):
    sd = module_or_sd.state_dict() if hasattr(module_or_sd, "state_dict") else module_or_sd
    return {k: sd[k].detach().to(dtype=dtype, device=device).clone().requires_grad_(grad) for k in KEYS}
