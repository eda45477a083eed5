"""Likelihood helpers of the reference's bits-per-dim path (ddpm_torch/functions.py:28-60, :99-101) — generic PyTorch
formulas used by ``GaussianDiffusion._loss_term_bpd`` / ``calc_all_bpd`` / ``loss_type="kl"``, parity-tested on CPU against
goldens written by the unmodified reference.
``calc_all_bpd`` of a native UNet (eps-prediction, fixed variance, CUDA input) does not call them: the engine's bits/dim step
(``bpd_elem`` in csrc/kernels_simt.cuh) repeats these operations in the same order in the epilogue of the UNet's final conv.
``loss_type="kl"`` training stays on these formulas (it would need the backward of the bound)."""
import math

import torch

_SQRT_2_OVER_PI = math.sqrt(2. / math.pi)


def flat_mean(x, start_dim=1):
    """functions.py:99-101"""
    return x.mean(dim=list(range(start_dim, x.ndim)))


def normal_kl(mean1, logvar1, mean2, logvar2):
    """KL( N(mean1, exp(logvar1)) || N(mean2, exp(logvar2)) ) element-wise, functions.py:29-34:
    0.5 * (-1 - d + (m1 - m2)^2 * exp(-lv2) + exp(d)),  d = lv1 - lv2."""
    d = logvar1 - logvar2
    sq = (mean1 - mean2) ** 2
    return ((-1.0 - d) + sq * torch.exp(-logvar2) + torch.exp(d)) * 0.5


def approx_std_normal_cdf(x):
    """tanh approximation of the standard normal CDF (Page 1977), functions.py:38-44"""
    return 0.5 * (1. + torch.tanh(_SQRT_2_OVER_PI * (x + 0.044715 * x ** 3)))


def discretized_gaussian_loglik(x, means, log_scale, precision=1. / 255, cutoff=(-0.999, 0.999), tol=1e-12):
    """log-probability of 8-bit data rescaled to [-1, 1] under a Gaussian discretised to bins of half-width ``precision``,
    with the outermost bins extended to +-infinity (functions.py:48-64)."""
    if isinstance(cutoff, float):
        cutoff = (-cutoff, cutoff)
    centered = x - means
    inv_std = torch.exp(-log_scale)
    one = torch.ones((), dtype=torch.float32, device=x.device)
    hi = torch.where(x > cutoff[1], one, approx_std_normal_cdf(inv_std * (centered + precision)))
    lo = torch.where(x < cutoff[0], one * 0, approx_std_normal_cdf(inv_std * (centered - precision)))
    return torch.log((hi - lo - tol).clamp(min=0) + tol)


def continuous_gaussian_loglik(x, mean, logvar):
    """functions.py:78-83: element-wise log N(x; mean, exp(logvar)), the decoder term of the toy models' bound."""
    x_centered = x - mean
    inv_var = torch.exp(-logvar)
    log_probs = x_centered.pow(2) * inv_var + math.log(2 * math.pi) + logvar
    return log_probs.mul(0.5).neg()
