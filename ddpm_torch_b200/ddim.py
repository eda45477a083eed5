"""Host-side mirror of the reference's ``ddim.py`` (DDIM sampler of Song et al. 2020) for the accelerated path:
same ``get_selection_schedule`` / ``DDIM(betas, model_mean_type, model_var_type, loss_type, eta, subsequence)`` /
``DDIM.from_ddpm`` / ``DDIM.p_sample`` surface; the S-step loop runs on the engine's sampler step."""
import math

import torch

from .diffusion import GaussianDiffusion, _coef_tables

__all__ = ["get_selection_schedule", "DDIM"]


def get_selection_schedule(schedule, size, timesteps):
    """ddim.py:30-44: linear = arange(0, T, T//size); quadratic = round(linspace(0, sqrt(0.8 T), size)^2)."""
    assert schedule in {"linear", "quadratic"}
    if schedule == "linear":
        return torch.arange(0, timesteps, timesteps // size)
    return torch.linspace(0, math.sqrt(timesteps * 0.8), size).pow(2).round().to(torch.int64)


class DDIM(GaussianDiffusion):
    _native_bpd = False           # calc_all_bpd over the sub-sequence tables keeps the generic formulas

    def __init__(self, betas, model_mean_type, model_var_type, loss_type, eta, subsequence):
        super().__init__(betas, model_mean_type, model_var_type, loss_type)
        self.eta = eta
        eta2 = eta ** 2
        if eta2 != 1. and model_var_type != "fixed-small":
            self.model_var_type = "fixed-small"          # ddim.py:54-59: DDIM with eta<1 implies the small variance
        # re-derive every table on the sub-sequence (ddim.py:61-92)
        self.__dict__.update(_coef_tables(alphas_bar=self.alphas_bar[subsequence], eta2=eta2))
        self._set_fixed_var(clip=True)
        self.subsequence = torch.as_tensor(subsequence)

    def _model_timesteps(self):
        return self.subsequence.to(torch.int64).clone()

    def _wrap_denoise(self, denoise_fn, device):
        sub = self.subsequence.to(device)
        return lambda x, t: denoise_fn(x, sub.gather(0, t))      # ddim.py:101

    @classmethod
    def from_ddpm(cls, diffusion, eta, subsequence):
        keys = ("betas", "model_mean_type", "model_var_type", "loss_type")
        return cls(**{k: diffusion.__dict__.get(k) for k in keys}, eta=eta, subsequence=subsequence)
