"""Mirror of ``ddpm_torch.toy`` for the 2-D toy models: ``Decoder`` and ``GaussianDiffusion`` on the toy engine
(csrc/toy_mlp.cuh).  ``Trainer``, ``Evaluator`` and ``DataStreamer`` are host code that does not depend on the denoiser, so the
reference's classes are used with these two."""
from ..diffusion import get_beta_schedule
from .diffusion import GaussianDiffusion
from .model import Decoder

__all__ = ["GaussianDiffusion", "get_beta_schedule", "Decoder"]
