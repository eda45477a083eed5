"""ddpm_torch_b200 — H100-native (sm_90a) drop-in for the hot path of tqch/ddpm-torch:
UNet forward/backward inside GaussianDiffusion.train_losses and the p_sample / DDIM loops.

Public surface mirrors the reference package (ddpm_torch/__init__.py:1-22, ddim.py:11) for the path in scope."""
from . import _lib  # noqa: F401
from .unet import UNet, ModelWrapper
from .diffusion import GaussianDiffusion, get_beta_schedule
from .ddim import DDIM, get_selection_schedule
from . import parallel
from . import optim
from . import postprocess
from . import checkpoint
from . import metrics
from .optim import EMA, FusedAdam

__all__ = ["UNet", "GaussianDiffusion", "get_beta_schedule", "DDIM", "get_selection_schedule", "EMA", "FusedAdam", "ModelWrapper"]
