"""``GaussianDiffusion`` of ddpm_torch/toy/diffusion.py: the image mirror with the toy overrides (no clip in ``p_mean_var``, a
continuous Gaussian decoder in ``_loss_term_bpd``).

For a bare native ``Decoder`` with eps-prediction, fixed variance and CUDA tensors:

* ``train_losses`` (mse) is one fused engine call (q_sample prologue, Decoder forward, per-row mse) with the matching fused backward;
* ``p_sample`` runs the whole chain in one launch (after the per-step table of the timestep path).  ``x_T`` and then one ``[B, D]``
  ``normal_`` per step are drawn in the reference loop's order (including the draw at t = 0, which the reference makes and discards),
  so the generator stream is the reference's.

Everything else takes the generic formulas, as the reference toy does."""
import ctypes as C
import math

import torch

from .. import _lib
from .. import diffusion
from ..functions import continuous_gaussian_loglik, flat_mean, normal_kl
from .model import Decoder


class GaussianDiffusion(diffusion.GaussianDiffusion):

    def p_mean_var(self, denoise_fn, x_t, t, clip_denoised, return_pred):
        """toy/diffusion.py:17-50: the image version with the clamp replaced by the identity."""
        return super().p_mean_var(denoise_fn, x_t, t, False, return_pred)

    def _loss_term_bpd(self, denoise_fn, x_0, x_t, t, clip_denoised, return_pred):
        """toy/diffusion.py:55-68: KL for t > 0, continuous Gaussian decoder NLL at t = 0, in bits."""
        true_mean, _, true_logvar = self.q_posterior_mean_var(x_0=x_0, x_t=x_t, t=t)
        model_mean, _, model_logvar, pred_x_0 = self.p_mean_var(denoise_fn, x_t=x_t, t=t, clip_denoised=clip_denoised, return_pred=True)
        kl = flat_mean(normal_kl(true_mean, true_logvar, model_mean, model_logvar)) / math.log(2.)
        nll = flat_mean(continuous_gaussian_loglik(x_0, model_mean, logvar=model_logvar).neg()) / math.log(2.)
        out = torch.where(t.to(kl.device) > 0, kl, nll)
        return (out, pred_x_0) if return_pred else out

    def _toy_native(self, denoise_fn, x):
        ok = (isinstance(denoise_fn, Decoder) and x.is_cuda and self.model_mean_type == "eps"
              and self.model_var_type in ("fixed-small", "fixed-large"))
        return denoise_fn if ok else None

    def train_losses(self, denoise_fn, x_0, t, noise=None):
        if noise is None:
            noise = torch.randn_like(x_0)
        model = self._toy_native(denoise_fn, x_0)
        if model is None or self.loss_type != "mse":
            return super().train_losses(denoise_fn, x_0, t, noise)
        model._check(x_0)
        t = t.to(device=x_0.device, dtype=torch.int64).contiguous()
        return _ToyTrainLossFn.apply(self, model, x_0.contiguous().float(), t, noise.contiguous().float(), *model.parameters())

    @torch.inference_mode()
    def p_sample(self, denoise_fn, shape=None, device=torch.device("cpu"), noise=None, seed=None, **kwargs):
        """toy/diffusion.py (diffusion.py:160-174) with the toy's p_mean_var."""
        device = torch.device(device)
        model = self._toy_native(denoise_fn, torch.empty(0, device=device))
        if model is None:
            return super().p_sample(denoise_fn, shape=shape, device=device, noise=noise, seed=seed, **kwargs)
        gen = torch.Generator(device).manual_seed(seed) if seed is not None else None
        x = torch.empty(shape, device=device).normal_(generator=gen) if noise is None else noise.to(device).float().clone()
        x = x.contiguous()
        model._check(x)
        S = self.timesteps
        z = torch.empty((S,) + tuple(x.shape), device=device)
        for k in range(S):
            z[k].normal_(generator=gen)
        return sample_chain(model, self._toy_coef_rows(device), x, z)

    def _toy_coef_rows(self, device):
        """[S, 6] fp32 {sqrt_recip_ab, sqrt_recip_m1_ab, coef1, coef2, sigma, t > 0} on ``device``: each entry is the fp32 value
        ``_extract`` gives the generic ``p_sample_step``, and sigma is ``exp(0.5 * logvar)`` computed there on the same device."""
        f = lambda a: torch.as_tensor(a, dtype=torch.float32, device=device)
        S = self.timesteps
        nz = (torch.arange(S, device=device) > 0).float()
        return torch.stack([f(self.sqrt_recip_alphas_bar), f(self.sqrt_recip_m1_alphas_bar), f(self.posterior_mean_coef1),
                            f(self.posterior_mean_coef2), torch.exp(0.5 * f(self.fixed_model_logvar)), nz], dim=1).contiguous()


def sample_chain(model, coef, x, z):
    """All S = len(coef) steps of p_sample on the engine: ``x`` [B, D] is updated in place with ``z[k]`` at t = S-1-k."""
    B, S = x.shape[0], coef.shape[0]
    dev = x.device
    ws = model._workspace(S, False, dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().ddpm_toy_sample(C.byref(model._cfg()), C.byref(model._param_table()), x.data_ptr(), B, S, coef.data_ptr(),
                                              z.contiguous().data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)), "toy_sample")
    return x


class _ToyTrainLossFn(torch.autograd.Function):
    """losses[b] = mean((noise - Decoder(q_sample(x0, t, noise), t))^2) through ddpm_toy_train_forward / ddpm_toy_train_backward."""

    @staticmethod
    def forward(ctx, diff, model, x0, t, noise, *params):
        B = x0.shape[0]
        dev = x0.device
        ta, ts = diff._dev_tables(dev)
        losses = torch.empty(B, dtype=torch.float32, device=dev)
        ws = model._workspace(B, True, dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ddpm_toy_train_forward(C.byref(model._cfg()), C.byref(model._param_table()), x0.data_ptr(), t.data_ptr(),
                                                         noise.data_ptr(), ta.data_ptr(), ts.data_ptr(), B, losses.data_ptr(),
                                                         ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)), "toy_train_forward")
        ctx.model, ctx.ws, ctx.keep = model, ws, (t, noise)
        return losses

    @staticmethod
    def backward(ctx, g):
        from .model import _split
        model = ctx.model
        t, noise = ctx.keep
        g = g.contiguous().float()
        dev = g.device
        flat = torch.empty(sum(p.numel() for p in model.parameters()), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ddpm_toy_train_backward(C.byref(model._cfg()), C.byref(model._param_table()), t.data_ptr(),
                                                          noise.data_ptr(), g.data_ptr(), g.shape[0], flat.data_ptr(), ctx.ws.data_ptr(),
                                                          ctx.ws.numel(), _lib.stream_ptr(dev)), "toy_train_backward")
        return (None, None, None, None, None, *_split(flat, model))
