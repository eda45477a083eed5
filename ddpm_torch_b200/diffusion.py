"""Host-side mirror of ``ddpm_torch.diffusion`` (reference diffusion.py) for the accelerated path.

``GaussianDiffusion`` keeps the reference's constructor, attribute names (fp64 coefficient tables) and method
signatures.  When ``denoise_fn`` is a ``ddpm_torch_b200.UNet`` (optionally wrapped in DDP / a ``.module`` holder) and
the configuration is the one every reference config uses (eps-prediction, fixed variance, mse loss):

* ``train_losses``  -> one fused engine call: q_sample prologue, UNet forward, per-sample MSE (and the matching
  fused backward through autograd),
* ``p_sample`` / ``p_sample_step`` -> the engine's sampler step (UNet forward + the alpha/beta update of
  diffusion.py:107-158 in one launch sequence, replayed from a CUDA graph once per timestep),
* ``calc_all_bpd`` -> the engine's bits/dim step (q_sample, UNet forward and the variational-bound terms of
  diffusion.py:203-215 in one launch sequence, replayed from a CUDA graph once per timestep).

Any other ``denoise_fn`` (wrappers, other modules) takes the generic formulas below, written with plain torch ops; the toy models'
native paths are in ``ddpm_torch_b200.toy``.
"""
import contextlib
import ctypes as C

import math

import torch

from . import _lib
from .unet import UNet


def get_beta_schedule(beta_schedule, beta_start, beta_end, timesteps, dtype=torch.float64):
    """Same schedules and fp64 arithmetic as diffusion.py:13-29."""
    lin = lambda a, b, n: torch.linspace(a, b, n, dtype=dtype)
    if beta_schedule == "linear":
        betas = lin(beta_start, beta_end, timesteps)
    elif beta_schedule == "quad":
        betas = lin(beta_start ** 0.5, beta_end ** 0.5, timesteps) ** 2
    elif beta_schedule in ("warmup10", "warmup50"):
        n = int(timesteps * (0.1 if beta_schedule == "warmup10" else 0.5))
        betas = torch.full((timesteps,), beta_end, dtype=dtype)
        betas[:n] = lin(beta_start, beta_end, n)
    elif beta_schedule == "const":
        betas = torch.full((timesteps,), beta_end, dtype=dtype)
    elif beta_schedule == "jsd":
        betas = 1. / lin(timesteps, 1, timesteps)
    else:
        raise NotImplementedError(beta_schedule)
    assert betas.shape == (timesteps,)
    return betas


def _native(denoise_fn):
    """Unwrap DDP / holders; return the engine-backed UNet or None."""
    m = denoise_fn
    for _ in range(3):
        if isinstance(m, UNet):
            return m
        m = getattr(m, "module", None)
        if m is None:
            return None
    return None


def _flat_mean(x):
    return x.mean(dim=list(range(1, x.ndim)))


def _coef_tables(betas=None, alphas_bar=None, eta2=None):
    """All fp64 coefficient tables as a dict keyed by the reference's attribute names.

    ``betas`` given: the full-chain tables of diffusion.py:52-67.  ``alphas_bar`` given (already restricted to a
    sub-sequence) with ``eta2 = eta**2``: the DDIM re-derivation of ddim.py:61-92.  Every expression keeps the reference's
    operand order, so the tables are bit-identical (tests/test_oracle_golden.py::test_mirror_tables_bit_exact)."""
    T = {}
    one = torch.ones(1, dtype=torch.float64)
    if alphas_bar is None:
        alphas = 1 - betas
        ab = torch.cumprod(alphas, dim=0)
        prev = torch.cat([one, ab[:-1]])
    else:
        ab = alphas_bar
        prev = torch.cat([one, ab[:-1]], dim=0)
        alphas = ab / prev
        betas = 1. - alphas
        T.update(betas=betas, alphas=alphas, alphas_bar_prev=prev, sqrt_alphas_bar_prev=prev.sqrt())
    rest = 1. - ab                                     # 1 - alpha_bar_t
    T.update(alphas_bar=ab, sqrt_alphas_bar=ab.sqrt(), sqrt_one_minus_alphas_bar=rest.sqrt(),
             sqrt_recip_alphas_bar=(1. / ab).sqrt(), sqrt_recip_m1_alphas_bar=(1. / ab - 1.).sqrt())
    if eta2 is None:
        pv = betas * (1. - prev) / rest
        T.update(posterior_var=pv, posterior_logvar_clipped=torch.log(torch.cat([pv[[1]], pv[1:]])),
                 posterior_mean_coef1=betas * prev.sqrt() / rest, posterior_mean_coef2=alphas.sqrt() * (1. - prev) / rest)
    else:
        pv = betas * (1. - prev) / rest * eta2
        c2 = (1 - ab - eta2 * betas).sqrt() * (1 - prev).sqrt() / rest
        T.update(posterior_var=pv, posterior_logvar_clipped=torch.log(torch.cat([pv[[1]], pv[1:]]).clip(min=1e-20)),
                 posterior_mean_coef2=c2, posterior_mean_coef1=prev.sqrt() * (1. - alphas.sqrt() * c2))
    return T


class GaussianDiffusion:
    def __init__(self, betas, model_mean_type, model_var_type, loss_type, **kwargs):
        assert isinstance(betas, torch.Tensor) and betas.dtype == torch.float64
        assert (betas > 0).all() and (betas <= 1).all()
        self.betas = betas
        self.model_mean_type, self.model_var_type, self.loss_type = model_mean_type, model_var_type, loss_type
        self.timesteps = len(betas)
        self.__dict__.update(_coef_tables(betas))
        self._set_fixed_var(clip=False)
        self._dev_cache = {}

    def _set_fixed_var(self, clip):
        large = torch.cat([self.posterior_var[[1]], self.betas[1:]])
        if clip:
            large = large.clip(min=1e-20)
        self.fixed_model_var, self.fixed_model_logvar = {
            "fixed-large": (self.betas, torch.log(large)),
            "fixed-small": (self.posterior_var, self.posterior_logvar_clipped),
        }.get(self.model_var_type, (None, None))

    # ------------------------------------------------------------------ generic (torch) formulas
    @staticmethod
    def _extract(arr, t, x, dtype=torch.float32, device=torch.device("cpu"), ndim=4):
        if x is not None:
            dtype, device, ndim = x.dtype, x.device, x.ndim
        out = torch.as_tensor(arr, dtype=dtype, device=device).gather(0, t)
        return out.reshape((-1,) + (1,) * (ndim - 1))

    def q_mean_var(self, x_0, t):
        return (self._extract(self.sqrt_alphas_bar, t, x_0) * x_0, self._extract(1. - self.alphas_bar, t, x_0),
                self._extract(torch.log(1 - self.alphas_bar), t, x_0))

    def q_sample(self, x_0, t, noise=None):
        if noise is None:
            noise = torch.randn_like(x_0)
        return self._extract(self.sqrt_alphas_bar, t, x_0) * x_0 + \
            self._extract(self.sqrt_one_minus_alphas_bar, t, x_0) * noise

    def q_posterior_mean_var(self, x_0, x_t, t):
        mean = self._extract(self.posterior_mean_coef1, t, x_0) * x_0 + self._extract(self.posterior_mean_coef2, t, x_0) * x_t
        return mean, self._extract(self.posterior_var, t, x_0), self._extract(self.posterior_logvar_clipped, t, x_0)

    def _pred_x_0_from_eps(self, x_t, eps, t):
        return self._extract(self.sqrt_recip_alphas_bar, t, x_t) * x_t - self._extract(self.sqrt_recip_m1_alphas_bar, t, x_t) * eps

    def _pred_x_0_from_mean(self, x_t, mean, t):
        c1, c2 = self._extract(self.posterior_mean_coef1, t, x_t), self._extract(self.posterior_mean_coef2, t, x_t)
        return mean / c1 - c2 / c1 * x_t

    def p_mean_var(self, denoise_fn, x_t, t, clip_denoised, return_pred):
        out = denoise_fn(x_t, t)
        if self.model_var_type == "learned":
            out, model_logvar = out.chunk(2, dim=1)
            model_var = torch.exp(model_logvar)
        elif self.model_var_type in ("fixed-small", "fixed-large"):
            model_var, model_logvar = self._extract(self.fixed_model_var, t, x_t), self._extract(self.fixed_model_logvar, t, x_t)
        else:
            raise NotImplementedError(self.model_var_type)
        clip = (lambda v: v.clamp(-1., 1.)) if clip_denoised else (lambda v: v)
        if self.model_mean_type == "mean":
            pred_x_0, model_mean = clip(self._pred_x_0_from_mean(x_t, out, t)), out
        elif self.model_mean_type == "x_0":
            pred_x_0 = clip(out)
            model_mean = self.q_posterior_mean_var(pred_x_0, x_t, t)[0]
        elif self.model_mean_type == "eps":
            pred_x_0 = clip(self._pred_x_0_from_eps(x_t, out, t))
            model_mean = self.q_posterior_mean_var(pred_x_0, x_t, t)[0]
        else:
            raise NotImplementedError(self.model_mean_type)
        return (model_mean, model_var, model_logvar, pred_x_0) if return_pred else (model_mean, model_var, model_logvar)

    def _fast_ok(self, denoise_fn):
        m = _native(denoise_fn)
        ok = m is not None and self.model_mean_type == "eps" and self.model_var_type in ("fixed-small", "fixed-large")
        return m if ok else None

    # ------------------------------------------------------------------ sampling
    def p_sample_step(self, denoise_fn, x_t, t, clip_denoised=True, return_pred=False, generator=None):
        model_mean, _, model_logvar, pred_x_0 = self.p_mean_var(denoise_fn, x_t, t, clip_denoised, True)
        noise = torch.empty_like(x_t).normal_(generator=generator)
        nonzero = (t > 0).reshape((-1,) + (1,) * (x_t.ndim - 1)).to(x_t)
        sample = model_mean + nonzero * torch.exp(0.5 * model_logvar) * noise
        return (sample, pred_x_0) if return_pred else sample

    def _coef_rows(self):
        """[S,6] fp32 rows {sqrt_recip_ab, sqrt_recip_m1_ab, c1, c2, exp(.5*logvar), t>0}; every entry goes through the
        same fp64 -> fp32 cast as ``_extract`` (diffusion.py:83) and sigma is exp(0.5*fp32(logvar)) as in :157."""
        f = lambda a: torch.as_tensor(a, dtype=torch.float32)
        S = len(self.betas)
        nz = (torch.arange(S) > 0).float()
        return torch.stack([f(self.sqrt_recip_alphas_bar), f(self.sqrt_recip_m1_alphas_bar), f(self.posterior_mean_coef1),
                            f(self.posterior_mean_coef2), torch.exp(0.5 * f(self.fixed_model_logvar)), nz], dim=1).contiguous()

    def _model_timesteps(self):
        return torch.arange(len(self.betas), dtype=torch.int64)

    @torch.inference_mode()
    def p_sample(self, denoise_fn, shape=None, device=torch.device("cpu"), noise=None, seed=None, rng="torch", use_graph=True, split=None):
        """diffusion.py:160-174.  ``rng="torch"`` consumes a torch.Generator exactly like the reference (bit-identical
        noise stream); ``rng="philox"`` draws the per-step noise inside the step kernel (one launch sequence per step)."""
        model = self._fast_ok(denoise_fn)
        B = (shape or noise.shape)[0]
        gen = torch.Generator(device).manual_seed(seed) if seed is not None else None
        x_t = torch.empty(shape, device=device).normal_(generator=gen) if noise is None else noise.to(device)
        S = len(self.betas)
        if model is None:
            t = torch.empty((B,), dtype=torch.int64, device=device)
            fn = self._wrap_denoise(denoise_fn, device)
            for ti in range(S - 1, -1, -1):
                t.fill_(ti)
                x_t = self.p_sample_step(fn, x_t, t, generator=gen)
            return x_t
        return _native_sample_loop(self, model, x_t.contiguous().float().clone(), gen, rng, seed, use_graph, split)

    def _wrap_denoise(self, denoise_fn, device):
        return denoise_fn

    @torch.inference_mode()
    def p_sample_progressive(self, denoise_fn, shape, device=torch.device("cpu"), noise=None, pred_freq=10, seed=None):
        """diffusion.py:176-198.  Native path: every step is the engine's sampler step, which also writes the clipped x_0
        prediction (ddpm_sampler_step_pred); predictions are copied out every ``pred_freq`` steps exactly as the reference does."""
        B = (shape or noise.shape)[0]
        gen = torch.Generator(device).manual_seed(seed) if seed is not None else None
        x_t = torch.empty(shape, device=device).normal_(generator=gen) if noise is None else noise.to(device)
        n = self.timesteps // pred_freq
        preds = torch.zeros((n, B) + tuple(shape[1:]), dtype=torch.float32)
        idx = n
        model = self._fast_ok(denoise_fn)
        if model is not None and x_t.is_cuda:
            L = _lib.lib()
            x_t = x_t.contiguous().float().clone()
            _, _, H, W = x_t.shape
            with _native_mode(model, x_t, "the sampler state"):
                h = model.prepare(B, H, W, training=False, force_repack=True)
                _sampler_tables(self, [h], self.timesteps - 1)
                z, pred = torch.empty_like(x_t), torch.empty_like(x_t)
                for ti in range(self.timesteps - 1, -1, -1):
                    z.normal_(generator=gen)
                    _lib.check(L.ddpm_sampler_step_pred(h, x_t.data_ptr(), z.data_ptr(), 0, pred.data_ptr(), _lib.stream_ptr()), "sampler_step")
                    if (ti + 1) % pred_freq == 0:
                        idx -= 1
                        preds[idx] = pred.cpu()
            return x_t.cpu(), preds
        t = torch.empty(B, dtype=torch.int64, device=device)
        fn = self._wrap_denoise(denoise_fn, device)
        for ti in range(self.timesteps - 1, -1, -1):
            t.fill_(ti)
            x_t, pred = self.p_sample_step(fn, x_t, t, return_pred=True, generator=gen)
            if (ti + 1) % pred_freq == 0:
                idx -= 1
                preds[idx] = pred.cpu()
        return x_t.cpu(), preds

    # ------------------------------------------------------------------ training
    def train_losses(self, denoise_fn, x_0, t, noise=None):
        if noise is None:
            noise = torch.randn_like(x_0)
        model = self._fast_ok(denoise_fn)
        if model is not None and self.loss_type == "mse" and x_0.is_cuda:
            return _TrainLossFn.apply(self, model, denoise_fn, x_0.contiguous().float(), t.contiguous(), noise.contiguous().float(),
                                      *model._params)
        x_t = self.q_sample(x_0, t, noise=noise)
        if self.loss_type == "kl":      # diffusion.py:226-228: weighted variational bound, generic torch path only
            return self._loss_term_bpd(denoise_fn, x_0=x_0, x_t=x_t, t=t, clip_denoised=False, return_pred=False)
        if self.loss_type != "mse":
            raise NotImplementedError(self.loss_type)
        assert self.model_var_type != "learned"
        target = {"mean": lambda: self.q_posterior_mean_var(x_0, x_t, t)[0], "x_0": lambda: x_0, "eps": lambda: noise}[self.model_mean_type]()
        return _flat_mean((target - denoise_fn(x_t, t)).pow(2))

    # ------------------------------------------------------------------ log-likelihood in bits per dimension (generic torch)
    def _loss_term_bpd(self, denoise_fn, x_0, x_t, t, clip_denoised, return_pred):
        """diffusion.py:203-215: L_t = KL(q(x_{t-1}|x_t,x_0) || p(x_{t-1}|x_t)) for t > 0, decoder NLL -log p(x_0|x_1) at t = 0."""
        from .functions import discretized_gaussian_loglik, flat_mean, normal_kl
        true_mean, _, true_logvar = self.q_posterior_mean_var(x_0=x_0, x_t=x_t, t=t)
        model_mean, _, model_logvar, pred_x_0 = self.p_mean_var(denoise_fn, x_t=x_t, t=t, clip_denoised=clip_denoised, return_pred=True)
        kl = flat_mean(normal_kl(true_mean, true_logvar, model_mean, model_logvar)) / math.log(2.)
        nll = flat_mean(-discretized_gaussian_loglik(x_0, model_mean, log_scale=0.5 * model_logvar)) / math.log(2.)
        out = torch.where(t.to(kl.device) > 0, kl, nll)
        return (out, pred_x_0) if return_pred else out

    def _prior_bpd(self, x_0):
        """diffusion.py:245-250: KL(q(x_T|x_0) || N(0, I)) in bits per dimension."""
        from .functions import flat_mean, normal_kl
        B, T = len(x_0), self.timesteps
        T_mean, _, T_logvar = self.q_mean_var(x_0=x_0, t=(T - 1) * torch.ones((B,), dtype=torch.int64, device=x_0.device))
        zero = torch.zeros((), dtype=T_mean.dtype, device=T_mean.device)
        return flat_mean(normal_kl(T_mean, T_logvar, zero, zero)) / math.log(2.)

    # DDIM re-derives the tables on a sub-sequence; its calc_all_bpd keeps the generic formulas
    _native_bpd = True

    def calc_all_bpd(self, denoise_fn, x_0, clip_denoised=True, *, noise=None, use_graph=True):
        """diffusion.py:252-270.  Upstream unpacks ``B, T = x_0.shape, self.timesteps`` (B becomes the shape tuple and
        ``torch.empty([B, ])`` raises); this is the evident intent, B = batch size.
        Returns (total_bpd [B], losses [B, T], prior_bpd [B], mses [B, T]), fp32 on the CPU as in the reference (:255-256).

        Native path (a native UNet, eps-prediction, fixed variance, CUDA ``x_0``): every timestep is one engine launch
        sequence (ddpm_bpd_step: q_sample in in_conv's loads, the UNet forward, the bound terms in the final conv's epilogue),
        captured once into a CUDA graph and replayed T times, with no host synchronisation until the [B, T] results are copied
        back.  Each step's noise is drawn like the generic loop's ``torch.randn_like(x_0)`` from the device's default
        generator, so after ``torch.manual_seed(s)`` both paths see the same x_t sequence.  ``noise`` (optional,
        [T, B, C, H, W]) replaces the draws: ``noise[ti]`` is used at step ti."""
        model = self._fast_ok(denoise_fn)
        if model is not None and x_0.is_cuda and self._native_bpd:
            losses, mses = _native_bpd_loop(self, model, x_0.contiguous().float(), clip_denoised, noise, use_graph)
        else:
            losses, mses = self._generic_bpd_terms(denoise_fn, x_0, clip_denoised, noise)
        prior_bpd = self._prior_bpd(x_0).cpu()
        total_bpd = torch.sum(losses, dim=1) + prior_bpd
        return total_bpd, losses, prior_bpd, mses

    def _generic_bpd_terms(self, denoise_fn, x_0, clip_denoised, noise):
        from .functions import flat_mean
        B, T = len(x_0), self.timesteps
        t = torch.empty([B, ], dtype=torch.int64, device=x_0.device)
        losses = torch.zeros([B, T], dtype=torch.float32, device=x_0.device)
        mses = torch.zeros([B, T], dtype=torch.float32, device=x_0.device)
        for ti in range(T - 1, -1, -1):
            t.fill_(ti)
            x_t = self.q_sample(x_0, t=t, noise=None if noise is None else noise[ti].to(x_0))
            loss, pred_x_0 = self._loss_term_bpd(denoise_fn, x_0, x_t=x_t, t=t, clip_denoised=clip_denoised, return_pred=True)
            losses[:, ti] = loss
            mses[:, ti] = flat_mean((pred_x_0 - x_0).pow(2))
        return losses.cpu(), mses.cpu()

    def _bpd_rows(self):
        """[T,9] fp32 rows {sqrt_ab, sqrt_1mab, sqrt_recip_ab, sqrt_recip_m1_ab, post_c1, post_c2, model_logvar, true_logvar,
        t>0} of ddpm_bpd_setup; every entry goes through the same fp64 -> fp32 cast as ``_extract`` (diffusion.py:83)."""
        f = lambda a: torch.as_tensor(a, dtype=torch.float32)
        nz = (torch.arange(self.timesteps) > 0).float()
        return torch.stack([f(self.sqrt_alphas_bar), f(self.sqrt_one_minus_alphas_bar), f(self.sqrt_recip_alphas_bar),
                            f(self.sqrt_recip_m1_alphas_bar), f(self.posterior_mean_coef1), f(self.posterior_mean_coef2),
                            f(self.fixed_model_logvar), f(self.posterior_logvar_clipped), nz], dim=1).contiguous()

    def _dev_tables(self, device):
        k = str(device)
        if k not in self._dev_cache:
            self._dev_cache[k] = (torch.as_tensor(self.sqrt_alphas_bar, dtype=torch.float32, device=device).contiguous(),
                                  torch.as_tensor(self.sqrt_one_minus_alphas_bar, dtype=torch.float32, device=device).contiguous())
        return self._dev_cache[k]


class _TrainLossFn(torch.autograd.Function):
    """losses[b] = mean((noise - UNet(q_sample(x0,t,noise), t))^2) through ddpm_train_forward / ddpm_train_backward."""

    @staticmethod
    def forward(ctx, diffusion, model, wrapper, x0, t, noise, *params):
        B, _, H, W = x0.shape
        train = torch.is_grad_enabled() or any(p.requires_grad for p in params)
        dev = model.flat_params.device
        if x0.device != dev:
            raise RuntimeError(f"UNet lives on {dev} but the batch is on {x0.device}")
        h = model.prepare(B, H, W, training=train)
        ta, ts = diffusion._dev_tables(dev)
        losses = torch.empty(B, dtype=torch.float32, device=dev)
        seed = model.next_dropout_seed() if (model.training and model.drop_rate > 0) else 0
        t = t.to(device=dev, dtype=torch.int64)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ddpm_train_forward(h, x0.data_ptr(), t.data_ptr(), noise.data_ptr(), ta.data_ptr(), ts.data_ptr(),
                                                     losses.data_ptr(), seed, _lib.stream_ptr(dev)), "train_forward")
        ctx.model = model
        ctx.wrapper = wrapper
        ctx.keep = (x0, t, noise)
        return losses

    @staticmethod
    def backward(ctx, g):
        model = ctx.model
        g = g.contiguous().float()
        dev = model.flat_params.device
        model._before_backward()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().ddpm_train_backward(model._h, g.data_ptr(), _lib.stream_ptr(dev)), "train_backward")
        _ddp_allreduce(ctx.wrapper, model)
        flat = model._grads.clone()
        return (None, None, None, None, None, None, *model.grad_views(flat))


def _ddp_allreduce(wrapper, model):
    """The fused path calls the inner UNet directly, so a DistributedDataParallel wrapper's ``forward`` never runs and its
    reducer stays disarmed (its autograd hooks return early) - the replicas would silently diverge under the reference flow
    ``DDP(model)`` + ``diffusion.train_losses(self.model, ...)`` (train.py:110, utils/train.py:144-153).  The engine owns the
    collective instead: ONE mean all-reduce of the flat gradient buffer over the wrapper's process group, issued here,
    before autograd hands the views to ``p.grad``.  (If the reducer happens to be armed, averaging already-equal
    gradients again is the identity.)"""
    import torch.distributed as dist
    if wrapper is model or not (dist.is_available() and dist.is_initialized()):
        return
    if not hasattr(wrapper, "process_group") and not hasattr(wrapper, "module"):
        return
    from .parallel import allreduce_grads_overlapped_
    allreduce_grads_overlapped_(model, group=getattr(wrapper, "process_group", None))     # chunk-wise, overlapped with the backward's tail


@contextlib.contextmanager
def _native_mode(model, x, what):
    """Scope of a native loop: every launch targets the model's device (generate.py:59 never calls set_device) and the model is
    in eval mode; the caller's train mode comes back on the way out.  ``x`` (named ``what`` in the error) must be on that device."""
    dev = model.flat_params.device
    if x.device != dev:
        raise RuntimeError(f"UNet lives on {dev} but {what} is on {x.device}")
    was_training = model.training
    model.eval()
    try:
        with torch.cuda.device(dev):
            yield
    finally:
        if was_training:
            model.train()


def _sampler_tables(diffusion, hs, first):
    """Upload the diffusion's sampler step tables to every handle in ``hs`` and arm each at step ``first``."""
    L = _lib.lib()
    coef, tmod = diffusion._coef_rows(), diffusion._model_timesteps().contiguous()
    for h in hs:
        _lib.check(L.ddpm_sampler_setup(h, coef.shape[0], tmod.data_ptr(), coef.data_ptr()), "sampler_setup")
        _lib.check(L.ddpm_sampler_reset(h, first, _lib.stream_ptr()), "sampler_reset")


def _capture(step, gen=None):
    """A CUDA graph of ``step()``, captured on a side stream (capture does not execute it).  ``gen``, a generator the step
    draws from, is registered with the graph, so every replay advances its Philox offset exactly like an eager draw."""
    graph = torch.cuda.CUDAGraph()
    if gen is not None:
        graph.register_generator_state(gen)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    return graph


def _graph_loop(model, key, n, step, x, gen=None, **outs):
    """``n`` steps of a native loop, each a noise draw into ``ent["z"]`` and ``step(ent)``: one eager step, then a CUDA graph of
    the step, cached on the model under ``key`` and replayed.  ``key`` ends with the ``ddpm_unet_graph_epoch`` of every handle
    the step launches on: the graph holds addresses in their workspaces and step tables, which stay put while the epochs do.
    The entry ``ent`` owns what the graph touches: ``x`` (refilled on every call), ``z``, an fp32 buffer per ``outs`` name and
    shape, and, for a seeded run, a generator registered with the graph that takes over ``gen``'s state."""
    ent = model._sampler_cache.get(key)
    if ent is None:
        if len(model._sampler_cache) >= 4:
            model._sampler_cache.clear()
        ent = model._sampler_cache[key] = {"x": torch.empty_like(x), "z": torch.empty_like(x), "graph": None,
                                           "gen": None if gen is None else torch.Generator(x.device),
                                           **{k: torch.empty(s, dtype=torch.float32, device=x.device) for k, s in outs.items()}}
    ent["x"].copy_(x)
    if gen is not None:
        ent["gen"].set_state(gen.get_state())      # continue the caller's stream (x_T may already have been drawn from it)

    def run():
        ent["z"].normal_(generator=ent["gen"])
        step(ent)

    if ent["graph"] is None:
        run()
        ent["graph"] = _capture(run, ent["gen"])
        n -= 1
    for _ in range(n):
        ent["graph"].replay()
    return ent


def _native_sample_loop(diffusion, model, x, gen, rng, seed, use_graph, split=None):
    """T sampler steps on the engine: per step {noise draw, step-table fetch, UNet forward with the alpha/beta update in the final
    conv's epilogue}; captured once, replayed T times - one graph launch per timestep.

    ``split=2`` (opt-in; DDPM_SAMPLER_SPLIT overrides the default of 1; not measured on H100): the batch is cut into two
    halves with their own plans, run on two forked streams inside the SAME captured graph, so that one half's HBM-bound
    GroupNorm kernels overlap the other half's tensor-core kernels.  Images and noise are per-sample, so the result is
    the same as the unsplit loop."""
    import os
    L = _lib.lib()
    B, _, H, W = x.shape
    if split is None:
        split = int(os.environ.get("DDPM_SAMPLER_SPLIT", "1"))
    if split not in (1, 2) or B % split:
        raise ValueError("sampler split must be 1 or 2 and divide the batch")
    Bh = B // split
    S = len(diffusion.betas)
    pseed = 0 if rng == "torch" else ((seed if seed is not None else torch.initial_seed()) | 1) & 0xFFFFFFFFFFFFFFFF
    with _native_mode(model, x, "the sampler state"):
        # weights are re-packed unconditionally at the head of every loop: the reference EMA swaps values with `p.data.copy_`
        # (utils/train.py:307-316), which no version counter sees; 0.2 ms against a T-step loop
        hs = [model.prepare(Bh, H, W, training=False, force_repack=True)] + [model.aux_plan(i, Bh, H, W, force=True) for i in range(1, split)]
        _sampler_tables(diffusion, hs, S - 1)
        forks = [torch.cuda.Stream() for _ in range(split - 1)]

        def step(x, z):
            cur = torch.cuda.current_stream()
            for s_ in forks:
                s_.wait_stream(cur)
            for i, h in enumerate(hs):
                st = cur if i == 0 else forks[i - 1]
                # the philox stream is keyed by (seed, element index): give each half its own key so halves do not repeat noise
                sd = 0 if pseed == 0 else (pseed + 2 * i) & 0xFFFFFFFFFFFFFFFF
                zi = None if z is None else z[i * Bh:(i + 1) * Bh].data_ptr()
                _lib.check(L.ddpm_sampler_step(h, x[i * Bh:(i + 1) * Bh].data_ptr(), zi, sd, C.c_void_p(st.cuda_stream)), "sampler_step")
            for s_ in forks:
                cur.wait_stream(s_)

        if use_graph and rng == "torch" and S > 1:
            # ONE graph launch per timestep: the noise draw, the step-table fetch, the UNet forward and the alpha/beta update fused
            # into the final conv's gather.  The graph is cached: generate.py calls p_sample once per batch, and re-capturing
            # ~150 kernels per call costs more than a dozen DDIM steps.
            key = (x.shape, split, S, gen is not None) + tuple(L.ddpm_unet_graph_epoch(h) for h in hs)
            return _graph_loop(model, key, S, lambda e: step(e["x"], e["z"]), x, gen)["x"].clone()
        if use_graph and S > 1:                     # in-kernel Philox noise: the seed is a launch argument, so the graph is per call
            step(x, None)
            graph = _capture(lambda: step(x, None))
            for _ in range(1, S):
                graph.replay()
            return x
        z = torch.empty_like(x) if rng == "torch" else None
        for _ in range(S):
            if z is not None:
                z.normal_(generator=gen)            # diffusion.py:155 - the reference's stream, drawn on the device
            step(x, z)
        return x


@torch.no_grad()
def _native_bpd_loop(diffusion, model, x0, clip_denoised, noise, use_graph):
    """The T timesteps of calc_all_bpd on the engine; returns CPU fp32 (losses [B, T], mses [B, T]).  Each step is
    {noise draw, step-table fetch, q_sample + UNet forward, bound terms in the final conv's epilogue, fixed-order per-image
    means}; with ``use_graph`` it is captured once per (shape, T, clip, handle epoch) and replayed T times."""
    L = _lib.lib()
    B, _, H, W = x0.shape
    T = diffusion.timesteps
    clip = int(bool(clip_denoised))
    with _native_mode(model, x0, "x_0"):
        if noise is not None and tuple(noise.shape) != (T,) + tuple(x0.shape):
            raise ValueError(f"noise must be [T, B, C, H, W] = {[T] + list(x0.shape)}, got {list(noise.shape)}")
        # weights are re-packed at the head of the loop, as in the sampler loops: the reference EMA swaps values with
        # `p.data.copy_` (utils/train.py:307-316), which no version counter sees
        h = model.prepare(B, H, W, training=False, force_repack=True)
        rows = diffusion._bpd_rows()
        _lib.check(L.ddpm_bpd_setup(h, T, rows.data_ptr()), "bpd_setup")
        _lib.check(L.ddpm_bpd_reset(h, T - 1, _lib.stream_ptr()), "bpd_reset")

        def step(x, z, losses, mses):
            _lib.check(L.ddpm_bpd_step(h, x.data_ptr(), z.data_ptr(), clip, losses.data_ptr(), mses.data_ptr(), _lib.stream_ptr()), "bpd_step")

        if noise is None and use_graph and T > 1:
            # the cached graph's persistent x_0 / noise / result buffers serve every batch of this shape; the default generator
            # advances its Philox offset on every replay exactly as an eager draw
            key = ("bpd", tuple(x0.shape), T, clip, L.ddpm_unet_graph_epoch(h))
            ent = _graph_loop(model, key, T, lambda e: step(e["x"], e["z"], e["losses"], e["mses"]), x0, losses=(B, T), mses=(B, T))
            return ent["losses"].cpu(), ent["mses"].cpu()
        losses = torch.empty((B, T), dtype=torch.float32, device=x0.device)
        mses = torch.empty_like(losses)
        if noise is not None:
            nz = noise.to(device=x0.device, dtype=torch.float32).contiguous()
            for ti in range(T - 1, -1, -1):
                step(x0, nz[ti], losses, mses)
        else:
            z = torch.empty_like(x0)
            for _ in range(T):
                z.normal_()                      # diffusion.py:93 torch.randn_like(x_0), same generator and order
                step(x0, z, losses, mses)
        return losses.cpu(), mses.cpu()
