"""CPU checks of the bits-per-dim evaluation surface: the ddpm_bpd_* entry points reject bad arguments before touching a
device, the per-step rows carry exactly the fp32 casts ``_extract`` makes, and the generic loop's ``noise=`` argument
replaces the per-step draws."""
import ctypes as C

import torch

from oracle import ddpm_ref as R


def _handle(L):
    from ddpm_torch_b200 import _lib
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels, u.levels, u.num_res_blocks = 3, 32, 3, 2, 1
    u.ch_mult[0], u.ch_mult[1] = 1, 2
    h = C.c_void_p()
    assert L.ddpm_unet_create(C.byref(u), C.byref(h)) == 0, L.ddpm_last_error()
    return h


def test_bpd_entry_points_validate_arguments_before_touching_the_device():
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    buf = (C.c_float * 64)()
    a = C.addressof(buf)
    h = _handle(L)
    try:
        assert L.ddpm_bpd_setup(None, 4, a) != 0 and b"null" in L.ddpm_last_error()
        assert L.ddpm_bpd_setup(h, 4, None) != 0 and b"null" in L.ddpm_last_error()
        assert L.ddpm_bpd_setup(h, 0, a) != 0 and b"T must" in L.ddpm_last_error()
        assert L.ddpm_bpd_setup(h, -3, a) != 0 and b"T must" in L.ddpm_last_error()
        assert L.ddpm_bpd_reset(None, 0, None) != 0
        assert L.ddpm_bpd_reset(h, 0, None) != 0 and b"plan" in L.ddpm_last_error()        # no plan yet
        assert L.ddpm_bpd_step(None, a, a, 1, a, a, None) != 0 and b"null" in L.ddpm_last_error()
        for args in ((None, a, a, a), (a, None, a, a), (a, a, None, a), (a, a, a, None)):
            x0, noise, losses, mses = args
            assert L.ddpm_bpd_step(h, x0, noise, 1, losses, mses, None) != 0 and b"null" in L.ddpm_last_error()
        assert L.ddpm_bpd_step(h, a, a, 1, a, a, None) != 0 and b"plan" in L.ddpm_last_error()
    finally:
        L.ddpm_unet_destroy(h)


def test_bpd_rows_are_the_extract_casts():
    import ddpm_torch_b200 as D
    betas = D.get_beta_schedule("linear", 1e-4, 0.02, 50)
    for vt in ("fixed-small", "fixed-large"):
        d = D.GaussianDiffusion(betas, "eps", vt, "mse")
        rows = d._bpd_rows()
        assert rows.shape == (50, 9) and rows.dtype == torch.float32 and rows.is_contiguous()
        t = torch.arange(50)
        names = ("sqrt_alphas_bar", "sqrt_one_minus_alphas_bar", "sqrt_recip_alphas_bar", "sqrt_recip_m1_alphas_bar",
                 "posterior_mean_coef1", "posterior_mean_coef2", "fixed_model_logvar", "posterior_logvar_clipped")
        for k, name in enumerate(names):
            assert torch.equal(rows[:, k], d._extract(getattr(d, name), t, None, ndim=1)), (vt, name)
        assert torch.equal(rows[:, 8], (t > 0).float())


def test_generic_loop_uses_given_noise_and_ddim_stays_generic():
    import ddpm_torch_b200 as D
    T = 8
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, T), "eps", "fixed-large", "kl")
    fn = R.toy_denoiser(3, 1, seed=5)
    g = torch.Generator().manual_seed(3)
    x0 = (torch.rand(2, 3, 8, 8, generator=g) * 2 - 1).mul(127.5).round().div(127.5)
    noise = torch.randn(T, 2, 3, 8, 8, generator=g)
    total, losses, prior, mses = d.calc_all_bpd(fn, x0, clip_denoised=False, noise=noise)
    t = torch.empty(2, dtype=torch.int64)
    for ti in range(T):
        t.fill_(ti)
        term, pred = d._loss_term_bpd(fn, x0, x_t=d.q_sample(x0, t, noise=noise[ti]), t=t, clip_denoised=False, return_pred=True)
        assert torch.equal(losses[:, ti], term) and torch.equal(mses[:, ti], (pred - x0).pow(2).mean(dim=(1, 2, 3)))
    assert torch.equal(total, losses.sum(1) + prior)
    assert all(v.device.type == "cpu" and v.dtype == torch.float32 for v in (total, losses, prior, mses))
    assert D.GaussianDiffusion._native_bpd and not D.DDIM._native_bpd
