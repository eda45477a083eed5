"""Image channel counts 1, 2 and 4 on the engine (every image-side kernel is instantiated per channel count), each next to
the C = 3 control of the same config.  Oracle = oracle/ddpm_ref.py on the same GPU in fp32 with TF32 off (pinned to the
unmodified reference at these channel counts by tests/test_image_channels_cpu.py); goldens = tests/golden/unet_channels.pt
(C = 3: unet_{tiny,small64}.pt and bpd_unet.pt).

Routes (asserted per case from the plan's tensor-core op count against the C = 3 plan of the same config):
  tiny (hid 32, 16x16): every image-side conv on CUDA cores - k_in_conv<C> (forward, q_sample prologue, quad statistics),
      k_corr3x3<C> (in_conv weight gradient), k_out_conv<C>, out_conv backward k_in_conv<C> / k_corr3x3<C>, and the separate
      tails k_psample_tail / k_bpd_tail<C>.
  small64 (hid 64, 32x32), C in {1, 2}: k_pack_in + k_im2col3<C> (q_sample prologue; sign -1 over d_eps), k_pack_tapco /
      k_pack_tapco_t with 9*C rows, k_out_gather<C> (plain, sampler and bits/dim epilogues), k_unpack_tap (both modes).
  small64, C = 4: tensor-core in_conv with the CUDA-core out_conv (9*4 > 32): k_psample_tail and k_bpd_tail<4> on an
      otherwise tensor-core plan, out_conv backward on CUDA cores beside the tensor-core in_conv weight gradient.
  small64, 1 -> 2 channels: in_conv at C = 1, out_conv at C = 2.

Tolerances (DESIGN.md section 2): eps rel-L2 <= 2e-2 (tiny) / 1e-2 (small64); loss relative <= 1e-2, flat gradient rel-L2
<= 5e-2, per-tensor cosine >= 0.995; per-tensor rel-L2 of the four image-side tensors <= IMG_TOL / IMG_TOL_SEAM (at most
twice the worst C = 3 value measured on H100); sampler step Linf <= 5e-2 * gain * max|eps| + 5e-4; bits/dim as
tests/test_bpd_gpu.py."""
import ctypes as C

import pytest
import torch

from oracle import ddpm_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
FIXTURE = "unet_channels.pt"
BASE = {"tiny": R.TINY_CFG, "small64": R.SMALL64_CFG}
EPS_TOL = {"tiny": 2e-2, "small64": 1e-2}
PAIRS = [(n, c) for n in ("tiny", "small64") for c in (1, 2, 3, 4)]
IMAGE_SIDE = ("in_conv.weight", "in_conv.bias", "out_conv.2.weight", "out_conv.2.bias")
# per-tensor rel-L2 of the image-side gradients: at most twice the worst C = 3 value measured on H100 (training: 1.86e-2 tiny,
# 4.79e-3 small64; autograd seam, small64: 1.24e-2)
IMG_TOL = {"tiny": 3.5e-2, "small64": 9.5e-3}
IMG_TOL_SEAM = 2.4e-2


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.cuda.empty_cache()


def flag_ok():
    from ddpm_torch_b200 import _lib
    assert _lib.lib().ddpm_device_error_flag() == 0


def case(golden, name, c):
    """Inputs / reference outputs of the (config, C) pair; C = 3 is the existing fixture of the config."""
    return golden(f"unet_{name}.pt") if c == 3 else golden(FIXTURE)["models"][f"{name}_c{c}"]


def build(cfg, seed, train=False):
    import ddpm_torch_b200 as D
    c = R.normalize_cfg(cfg)
    m = D.UNet(in_channels=c["in_channels"], hid_channels=c["hid_channels"], out_channels=c["out_channels"],
               ch_multipliers=c["ch_multipliers"], num_res_blocks=c["num_res_blocks"], apply_attn=c["apply_attn"], drop_rate=0.0)
    sd = R.make_state_dict(cfg, seed)
    m.load_state_dict(sd)
    m = m.to(DEV)
    m.train(train)
    return m, {k: v.to(DEV) for k, v in sd.items()}


def _stats(h):
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    ntc, nf = C.c_int(), C.c_int()
    L.ddpm_unet_plan_stats(h, None, None, C.byref(ntc), None, None, None)
    L.ddpm_unet_launch_counts(h, C.byref(nf), None, None)
    return ntc.value, nf.value


def _control_stats(name, B, H, training):
    """(tensor-core ops, forward launches) of the C = 3 plan of the same config and shape (dry plan)."""
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    import ddpm_torch_b200 as D
    c = R.normalize_cfg(BASE[name])
    m = D.UNet(3, c["hid_channels"], 3, c["ch_multipliers"], c["num_res_blocks"], c["apply_attn"])
    assert L.ddpm_unet_workspace_bytes(m._h, B, H, H, int(training)) > 0, L.ddpm_last_error()
    return _stats(m._h)


def check_route(m, name, cin, cout, B, H, training):
    """The plan the model just ran took the route the module docstring names for this (config, channel) pair."""
    ntc, nf = _stats(m._h)
    ntc3, nf3 = _control_stats(name, B, H, training)
    if name == "small64" and cout == 4:
        assert (ntc, nf) == (ntc3 - (3 if training else 1), nf3 - 1), ((ntc, nf), (ntc3, nf3))     # out_conv off the TC path
    else:
        assert (ntc, nf) == (ntc3, nf3), ((ntc, nf), (ntc3, nf3))


@pytest.mark.parametrize("name,c", PAIRS)
def test_forward_vs_oracle_and_golden(golden, name, c):
    fx = case(golden, name, c)
    cfg = fx["cfg"]
    assert cfg["in_channels"] == cfg["out_channels"] == c
    m, sd = build(cfg, fx["seed"])
    x, t = fx["x_t"].to(DEV), fx["t"].to(DEV)
    with torch.no_grad():
        eps = m(x, t)
        ref = R.unet_forward(sd, cfg, x, t)
    flag_ok()
    check_route(m, name, c, c, x.shape[0], x.shape[-1], False)
    r1, r2 = rel(eps, ref), rel(eps.cpu(), fx["eps"])
    print(f"\n[{name} C={c}] eps rel-L2 vs oracle {r1:.3e}, vs reference golden {r2:.3e}")
    assert eps.shape == (x.shape[0], c) + tuple(x.shape[2:])
    assert r1 < EPS_TOL[name] and r2 < EPS_TOL[name]


def grads_vs_oracle(m, sd, cfg, tag, ref_norms, run_engine, run_oracle, image_tol):
    """Every gradient tensor of the engine vs the oracle (flat rel-L2, per-tensor cosine), the four image-side tensors by
    their own rel-L2, and the reference's gradient norms."""
    run_engine()
    flag_ok()
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    run_oracle(sdg)
    gm = torch.cat([p.grad.flatten() for p in m.parameters()])
    gr = torch.cat([sdg[k].grad.flatten() for k, _ in m.named_parameters()])
    worst = (1.0, "")
    for k, p in m.named_parameters():
        a, b = p.grad.flatten().double(), sdg[k].grad.flatten().double()
        if b.norm() < 1e-6 * gr.norm():
            continue
        cos = (a @ b / (a.norm() * b.norm()).clamp_min(1e-30)).item()
        if cos < worst[0]:
            worst = (cos, k)
    grads = dict(m.named_parameters())
    img = {k: rel(grads[k].grad, sdg[k].grad) for k in IMAGE_SIDE}
    print(f"[{tag}] flat grad rel-L2 {rel(gm, gr):.3e}; worst per-tensor cosine {worst[0]:.5f} ({worst[1]}); image-side rel-L2 "
          + ", ".join(f"{k} {v:.2e}" for k, v in img.items()))
    assert rel(gm, gr) < 5e-2 and worst[0] > 0.995, (rel(gm, gr), worst)
    assert max(img.values()) <= image_tol, img
    for k, p in m.named_parameters():
        gn = ref_norms[k] if ref_norms else 0.0
        if gn > 1e-3:
            assert abs(p.grad.norm().item() - gn) / gn < 0.1, k


@pytest.mark.parametrize("name,c", PAIRS)
def test_train_losses_and_grads(golden, name, c):
    """ddpm_train_forward (q_sample fused into in_conv's loads) + ddpm_train_backward against the oracle."""
    import ddpm_torch_b200 as D
    fx = case(golden, name, c)
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"], train=True)
    x0, t, noise = fx["x0"].to(DEV), fx["t"].to(DEV), fx["noise"].to(DEV)
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    rd = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, 1000), "fixed-large")
    out = {}

    def engine():
        out["l"] = diff.train_losses(m, x0, t, noise)
        out["l"].mean().backward()

    def oracle(sdg):
        out["r"] = rd.train_losses(lambda x, tt: R.unet_forward(sdg, cfg, x, tt), x0, t, noise)
        out["r"].mean().backward()

    grads_vs_oracle(m, sd, cfg, f"{name} C={c} train", fx["grad_norm"], engine, oracle, IMG_TOL[name])
    check_route(m, name, c, c, x0.shape[0], x0.shape[-1], True)
    lr = (out["l"] - out["r"]).abs().max().item() / out["r"].abs().max().item()
    lg = (out["l"].detach().cpu() - fx["losses"]).abs().max().item() / fx["losses"].abs().max().item()
    print(f"[{name} C={c} train] loss rel err vs oracle {lr:.3e}, vs reference golden {lg:.3e}")
    assert lr < 1e-2 and lg < 1e-2


@pytest.mark.parametrize("model", ["small64_c3", "small64_c1to2"])
def test_autograd_seam(golden, model):
    """model(x, t) under autograd with an arbitrary upstream gradient, (out * g).sum().backward(), as
    tests/test_unet_gpu.py::test_plain_forward_backward_autograd does: the C = 3 control and in_channels = 1, out_channels = 2
    (a 1-channel dataset with a learned variance, train.py:63).  The eps-prediction training and sampler entry points refuse
    the 1 -> 2 model instead of mixing the two channel counts."""
    import ddpm_torch_b200 as D
    fx = golden("unet_small64.pt") if model == "small64_c3" else golden(FIXTURE)["models"][model]
    cfg = fx["cfg"]
    cin, cout = cfg["in_channels"], cfg["out_channels"]
    m, sd = build(cfg, fx["seed"], train=True)
    x, t = fx["x_t"].to(DEV), fx["t"].to(DEV)
    g = fx["g"].to(DEV) if "g" in fx else torch.randn(x.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    with torch.no_grad():
        eps = m(x, t)
        ref = R.unet_forward(sd, cfg, x, t)
    r1, r2 = rel(eps, ref), rel(eps.cpu(), fx["eps"])
    print(f"\n[small64 C={cin}->{cout}] eps rel-L2 vs oracle {r1:.3e}, vs reference golden {r2:.3e}")
    assert eps.shape == (x.shape[0], cout) + tuple(x.shape[2:]) and r1 < EPS_TOL["small64"] and r2 < EPS_TOL["small64"]

    def engine():
        (m(x, t) * g).sum().backward()

    def oracle(sdg):
        (R.unet_forward(sdg, cfg, x, t) * g).sum().backward()

    grads_vs_oracle(m, sd, cfg, f"small64 C={cin}->{cout} autograd", fx["grad_norm"] if "g" in fx else None, engine, oracle,
                    IMG_TOL_SEAM)
    check_route(m, "small64", cin, cout, x.shape[0], x.shape[-1], True)
    if cin != cout:
        d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 10), "eps", "fixed-large", "mse")
        with pytest.raises(RuntimeError, match="out_channels == in_channels"):
            d.train_losses(m, x, t, torch.randn_like(x))
        with pytest.raises(RuntimeError, match="out_channels == in_channels"):
            d.p_sample(m, shape=tuple(x.shape), device=torch.device(DEV), noise=x, seed=1, use_graph=False)
    flag_ok()


def _native_step(m, d, x_t, t_idx, z):
    """ONE call of ddpm_sampler_step (prep + UNet forward + alpha/beta update) at step index t_idx."""
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    B, _, H, W = x_t.shape
    h = m.prepare(B, H, W, training=False, force_repack=True)
    coef, tmod = d._coef_rows(), d._model_timesteps().contiguous()
    _lib.check(L.ddpm_sampler_setup(h, coef.shape[0], tmod.data_ptr(), coef.data_ptr()))
    st = _lib.stream_ptr()
    _lib.check(L.ddpm_sampler_reset(h, t_idx, st))
    x = x_t.clone().contiguous()
    _lib.check(L.ddpm_sampler_step(h, x.data_ptr(), z.data_ptr(), 0, st))
    return x


@pytest.mark.parametrize("name,c", PAIRS)
def test_native_sampler_step_teacher_forced(golden, name, c):
    """ddpm_sampler_step itself (the fused gather epilogue for small64 C <= 3, k_psample_tail otherwise) against
    RefDiffusion.p_sample_step over the oracle's eps; bound as tests/test_bench_shapes_gpu.py."""
    import ddpm_torch_b200 as D
    fx = case(golden, name, c)
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    betas = D.get_beta_schedule("linear", 1e-4, 0.02, 1000)
    x_t = fx["x_t"].to(DEV)
    B = x_t.shape[0]
    z = torch.empty_like(x_t).normal_(generator=torch.Generator(DEV).manual_seed(3))
    for vt in ("fixed-large", "fixed-small"):
        d = D.GaussianDiffusion(betas, "eps", vt, "mse")
        rd = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, 1000), vt)
        for tv in (0, 1, 500, 999):
            tt = torch.full((B,), tv, dtype=torch.int64, device=DEV)
            xs = _native_step(m, d, x_t, tv, z)
            with torch.no_grad():
                eps_ref = R.unet_forward(sd, cfg, x_t, tt)
                ref = rd.p_sample_step(lambda a, q: eps_ref, x_t, tt, z)
            gain = float(d.posterior_mean_coef1[tv] * d.sqrt_recip_m1_alphas_bar[tv])
            bound = 5e-2 * gain * eps_ref.abs().max().item() + 5e-4
            err = (xs - ref).abs().max().item()
            print(f"[{name} C={c} {vt} t={tv}] native step Linf {err:.3e} (bound {bound:.3e})")
            assert err < bound, (vt, tv, err, bound)
    check_route(m, name, c, c, B, x_t.shape[-1], False)
    flag_ok()


def _bpd_golden(golden, name, c):
    if c == 3:
        fx = golden("bpd_unet.pt")
        mx = fx["models"][name]
        return mx["cfg"], mx["seed"], fx["T"], mx["x0"], mx["noise"], mx["cases"]
    mx = golden(FIXTURE)["models"][f"{name}_c{c}"]
    bp = mx["bpd"]
    return mx["cfg"], mx["seed"], bp["T"], bp["x0"], bp["noise"], bp["cases"]


@pytest.mark.parametrize("name,c", [(n, c) for n in ("tiny", "small64") for c in (1, 3, 4)])
def test_native_bpd_matches_reference_golden(golden, name, c):
    """Native calc_all_bpd with the reference's per-step noise; bounds of tests/test_bpd_gpu.py."""
    import ddpm_torch_b200 as D
    cfg, seed, T, x0c, noise, cases = _bpd_golden(golden, name, c)
    m, _ = build(cfg, seed)
    x0 = x0c.to(DEV)
    for (vt, clip), ref in cases.items():
        d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, T), "eps", vt, "mse")
        total, losses, prior, mses = d.calc_all_bpd(m, x0, clip_denoised=clip, noise=noise)
        ref_total = ref["losses"].sum(1) + d._prior_bpd(x0c)
        el, em, et = rel(losses, ref["losses"]), rel(mses, ref["mses"]), ((total - ref_total).abs() / ref_total.abs()).max().item()
        print(f"\n[bpd golden {name} C={c} {vt} clip={clip}] losses rel-L2 {el:.2e}  mses rel-L2 {em:.2e}  total rel {et:.2e}")
        assert el <= 2e-2 and em <= 2e-2 and et <= 1e-2
    check_route(m, name, c, c, x0.shape[0], x0.shape[-1], False)
    flag_ok()


def bpd_data(B, c, HW, seed):
    """8-bit data with a band of saturated pixels: row 0 at exactly +1, row 1 at exactly -1 (the decoder's edge bins)."""
    g = torch.Generator().manual_seed(seed)
    x0 = (torch.rand(B, c, HW, HW, generator=g) * 2 - 1).mul(127.5).round().div(127.5)
    x0[:, :, 0, :] = 1.0
    x0[:, :, 1, :] = -1.0
    return x0.to(DEV)


@pytest.mark.parametrize("name,c", PAIRS)
def test_native_bpd_matches_generic_loop_on_same_engine(name, c):
    """Native calc_all_bpd against the generic torch loop over the SAME engine forward, same seed: only the per-image
    reduction order and the forward's run-to-run drift differ, so this pins the epilogue arithmetic and its C*H*W
    normalisation.  Bounds of tests/test_bpd_gpu.py (per term rtol 1e-3 / atol 1e-5, total relative <= 1e-4, mses rtol 1e-2).
    64x64 images: the forward is not bit-reproducible, and a per-image mean over 16x16 pixels of one channel keeps enough of
    that drift to cross the per-term bound now and then (measured on H100 up to 1.5x it for tiny C = 1); 4096 pixels average
    it down."""
    import ddpm_torch_b200 as D
    HW = 64
    cfg = dict(BASE[name], in_channels=c, out_channels=c)
    m, _ = build(cfg, 90 + c)
    x0 = bpd_data(2, c, HW, 17 + c)
    for vt, clip in (("fixed-large", True), ("fixed-small", False)):
        d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 100), "eps", vt, "mse")
        torch.manual_seed(1234)
        total, losses, prior, mses = d.calc_all_bpd(m, x0, clip_denoised=clip)
        torch.manual_seed(1234)
        with torch.no_grad():
            g_total, g_losses, g_prior, g_mses = d.calc_all_bpd(lambda x, t: m(x, t), x0, clip_denoised=clip)
        err = ((losses - g_losses).abs() / (1e-5 + 1e-3 * g_losses.abs())).max().item()
        tot = ((total - g_total).abs() / g_total.abs()).max().item()
        print(f"\n[bpd vs generic {name} C={c} {vt} clip={clip}] max term err / (atol + rtol |term|) {err:.3f}; total rel {tot:.2e}")
        torch.testing.assert_close(losses, g_losses, rtol=1e-3, atol=1e-5)
        assert torch.equal(prior, g_prior)
        assert tot <= 1e-4
        torch.testing.assert_close(mses, g_mses, rtol=1e-2, atol=1e-5)
    check_route(m, name, c, c, 2, HW, False)
    flag_ok()


def test_to_uint8_nhwc_two_channels_bit_exact():
    """generate.py:129 at C = 2 (the instantiation tests/test_optim.py does not reach): ties, out-of-range values and the
    exact end points, against the literal reference expression on the CPU."""
    from ddpm_torch_b200.postprocess import to_uint8_nhwc
    for shape in ((3, 2, 16, 16), (2, 2, 7, 5)):
        x = torch.randn(shape, generator=torch.Generator().manual_seed(9)) * 0.8
        flat = x.view(-1)
        ties = (torch.arange(0, 256, dtype=torch.float32) + 0.5 - 127.5) / 127.5
        n = min(flat.numel() // 2, ties.numel())
        flat[:n] = ties[:n]
        flat[n:n + 6] = torch.tensor([-1.0, 1.0, -3.0, 3.0, 0.0, 1.0 - 2 ** -24])
        ref = R.to_uint8_nhwc(x)
        out = to_uint8_nhwc(x.cuda())
        assert out.dtype == torch.uint8 and out.shape == ref.shape and out.is_contiguous()
        assert torch.equal(out.cpu(), ref.contiguous())
    flag_ok()
