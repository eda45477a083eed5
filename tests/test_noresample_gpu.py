"""UNets built with resample_with_conv=False on the engine: AvgPool2d(2) down (k_upsample2x_bwd at scale 1/4, with the quad
statistics of its output where C % 32 == 0 and the pooled map has a multiple of 32 pixels), materialised nearest x2 up
(k_upsample2x, statistics 4x those of its input), and their adjoints (the same two kernels the other way round).

Oracle = tests/noresample_ref.py on the same GPU in fp32 with TF32 off (pinned to the unmodified reference by
tests/test_noresample_cpu.py); golden = tests/golden/unet_noresample.pt.  Cases: tiny (hid 32, 16x16: CUDA-core convs, no
statistics route at C = 32), small64 (hid 64, 32x32: tensor-core convs, pool at C = 64, upsample at C = 128) and the CIFAR-10
config (32x32, 4 levels: pools at 16x16 / 8x8 / 4x4, the 4x4 one without statistics, upsamples at C = 256).

Tolerances (DESIGN.md section 2): eps rel-L2 <= 2e-2 (tiny) / 1e-2; loss relative <= 1e-2; flat gradient rel-L2 <= 5e-2 and
per-tensor cosine >= 0.995; sampler step Linf <= 5e-2 * gain * max|eps| + 5e-4; sampler loops on a T = 20 / 10 chain Linf <= 5e-2;
bits/dim as tests/test_bpd_gpu.py."""
import pytest
import torch

import noresample_ref as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
FIXTURE = "unet_noresample.pt"
NAMES = [c[0] for c in N.CASES]
EPS_TOL = {"tiny": 2e-2, "small64": 1e-2, "cifar10": 1e-2}


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


def build(cfg, seed, train=False):
    import ddpm_torch_b200 as D
    c = N.normalize_cfg(cfg)
    m = D.UNet(in_channels=c["in_channels"], hid_channels=c["hid_channels"], out_channels=c["out_channels"],
               ch_multipliers=c["ch_multipliers"], num_res_blocks=c["num_res_blocks"], apply_attn=c["apply_attn"], drop_rate=0.0,
               resample_with_conv=False)
    sd = N.make_state_dict(cfg, seed)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    m.train(train)
    return m, {k: v.to(DEV) for k, v in sd.items()}


def oracle(sd, cfg):
    return lambda x, t: N.unet_forward(sd, cfg, x, t)


@pytest.mark.parametrize("name", NAMES)
def test_forward_vs_oracle_and_golden(golden, name):
    fx = golden(FIXTURE)["models"][name]
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    x, t = fx["x_t"].to(DEV), fx["t"].to(DEV)
    with torch.no_grad():
        eps = m(x, t)
        ref = N.unet_forward(sd, cfg, x, t)
    flag_ok()
    r1, r2 = rel(eps, ref), rel(eps.cpu(), fx["eps"])
    print(f"\n[{name}] eps rel-L2 vs oracle {r1:.3e}, vs reference golden {r2:.3e}")
    assert r1 < EPS_TOL[name] and r2 < EPS_TOL[name]


def grads_vs_oracle(m, sd, tag, ref_norms, run_engine, run_oracle):
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
    print(f"[{tag}] flat grad rel-L2 {rel(gm, gr):.3e}; worst per-tensor cosine {worst[0]:.5f} ({worst[1]})")
    assert rel(gm, gr) < 5e-2 and worst[0] > 0.995, (rel(gm, gr), worst)
    for k, p in m.named_parameters():
        gn = ref_norms[k] if ref_norms else 0.0
        if gn > 1e-3:
            assert abs(p.grad.norm().item() - gn) / gn < 0.1, k


@pytest.mark.parametrize("name", NAMES)
def test_train_losses_and_grads(golden, name):
    """ddpm_train_forward + ddpm_train_backward (the pool's adjoint accumulates into the skip's gradient) against the oracle."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"][name]
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"], train=True)
    x0, t, noise = fx["x0"].to(DEV), fx["t"].to(DEV), fx["noise"].to(DEV)
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    rd = N.R.RefDiffusion(N.R.get_beta_schedule("linear", 1e-4, 0.02, 1000), "fixed-large")
    out = {}

    def engine():
        out["l"] = diff.train_losses(m, x0, t, noise)
        out["l"].mean().backward()

    def run_oracle(sdg):
        out["r"] = rd.train_losses(oracle(sdg, cfg), x0, t, noise)
        out["r"].mean().backward()

    grads_vs_oracle(m, sd, f"{name} train", fx["grad_norm"], engine, run_oracle)
    lr = (out["l"] - out["r"]).abs().max().item() / out["r"].abs().max().item()
    lg = (out["l"].detach().cpu() - fx["losses"]).abs().max().item() / fx["losses"].abs().max().item()
    print(f"[{name} train] loss rel err vs oracle {lr:.3e}, vs reference golden {lg:.3e}")
    assert lr < 1e-2 and lg < 1e-2


@pytest.mark.parametrize("name", NAMES)
def test_autograd_seam(golden, name):
    """model(x, t) under autograd with an arbitrary upstream gradient: ddpm_unet_forward / ddpm_unet_backward."""
    fx = golden(FIXTURE)["models"][name]
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"], train=True)
    x, t = fx["x_t"].to(DEV), fx["t"].to(DEV)
    g = torch.randn(x.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(3))

    def engine():
        (m(x, t) * g).sum().backward()

    def run_oracle(sdg):
        (N.unet_forward(sdg, cfg, x, t) * g).sum().backward()

    grads_vs_oracle(m, sd, f"{name} autograd", None, engine, run_oracle)
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


@pytest.mark.parametrize("name", NAMES)
def test_native_sampler_step_teacher_forced(golden, name):
    """ddpm_sampler_step against RefDiffusion.p_sample_step over the oracle's eps; bound as tests/test_bench_shapes_gpu.py."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"][name]
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    betas = D.get_beta_schedule("linear", 1e-4, 0.02, 1000)
    x_t = fx["x_t"].to(DEV)
    B = x_t.shape[0]
    z = torch.empty_like(x_t).normal_(generator=torch.Generator(DEV).manual_seed(3))
    for vt in ("fixed-large", "fixed-small"):
        d = D.GaussianDiffusion(betas, "eps", vt, "mse")
        rd = N.R.RefDiffusion(N.R.get_beta_schedule("linear", 1e-4, 0.02, 1000), vt)
        for tv in (0, 1, 500, 999):
            tt = torch.full((B,), tv, dtype=torch.int64, device=DEV)
            xs = _native_step(m, d, x_t, tv, z)
            with torch.no_grad():
                eps_ref = N.unet_forward(sd, cfg, x_t, tt)
                ref = rd.p_sample_step(lambda a, q: eps_ref, x_t, tt, z)
            gain = float(d.posterior_mean_coef1[tv] * d.sqrt_recip_m1_alphas_bar[tv])
            bound = 5e-2 * gain * eps_ref.abs().max().item() + 5e-4
            err = (xs - ref).abs().max().item()
            print(f"[{name} {vt} t={tv}] native step Linf {err:.3e} (bound {bound:.3e})")
            assert err < bound, (vt, tv, err, bound)
    flag_ok()


@pytest.mark.parametrize("name", ["small64", "cifar10"])
def test_ddim_loop_graph_and_eager(golden, name):
    """5-step DDIM loops (eta 0 and 1) on a T = 20 chain, CUDA graph and eager: pixel Linf <= 5e-2."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"][name]
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    T, S = 20, 5
    betas = D.get_beta_schedule("linear", 1e-4, 0.02, T)
    x_T = fx["noise"].to(DEV)
    for eta in (0.0, 1.0):
        sub = D.get_selection_schedule("linear", S, T)
        dd = D.DDIM.from_ddpm(D.GaussianDiffusion(betas, "eps", "fixed-small", "mse"), eta=eta, subsequence=sub)
        rd = N.R.RefDiffusion(N.R.get_beta_schedule("linear", 1e-4, 0.02, T), "fixed-small", eta=eta, subsequence=sub)
        gz = torch.Generator(DEV).manual_seed(11)
        zs = [torch.empty_like(x_T).normal_(generator=gz) for _ in range(S)]
        with torch.no_grad():
            ref = rd.p_sample(oracle(sd, cfg), x_T, zs)
        for use_graph in (True, False):
            xs = dd.p_sample(m, shape=tuple(x_T.shape), device=torch.device(DEV), noise=x_T, seed=11, use_graph=use_graph)
            err = (xs - ref).abs().max().item()
            print(f"\n[{name} ddim T={T} S={S} eta={eta} graph={use_graph}] pixel Linf {err:.3e}")
            assert err < 5e-2
    flag_ok()


def test_native_bpd_matches_reference_golden(golden):
    """Native calc_all_bpd with the reference's per-step noise; bounds of tests/test_bpd_gpu.py."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"][N.BPD_CASE]
    bp = fx["bpd"]
    m, _ = build(fx["cfg"], fx["seed"])
    x0 = bp["x0"].to(DEV)
    for (vt, clip), ref in bp["cases"].items():
        d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, bp["T"]), "eps", vt, "mse")
        total, losses, prior, mses = d.calc_all_bpd(m, x0, clip_denoised=clip, noise=bp["noise"])
        ref_total = ref["losses"].sum(1) + d._prior_bpd(bp["x0"])
        el, em = rel(losses.cpu(), ref["losses"]), rel(mses.cpu(), ref["mses"])
        et = ((total.cpu() - ref_total).abs() / ref_total.abs()).max().item()
        print(f"\n[bpd golden {vt} clip={clip}] losses rel-L2 {el:.2e}  mses rel-L2 {em:.2e}  total rel {et:.2e}")
        assert el <= 2e-2 and em <= 2e-2 and et <= 1e-2
    flag_ok()


@pytest.mark.parametrize("name", ["small64", "cifar10"])
def test_native_bpd_matches_generic_loop_on_same_engine(name):
    """Native calc_all_bpd against the generic torch loop over the same engine forward (bounds of tests/test_bpd_gpu.py)."""
    import ddpm_torch_b200 as D
    cfg = {c[0]: c[1] for c in N.CASES}[name]
    m, _ = build(cfg, 95)
    g = torch.Generator().manual_seed(17)
    x0 = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).mul(127.5).round().div(127.5).to(DEV)
    for vt, clip in (("fixed-large", True), ("fixed-small", False)):
        d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 100), "eps", vt, "mse")
        torch.manual_seed(1234)
        total, losses, prior, mses = d.calc_all_bpd(m, x0, clip_denoised=clip)
        torch.manual_seed(1234)
        with torch.no_grad():
            g_total, g_losses, g_prior, g_mses = d.calc_all_bpd(lambda x, t: m(x, t), x0, clip_denoised=clip)
        tot = ((total - g_total).abs() / g_total.abs()).max().item()
        print(f"\n[{name} bpd vs generic {vt} clip={clip}] total rel {tot:.2e}")
        torch.testing.assert_close(losses, g_losses, rtol=1e-3, atol=1e-5)
        assert torch.equal(prior, g_prior)
        assert tot <= 1e-4
        torch.testing.assert_close(mses, g_mses, rtol=1e-2, atol=1e-5)
    flag_ok()


def test_cifar_bs128_train_step():
    """The CIFAR-10 training step at bs = 128 (the plan bench_resample.py times), dropout 0, against the oracle."""
    import ddpm_torch_b200 as D
    m, sd = build(N.CIFAR10_CFG, 7, train=True)
    g = torch.Generator(DEV).manual_seed(128)
    x0 = torch.rand(128, 3, 32, 32, device=DEV, generator=g) * 2 - 1
    t = torch.randint(1000, (128,), device=DEV, generator=g)
    noise = torch.randn(128, 3, 32, 32, device=DEV, generator=g)
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    rd = N.R.RefDiffusion(N.R.get_beta_schedule("linear", 1e-4, 0.02, 1000), "fixed-large")
    out = {}

    def engine():
        out["l"] = diff.train_losses(m, x0, t, noise)
        out["l"].mean().backward()

    def run_oracle(sdg):
        ls = []
        for i in range(0, 128, 32):
            s = slice(i, i + 32)
            l = rd.train_losses(oracle(sdg, N.CIFAR10_CFG), x0[s], t[s], noise[s])
            (l.sum() / 128).backward()
            ls.append(l.detach())
        out["r"] = torch.cat(ls)

    grads_vs_oracle(m, sd, "cifar10 bs=128 train", None, engine, run_oracle)
    lr = (out["l"] - out["r"]).abs().max().item() / out["r"].abs().max().item()
    print(f"[cifar10 bs=128 train] loss rel err {lr:.3e}")
    assert lr < 1e-2


def test_cifar_bs256_ancestral_loop_and_split_sampler():
    """bs = 256 inference plan: the native ancestral loop (10-step chain, graph) against the oracle, and the two-stream split
    sampler, whose second half runs on an auxiliary engine handle created with the same resample_with_conv flag."""
    import ddpm_torch_b200 as D
    cfg = N.CIFAR10_CFG
    m, sd = build(cfg, 8)
    S = 10
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, S), "eps", "fixed-large", "mse")
    rd = N.R.RefDiffusion(N.R.get_beta_schedule("linear", 1e-4, 0.02, S), "fixed-large")
    x_T = torch.randn(256, 3, 32, 32, device=DEV, generator=torch.Generator(DEV).manual_seed(5))
    gz = torch.Generator(DEV).manual_seed(77)
    zs = [torch.empty_like(x_T).normal_(generator=gz) for _ in range(S)]
    with torch.no_grad():
        xr = x_T
        for k, ti in enumerate(range(S - 1, -1, -1)):
            tt = torch.full((256,), ti, dtype=torch.int64, device=DEV)
            xr = torch.cat([rd.p_sample_step(oracle(sd, cfg), xr[i:i + 64], tt[i:i + 64], zs[k][i:i + 64]) for i in range(0, 256, 64)])
    for split in (1, 2):
        xs = d.p_sample(m, shape=tuple(x_T.shape), device=torch.device(DEV), noise=x_T, seed=77, use_graph=True, split=split)
        err = (xs - xr).abs().max().item()
        print(f"\n[cifar10 bs=256 ancestral, {S} steps, split={split}] pixel Linf {err:.3e}")
        assert err < 5e-2
    flag_ok()
