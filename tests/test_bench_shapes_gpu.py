"""Parity AT THE BENCHMARKED SHAPES (VERDICT r1 "next round" item 1): the plans bench.py times are batch-size dependent
(N128-fill vs split-K, GroupNorm grids, tensor-core timestep projections), so the bs=4 / bs=64 fixtures do not cover them.

Oracle = oracle/ddpm_ref.py run on the same GPU in fp32 with TF32 off, on identical seeded inputs and weights.
Tolerances (bf16 operands / bf16 inter-kernel activations, fp32 accumulation): eps rel-L2 <= 1e-2; loss relative <= 1e-2;
flat gradient rel-L2 <= 5e-2 and per-tensor cosine >= 0.995; sampler pixel Linf <= 5e-2 on chains whose error gain is O(1)
(short beta schedules; the T=1000 chain multiplies an eps error by sqrt(1/alpha_bar - 1) ~ 157 at t=999, see test_unet_gpu)."""
import ctypes as C

import pytest
import torch

from oracle import ddpm_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.cuda.empty_cache()


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


def flag_ok():
    from ddpm_torch_b200 import _lib
    assert _lib.lib().ddpm_device_error_flag() == 0


def grads_vs_oracle(m, sd, cfg, x0, t, noise, tag, chunk=None):
    """train_losses + all parameter gradients of the engine vs the oracle.  ``chunk`` splits the ORACLE's batch (the loss is a
    mean of per-sample terms, so gradients add) to bound its fp32 autograd memory."""
    import ddpm_torch_b200 as D
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    losses = diff.train_losses(m, x0, t, noise)
    losses.mean().backward()
    flag_ok()
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    rd = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, 1000), "fixed-large")
    B = x0.shape[0]
    chunk = chunk or B
    lref = []
    for i in range(0, B, chunk):
        s = slice(i, i + chunk)
        l = rd.train_losses(lambda x, tt: R.unet_forward(sdg, cfg, x, tt), x0[s], t[s], noise[s])
        (l.sum() / B).backward()
        lref.append(l.detach())
    lref = torch.cat(lref)
    lr = (losses - lref).abs().max().item() / lref.abs().max().item()
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
    print(f"\n[{tag}] loss rel err {lr:.3e}; flat grad rel-L2 {rel(gm, gr):.3e}; worst per-tensor cosine {worst[0]:.5f} ({worst[1]})")
    assert lr < 1e-2 and rel(gm, gr) < 5e-2 and worst[0] > 0.995, (lr, rel(gm, gr), worst)


def test_cifar_bs128_train_step_plan(golden):
    """BASELINE config 2 — the exact plan bench.py times (bs=128, 32x32, training), dropout 0."""
    fx = golden("unet_cifar10_bs4.pt")
    m, sd = build(fx["cfg"], fx["seed"], train=True)
    g = torch.Generator(DEV).manual_seed(128)
    x0 = torch.rand(128, 3, 32, 32, device=DEV, generator=g) * 2 - 1
    t = torch.randint(1000, (128,), device=DEV, generator=g)
    noise = torch.randn(128, 3, 32, 32, device=DEV, generator=g)
    grads_vs_oracle(m, sd, fx["cfg"], x0, t, noise, "cifar10 bs=128 train", chunk=32)


def test_cifar_bs256_forward_and_native_ancestral_loop(golden):
    """BASELINE config 3 — bs=256 inference plan: one forward vs the oracle, then the NATIVE ancestral fixed-large loop
    (GaussianDiffusion.p_sample -> ddpm_sampler_step, graph and eager) on a 10-step beta schedule with the same CUDA
    generator on both sides."""
    import ddpm_torch_b200 as D
    fx = golden("unet_cifar10_bs4.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    g = torch.Generator(DEV).manual_seed(256)
    x = torch.randn(256, 3, 32, 32, device=DEV, generator=g)
    t = torch.randint(1000, (256,), device=DEV, generator=g)
    with torch.no_grad():
        eps = m(x, t)
        ref = torch.cat([R.unet_forward(sd, cfg, x[i:i + 64], t[i:i + 64]) for i in range(0, 256, 64)])
    flag_ok()
    r = rel(eps, ref)
    print(f"\n[cifar10 bs=256 fwd] eps rel-L2 {r:.3e}, max-abs {(eps - ref).abs().max().item():.3e} (ref max {ref.abs().max().item():.3e})")
    assert r < 1e-2
    S = 10
    betas = D.get_beta_schedule("linear", 1e-4, 0.02, S)
    d = D.GaussianDiffusion(betas, "eps", "fixed-large", "mse")
    rd = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, S), "fixed-large")
    x_T = torch.randn(256, 3, 32, 32, device=DEV, generator=torch.Generator(DEV).manual_seed(5))
    gz = torch.Generator(DEV).manual_seed(77)
    zs = [torch.empty_like(x_T).normal_(generator=gz) for _ in range(S)]
    with torch.no_grad():
        xr = x_T
        for k, ti in enumerate(range(S - 1, -1, -1)):
            tt = torch.full((256,), ti, dtype=torch.int64, device=DEV)
            xr = torch.cat([rd.p_sample_step(lambda a, q: R.unet_forward(sd, cfg, a, q), xr[i:i + 64], tt[i:i + 64], zs[k][i:i + 64])
                            for i in range(0, 256, 64)])
    for use_graph in (True, False):
        xs = d.p_sample(m, shape=tuple(x_T.shape), device=torch.device(DEV), noise=x_T, seed=77, use_graph=use_graph)
        dlt = (xs - xr).abs()
        print(f"[cifar10 bs=256 native ancestral fixed-large, {S} steps, graph={use_graph}] pixel Linf {dlt.max().item():.3e}, L1 {dlt.mean().item():.3e}")
        assert dlt.max().item() < 5e-2
    flag_ok()


def test_celebahq_256_fwd_bwd(golden):
    """BASELINE config 4 shape: celebahq.json UNet (113.7M params) at 256x256, bs=2: loss, all gradients."""
    fx = golden("unet_celebahq_bs1.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"], train=True)
    g = torch.Generator(DEV).manual_seed(9)
    x0 = torch.rand(2, 3, 256, 256, device=DEV, generator=g) * 2 - 1
    t = torch.randint(1000, (2,), device=DEV, generator=g)
    noise = torch.randn(2, 3, 256, 256, device=DEV, generator=g)
    grads_vs_oracle(m, sd, cfg, x0, t, noise, "celebahq 256x256 bs=2 train", chunk=1)


def _native_step(m, d, x_t, t_idx, z):
    """ONE call of ddpm_sampler_step (prep + UNet forward + alpha/beta tail) at step index t_idx."""
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


@pytest.mark.parametrize("name", ["tiny", "cifar10_bs4"])
def test_native_sampler_step_teacher_forced_linf(golden, name):
    """ddpm_sampler_step ITSELF (not the generic torch tail), teacher-forced, with a pixel Linf bound.  With random weights
    the clamp of x0_hat at +-1 is exercised on most pixels at large t; the bound is over ALL pixels:
    5e-2 * max|eps| (the eps-prediction Linf budget) times the step's own error gain  c1 * sqrt(1/ab - 1)  (the factor between
    an eps error and an x_{t-1} error, diffusion.py:145-148,99-105; 0.01-0.02 on the T=1000 chain)."""
    import ddpm_torch_b200 as D
    fx = golden(f"unet_{name}.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    betas = D.get_beta_schedule("linear", 1e-4, 0.02, 1000)
    x_t = fx["x_t"].to(DEV)
    B = x_t.shape[0]
    z = torch.empty_like(x_t).normal_(generator=torch.Generator(DEV).manual_seed(3))
    for vt in ("fixed-large", "fixed-small"):
        d = D.GaussianDiffusion(betas, "eps", vt, "mse")
        rd = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, 1000), vt)
        for tv in (0, 1, 50, 200, 500, 999):
            tt = torch.full((B,), tv, dtype=torch.int64, device=DEV)
            xs = _native_step(m, d, x_t, tv, z)
            with torch.no_grad():
                eps_ref = R.unet_forward(sd, cfg, x_t, tt)
                ref = rd.p_sample_step(lambda a, q: eps_ref, x_t, tt, z)
            gain = float(d.posterior_mean_coef1[tv] * d.sqrt_recip_m1_alphas_bar[tv])
            bound = 5e-2 * gain * eps_ref.abs().max().item() + 5e-4      # eps Linf error budget x gain + fp32 floor of the tail
            err = (xs - ref).abs().max().item()
            print(f"[{name} {vt} t={tv}] native step Linf {err:.3e} (bound {bound:.3e}, eps-error gain {gain:.3f})")
            assert err < bound, (vt, tv, err, bound)
    flag_ok()


def test_ddim_short_chain_linf(golden):
    """DDIM loops (graph + eager) on a T=20 chain (error gain O(1)): pixel Linf bound 5e-2."""
    import ddpm_torch_b200 as D
    fx = golden("unet_cifar10_bs4.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    T, S = 20, 5
    betas = D.get_beta_schedule("linear", 1e-4, 0.02, T)
    x_T = fx["noise"].to(DEV)
    for sched, eta in (("linear", 0.0), ("quadratic", 0.0), ("linear", 1.0)):
        sub = D.get_selection_schedule(sched, S, T)
        dd = D.DDIM.from_ddpm(D.GaussianDiffusion(betas, "eps", "fixed-small", "mse"), eta=eta, subsequence=sub)
        rd = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, T), "fixed-small", eta=eta, subsequence=sub)
        gz = torch.Generator(DEV).manual_seed(11)
        zs = [torch.empty_like(x_T).normal_(generator=gz) for _ in range(S)]
        with torch.no_grad():
            ref = rd.p_sample(lambda a, q: R.unet_forward(sd, cfg, a, q), x_T, zs)
        for use_graph in (True, False):
            xs = dd.p_sample(m, shape=tuple(x_T.shape), device=torch.device(DEV), noise=x_T, seed=11, use_graph=use_graph)
            err = (xs - ref).abs().max().item()
            print(f"\n[ddim T={T} S={S} {sched} eta={eta} graph={use_graph}] pixel Linf {err:.3e}")
            assert err < 5e-2
    flag_ok()


def test_reference_ema_data_copy_swap_is_seen_by_sampler(golden):
    """utils/train.py:307-316: the reference EMA swaps weights with ``p.data.copy_`` (no version counter moves).  A sampler
    loop on a REUSED eval plan must run with the swapped-in weights, and with the originals after the swap back."""
    import ddpm_torch_b200 as D
    fx = golden("unet_tiny.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    sd2 = {k: v.to(DEV) for k, v in R.make_state_dict(cfg, fx["seed"] + 1).items()}
    T = 6
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, T), "eps", "fixed-small", "mse")
    rd = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, T), "fixed-small")
    x_T = fx["noise"].to(DEV)
    gz = torch.Generator(DEV).manual_seed(2)
    zs = [torch.empty_like(x_T).normal_(generator=gz) for _ in range(T)]

    def oracle(w):
        with torch.no_grad():
            return rd.p_sample(lambda a, q: R.unet_forward(w, cfg, a, q), x_T, zs)

    def native():
        return d.p_sample(m, shape=tuple(x_T.shape), device=torch.device(DEV), noise=x_T, seed=2)

    a0 = native()
    assert (a0 - oracle(sd)).abs().max().item() < 5e-2
    backup = {k: p.detach().clone() for k, p in m.named_parameters()}
    for k, p in m.named_parameters():
        p.data.copy_(sd2[k])                       # EMA.apply(), reference style
    a1 = native()
    e1 = (a1 - oracle(sd2)).abs().max().item()
    print(f"\n[ema swap] after .data.copy_: Linf vs oracle(new weights) {e1:.3e}; vs stale output {(a1 - a0).abs().max().item():.3e}")
    assert e1 < 5e-2 and (a1 - a0).abs().max().item() > 1e-2
    for k, p in m.named_parameters():
        p.data.copy_(backup[k])                    # EMA.restore()
    assert (native() - oracle(sd)).abs().max().item() < 5e-2
    flag_ok()


def test_cuda_model_load_state_dict_then_forward(golden):
    """ADVICE r1: after .cuda() the parameters do not share the flat buffer's version counter; load_state_dict / p.copy_ on a
    CUDA model followed by a forward on the SAME plan must use the new weights."""
    fx = golden("unet_tiny.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    x, t = fx["x_t"].to(DEV), fx["t"].to(DEV)
    with torch.no_grad():
        e0 = m(x, t)
    sd2 = R.make_state_dict(cfg, fx["seed"] + 7)
    m.load_state_dict(sd2)
    with torch.no_grad():
        e1 = m(x, t)
        ref = R.unet_forward({k: v.to(DEV) for k, v in sd2.items()}, cfg, x, t)
    assert rel(e1, ref) < 1e-2 and rel(e1, e0) > 0.1
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(sd[k])
        e2 = m(x, t)
    assert rel(e2, e0) < 1e-2
    flag_ok()


def test_gradient_accumulation_matches_reference_semantics(golden):
    """--num-accum (utils/train.py:149-165): two backward passes before one optimizer step ADD UP in flat_grads."""
    import ddpm_torch_b200 as D
    fx = golden("unet_tiny.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"], train=True)
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    g = torch.Generator(DEV).manual_seed(4)
    H = fx["x0"].shape[-1]
    xs = [torch.randn(4, 3, H, H, device=DEV, generator=g) for _ in range(2)]
    ts = [torch.randint(1000, (4,), device=DEV, generator=g) for _ in range(2)]
    ns = [torch.randn(4, 3, H, H, device=DEV, generator=g) for _ in range(2)]
    m.zero_grad()
    for i in range(2):
        diff.train_losses(m, xs[i], ts[i], ns[i]).mean().div(2).backward()
    acc = m.flat_grads.clone()
    pg = torch.cat([p.grad.flatten() for p in m.parameters()])
    singles = []
    for i in range(2):
        m.zero_grad()
        diff.train_losses(m, xs[i], ts[i], ns[i]).mean().div(2).backward()
        singles.append(m.flat_grads.clone())
    want = singles[0] + singles[1]
    r = rel(acc, want)
    views = torch.cat([v.flatten() for v in m.grad_views(acc)])
    print(f"\n[grad accumulation] flat_grads vs sum of single passes rel-L2 {r:.3e}; p.grad vs flat views {rel(pg, views):.3e}")
    assert r < 1e-2 and rel(pg, views) < 1e-2 and rel(acc, singles[1]) > 0.1
    flag_ok()


def test_native_p_sample_progressive(golden):
    """diffusion.py:176-198 on the engine (ddpm_sampler_step_pred): final sample and the x_0 predictions every pred_freq steps
    against the generic torch loop of the same class driven by the oracle network, same seed (same CUDA noise stream)."""
    import ddpm_torch_b200 as D
    fx = golden("unet_tiny.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    T = 12
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, T), "eps", "fixed-large", "mse")
    shape = tuple(fx["noise"].shape)
    xs, preds = d.p_sample_progressive(m, shape, device=torch.device(DEV), pred_freq=3, seed=5)
    with torch.no_grad():
        xr, pr = d.p_sample_progressive(lambda a, q: R.unet_forward(sd, cfg, a, q), shape, device=torch.device(DEV), pred_freq=3, seed=5)
    e1, e2 = (xs - xr).abs().max().item(), (preds - pr).abs().max().item()
    print(f"\n[progressive T={T}] final Linf {e1:.3e}; x0-prediction Linf {e2:.3e}; preds shape {tuple(preds.shape)}")
    assert preds.shape == pr.shape == (T // 3,) + shape and e1 < 5e-2 and e2 < 5e-2
    flag_ok()


CELEBA64_CFG = dict(in_channels=3, hid_channels=128, out_channels=3, ch_multipliers=(1, 2, 2, 2), num_res_blocks=2,
                    apply_attn=(False, False, True, False), drop_rate=0.0)          # configs/celeba.json


def test_celeba64_config_fwd_bwd():
    """configs/celeba.json (CelebA 64x64, attention at the 16x16 level = level 2): loss and all gradients at bs=8."""
    m, sd = build(CELEBA64_CFG, 77, train=True)
    g = torch.Generator(DEV).manual_seed(64)
    x0 = torch.rand(8, 3, 64, 64, device=DEV, generator=g) * 2 - 1
    t = torch.randint(1000, (8,), device=DEV, generator=g)
    noise = torch.randn(8, 3, 64, 64, device=DEV, generator=g)
    grads_vs_oracle(m, sd, CELEBA64_CFG, x0, t, noise, "celeba 64x64 bs=8 train", chunk=4)


WIDE_ATTN_CFG = dict(in_channels=3, hid_channels=256, out_channels=3, ch_multipliers=(1, 2, 4), num_res_blocks=2,
                     apply_attn=(False, False, True), drop_rate=0.0)


def test_wide_attention_config_fwd_bwd():
    """hid 256, ch_mult (1, 2, 4), attention at the 1024-channel level: project_in's bias gradient is a column sum over
    3 * 1024 channels (k_colsum in 2048-channel slices) and the up path's widest GroupNorm concat is 1024 + 1024.
    Loss and all gradients at bs=2, 32x32."""
    m, sd = build(WIDE_ATTN_CFG, 31, train=True)
    g = torch.Generator(DEV).manual_seed(31)
    x0 = torch.rand(2, 3, 32, 32, device=DEV, generator=g) * 2 - 1
    t = torch.randint(1000, (2,), device=DEV, generator=g)
    noise = torch.randn(2, 3, 32, 32, device=DEV, generator=g)
    grads_vs_oracle(m, sd, WIDE_ATTN_CFG, x0, t, noise, "hid 256 (1, 2, 4) attention at 1024 channels, bs=2 train")


def test_gradient_chunks_tile_the_flat_buffer(golden):
    """data-parallel seam: the backward completes the flat gradient buffer in contiguous chunks (ddpm_unet_grad_chunks) that
    tile it exactly; waiting for a chunk's event on another stream and reading the chunk there sees the final gradients."""
    import ddpm_torch_b200 as D
    from ddpm_torch_b200 import _lib, parallel
    fx = golden("unet_cifar10_bs4.pt")
    m, sd = build(fx["cfg"], fx["seed"], train=True)
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    x0, t, noise = fx["x0"].to(DEV), fx["t"].to(DEV), fx["noise"].to(DEV)
    diff.train_losses(m, x0, t, noise).mean().backward()
    ref = m.flat_grads.clone()
    chunks = parallel.grad_chunks(m)
    print(f"\n[grad chunks] {len(chunks)} chunks: " + ", ".join(f"[{lo / 1e6:.2f}M, {hi / 1e6:.2f}M)" for lo, hi in chunks))
    assert len(chunks) >= 3
    cover = sorted(chunks)
    assert cover[0][0] == 0 and cover[-1][1] == m.flat_grads.numel() and all(a[1] == b[0] for a, b in zip(cover, cover[1:]))
    # second backward: copy every chunk out on a side stream as soon as its event fires
    m.zero_grad()
    L = _lib.lib()
    loss = diff.train_losses(m, x0, t, noise).mean()
    got = torch.zeros_like(ref)
    loss.backward()
    side = torch.cuda.Stream()
    for i, (lo, hi) in enumerate(chunks):
        _lib.check(L.ddpm_unet_wait_grad_chunk(m._h, i, side.cuda_stream))
        with torch.cuda.stream(side):
            got[lo:hi].copy_(m._grads[lo:hi])
    side.synchronize()
    torch.cuda.synchronize()
    r = rel(got, ref)
    print(f"[grad chunks] chunk-wise copy vs first backward rel-L2 {r:.3e}")
    assert r < 1e-2
    flag_ok()


def test_operand_path_groupnorm_optin(golden, monkeypatch):
    """DDPM_XF=1 (opt-in): inference plans fold norm + SiLU into the consumer
    conv's operand path (transform warps of the CTA-pair kernel).  Same parity bar as the default path."""
    monkeypatch.setenv("DDPM_XF", "1")
    fx = golden("unet_cifar10_bs4.pt")
    cfg = fx["cfg"]
    m, sd = build(cfg, fx["seed"])
    g = torch.Generator(DEV).manual_seed(3)
    x = torch.randn(8, 3, 32, 32, device=DEV, generator=g); t = torch.randint(1000, (8,), device=DEV, generator=g)
    with torch.no_grad():
        eps = m(x, t)
        ref = R.unet_forward(sd, cfg, x, t)
    r = rel(eps, ref)
    print(f"\n[DDPM_XF=1] eps rel-L2 {r:.3e}")
    assert r < 1e-2
    flag_ok()


def test_fused_attention_backward_optin(golden, monkeypatch):
    """DDPM_FUSED_ATTN_BWD=1 (opt-in): dP -> softmax backward -> dQ of
    the 16x16 attention blocks as one launch.  Same parity bar as the default training plan."""
    monkeypatch.setenv("DDPM_FUSED_ATTN_BWD", "1")
    fx = golden("unet_cifar10_bs4.pt")
    m, sd = build(fx["cfg"], fx["seed"], train=True)
    g = torch.Generator(DEV).manual_seed(77)
    x0 = torch.rand(8, 3, 32, 32, device=DEV, generator=g) * 2 - 1
    t = torch.randint(1000, (8,), device=DEV, generator=g)
    noise = torch.randn(8, 3, 32, 32, device=DEV, generator=g)
    grads_vs_oracle(m, sd, fx["cfg"], x0, t, noise, "cifar10 bs=8 train, fused attention backward")


def test_run_to_run_gradient_drift_is_bounded(golden):
    """The engine's reductions (split-K fp32 REDs of the weight gradients, GroupNorm / column-sum atomics) are order-dependent, so
    two passes over identical inputs are not bit-identical (the reference is).  Bound the drift at the benchmarked shape: it has to
    stay an order of magnitude inside the parity budget against the oracle (flat-gradient rel-L2 5e-2, loss 1e-2)."""
    import ddpm_torch_b200 as D
    fx = golden("unet_cifar10_bs4.pt")
    m, _ = build(fx["cfg"], fx["seed"], train=True)
    g = torch.Generator(DEV).manual_seed(321)
    x0 = torch.rand(128, 3, 32, 32, device=DEV, generator=g) * 2 - 1
    t = torch.randint(1000, (128,), device=DEV, generator=g)
    noise = torch.randn(128, 3, 32, 32, device=DEV, generator=g)
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    runs = []
    for _ in range(3):
        m.zero_grad()
        losses = diff.train_losses(m, x0, t, noise)
        losses.mean().backward()
        runs.append((losses.detach().clone(), torch.cat([p.grad.flatten() for p in m.parameters()]).clone()))
    flag_ok()
    dl = max((runs[i][0] - runs[0][0]).abs().max().item() / runs[0][0].abs().max().item() for i in (1, 2))
    dg = max(rel(runs[i][1], runs[0][1]) for i in (1, 2))
    print(f"\n[run-to-run, cifar10 bs=128 train] loss drift {dl:.3e}; flat-gradient drift rel-L2 {dg:.3e}")
    assert dl < 2e-3 and dg < 1e-2
