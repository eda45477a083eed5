"""The sampler step and the training tails of the engine with the UNet taken out of the arithmetic: out_conv.weight = 0 and
out_conv.bias = BETA make eps == BETA per channel EXACTLY on both out_conv routes (tensor-core gather: the packed zeros give T = 0,
then + bias; CUDA-core k_out_conv: bias + sum a * 0).  What remains is the step / loss arithmetic itself:
  step    psample_update (kernels_simt.cuh) in k_out_gather's fused epilogue (small64, CIFAR-10) and in k_psample_tail (tiny: its
          out_conv runs on the CUDA cores), fed by k_sampler_prep's row for the step.  It repeats the fp32 operations of the mirror's
          generic p_sample_step (diffusion.py) in the same order, and sigma comes from the same CPU exp as the mirror's, so x_{t-1}
          and pred_x0 must equal the mirror's, run on the CPU with denoise_fn = BETA and the same z, BIT FOR BIT.
  chains  p_sample (DDPM, T = 20, both variances; DDIM on 20 of 1000 steps with eta in {0, 0.5, 1}), graph and eager, split 1 and
          2, against the mirror's CPU loop fed the same torch.Generator stream: bit-identical at the end.  This checks
          k_sampler_prep's counter walk and row selection.  Also DDPM T = 20 and DDIM on 10 steps alternating on one model: a
          new chain length captures a new step graph, the same length replays the cached one.
  philox  rng = "philox" with BETA = 0 and x_t = 0 writes x_{t-1} = fl(sigma z): z at CIFAR-10 shape, B = 256 (786k samples per
          step), fixed seeds.  Mean and variance within 5 sigma of N(0, 1), KS p > 1e-3, |z| <= sqrt(-2 ln 2^-32) (u1 >= 2^-32;
          1e-5 relative for __logf and the division by sigma), correlation of consecutive steps and of the two split halves' seeds
          within 5 / sqrt(n), same seed bit-identical, another seed different.
  train   train_losses = mean((noise - BETA_c)^2) against fp64 within the bound of k_mse's sums (per-thread serial sums of
          per_img / 256 terms, a warp and an 8-way sum: (per_img / 256 + 13 + 3) 2^-23 of the loss, the 3 for d and d^2);
          (losses . w).sum().backward() with a different w per image gives exactly zero gradients outside out_conv.2, and
          out_conv.2.bias.grad = sum_b w_b sum_p 2 (BETA_c - noise) / per_img within (B HW + 4) 2^-23 of the sum of |terms|.
  q_sample  with real weights, per-image t shuffled over {0, 1, 998, 999, ...}: train_losses against mean((noise - m(x_t, t))^2)
          with x_t the mirror's fp32 q_sample, on the same training plan.  The prologue repeats those fp32 operations, so the only
          difference is the forward's run-to-run drift: bound 4x the spread of three m(x_t, t) calls + 1e-6."""
import math

import pytest
import torch

from oracle import ddpm_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
BETA = torch.tensor([0.3, -0.7, 1.9])
CFGS = {"tiny": (R.TINY_CFG, 16), "small64": (R.SMALL64_CFG, 32), "cifar10": (R.CIFAR10_CFG, 32)}


def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def st():
    from ddpm_torch_b200 import _lib
    return _lib.stream_ptr()


def ok(rc):
    assert rc == 0, L().ddpm_last_error()


def model(name, beta=BETA, pinned=True, seed=0):
    import ddpm_torch_b200 as D
    cfg, HW = CFGS[name]
    c = R.normalize_cfg(cfg)
    m = D.UNet(c["in_channels"], c["hid_channels"], c["out_channels"], c["ch_multipliers"], c["num_res_blocks"],
               c["apply_attn"], drop_rate=0.0)
    m.load_state_dict(R.make_state_dict(cfg, seed))
    if pinned:
        P = dict(m.named_parameters())
        with torch.no_grad():
            P["out_conv.2.weight"].zero_()
            P["out_conv.2.bias"].copy_(beta)
    return m.to(DEV), HW


def diffusion(var, T=1000):
    import ddpm_torch_b200 as D
    return D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, T), "eps", var, "mse")


def pinned_fn(beta=BETA):
    return lambda x, t: beta.view(1, -1, 1, 1).expand_as(x).to(x.device).contiguous()


def clip_edges(diff, ti, x):
    """rows of x_t whose fp32 c0 x_t - c1 BETA lands exactly on -1, +1, and just past / inside them"""
    c = diff._coef_rows()[ti]
    c0, c1 = c[0], c[1]
    for ch in range(3):
        for k, v in enumerate((1.0, -1.0, 1.0000001, -1.0000001, 0.9999999, -0.9999999, 1.5, -1.5)):
            xv = ((v + c1 * BETA[ch]) / c0).float()
            for _ in range(64):                 # walk x_t by ulps until the fp32 expression gives v, when it can
                got = (c0 * xv - c1 * BETA[ch]).item()
                if got == v or abs(v) == 1.5:
                    break
                xv = torch.nextafter(xv, torch.tensor(math.inf if got < v else -math.inf))
            x[0, ch, 0, k] = xv
    return x


@pytest.mark.parametrize("name", sorted(CFGS))
@pytest.mark.parametrize("var", ["fixed-large", "fixed-small"])
def test_sampler_step_bit_exact(name, var):
    m, HW = model(name)
    diff = diffusion(var)
    B = 4
    m.eval()
    h = m.prepare(B, HW, HW, False, force_repack=True)
    coef, tmod = diff._coef_rows(), diff._model_timesteps().contiguous()
    ok(L().ddpm_sampler_setup(h, coef.shape[0], tmod.data_ptr(), coef.data_ptr()))
    for ti in (0, 1, 500, 999):
        g = torch.Generator().manual_seed(ti)
        x = clip_edges(diff, ti, torch.randn(B, 3, HW, HW, generator=g) * 3)
        t = torch.full((B,), ti, dtype=torch.int64)
        ref, ref_pred = diff.p_sample_step(pinned_fn(), x, t, return_pred=True, generator=torch.Generator().manual_seed(7 + ti))
        z = torch.empty_like(x).normal_(generator=torch.Generator().manual_seed(7 + ti))      # the draw p_sample_step made
        xd, pd = x.to(DEV), torch.full((B, 3, HW, HW), float("nan"), device=DEV)
        ok(L().ddpm_sampler_reset(h, ti, st()))
        ok(L().ddpm_sampler_step_pred(h, xd.data_ptr(), z.to(DEV).data_ptr(), 0, pd.data_ptr(), st()))
        torch.cuda.synchronize()
        assert torch.equal(pd.cpu(), ref_pred), f"{name} {var} t={ti}: pred_x0 differs (max {(pd.cpu() - ref_pred).abs().max():.3e})"
        assert torch.equal(xd.cpu(), ref), f"{name} {var} t={ti}: x_(t-1) differs (max {(xd.cpu() - ref).abs().max():.3e})"
        hit = ref_pred.abs() == 1
        assert hit.any() and (ref_pred.abs() <= 1).all()
        if ti == 0:                          # no noise term at t = 0: a different z gives the same bits
            xd2 = x.to(DEV)
            ok(L().ddpm_sampler_reset(h, ti, st()))
            ok(L().ddpm_sampler_step(h, xd2.data_ptr(), (z * 1e3).to(DEV).data_ptr(), 0, st()))
            torch.cuda.synchronize()
            assert torch.equal(xd2, xd)
    assert L().ddpm_device_error_flag() == 0


def mirror_chain(diff, x_T, seed, fn):
    """the mirror's generic loop on the CPU, fed the device generator's per-step draws (what the native loop draws)"""
    gen = torch.Generator(DEV).manual_seed(seed)
    x = x_T.clone()
    B = x.shape[0]
    for ti in range(len(diff.betas) - 1, -1, -1):
        z = torch.empty(x.shape, device=DEV).normal_(generator=gen).cpu()
        t = torch.full((B,), ti, dtype=torch.int64)
        mean, _, logvar, _ = diff.p_mean_var(fn, x, t, True, True)
        nonzero = (t > 0).reshape((-1, 1, 1, 1)).to(x)
        x = mean + nonzero * torch.exp(0.5 * logvar) * z                 # diffusion.py p_sample_step
    return x


def chain(kind):
    """ddpm-large / ddpm-small: DDPM with T = 20; ddim<eta>[/<S>]: DDIM on S (default 20) of 1000 steps"""
    from ddpm_torch_b200.ddim import DDIM, get_selection_schedule
    if kind.startswith("ddpm"):
        return diffusion("fixed-large" if kind.endswith("large") else "fixed-small", T=20)
    eta, _, S = kind[4:].partition("/")
    return DDIM.from_ddpm(diffusion("fixed-large"), eta=float(eta), subsequence=get_selection_schedule("linear", int(S or 20), 1000))


# chains run in order on one model: each change of chain length reallocates the handles' step tables, so the step graph cached
# by the previous call of that length must be captured anew rather than replayed; DDIM with a new eta keeps the length and the graph
REALLOC = ("ddpm-large", "ddim0/10", "ddpm-large", "ddim0/10", "ddim1/10")


@pytest.mark.parametrize("kinds", [(k,) for k in ("ddpm-large", "ddpm-small", "ddim0", "ddim0.5", "ddim1")] + [REALLOC], ids=",".join)
def test_chains_bit_exact(kinds):
    m, HW = model("small64")
    B = 4
    x_T = torch.randn(B, 3, HW, HW, generator=torch.Generator().manual_seed(3))
    diffs = [chain(k) for k in kinds]
    refs = [mirror_chain(diff, x_T, 11, pinned_fn()) for diff in diffs]
    for use_graph in (True, False):
        for split in (1, 2):
            for j, (kind, diff, ref) in enumerate(zip(kinds, diffs, refs)):
                before = {k: e["graph"] for k, e in m._sampler_cache.items()}
                out = diff.p_sample(m, (B, 3, HW, HW), device=DEV, noise=x_T.to(DEV), seed=11, use_graph=use_graph, split=split)
                assert torch.equal(out.cpu(), ref), f"{kind} graph={use_graph} split={split}: max {(out.cpu() - ref).abs().max():.3e}"
                if use_graph:
                    new = [e["graph"] for k, e in m._sampler_cache.items() if k not in before]
                    recapture = j == 0 or len(diffs[j - 1].betas) != len(diff.betas)
                    assert len(new) == int(recapture), f"{kind} split={split}: {len(new)} graphs captured"
                    assert all(g is not old for g in new for old in before.values())
                    assert all(m._sampler_cache[k]["graph"] is g for k, g in before.items() if k in m._sampler_cache)
    assert L().ddpm_device_error_flag() == 0


def test_philox_noise_is_standard_normal_and_independent():
    from scipy import stats
    m, HW = model("cifar10", beta=torch.zeros(3))
    diff = diffusion("fixed-large")
    B = 256
    m.eval()
    h = m.prepare(B, HW, HW, False, force_repack=True)
    coef, tmod = diff._coef_rows(), diff._model_timesteps().contiguous()
    ok(L().ddpm_sampler_setup(h, coef.shape[0], tmod.data_ptr(), coef.data_ptr()))
    x = torch.zeros(B, 3, HW, HW, device=DEV)

    def draws(seed, first, n):
        ok(L().ddpm_sampler_reset(h, first, st()))
        out = []
        for k in range(n):
            x.zero_()
            ok(L().ddpm_sampler_step(h, x.data_ptr(), None, seed, st()))
            out.append((x.double() / float(coef[first - k, 4])).flatten())
        torch.cuda.synchronize()
        return out

    seed = 0x5EED0001
    z = draws(seed, 999, 3)
    n = z[0].numel()
    zmax = math.sqrt(-2 * math.log(2.0 ** -32)) * (1 + 1e-5)
    for k, zk in enumerate(z):
        mu, var = zk.mean().item(), zk.var().item()
        p = stats.kstest(zk.cpu().numpy(), "norm").pvalue
        print(f"[philox step {k}] n {n} mean {mu:.2e} var {var:.5f} KS p {p:.3f} max|z| {zk.abs().max().item():.3f}")
        assert abs(mu) <= 5 / math.sqrt(n) and abs(var - 1) <= 5 * math.sqrt(2 / n)
        assert p > 1e-3
        assert zk.abs().max().item() <= zmax
    corr = lambda a, b: (((a - a.mean()) * (b - b.mean())).mean() / (a.std() * b.std())).item()
    for a, b in ((0, 1), (1, 2)):
        assert abs(corr(z[a], z[b])) <= 5 / math.sqrt(n), f"steps {a}, {b} correlated"
    half = draws((seed + 2) & 0xFFFFFFFFFFFFFFFF, 999, 1)[0]            # the second half of split = 2 (diffusion.py)
    print(f"[philox] corr consecutive {corr(z[0], z[1]):.2e}, split halves {corr(z[0], half):.2e}")
    assert abs(corr(z[0], half)) <= 5 / math.sqrt(n)
    assert torch.equal(draws(seed, 999, 1)[0], z[0])
    assert not torch.equal(half, z[0])
    assert L().ddpm_device_error_flag() == 0


def test_training_tail_with_eps_pinned():
    m, HW = model("small64")
    m.train()
    diff = diffusion("fixed-large")
    B = 4
    g = torch.Generator(DEV).manual_seed(5)
    x0 = torch.rand(B, 3, HW, HW, device=DEV, generator=g) * 2 - 1
    t = torch.tensor([999, 0, 500, 1], device=DEV)
    noise = torch.randn(B, 3, HW, HW, device=DEV, generator=g)
    losses = diff.train_losses(m, x0, t, noise)
    per_img = 3 * HW * HW
    d = noise.double() - BETA.double().to(DEV).view(1, 3, 1, 1)
    ref = d.pow(2).flatten(1).mean(1)
    bound = (per_img / 256 + 16) * 2.0 ** -23 * ref
    r = ((losses.double() - ref).abs() / bound).max().item()
    print(f"[train loss] worst error / bound {r:.3f}")
    assert r <= 1
    w = torch.tensor([1.0, -0.5, 2.0, 0.25], device=DEV)
    m.zero_grad()
    (losses * w).sum().backward()
    for n, p in m.named_parameters():
        if n.startswith("out_conv.2."):
            continue
        assert p.grad is not None and torch.equal(p.grad, torch.zeros_like(p.grad)), f"{n}: non-zero gradient with eps pinned"
    terms = w.double().view(B, 1, 1, 1) * 2 * (BETA.double().to(DEV).view(1, 3, 1, 1) - noise.double()) / per_img
    gb = terms.sum((0, 2, 3))
    bnd = (B * HW * HW + 4) * 2.0 ** -23 * terms.abs().sum((0, 2, 3))
    r = ((dict(m.named_parameters())["out_conv.2.bias"].grad.double() - gb).abs() / bnd).max().item()
    print(f"[train bias grad] worst error / bound {r:.3f}")
    assert r <= 1
    assert L().ddpm_device_error_flag() == 0


def test_q_sample_prologue_with_per_image_t():
    m, HW = model("small64", pinned=False, seed=4)
    m.train()
    diff = diffusion("fixed-large")
    B = 8
    g = torch.Generator(DEV).manual_seed(8)
    x0 = torch.rand(B, 3, HW, HW, device=DEV, generator=g) * 2 - 1
    t = torch.tensor([999, 0, 500, 1, 998, 250, 10, 750], device=DEV)
    noise = torch.randn(B, 3, HW, HW, device=DEV, generator=g)
    with torch.no_grad():
        losses = diff.train_losses(m, x0, t, noise)
        xt = diff.q_sample(x0, t, noise)                              # the mirror's fp32 q_sample
        refs = torch.stack([(noise - m._forward_nograd(xt, t, training_plan=True)).pow(2).flatten(1).mean(1) for _ in range(3)])
    spread = (refs.max(0).values - refs.min(0).values)
    err = (losses - refs[0]).abs()
    print(f"[q_sample prologue] max |loss - ref| {err.max().item():.3e}, spread {spread.max().item():.3e}")
    assert (err <= 4 * spread + 1e-6).all(), (err, spread)
    assert L().ddpm_device_error_flag() == 0
