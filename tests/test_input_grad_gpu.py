"""Gradients with respect to the UNet's input x on the engine: model(x, t) under autograd returns dx (ddpm_unet_backward_ex),
and a frozen model's backward computes dx alone, without weight gradients and without touching the flat gradient buffer.

Oracle = oracle/ddpm_ref.py (tests/noresample_ref.py for resample_with_conv=False) under torch.autograd on the same GPU in fp32
with TF32 off; golden = tests/golden/unet_input_grad.pt (the unmodified reference, pinned by tests/test_input_grad_cpu.py).

Bounds (DESIGN.md section 2): dx per-image cosine >= 0.995 and whole-tensor rel-L2 <= DX_TOL (twice the worst value measured on
the H100, 1.40e-2 for tiny C = 1; never looser than the flat-gradient bound 5e-2); guidance gradient per-image cosine >= 0.99.
Mode agreement and graph replay: within run-to-run drift, i.e. the bound 1e-2 of
tests/test_unet_gpu.py::test_run_to_run_gradient_drift_is_bounded or 1.5x the drift of two runs of the same mode measured in the
test, whichever is larger.  The GroupNorm-backward column sums use fp32 atomics, so two identical backwards already differ: with
the random cotangents used here dx drifts by about 1e-2 rel-L2 between two runs of one mode on the H100 (measured 1.01e-2 - 1.05e-2)."""
import ctypes as C

import pytest
import torch

import noresample_ref as N
from oracle import ddpm_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
FIXTURE = "unet_input_grad.pt"
NAMES = ["tiny_c1", "tiny_c3", "tiny_c4", "small64_c1", "small64_c2", "small64_c3", "cifar10", "small64_c1to2", "small64_noresample"]
DX_TOL = 2.8e-2
DRIFT = 1e-2


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def cos_per_image(a, b):
    a, b = a.flatten(1).double(), b.flatten(1).double()
    return ((a * b).sum(1) / (a.norm(dim=1) * b.norm(dim=1)).clamp_min(1e-30)).min().item()


@pytest.fixture(autouse=True)
def _no_tf32_and_flag():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    from ddpm_torch_b200 import _lib
    assert _lib.lib().ddpm_device_error_flag() == 0
    torch.cuda.empty_cache()


def build(fx_or_cfg, seed=None, resample=True, drop_rate=None):
    """Engine model and oracle forward over the same weights, on the GPU, eval mode, parameters frozen."""
    import ddpm_torch_b200 as D
    if isinstance(fx_or_cfg, dict) and "cfg" in fx_or_cfg:
        cfg, seed, resample = fx_or_cfg["cfg"], fx_or_cfg["seed"], fx_or_cfg["resample_with_conv"]
    else:
        cfg = fx_or_cfg
    if drop_rate is not None:
        cfg = dict(cfg, drop_rate=drop_rate)
    c = R.normalize_cfg(dict(cfg, resample_with_conv=True))
    m = D.UNet(c["in_channels"], c["hid_channels"], c["out_channels"], c["ch_multipliers"], c["num_res_blocks"], c["apply_attn"],
               drop_rate=c["drop_rate"], resample_with_conv=resample)
    sd = (R if resample else N).make_state_dict(cfg, seed)
    m.load_state_dict(sd)
    m = m.to(DEV).eval().requires_grad_(False)
    sd = {k: v.to(DEV) for k, v in sd.items()}
    fwd = (lambda x, t: R.unet_forward(sd, cfg, x, t)) if resample else (lambda x, t: N.unet_forward(sd, cfg, x, t))
    return m, fwd


def engine_dx(m, x, t, g):
    xg = x.clone().requires_grad_(True)
    (dx,) = torch.autograd.grad((m(xg, t) * g).sum(), xg)
    return dx


def oracle_dx(fwd, x, t, g):
    xg = x.clone().requires_grad_(True)
    (dx,) = torch.autograd.grad((fwd(xg, t) * g).sum(), xg)
    return dx


def drift_bound(a, b):
    """Bound for two runs that may differ only by run-to-run drift, given two runs a, b of the same mode."""
    return max(DRIFT, 1.5 * rel(a, b))


def launches(m, want_dx, params):
    from ddpm_torch_b200 import _lib
    n = _lib.lib().ddpm_unet_backward_launches(m._h, want_dx, params)
    assert n > 0
    return n


# ------------------------------------------------------------------------------------------------ 1. dx vs oracle / golden
@pytest.mark.parametrize("name", NAMES)
def test_dx_vs_oracle_and_golden(golden, name):
    fx = golden(FIXTURE)["models"][name]
    m, fwd = build(fx)
    x, t, g = fx["x"].to(DEV), fx["t"].to(DEV), fx["g"].to(DEV)
    dx = engine_dx(m, x, t, g)
    assert m._grads is not None and m._bwd_since_zero == 0           # input-only: no accumulation bookkeeping
    ref = oracle_dx(fwd, x, t, g)
    c = R.normalize_cfg(dict(fx["cfg"], resample_with_conv=True))
    tc = c["hid_channels"] % 64 == 0 and 9 * c["in_channels"] <= 32
    assert launches(m, 1, 1) - launches(m, 0, 1) == (3 if tc else 2)   # route: pack + GEMM + gather, or pack + k_out_conv
    r_o, r_g = rel(dx, ref), rel(dx.cpu(), fx["dx"])
    c_o, c_g = cos_per_image(dx, ref), cos_per_image(dx.cpu(), fx["dx"])
    nrm = (dx.flatten(1).norm(dim=1).cpu() / fx["dx_norm"] - 1).abs().max().item()
    print(f"\n[dx {name} {'tc' if tc else 'simt'}] rel-L2 vs oracle {r_o:.3e} vs golden {r_g:.3e}; min cosine {min(c_o, c_g):.5f}; "
          f"per-image norm rel err {nrm:.2e}")
    assert dx.shape == x.shape
    assert c_o >= 0.995 and c_g >= 0.995
    assert r_o <= DX_TOL and r_g <= DX_TOL


# ------------------------------------------------------------------------------------------------ 2. mode agreement
def test_modes_agree(golden):
    """x only (frozen parameters), parameters only, and both: the shared outputs agree within run-to-run drift, and
    parameters-only still meets the autograd seam's bound against the oracle."""
    fx = golden(FIXTURE)["models"]["small64_c3"]
    m, _ = build(fx)
    cfg = fx["cfg"]
    sd = {k: v.to(DEV) for k, v in R.make_state_dict(cfg, fx["seed"]).items()}
    x, t, g = fx["x"].to(DEV), fx["t"].to(DEV), fx["g"].to(DEV)
    dx_x, dx_x2 = engine_dx(m, x, t, g), engine_dx(m, x, t, g)

    def with_params(want_x):
        m.requires_grad_(True)
        m.zero_grad(set_to_none=True)
        xg = x.clone().requires_grad_(want_x)
        (m(xg, t) * g).sum().backward()
        gp = torch.cat([p.grad.flatten() for p in m.parameters()])
        m.requires_grad_(False)
        return gp, xg.grad

    gp_p, none = with_params(False)
    assert none is None
    gp_p2, _ = with_params(False)
    gp_b, dx_b = with_params(True)
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    (R.unet_forward(sdg, cfg, x, t) * g).sum().backward()
    gr = torch.cat([sdg[k].grad.flatten() for k, _ in m.named_parameters()])
    print(f"\n[modes] params both vs params-only {rel(gp_b, gp_p):.2e} (same-mode drift {rel(gp_p2, gp_p):.2e}); dx both vs x-only "
          f"{rel(dx_b, dx_x):.2e} (same-mode drift {rel(dx_x2, dx_x):.2e}); params-only vs oracle {rel(gp_p, gr):.2e}")
    assert rel(gp_b, gp_p) <= drift_bound(gp_p2, gp_p) and rel(dx_b, dx_x) <= drift_bound(dx_x2, dx_x)
    assert rel(gp_p, gr) < 5e-2


# ------------------------------------------------------------------------------------------------ 3. training state untouched
def test_input_only_backward_leaves_flat_gradients_alone(golden):
    """A sentinel in the flat gradient buffer survives an input-only backward bit for bit (no memset, no dgamma/dbeta or
    bias-sum atomics, no weight-gradient write), and the accumulation bookkeeping is untouched."""
    fx = golden(FIXTURE)["models"]["cifar10"]
    m, _ = build(fx)
    x, t, g = fx["x"].to(DEV), fx["t"].to(DEV), fx["g"].to(DEV)
    engine_dx(m, x, t, g)                       # plans and allocates the gradient buffer
    m._grads.copy_(torch.linspace(-3.0, 3.0, m._grads.numel(), device=DEV))
    sentinel = m._grads.clone()
    dx = engine_dx(m, x, t, g)
    torch.cuda.synchronize()
    assert torch.equal(m._grads, sentinel)
    assert m._bwd_since_zero == 0 and m._acc is None and not m._acc_pending
    assert torch.isfinite(dx).all()


def test_input_only_probe_between_training_backwards(golden):
    """train_losses backward -> frozen model(x, t) input-only backward -> train_losses backward accumulates the same flat
    gradients as the two training backwards alone (gradient accumulation with a guidance probe in the middle)."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"]["small64_c3"]
    m, _ = build(fx)
    diff = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    gen = torch.Generator(DEV).manual_seed(11)
    B = 4
    x0 = torch.randn(B, 3, 32, 32, device=DEV, generator=gen); t = torch.randint(1000, (B,), device=DEV, generator=gen)
    nz = torch.randn(B, 3, 32, 32, device=DEV, generator=gen)
    xp = torch.randn(B, 3, 32, 32, device=DEV, generator=gen); gp = torch.randn(B, 3, 32, 32, device=DEV, generator=gen)

    def run(probe):
        m.requires_grad_(True)
        m.zero_grad(set_to_none=True)
        diff.train_losses(m, x0, t, nz).mean().backward()
        if probe:
            m.requires_grad_(False)
            engine_dx(m, xp, t, gp)
            m.requires_grad_(True)
        diff.train_losses(m, x0, t, nz).mean().backward()
        flat = m.flat_grads.clone()
        pg = torch.cat([p.grad.flatten() for p in m.parameters()])
        m.zero_grad(set_to_none=True)
        m.requires_grad_(False)
        return flat, pg

    f_ref, p_ref = run(False)
    f_probe, p_probe = run(True)
    print(f"\n[probe] flat grads rel-L2 {rel(f_probe, f_ref):.2e}; p.grad rel-L2 {rel(p_probe, p_ref):.2e}")
    assert rel(f_probe, f_ref) <= DRIFT and rel(p_probe, p_ref) <= DRIFT


# ------------------------------------------------------------------------------------------------ 4. dropout
def test_dropout_input_gradient_directional_derivative():
    """Train mode with dropout: the backward re-uses the forward's saved masks; with the seed held, L(x - e*dx) ~= L(x) - e*|dx|^2."""
    cfg = dict(R.SMALL64_CFG)
    m, _ = build(cfg, 7, drop_rate=0.1)
    m.train()
    gen = torch.Generator(DEV).manual_seed(3)
    x = torch.randn(8, 3, 32, 32, device=DEV, generator=gen); t = torch.randint(1000, (8,), device=DEV, generator=gen)
    target = torch.randn(8, 3, 32, 32, device=DEV, generator=gen)

    def loss(xx):
        m._drop_calls = 41                        # same dropout seed on every evaluation, always through the training plan
        return (m(xx if xx.requires_grad else xx.detach().requires_grad_(True), t) - target).pow(2).mean()

    xg = x.clone().requires_grad_(True)
    l0 = loss(xg)
    (dx,) = torch.autograd.grad(l0, xg)
    d2 = (dx.double() ** 2).sum().item()
    l0b = loss(x).item()
    assert abs(l0b - l0.item()) < 2e-3 * abs(l0.item())         # same seed -> same masks
    e = 0.05 * l0.item() / d2
    l1 = loss(x - e * dx).item()
    pred, got = e * d2, l0.item() - l1
    print(f"\n[dropout dx] L0 {l0.item():.5f} predicted decrease {pred:.5f} measured {got:.5f}")
    assert 0.7 * pred < got < 1.3 * pred


# ------------------------------------------------------------------------------------------------ 5. guidance
def _guide_loss(pred, y, mask):
    return (mask * (pred - y)).pow(2).flatten(1).sum(1)


def test_guidance_gradient_vs_oracle_and_golden(golden):
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"]["cifar10"]
    gd = fx["guide"]
    m, fwd = build(fx)
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, 1000), "eps", "fixed-large", "mse")
    x, t, y, mask = fx["x"].to(DEV), gd["t"].to(DEV), gd["y"].to(DEV), gd["mask"].to(DEV)
    out = {}
    for tag, fn in (("engine", m), ("oracle", fwd)):
        xg = x.clone().requires_grad_(True)
        pred = d.p_mean_var(fn, xg, t, clip_denoised=False, return_pred=True)[-1]
        (out[tag],) = torch.autograd.grad(_guide_loss(pred, y, mask).sum(), xg)
    c_o, c_g = cos_per_image(out["engine"], out["oracle"]), cos_per_image(out["engine"].cpu(), gd["grad"])
    print(f"\n[guidance] per-image cosine vs oracle {c_o:.5f}, vs golden {c_g:.5f}; rel-L2 vs golden {rel(out['engine'].cpu(), gd['grad']):.2e}")
    assert c_o >= 0.99 and c_g >= 0.99


def test_guided_ancestral_loop_reduces_guidance_loss(golden):
    """10 ancestral steps at CIFAR-10 B = 4 with a reconstruction-guidance step on x_t after every p_mean_var (x0_hat from eps,
    masked L2 to y); the same noise without guidance is the control."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"]["cifar10"]
    gd = fx["guide"]
    m, _ = build(fx)
    T = 10
    d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, T), "eps", "fixed-large", "mse")
    y, mask = gd["y"].to(DEV), gd["mask"].to(DEV)
    gen = torch.Generator(DEV).manual_seed(5)
    x_T = torch.randn(4, 3, 32, 32, device=DEV, generator=gen)
    zs = torch.randn(T, 4, 3, 32, 32, device=DEV, generator=gen)

    def loop(scale):
        x = x_T.clone()
        for i in range(T - 1, -1, -1):
            t = torch.full((4,), i, dtype=torch.int64, device=DEV)
            xg = x.requires_grad_(True)
            mean, _, logvar, pred = d.p_mean_var(m, xg, t, clip_denoised=False, return_pred=True)
            (gx,) = torch.autograd.grad(_guide_loss(pred, y, mask).sum(), xg)
            with torch.no_grad():
                step = gx / gx.flatten(1).pow(2).mean(1).sqrt().clamp_min(1e-12).view(-1, 1, 1, 1)   # unit RMS per image
                x = mean + (i > 0) * torch.exp(0.5 * logvar) * zs[i] - scale * step
        return _guide_loss(x, y, mask)

    base, guided = loop(0.0), loop(0.2)
    print(f"\n[guided loop] guidance loss per image: unguided {base.tolist()} guided {guided.tolist()}")
    assert torch.isfinite(guided).all() and (guided < base).all()


# ------------------------------------------------------------------------------------------------ 6. graph, chunks
def test_graph_capture_and_grad_chunks(golden):
    """A captured forward + input-only backward replays to the eager dx within drift; after an input-only backward,
    ddpm_unet_wait_grad_chunk refuses (no chunk event was recorded) until a backward with parameter gradients."""
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    fx = golden(FIXTURE)["models"]["cifar10"]
    m, _ = build(fx)
    x, t, g = fx["x"].to(DEV), fx["t"].to(DEV).contiguous(), fx["g"].to(DEV).contiguous()
    dx_eager, dx_eager2 = engine_dx(m, x, t, g), engine_dx(m, x, t, g)
    B, _, H, W = x.shape
    h = m.prepare(B, H, W, training=True)
    eps = torch.empty(B, 3, H, W, device=DEV); dx = torch.empty_like(x)
    st = _lib.stream_ptr()
    _lib.check(L.ddpm_unet_forward(h, x.data_ptr(), t.data_ptr(), eps.data_ptr(), 0, st))   # consumes the pending repack
    _lib.check(L.ddpm_unet_backward_ex(h, g.data_ptr(), dx.data_ptr(), 0, st))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            cs = _lib.stream_ptr()
            _lib.check(L.ddpm_unet_forward(h, x.data_ptr(), t.data_ptr(), eps.data_ptr(), 0, cs))
            _lib.check(L.ddpm_unet_backward_ex(h, g.data_ptr(), dx.data_ptr(), 0, cs))
    torch.cuda.current_stream().wait_stream(s)
    dx.zero_()
    graph.replay()
    torch.cuda.synchronize()
    print(f"\n[graph] replayed dx vs eager rel-L2 {rel(dx, dx_eager):.2e} (eager drift {rel(dx_eager2, dx_eager):.2e})")
    assert rel(dx, dx_eager) <= drift_bound(dx_eager2, dx_eager)
    n = L.ddpm_unet_grad_chunks(h, 0, None, None)
    assert n > 0
    assert L.ddpm_unet_wait_grad_chunk(h, 0, st) != 0
    assert b"no parameter gradients" in L.ddpm_last_error()
    _lib.check(L.ddpm_unet_backward(h, g.data_ptr(), st))
    assert all(L.ddpm_unet_wait_grad_chunk(h, i, st) == 0 for i in range(n))
    torch.cuda.synchronize()
