"""The toy engine (csrc/toy_mlp.cuh) against the fp64 restatement of the reference Decoder (tests/toy_ref.py) on the H100:
forward over the supported shapes, the fused training loss and gradients, dx through model(x, t), determinism, weight updates
without a repack, the sampler chain (bit-exact tail with eps pinned; approximate against the generic loop) and the reference
Trainer / Evaluator end to end."""
import copy
import importlib.util
import math

import numpy as np
import pytest
import torch

from ddpm_torch_b200 import toy as T

from toy_ref import KEYS, decoder_forward, params_of

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _model(D, M, L, seed=0):
    torch.manual_seed(seed)
    m = T.Decoder(D, M, L)
    with torch.no_grad():                      # non-trivial LayerNorm affine and biases
        for n, p in m.named_parameters():
            if n.endswith("bias") or "norm" in n:
                p.add_(0.1 * torch.randn_like(p))
    return m.to(DEV)


def _diff(T_=100):
    return T.GaussianDiffusion(T.get_beta_schedule("linear", 0.001, 0.2, T_), "eps", "fixed-large", "mse")


def _ts(B, kind, T_=100, g=None):
    if kind == "random":
        return torch.randint(T_, (B,), generator=g).to(DEV)
    return torch.full((B,), {"0": 0, "1": 1, "T-1": T_ - 1}[kind], dtype=torch.int64, device=DEV)


@pytest.mark.parametrize("B", [1, 63, 64, 65, 1000, 30000])
@pytest.mark.parametrize("M,L,D", [(64, 1, 1), (64, 3, 4), (128, 1, 2), (128, 3, 2), (128, 3, 4), (64, 3, 2)])
def test_forward_vs_fp64(B, M, L, D):
    m = _model(D, M, L, seed=B + M + L + D)
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B, D, generator=g).to(DEV)
    p = params_of(m, device=DEV)
    for kind in ("0", "1", "T-1", "random"):
        t = _ts(B, kind, g=g)
        with torch.no_grad():
            out = m(x, t)
        ref = decoder_forward(p, L, x.double(), t)
        err = _rel(out, ref)
        assert err <= 2e-2, (kind, err)
        # per-row direction, on rows whose output is not near zero (there bf16 operand rounding dominates the angle)
        cos = torch.nn.functional.cosine_similarity(out.double(), ref, dim=1)
        big = ref.norm(dim=1) >= 0.5 * ref.norm(dim=1).median()
        if D > 1 and big.any():
            assert cos[big].min().item() >= 0.99, (kind, cos[big].min().item())


@pytest.mark.parametrize("B,M,L,D", [(1000, 128, 3, 2), (65, 64, 1, 1), (257, 64, 3, 4)])
def test_train_loss_and_gradients(B, M, L, D):
    m = _model(D, M, L, seed=3)
    d = _diff()
    g = torch.Generator().manual_seed(1)
    x0 = torch.randn(B, D, generator=g).to(DEV)
    t = torch.randint(100, (B,), generator=g).to(DEV)
    noise = torch.randn(B, D, generator=g).to(DEV)
    loss = d.train_losses(m, x0, t, noise)
    loss.mean().backward()
    p = params_of(m, device=DEV, grad=True)
    x_t = d.q_sample(x0, t, noise=noise).double()
    lref = ((noise.double() - decoder_forward(p, L, x_t, t)) ** 2).mean(1)
    lref.mean().backward()
    # per-row, relative to the larger of the row's loss and the batch mean (a row whose output nearly matches its noise has a
    # loss near zero, and bf16 rounding of the output is then a large fraction of it)
    assert ((loss.double() - lref).abs() / torch.maximum(lref, lref.mean())).max().item() <= 3e-2     # measured <= 1.6e-2
    got = torch.cat([q.grad.flatten() for q in m.parameters()])
    ref = torch.cat([p[k].grad.flatten() for k in KEYS])
    assert _rel(got, ref) <= 5e-2
    for (k, q) in zip(KEYS, m.parameters()):
        cos = torch.nn.functional.cosine_similarity(q.grad.double().flatten(), p[k].grad.flatten(), dim=0).item()
        assert cos >= 0.995, k


@pytest.mark.parametrize("B", [1, 100, 1000])
def test_model_backward_with_dx(B):
    m = _model(2, 128, 3, seed=5)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, 2, generator=g).to(DEV).requires_grad_(True)
    t = torch.randint(100, (B,), generator=g).to(DEV)
    w = torch.randn(B, 2, generator=g).to(DEV)
    (m(x, t) * w).sum().backward()
    p = params_of(m, device=DEV, grad=True)
    xr = x.detach().double().requires_grad_(True)
    (decoder_forward(p, 3, xr, t) * w.double()).sum().backward()
    # dx is the [M] -> [D] projection of the residual-stream gradient through in_fc: most of that gradient cancels, so the bf16
    # rounding of the backward GEMM operands is a larger fraction of dx than of the weight gradients (measured 5.9e-2 at B = 1000)
    assert _rel(x.grad, xr.grad) <= 1e-1
    assert _rel(torch.cat([q.grad.flatten() for q in m.parameters()]), torch.cat([p[k].grad.flatten() for k in KEYS])) <= 5e-2


def test_training_step_is_bit_reproducible():
    m = _model(2, 128, 3, seed=9)
    d = _diff()
    g = torch.Generator().manual_seed(3)
    x0, t, noise = torch.randn(1000, 2, generator=g).to(DEV), torch.randint(100, (1000,), generator=g).to(DEV), torch.randn(1000, 2, generator=g).to(DEV)
    grads = []
    for _ in range(2):
        m.zero_grad()
        d.train_losses(m, x0, t, noise).mean().backward()
        grads.append(torch.cat([q.grad.flatten() for q in m.parameters()]))
    assert torch.equal(grads[0], grads[1])


@pytest.mark.parametrize("fused", [False, True])
def test_outputs_follow_weight_updates(fused):
    m = _model(2, 128, 3, seed=11)
    d = _diff()
    opt = torch.optim.Adam(m.parameters(), lr=1e-2, fused=fused)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(500, 2, generator=g).to(DEV)
    t = torch.randint(100, (500,), generator=g).to(DEV)
    for _ in range(3):
        opt.zero_grad()
        d.train_losses(m, x, t).mean().backward()
        opt.step()
        with torch.no_grad():
            assert _rel(m(x, t), decoder_forward(params_of(m, device=DEV), 3, x.double(), t)) <= 1e-2
    other = _model(2, 128, 3, seed=12)
    m.load_state_dict(other.state_dict())
    with torch.no_grad():
        assert _rel(m(x, t), decoder_forward(params_of(other, device=DEV), 3, x.double(), t)) <= 1e-2
        for q, r in zip(m.parameters(), _model(2, 128, 3, seed=13).parameters()):
            q.data.copy_(r.data)
        assert _rel(m(x, t), decoder_forward(params_of(m, device=DEV), 3, x.double(), t)) <= 1e-2


@pytest.mark.parametrize("M,L,D", [(128, 3, 2), (64, 1, 1)])
def test_sampler_tail_exact_with_eps_pinned(M, L, D):
    m = _model(D, M, L, seed=21)
    with torch.no_grad():
        m.out_fc.weight.zero_()
        m.out_fc.bias.fill_(0.37)
    d = _diff()
    B = 777
    xT = 3.0 * torch.randn(B, D, device=DEV)                      # beyond +-1: a clip would show
    nat = d.p_sample(m, shape=(B, D), device=DEV, noise=xT, seed=5)
    gen = torch.Generator(DEV).manual_seed(5)
    x = xT.clone()
    tt = torch.empty(B, dtype=torch.int64, device=DEV)
    with torch.no_grad():
        for ti in range(d.timesteps - 1, -1, -1):
            tt.fill_(ti)
            x = d.p_sample_step(m, x, tt, generator=gen)
    assert torch.equal(nat, x)
    assert x.abs().max().item() > 1.0


def test_sampler_default_config_vs_generic_loop():
    ref_mod = _reference_functions()
    m = _model(2, 128, 3, seed=31)
    d = _diff()
    B, S = 30000, d.timesteps
    # teacher-forced single steps: the chain kernel with S = 1 rows of the table is the generic step on the same x and z
    g = torch.Generator().manual_seed(0)
    x = 2 * torch.randn(B, 2, generator=g).to(DEV)
    z = torch.randn(S, B, 2, generator=g).to(DEV)
    coef = d._toy_coef_rows(DEV)
    worst = 0.0
    for ti in (S - 1, S // 2, 1, 0):
        # one native step at t = ti: a table of ti+1 rows whose lower rows are the identity update (coef2 = 1, the rest 0)
        ident = torch.zeros(ti + 1, 6, device=DEV)
        ident[:, 3] = 1.0
        ident[ti] = coef[ti]
        zz = torch.zeros(ti + 1, B, 2, device=DEV)
        zz[0] = z[0]
        x1 = T.diffusion.sample_chain(m, ident, x.clone(), zz)
        tt = torch.full((B,), ti, dtype=torch.int64, device=DEV)
        with torch.no_grad():
            gen_step = d.p_mean_var(m, x, tt, True, False)[0] + coef[ti, 5] * coef[ti, 4] * z[0]
        worst = max(worst, (x1 - gen_step).abs().max().item())
    assert worst <= 5e-2, worst
    # full chains from the same generator
    nat = d.p_sample(m, shape=(B, 2), device=DEV, seed=7).cpu().numpy()
    gen = [_generic_chain(d, m, B, seed) for seed in (7, 8)]
    close = (np.abs(nat - gen[0]).max(axis=1) <= 5e-2).mean()
    assert close >= 0.99, close
    if ref_mod is not None:
        h = lambda a: ref_mod.hist2d(a, bins=64, value_range=4)
        kl_nat = ref_mod.discrete_klv2d(h(gen[0]), h(nat))
        kl_gen = ref_mod.discrete_klv2d(h(gen[0]), h(gen[1]))
        assert kl_nat <= max(kl_gen, 1e-3) * 1.5, (kl_nat, kl_gen)


def _generic_chain(d, m, B, seed):
    gen = torch.Generator(DEV).manual_seed(seed)
    x = torch.empty((B, 2), device=DEV).normal_(generator=gen)
    tt = torch.empty(B, dtype=torch.int64, device=DEV)
    with torch.no_grad():
        for ti in range(d.timesteps - 1, -1, -1):
            tt.fill_(ti)
            x = d.p_sample_step(m, x, tt, generator=gen)
    return x.cpu().numpy()


def _reference_functions():
    from oracle import ref_loader
    if not ref_loader.available():
        return None
    ddpm_torch, _ = ref_loader.load()
    return ddpm_torch.functions


def test_reference_trainer_end_to_end(tmp_path, monkeypatch):
    if importlib.util.find_spec("sklearn") is None:
        pytest.skip("the reference's ddpm_torch/toy/__init__.py imports toy_data.py, which needs scikit-learn")
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip("reference not staged")
    ref_loader.load()
    from ddpm_torch.toy import DataStreamer, Trainer, Evaluator
    from ddpm_torch.utils import infer_range
    torch.manual_seed(0)
    loader = DataStreamer("gaussian8", batch_size=1000, num_batches=5)
    d = _diff()
    m = T.Decoder(2, 128, 3).to(DEV)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    tr = Trainer(model=m, optimizer=opt, diffusion=d, epochs=1, trainloader=loader, device=torch.device(DEV), eval_intv=1, chkpt_intv=1)
    xlim, ylim = infer_range(loader.dataset)
    it = iter(loader)
    ev = Evaluator(true_data=np.concatenate([next(it) for _ in range(3)]), eval_batch_size=3000, max_eval_count=3000, value_range=(xlim, ylim))
    path = str(tmp_path / "toy.pt")
    tr.train(ev, chkpt_path=path, image_dir=None)
    res = ev.eval(lambda n: d.p_sample(m, shape=(n, 2), device=DEV).cpu().numpy())
    assert all(np.all(np.isfinite(v)) for v in res.values())
    before = copy.deepcopy(m.state_dict())
    # the reference's load_checkpoint predates torch's weights_only default (its checkpoint holds the scheduler object's state)
    load = torch.load
    monkeypatch.setattr(torch, "load", lambda *a, **k: load(*a, **{**k, "weights_only": False}))
    with torch.no_grad():
        for q in m.parameters():
            q.zero_()
    tr.load_checkpoint(path)
    for k, v in before.items():
        assert torch.equal(m.state_dict()[k], v)
