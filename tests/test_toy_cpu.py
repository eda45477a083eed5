"""The toy mirror (ddpm_torch_b200.toy) on the CPU: module tree, tied weights, same-seed initialisation, the generic toy formulas
against goldens written by the unmodified reference (tools/gen_golden_toy.py), the C ABI's refusals and the kernels' SASS."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import toy as T
from ddpm_torch_b200.toy.model import ToyCfg

from toy_ref import KEYS, decoder_forward, params_of

HERE = os.path.dirname(os.path.abspath(__file__))
G = torch.load(os.path.join(HERE, "golden", "toy.pt"), weights_only=False)
CASES = ["default", "small"]


def _diffusion():
    betas = T.get_beta_schedule("linear", 0.001, 0.2, G["T"])
    return T.GaussianDiffusion(betas, "eps", "fixed-large", "mse")


@pytest.mark.parametrize("case", CASES)
def test_module_tree_keys_and_ties(case):
    D, M, L, _ = G[case]["cfg"]
    m = T.Decoder(D, M, L)
    ref = G[case]["state_dict"]
    assert list(m.state_dict().keys()) == list(ref.keys())
    assert [n for n, _ in m.named_parameters()] == KEYS
    assert len(m.state_dict()) == 7 + 8 * L and len(list(m.parameters())) == 15
    sd = m.state_dict()
    for l in range(1, L):
        for k in KEYS[1:9]:
            assert sd[k.replace("temp_fc.0.", f"temp_fc.{l}.")].data_ptr() == sd[k].data_ptr()
    m.load_state_dict(ref, strict=True)


@pytest.mark.parametrize("case", CASES)
def test_same_seed_init_bit_exact(case):
    D, M, L, seed = G[case]["cfg"]
    torch.manual_seed(seed)
    m = T.Decoder(D, M, L)
    for k, v in G[case]["state_dict"].items():
        assert torch.equal(m.state_dict()[k], v), k


@pytest.mark.parametrize("case", CASES)
def test_restatement_pinned_to_goldens(case):
    g = G[case]
    L = g["cfg"][2]
    p32 = params_of(g["state_dict"], torch.float32)
    out32 = decoder_forward(p32, L, g["x"], g["t"])
    assert torch.allclose(out32, g["out"], rtol=1e-5, atol=1e-6)
    p64 = params_of(g["state_dict"], grad=True)
    out64 = decoder_forward(p64, L, g["x"].double(), g["t"])
    assert ((out64 - g["out"].double()).norm() / g["out"].double().norm()).item() < 1e-5
    loss = ((g["noise"].double() - decoder_forward(p64, L, _diffusion().q_sample(g["x"], g["t"], g["noise"]).double(), g["t"])) ** 2).mean(1)
    assert torch.allclose(loss.float(), g["losses"], rtol=1e-4, atol=1e-7)
    loss.mean().backward()
    for k, ref in zip(KEYS, g["grads"]):
        got = p64[k].grad
        assert ((got - ref.double()).norm() / ref.double().norm().clamp_min(1e-30)).item() < 1e-4, k


@pytest.mark.parametrize("case", CASES)
def test_generic_toy_formulas_reproduce_goldens(case):
    g = G[case]
    L = g["cfg"][2]
    p = params_of(g["state_dict"], torch.float32)
    fn = lambda x, t: decoder_forward(p, L, x, t)
    d = _diffusion()
    with torch.no_grad():
        mean, _, logvar, pred = d.p_mean_var(fn, g["x"], g["t"], clip_denoised=True, return_pred=True)
        step = mean + (g["t"] > 0).float().reshape(-1, 1) * torch.exp(0.5 * logvar) * g["z"]
        x_t = d.q_sample(g["x"], g["t"], noise=g["noise"])
        bpd = d._loss_term_bpd(fn, x_0=g["x"], x_t=x_t, t=g["t"], clip_denoised=True, return_pred=False)
    assert torch.allclose(pred, g["pred_x_0"], rtol=1e-4, atol=1e-5)
    assert (pred.abs() > 1).any()                                  # no clip: predictions beyond +-1 survive
    assert torch.allclose(step, g["step"], rtol=1e-4, atol=1e-5)
    assert torch.allclose(bpd, g["bpd"], rtol=1e-4, atol=1e-5)
    assert (g["t"] == 0).any() and (g["t"] > 0).any()


def test_cpu_model_raises_at_call_time():
    m = T.Decoder(2, 64, 1)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(3, 2), torch.zeros(3, dtype=torch.int64))


def test_exports_and_refusals():
    L = _lib.lib()
    for name in ("ddpm_toy_num_params", "ddpm_toy_workspace_bytes", "ddpm_toy_ws_layout", "ddpm_toy_forward", "ddpm_toy_train_forward",
                 "ddpm_toy_backward", "ddpm_toy_train_backward", "ddpm_toy_sample"):
        assert name in _lib.EXPORTS
        getattr(L, name)
    assert L.ddpm_toy_num_params(C.byref(ToyCfg(2, 128, 3))) == 67074
    assert L.ddpm_toy_num_params(C.byref(ToyCfg(1, 64, 1))) == sum(p.numel() for p in T.Decoder(1, 64, 1).parameters())
    for cfg, rows, msg in [((2, 96, 3), 10, "mid_features"), ((2, 256, 3), 10, "mid_features"), ((5, 128, 3), 10, "in_features"),
                           ((0, 128, 3), 10, "in_features"), ((2, 128, 0), 10, "num_temporal_layers"), ((2, 128, 3), 0, "rows")]:
        assert L.ddpm_toy_workspace_bytes(C.byref(ToyCfg(*cfg)), rows, 1) < 0
        assert msg in L.ddpm_last_error().decode()
    # refused before any launch: null workspace / pointers never reach the device
    assert L.ddpm_toy_forward(C.byref(ToyCfg(2, 128, 3)), None, None, None, 4, None, 0, None, 0, None) != 0
    assert L.ddpm_toy_sample(C.byref(ToyCfg(2, 64, 1)), None, None, 4, 0, None, None, None, 0, None) != 0


def test_toy_kernels_are_wgmma():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    txt = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    per, cur = {}, None
    for ln in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1); per[cur] = set(); continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", ln)
        if m and cur:
            per[cur].add(m.group(1))
    toy = {fn: ops for fn, ops in per.items() if "toy_" in fn}
    for kind in ("toy_fwd_kernel", "toy_bwd_kernel", "toy_temb_kernel", "toy_temb_bwd_kernel", "toy_sample_kernel"):
        hits = [ops for fn, ops in toy.items() if kind in fn]
        assert len(hits) == 2, kind                                # mid_features 64 and 128
        assert all(any(o.startswith("HGMMA") for o in ops) for ops in hits), kind
    assert not any(o.startswith("HMMA") for ops in toy.values() for o in ops)
