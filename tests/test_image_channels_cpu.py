"""Image channel counts other than 3 (the engine accepts 1..4 input and output channels), without a GPU:

1. The oracle (oracle/ddpm_ref.py) against the UNMODIFIED reference at C in {1, 2, 4} and for a 1 -> 2 channel model
   (tests/golden/unet_channels.pt, tools/gen_golden_unet_channels.py): x_t bit-exact, eps rel-L2 < 1e-5, per-sample losses
   and gradient norms at the tolerances of test_oracle_golden.py; the bits/dim terms of the host mirror's generic loop over
   the oracle network at C in {1, 4}.  The GPU tests of tests/test_image_channels_gpu.py lean on this oracle.
2. The planner's route per channel count (dry plans, no device): which image-side convs run on the tensor cores.
3. Models whose output channel count differs from the input's are refused by the training and sampler entry points
   before anything runs on the device (the loss and the update are element-wise against the input)."""
import ctypes as C

import pytest
import torch

from oracle import ddpm_ref as R

FIXTURE = "unet_channels.pt"
MODELS = ["tiny_c1", "tiny_c2", "tiny_c4", "small64_c1", "small64_c2", "small64_c4"]


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def check_grad_norms(sd, ref):
    for k, p in sd.items():
        assert abs(p.grad.norm().item() - ref[k]) <= 2e-4 * max(ref[k], 1e-3), k


@pytest.mark.parametrize("name", MODELS)
def test_oracle_forward_loss_backward_match_reference(golden, name):
    fx = golden(FIXTURE)["models"][name]
    cfg, C_ = fx["cfg"], fx["cfg"]["in_channels"]
    assert fx["x0"].shape == (fx["B"], C_, fx["H"], fx["W"]) and fx["eps"].shape == fx["x0"].shape
    sd = {k: v.requires_grad_(True) for k, v in R.make_state_dict(cfg, fx["seed"]).items()}
    d = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, 1000), "fixed-large")
    x_t = d.q_sample(fx["x0"], fx["t"], fx["noise"])
    assert torch.equal(x_t, fx["x_t"])
    fn = lambda x, t: R.unet_forward(sd, cfg, x, t)
    with torch.no_grad():
        eps = fn(x_t, fx["t"])
    assert rel_l2(eps, fx["eps"]) < 1e-5
    assert (eps - fx["eps"]).abs().max().item() < 5e-5
    losses = d.train_losses(fn, fx["x0"], fx["t"], fx["noise"])
    assert torch.allclose(losses, fx["losses"], rtol=1e-5, atol=1e-6)
    losses.mean().backward()
    check_grad_norms(sd, fx["grad_norm"])


def test_oracle_asymmetric_model_matches_reference(golden):
    fx = golden(FIXTURE)["models"]["small64_c1to2"]
    cfg = fx["cfg"]
    assert (cfg["in_channels"], cfg["out_channels"]) == (1, 2)
    sd = {k: v.requires_grad_(True) for k, v in R.make_state_dict(cfg, fx["seed"]).items()}
    assert sd["in_conv.weight"].shape[1] == 1 and sd["out_conv.2.weight"].shape[0] == 2
    out = R.unet_forward(sd, cfg, fx["x_t"], fx["t"])
    assert out.shape == fx["eps"].shape == (fx["B"], 2, fx["H"], fx["W"])
    assert rel_l2(out, fx["eps"]) < 1e-5
    (out * fx["g"]).sum().backward()
    check_grad_norms(sd, fx["grad_norm"])


@pytest.mark.parametrize("name", [m for m in MODELS if not m.endswith("_c2")])
def test_oracle_bpd_terms_match_reference(golden, name):
    """The generic bits/dim loop of the host mirror (the same torch formulas as the reference) over the oracle network."""
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"][name]
    bp = fx["bpd"]
    cfg = fx["cfg"]
    sd = R.make_state_dict(cfg, fx["seed"])
    x0 = bp["x0"]
    assert (x0 == 1).any() and (x0 == -1).any()                     # the decoder's edge bins are reached
    for (vt, clip), ref in bp["cases"].items():
        d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, bp["T"]), "eps", vt, "mse")
        with torch.no_grad():
            losses, mses = d._generic_bpd_terms(lambda x, t: R.unet_forward(sd, cfg, x, t), x0, clip, bp["noise"])
        torch.testing.assert_close(losses, ref["losses"], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(mses, ref["mses"], rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------ planner routes
def _plan_stats(cfg, B, HW, training):
    """Dry plan (no device): (tensor-core op count, forward launches, backward launches)."""
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    c = R.normalize_cfg(cfg)
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = c["in_channels"], c["hid_channels"], c["out_channels"]
    u.levels, u.num_res_blocks, u.temb_dim, u.drop_rate = len(c["ch_multipliers"]), c["num_res_blocks"], 0, c["drop_rate"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    h = C.c_void_p()
    assert L.ddpm_unet_create(C.byref(u), C.byref(h)) == 0, L.ddpm_last_error()
    try:
        assert L.ddpm_unet_workspace_bytes(h, B, HW, HW, int(training)) > 0, L.ddpm_last_error()
        ntc, nf, nb = C.c_int(), C.c_int(), C.c_int()
        L.ddpm_unet_plan_stats(h, None, None, C.byref(ntc), None, None, None)
        L.ddpm_unet_launch_counts(h, C.byref(nf), C.byref(nb), None)
        return ntc.value, nf.value, nb.value
    finally:
        L.ddpm_unet_destroy(h)


@pytest.mark.parametrize("training", [False, True])
def test_planner_routes_per_channel_count(training):
    """tiny (hid 32): no image-side conv is eligible for the tensor cores, at any C.  small64 (hid 64, 32x32): in_conv on
    the tensor cores for every C (9*C <= 64); out_conv on the tensor cores for C <= 3 (9*C <= 32), on CUDA cores at C = 4."""
    st = lambda base, HW, cin, cout: _plan_stats(dict(base, in_channels=cin, out_channels=cout), 2, HW, training)
    tiny = {c: st(R.TINY_CFG, 16, c, c) for c in (1, 2, 3, 4)}
    assert len(set(tiny.values())) == 1, tiny
    small = {c: st(R.SMALL64_CFG, 32, c, c) for c in (1, 2, 3, 4)}
    assert small[1] == small[2] == small[3], small
    assert st(R.SMALL64_CFG, 32, 1, 2) == small[3]
    # C = 4 loses exactly the out_conv GEMM (and in training its data- and weight-gradient GEMMs) and the gather launch;
    # in_conv stays on the tensor cores
    assert small[4][0] == small[3][0] - (3 if training else 1), small
    assert small[4][1] == small[3][1] - 1, small


def test_asymmetric_model_refused_by_train_and_sampler_entry_points():
    from ddpm_torch_b200 import _lib
    L = _lib.lib()
    c = R.normalize_cfg(dict(R.SMALL64_CFG, in_channels=1, out_channels=2))
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = 1, c["hid_channels"], 2
    u.levels, u.num_res_blocks = len(c["ch_multipliers"]), c["num_res_blocks"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    h = C.c_void_p()
    assert L.ddpm_unet_create(C.byref(u), C.byref(h)) == 0, L.ddpm_last_error()
    try:
        assert L.ddpm_train_forward(h, None, None, None, None, None, None, 0, None) != 0
        assert b"out_channels == in_channels" in L.ddpm_last_error()
        assert L.ddpm_sampler_step(h, None, None, 0, None) != 0
        assert b"out_channels == in_channels" in L.ddpm_last_error()
        assert L.ddpm_sampler_step_pred(h, None, None, 0, None, None) != 0
        assert b"out_channels == in_channels" in L.ddpm_last_error()
    finally:
        L.ddpm_unet_destroy(h)
