"""UNets built with resample_with_conv=False (AvgPool2d(2) down, bare nearest x2 up, no resample convs; unet.py:164-170,199-202),
without a GPU:

1. The oracle of this variant (tests/noresample_ref.py) against the UNMODIFIED reference (tests/golden/unet_noresample.pt,
   tools/gen_golden_noresample.py): x_t bit-exact, eps rel-L2 < 1e-5, per-sample losses and gradient norms at the tolerances
   of test_oracle_golden.py, and the bits/dim terms of the host mirror's generic loop.  tests/test_noresample_gpu.py leans on it.
2. The boundary: the mirror's state_dict and the engine's parameter inventory are the reference's (names, shapes, order),
   a reference state dict loads strict, ddpm_unet_create_ex refuses flags other than 0 / 1, the dry plan's FLOPs are the
   reference model's, and the forward launch counts are the ones derived below."""
import ctypes as C
import math

import pytest
import torch

import noresample_ref as N
from oracle import ddpm_ref as R

FIXTURE = "unet_noresample.pt"
NAMES = [c[0] for c in N.CASES]


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _cfg_struct(cfg):
    from ddpm_torch_b200 import _lib
    c = N.normalize_cfg(cfg)
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = c["in_channels"], c["hid_channels"], c["out_channels"]
    u.levels, u.num_res_blocks, u.temb_dim, u.drop_rate = len(c["ch_multipliers"]), c["num_res_blocks"], 0, c["drop_rate"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    return u


def _handle(L, cfg, flag=0):
    u = _cfg_struct(cfg)
    h = C.c_void_p()
    assert L.ddpm_unet_create_ex(C.byref(u), flag, C.byref(h)) == 0, L.ddpm_last_error()
    return h


def _mirror(cfg):
    import ddpm_torch_b200 as D
    c = N.normalize_cfg(cfg)
    return D.UNet(c["in_channels"], c["hid_channels"], c["out_channels"], c["ch_multipliers"], c["num_res_blocks"],
                  c["apply_attn"], drop_rate=c["drop_rate"], resample_with_conv=False)


# ------------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize("name", NAMES)
def test_oracle_forward_loss_backward_match_reference(golden, name):
    fx = golden(FIXTURE)["models"][name]
    cfg = fx["cfg"]
    assert [(k, tuple(s)) for k, s in N.param_shapes(cfg).items()] == [(k, tuple(s)) for k, s in fx["keys"]]
    sd = {k: v.requires_grad_(True) for k, v in N.make_state_dict(cfg, fx["seed"]).items()}
    d = R.RefDiffusion(R.get_beta_schedule("linear", 1e-4, 0.02, 1000), "fixed-large")
    x_t = d.q_sample(fx["x0"], fx["t"], fx["noise"])
    assert torch.equal(x_t, fx["x_t"])
    fn = lambda x, t: N.unet_forward(sd, cfg, x, t)
    with torch.no_grad():
        eps = fn(x_t, fx["t"])
    assert rel_l2(eps, fx["eps"]) < 1e-5
    losses = d.train_losses(fn, fx["x0"], fx["t"], fx["noise"])
    assert torch.allclose(losses, fx["losses"], rtol=1e-5, atol=1e-6)
    losses.mean().backward()
    for k, p in sd.items():
        ref = fx["grad_norm"][k]
        assert abs(p.grad.norm().item() - ref) <= 2e-4 * max(ref, 1e-3), k


def test_oracle_bpd_terms_match_reference(golden):
    import ddpm_torch_b200 as D
    fx = golden(FIXTURE)["models"][N.BPD_CASE]
    bp, cfg = fx["bpd"], fx["cfg"]
    sd = N.make_state_dict(cfg, fx["seed"])
    for (vt, clip), ref in bp["cases"].items():
        d = D.GaussianDiffusion(D.get_beta_schedule("linear", 1e-4, 0.02, bp["T"]), "eps", vt, "mse")
        with torch.no_grad():
            losses, mses = d._generic_bpd_terms(lambda x, t: N.unet_forward(sd, cfg, x, t), bp["x0"], clip, bp["noise"])
        torch.testing.assert_close(losses, ref["losses"], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(mses, ref["mses"], rtol=1e-5, atol=1e-6)


def test_variant_drops_exactly_the_resample_convs():
    """The variant drops exactly the six (CIFAR-10) resample convs: 3,097,984 of 35,746,307 parameters, 1.76 of 12.44 GFLOP."""
    full, var = R.param_shapes(R.CIFAR10_CFG), N.param_shapes(N.CIFAR10_CFG)
    assert [k for k in full if k not in var] == N.resample_keys(N.CIFAR10_CFG)
    n = lambda s: sum(math.prod(v) for v in s.values())
    assert n(full) - n(var) == 3_097_984 and n(var) == 35_746_307 - 3_097_984
    assert abs((R.fwd_flops_per_image(R.CIFAR10_CFG, 32, 32) - N.fwd_flops_per_image(N.CIFAR10_CFG, 32, 32)) / 1e9 - 1.755) < 1e-3


# ------------------------------------------------------------------------------------------------ boundary
@pytest.mark.parametrize("name", NAMES)
def test_mirror_state_dict_is_the_reference_state_dict(golden, name):
    fx = golden(FIXTURE)["models"][name]
    m = _mirror(fx["cfg"])
    assert m.resample_with_conv is False
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in fx["keys"]]
    sd = N.make_state_dict(fx["cfg"], fx["seed"])
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    # the flat buffer holds what was loaded: every parameter is a view of it
    assert all(p.data_ptr() == m.flat_params.data_ptr() + 4 * off for p, (_, _, off) in zip(m.parameters(), m._meta))


@pytest.mark.parametrize("name", NAMES)
def test_engine_param_inventory(L, golden, name):
    fx = golden(FIXTURE)["models"][name]
    h = _handle(L, fx["cfg"])
    try:
        assert L.ddpm_unet_num_params(h) == len(fx["keys"])
        for i, (k, s) in enumerate(fx["keys"]):
            nm, nd, dims, off = C.c_char_p(), C.c_int(), (C.c_int * 4)(), C.c_longlong()
            assert L.ddpm_unet_param_info(h, i, C.byref(nm), C.byref(nd), C.byref(dims), C.byref(off)) == 0
            assert nm.value.decode() == k and tuple(dims[:nd.value]) == tuple(s)
            assert off.value % 64 == 0
    finally:
        L.ddpm_unet_destroy(h)


def test_create_ex_flag(L):
    u = _cfg_struct(N.TINY_CFG)
    for bad in (-1, 2, 3, 255):
        h = C.c_void_p()
        assert L.ddpm_unet_create_ex(C.byref(u), bad, C.byref(h)) != 0
        assert b"resample_with_conv" in L.ddpm_last_error()
        assert not h.value
    # flag 1 is ddpm_unet_create: the same inventory as the conv-resample reference model
    for create in (lambda h: L.ddpm_unet_create(C.byref(u), C.byref(h)), lambda h: L.ddpm_unet_create_ex(C.byref(u), 1, C.byref(h))):
        h = C.c_void_p()
        assert create(h) == 0
        try:
            assert L.ddpm_unet_num_params(h) == len(R.param_shapes(R.TINY_CFG))
        finally:
            L.ddpm_unet_destroy(h)


def _plan(L, cfg, B, HW, training):
    h = _handle(L, cfg)
    try:
        assert L.ddpm_unet_workspace_bytes(h, B, HW, HW, int(training)) > 0, L.ddpm_last_error()
        ff, f, b, p = C.c_double(), C.c_int(), C.c_int(), C.c_int()
        L.ddpm_unet_plan_stats(h, None, None, None, None, C.byref(ff), None)
        L.ddpm_unet_launch_counts(h, C.byref(f), C.byref(b), C.byref(p))
        return ff.value, f.value, b.value, p.value
    finally:
        L.ddpm_unet_destroy(h)


@pytest.mark.parametrize("cfg,B,HW", [(N.TINY_CFG, 2, 16), (N.SMALL64_CFG, 4, 32), (N.CIFAR10_CFG, 128, 32)])
@pytest.mark.parametrize("training", [False, True])
def test_plan_flops_equal_reference_model(L, cfg, B, HW, training):
    ff, _, _, _ = _plan(L, cfg, B, HW, training)
    ref = N.fwd_flops_per_image(cfg, HW, HW)
    assert abs(ff / B - ref) / ref < 1e-6


# Forward launches of the conv-resample plan of the same shape, minus what the variant removes.  Every pool and upsample is one
# launch; a stride-2 down conv is one launch (two when it runs split-K), a training / small-map up path is an upsample plus a 3x3
# conv (one launch, two split-K), and the inference up path at C % 256 == 0 is four folded GEMMs.  Every GroupNorm keeps its
# route or gains the one-pass route from quad statistics (where the conv producer ran split-K, which delivers none), so no
# GroupNorm statistics launch is added:
#   tiny              78 = 77 + (down conv 1 -> pool 1) + (upsample 1 + conv 1 -> upsample 1)
#   small64           76 = 75 + (1 -> 1) + (2 -> 1)
#   CIFAR-10 B = 128  train 146 = 142 + (1 + 1 + 2 -> 3 pools) + 3 x (2 -> 1)
#                     infer 152 = 142 + (4 -> 3) + 3 x (4 folded GEMMs -> 1)
#   CIFAR-10 B = 2    train 160 = 151 + (2 + 2 + 2 -> 3) + (3 + 2 + 2 -> 3 upsamples) + 2 x (statistics + apply -> apply)
#                     infer 165 = 151 + (6 -> 3) + 3 x (4 -> 1) + 2 x (2 -> 1)
LAUNCHES = {  # (name, B, training): (forward, backward, repack) launches of the resample_with_conv=False plan
    ("tiny", 2, False): (77, 0, 1), ("tiny", 2, True): (77, 153, 1),
    ("small64", 2, False): (75, 0, 3), ("small64", 2, True): (75, 160, 4),
    ("cifar10", 2, False): (151, 0, 3), ("cifar10", 2, True): (151, 365, 4),
    ("cifar10", 128, False): (142, 0, 4), ("cifar10", 128, True): (142, 354, 5),
}


@pytest.mark.parametrize("key", sorted(LAUNCHES))
def test_launch_counts(L, key):
    name, B, training = key
    cfg, HW = {c[0]: (c[1], c[3]) for c in N.CASES}[name]
    _, f, b, p = _plan(L, cfg, B, HW, training)
    assert (f, b, p) == LAUNCHES[key]
