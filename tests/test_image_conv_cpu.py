"""CPU-only checks of the image-side convolution probes (ddpm_unet_image_layout / _forward / _backward) and of the planner's
routes for in_conv, its weight gradient, out_conv.2 and the input gradient dx (unet_engine_impl.cuh, plan()):

  in_conv forward     tensor cores (k_pack_in + k_im2col3 + a K = 64 GEMM) when hid % 64 == 0 and the map is a power-of-two
                      geometry (conv_tc_geom), else k_in_conv
  in_conv wgrad       the same rule (an MN-major GEMM over the im2col + k_unpack_tap mode 1 + the column sum), else k_corr3x3
  out_conv.2          tensor cores (k_pack_tapco + a 1x1 GEMM to the 9*Cout tap outputs + k_out_gather) when additionally
                      9 * Cout <= 32, else k_out_conv; its backward follows the forward's route
  dx                  tensor cores (k_pack_tapflip + out_conv's GEMM shape + k_out_gather) when 9 * Cin <= 32, else
                      k_flip_transpose_w + k_out_conv
  h0 quad statistics  written by in_conv when hid % 32 == 0 and H * W % 32 == 0

The cases of tests/test_image_conv_gpu.py are declared here, and this file checks on dry plans that together they reach every
route both ways.  Also: the exports, argument refusals before any device work, and the default plans' launch counts."""
import ctypes as C

import pytest
import torch

from oracle import ddpm_ref as R

FAKE = 1 << 20          # a 16-byte aligned non-null address: every call below fails on the host before it could be used


def _cfg(hid, cin=3, cout=3, mult=(1, 2)):
    return dict(in_channels=cin, hid_channels=hid, out_channels=cout, ch_multipliers=mult, num_res_blocks=1,
                apply_attn=(False,) * len(mult), drop_rate=0.0)


# name -> (cfg, B, H, W): the shapes of test_image_conv_gpu.py.  Only hid, Cin, Cout, B, H and W reach the image-side ops; the
# rest of a config just has to plan (the off-power-of-two CIFAR-10 shapes use a two-level network without attention).
CASES = {
    "tiny_b1": (R.TINY_CFG, 1, 16, 16),
    "tiny_b3": (R.TINY_CFG, 3, 16, 16),
    "small64_c1": (dict(R.SMALL64_CFG, in_channels=1, out_channels=1), 3, 32, 32),
    "small64_c2": (dict(R.SMALL64_CFG, in_channels=2, out_channels=2), 3, 32, 32),
    "small64_c3": (R.SMALL64_CFG, 3, 32, 32),
    "small64_c1to2": (dict(R.SMALL64_CFG, in_channels=1, out_channels=2), 3, 32, 32),
    "small64_c4": (dict(R.SMALL64_CFG, in_channels=4, out_channels=4), 3, 32, 32),
    "cifar10_b1": (R.CIFAR10_CFG, 1, 32, 32),
    "cifar10_b128": (R.CIFAR10_CFG, 128, 32, 32),
    "hid128_40x40": (_cfg(128), 2, 40, 40),
    "hid128_24x48": (_cfg(128), 2, 24, 48),
    "tail32_12x12": (_cfg(32), 1, 12, 12),
    "tail128_20x12": (_cfg(128), 3, 20, 12),
    "hid96": (_cfg(96), 2, 32, 32),
    "hid256_32x32": (_cfg(256, mult=(1, 1)), 2, 32, 32),
    "hid256_40x40": (_cfg(256, mult=(1, 1)), 2, 40, 40),
    "celebahq": (R.CELEBAHQ_CFG, 1, 256, 256),
}


def pow2(v):
    return v > 0 and v & (v - 1) == 0


def expected_layout(cfg, H, W, training):
    """(in route, in_conv wgrad route, out_conv route, dx route, h0 quad statistics) by the planner's rules as written"""
    c = R.normalize_cfg(cfg)
    hid, cin, cout = c["hid_channels"], c["in_channels"], c["out_channels"]
    geom = pow2(H) and pow2(W)                    # conv_tc_geom: both TMA boxes exist exactly for power-of-two maps
    tc_in = hid % 64 == 0 and geom
    tc_out = tc_in and 9 * cout <= 32
    tc_dx = tc_in and 9 * cin <= 32
    qs = hid % 32 == 0 and (H * W) % 32 == 0
    return (int(tc_in), int(tc_in) if training else -1, int(tc_out), int(tc_dx) if training else -1, int(qs))


@pytest.fixture(scope="module")
def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _handle(L, cfg):
    from ddpm_torch_b200 import _lib
    c = R.normalize_cfg(cfg)
    u = _lib.UnetCfg()
    u.in_channels, u.hid_channels, u.out_channels = c["in_channels"], c["hid_channels"], c["out_channels"]
    u.levels, u.num_res_blocks, u.temb_dim, u.drop_rate = len(c["ch_multipliers"]), c["num_res_blocks"], 0, c["drop_rate"]
    for i, m in enumerate(c["ch_multipliers"]):
        u.ch_mult[i] = m; u.attn[i] = int(c["apply_attn"][i])
    h = C.c_void_p()
    assert L.ddpm_unet_create(C.byref(u), C.byref(h)) == 0, L.ddpm_last_error()
    return h


def layout(L, h):
    """(in route, in_conv wgrad route, out_conv route, dx route, h0 quad statistics) of a planned or dry-planned handle"""
    v = [C.c_int(-7) for _ in range(5)]
    assert L.ddpm_unet_image_layout(h, *[C.byref(x) for x in v]) == 0, L.ddpm_last_error()
    return tuple(x.value for x in v)


def dry_layout(L, cfg, B, H, W, training):
    h = _handle(L, cfg)
    try:
        assert L.ddpm_unet_workspace_bytes(h, B, H, W, training) > 0, L.ddpm_last_error()
        return layout(L, h)
    finally:
        L.ddpm_unet_destroy(h)


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("training", [0, 1])
def test_layout_follows_the_planner_rules(L, name, training):
    cfg, B, H, W = CASES[name]
    assert dry_layout(L, cfg, B, H, W, training) == expected_layout(cfg, H, W, training)


def test_cases_reach_every_route_both_ways(L):
    seen = [set() for _ in range(5)]
    for cfg, B, H, W in CASES.values():
        for i, r in enumerate(dry_layout(L, cfg, B, H, W, 1)):
            seen[i].add(r)
    assert all(s == {0, 1} for s in seen), seen
    # the CUDA-core out_conv at 4 output channels and the 256-channel limit of k_out_conv / k_corr3x3 are among them
    assert dry_layout(L, *CASES["small64_c4"][:2], 32, 32, 1) == (1, 1, 0, 0, 1)
    assert dry_layout(L, *CASES["hid256_40x40"][:2], 40, 40, 1)[:4] == (0, 0, 0, 0)


@pytest.mark.parametrize("hid", [32, 64, 96, 128])
@pytest.mark.parametrize("HW", [(4, 4), (8, 8), (16, 48), (48, 16), (12, 12), (64, 64), (128, 32)])
def test_layout_on_more_geometries(L, hid, HW):
    for cin, cout in ((1, 1), (3, 3), (4, 4), (4, 3), (3, 4)):
        cfg = _cfg(hid, cin, cout, mult=(1,))
        for training in (0, 1):
            assert dry_layout(L, cfg, 2, *HW, training) == expected_layout(cfg, *HW, training), (cin, cout, training)


def test_entry_points_exported(L):
    from ddpm_torch_b200 import _lib
    for n in ("ddpm_unet_image_layout", "ddpm_unet_image_forward", "ddpm_unet_image_backward"):
        assert n in _lib.EXPORTS and hasattr(L, n)


def test_probes_validate_arguments(L):
    F_ = FAKE
    assert L.ddpm_unet_image_layout(None, None, None, None, None, None) != 0
    assert b"null handle" in L.ddpm_last_error()
    assert L.ddpm_unet_image_forward(None, F_, None, None, None, None, F_, None, None, None, F_, None) != 0
    assert b"null handle" in L.ddpm_last_error()
    assert L.ddpm_unet_image_backward(None, F_, F_, None, None, None) != 0
    assert b"null handle" in L.ddpm_last_error()
    h = _handle(L, R.TINY_CFG)
    try:
        assert L.ddpm_unet_image_layout(h, None, None, None, None, None) != 0
        assert b"no plan" in L.ddpm_last_error()
        fwd = lambda *a: L.ddpm_unet_image_forward(h, *a, None)
        assert fwd(None, None, None, None, None, F_, None, None, None, F_) != 0
        assert b"are required" in L.ddpm_last_error()
        assert fwd(F_, None, None, None, None, None, None, None, None, F_) != 0
        assert b"are required" in L.ddpm_last_error()
        assert fwd(F_, None, None, None, None, F_, None, None, None, None) != 0
        assert b"are required" in L.ddpm_last_error()
        # noise without t or either table
        for t, ta, ts in ((None, F_, F_), (F_, None, F_), (F_, F_, None)):
            assert fwd(F_, t, F_, ta, ts, F_, None, None, None, F_) != 0
            assert b"noise needs t, tab_a and tab_s" in L.ddpm_last_error()
        assert fwd(F_, None, None, None, None, F_, F_, None, None, F_) != 0
        assert b"xt_out needs noise" in L.ddpm_last_error()
        assert L.ddpm_unet_image_backward(h, None, F_, None, None, None) != 0
        assert b"are required" in L.ddpm_last_error()
        assert L.ddpm_unet_image_backward(h, F_, None, None, None, None) != 0
        assert b"are required" in L.ddpm_last_error()
        # a dry plan gives a layout but no device buffers: both probes refuse it
        assert L.ddpm_unet_workspace_bytes(h, 3, 16, 16, 1) > 0
        assert layout(L, h) == (0, 0, 0, 0, 1)
        assert fwd(F_, None, None, None, None, F_, None, None, None, F_) != 0
        assert b"has not been called" in L.ddpm_last_error()
        assert L.ddpm_unet_image_backward(h, F_, F_, None, None, None) != 0
        assert b"has not been called" in L.ddpm_last_error()
    finally:
        L.ddpm_unet_destroy(h)


def test_no_gpu_means_the_probes_refuse(L):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = _handle(L, R.TINY_CFG)
    try:
        assert L.ddpm_unet_plan(h, 3, 16, 16, 1, FAKE, FAKE, FAKE, 1 << 30) != 0
        assert L.ddpm_unet_image_forward(h, FAKE, None, None, None, None, FAKE, None, None, None, FAKE, None) != 0
        assert L.ddpm_unet_image_backward(h, FAKE, FAKE, None, None, None) != 0
    finally:
        L.ddpm_unet_destroy(h)


# the default plans' launch counts (the probes add no op to any plan): CIFAR-10 bs = 128 training is 146 / 378 / 5
@pytest.mark.parametrize("name,B,HW,want", [("cifar10", 128, 32, (146, 378, 5)), ("tiny", 3, 16, (78, 158, 1)),
                                            ("small64", 3, 32, (76, 168, 4))])
def test_default_plans_launch_counts_unchanged(L, name, B, HW, want):
    cfg = {"cifar10": R.CIFAR10_CFG, "tiny": R.TINY_CFG, "small64": R.SMALL64_CFG}[name]
    h = _handle(L, cfg)
    try:
        assert L.ddpm_unet_workspace_bytes(h, B, HW, HW, 1) > 0, L.ddpm_last_error()
        f, b, p = C.c_int(), C.c_int(), C.c_int()
        L.ddpm_unet_launch_counts(h, C.byref(f), C.byref(b), C.byref(p))
        got = (f.value, b.value, p.value)
        layout(L, h)                               # reading the layout changes nothing
        L.ddpm_unet_launch_counts(h, C.byref(f), C.byref(b), C.byref(p))
        assert (f.value, b.value, p.value) == got == want
    finally:
        L.ddpm_unet_destroy(h)
