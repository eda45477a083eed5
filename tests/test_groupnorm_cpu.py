"""CPU-only checks of the GroupNorm / column-sum operators of the C ABI and of the GroupNorm channel limit of the planner:
every argument error is reported before any device work, and a plan whose GroupNorm concat exceeds 2048 channels is refused
at plan time with the layer's name."""
import ctypes as C

import pytest

from oracle import ddpm_ref as R

FAKE = 1 << 20          # a 16-byte aligned non-null address: every call below fails on the host before it could be used


@pytest.fixture(scope="module")
def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _fwd(**kw):
    from ddpm_torch_b200 import _lib
    d = _lib.GnDesc()
    d.route, d.B, d.HW, d.C0, d.C1 = 1, 2, 256, 64, 0
    d.x0 = d.gamma = d.beta = d.y = d.K = d.scratch = FAKE
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _bwd(**kw):
    from ddpm_torch_b200 import _lib
    d = _lib.GnBwdDesc()
    d.B, d.HW, d.C0, d.C1 = 2, 256, 64, 0
    d.x0 = d.dy = d.K = d.gamma = d.dgamma = d.dbeta = d.dx0 = d.scratch = FAKE
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("kw,msg", [
    (dict(C0=60), b"multiples of 8"),
    (dict(C0=64, C1=4, x1=FAKE), b"multiples of 8"),
    (dict(C0=40, C1=8, x1=FAKE), b"multiple of 32"),
    (dict(C0=1536, C1=1024, x1=FAKE), b"2048"),
    (dict(C0=64, C1=64), b"null source"),
    (dict(x0=FAKE + 8), b"aligned"),
    (dict(route=0), b"route"),
    (dict(route=5), b"route"),
    (dict(route=2, HW=65), b"HW <= 64"),
    (dict(route=3, C0=64), b"128"),
    (dict(route=4, C0=96, C1=64, x1=FAKE), b"128"),
    (dict(route=3, C0=128), b"quad statistics"),
    (dict(route=4, C0=128, C1=128, x1=FAKE, qs0=FAKE), b"quad statistics"),
    (dict(route=1, scratch=None), b"null buffer"),
    (dict(route=2, HW=16, y=None), b"null buffer"),
    (dict(K=None), b"null buffer"),
    (dict(drop_p=1.0), b"drop_p"),
    (dict(B=0), b"B >= 1"),
])
def test_groupnorm_fwd_validates_arguments(L, kw, msg):
    d = _fwd(**kw)
    assert L.ddpm_groupnorm_fwd_run(C.byref(d), None) != 0
    assert msg in L.ddpm_last_error(), L.ddpm_last_error()


@pytest.mark.parametrize("kw,msg", [
    (dict(C0=36, C1=28, x1=FAKE, dx1=FAKE), b"multiples of 8"),
    (dict(C0=2048, C1=32, x1=FAKE, dx1=FAKE), b"2048"),
    (dict(C0=64, C1=64, x1=FAKE), b"null buffer"),          # second source without its destination
    (dict(scratch=None), b"null buffer"),
    (dict(drop_p=0.1), b"mask"),                            # dropout backward without the forward's keep bits
    (dict(cs_per_img=FAKE, cs_ld=32), b"cs_ld"),
    (dict(addend=FAKE + 4), b"aligned"),
])
def test_groupnorm_bwd_validates_arguments(L, kw, msg):
    d = _bwd(**kw)
    assert L.ddpm_groupnorm_bwd_run(C.byref(d), None) != 0
    assert msg in L.ddpm_last_error(), L.ddpm_last_error()


def test_colsum_validates_arguments(L):
    cases = [((None, None, 0, FAKE, None, 1, 64, 128, 128), b"null dy"),
             ((FAKE, None, 0, FAKE, None, 1, 64, 124, 124), b"multiple of 8"),
             ((FAKE, None, 0, FAKE, None, 1, 64, 128, 129), b"C_valid"),
             ((FAKE, FAKE, 64, FAKE, None, 1, 64, 128, 128), b"ld"),
             ((FAKE, None, 0, FAKE, None, 0, 64, 128, 128), b"B >= 1")]
    for args, msg in cases:
        assert L.ddpm_colsum_run(*args, None) != 0
        assert msg in L.ddpm_last_error(), (args, L.ddpm_last_error())


def test_scratch_bytes_cover_both_directions(L):
    for B, Ch in ((1, 32), (3, 384), (128, 2048)):
        n = L.ddpm_gn_scratch_bytes(B, Ch)
        assert n >= B * 64 * 8 + B * 4 and n >= 2 * (B * 2 * Ch * 4) + B * 4
    assert L.ddpm_gn_scratch_bytes(0, 32) < 0


WIDE_ATTN_CFG = dict(in_channels=3, hid_channels=256, out_channels=3, ch_multipliers=(1, 2, 4), num_res_blocks=2,
                     apply_attn=(False, False, True), drop_rate=0.1)


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


def test_wide_attention_plan_is_accepted(L):
    """hid 256, ch_mult (1, 2, 4), attention at the 1024-channel level: project_in's bias gradient sums 3 * 1024 columns, wider
    than one block of the column-sum kernel; the widest GroupNorm concat is 1024 + 1024."""
    h = _handle(L, WIDE_ATTN_CFG)
    for training in (1, 0):
        assert L.ddpm_unet_workspace_bytes(h, 2, 32, 32, training) > 0, L.ddpm_last_error()
    L.ddpm_unet_destroy(h)


@pytest.mark.parametrize("mults,layer", [((1, 2, 4, 8), b"upsamples.level_3.0.norm1"),
                                         ((1, 2, 8), b"upsamples.level_2.0.norm1")])
def test_groupnorm_wider_than_2048_channels_is_refused_at_plan_time(L, mults, layer):
    cfg = dict(WIDE_ATTN_CFG, ch_multipliers=mults, apply_attn=(False,) * len(mults))
    h = _handle(L, cfg)
    for training in (1, 0):
        assert L.ddpm_unet_workspace_bytes(h, 2, 32, 32, training) < 0
        err = L.ddpm_last_error()
        assert layer in err and b"4096 channels" in err and b"2048" in err, err
    L.ddpm_unet_destroy(h)
