"""CPU-only checks of the timestep-path probes (ddpm_unet_temb_layout / _forward / _backward) and of the planner's timestep
route: which batch sizes put the per-block projections on the tensor cores, the layout of TP [B][tp_ld] (every ResBlock's `fc`
exactly once, in the order the forward runs the ResBlocks (the reference's parameter order, except that the up path
runs its levels from the deepest one), at column offset i * maxc with cout = the fc.weight rows), the exports, and
argument errors reported before any device work."""
import ctypes as C

import pytest
import torch

from oracle import ddpm_ref as R

FAKE = 1 << 20          # a 16-byte aligned non-null address: every call below fails on the host before it could be used


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
    """(route, has_uniform, E, tp_ld, maxc, [(block, off, cout)]) of a planned or dry-planned handle."""
    r, u, E, ld, mc = C.c_int(), C.c_int(), C.c_int(), C.c_int(), C.c_int()
    n = L.ddpm_unet_temb_layout(h, 0, C.byref(r), C.byref(u), C.byref(E), C.byref(ld), C.byref(mc), None, None, None)
    assert n > 0, L.ddpm_last_error()
    off, cout, blk = (C.c_int * n)(), (C.c_int * n)(), (C.c_char_p * n)()
    assert L.ddpm_unet_temb_layout(h, n, None, None, None, None, None, off, cout, blk) == n
    return r.value, u.value, E.value, ld.value, mc.value, [(blk[i].decode(), off[i], cout[i]) for i in range(n)]


def dry_layout(L, cfg, B, HW, training):
    h = _handle(L, cfg)
    try:
        assert L.ddpm_unet_workspace_bytes(h, B, HW, HW, training) > 0, L.ddpm_last_error()
        return layout(L, h)
    finally:
        L.ddpm_unet_destroy(h)


# config -> (blocks, maxc, E, tp_ld)
SHAPES = {"tiny": (R.TINY_CFG, 16, 8, 64, 128, 512), "cifar10": (R.CIFAR10_CFG, 32, 22, 256, 512, 5632),
          "celebahq": (R.CELEBAHQ_CFG, 256, 32, 512, 512, 16384)}
TC_B = (64, 128, 256)
SIMT_B = (1, 3, 4, 63, 96, 127)


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("training", [0, 1])
def test_route_follows_batch_size(L, name, training):
    cfg, HW = SHAPES[name][:2]
    for B in TC_B + SIMT_B:
        route, has_uni = dry_layout(L, cfg, B, HW, training)[:2]
        assert route == (1 if B in TC_B else 0), (name, B)
        assert has_uni == 1, (name, B)          # tp_ld is a multiple of 4: the one-row route and broadcast exist at every B


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_layout_covers_every_fc_once_in_reference_order(L, name):
    cfg, HW, nblocks, maxc, E, tp_ld = SHAPES[name]
    _, _, e, ld, mc, blocks = dry_layout(L, cfg, 4, HW, 1)
    assert (len(blocks), mc, e, ld) == (nblocks, maxc, E, tp_ld)
    shapes = R.param_shapes(cfg)
    fcs = [k[:-len(".fc.weight")] for k in shapes if k.endswith(".fc.weight")]
    names = [b for b, _, _ in blocks]
    assert sorted(names) == sorted(fcs) and len(set(names)) == len(names)
    # the forward's order: the reference's parameter order, except that the up path runs its levels from the deepest one
    up = [b for b in fcs if b.startswith("upsamples.")]
    up.sort(key=lambda b: -int(b.split(".")[1][len("level_"):]))
    assert names == [b for b in fcs if not b.startswith("upsamples.")] + up
    for i, (b, off, cout) in enumerate(blocks):
        assert off == i * maxc
        assert shapes[b + ".fc.weight"] == (cout, E) and cout <= maxc
    assert max(c for _, _, c in blocks) == maxc


def test_layout_counts_blocks_even_with_short_arrays(L):
    h = _handle(L, R.CIFAR10_CFG)
    try:
        assert L.ddpm_unet_workspace_bytes(h, 3, 32, 32, 0) > 0
        off = (C.c_int * 2)(-1, -1)
        assert L.ddpm_unet_temb_layout(h, 1, None, None, None, None, None, off, None, None) == 22
        assert list(off) == [0, -1]              # max_n bounds the writes
    finally:
        L.ddpm_unet_destroy(h)


def test_entry_points_exported(L):
    from ddpm_torch_b200 import _lib
    for n in ("ddpm_unet_temb_layout", "ddpm_unet_temb_forward", "ddpm_unet_temb_backward"):
        assert n in _lib.EXPORTS and hasattr(L, n)


def test_probes_validate_arguments(L):
    assert L.ddpm_unet_temb_layout(None, 0, None, None, None, None, None, None, None, None) != 0
    assert b"null handle" in L.ddpm_last_error()
    assert L.ddpm_unet_temb_forward(None, FAKE, 0, None, None, None, None, None) != 0
    assert L.ddpm_unet_temb_backward(None, FAKE, None, None, None) != 0
    h = _handle(L, R.TINY_CFG)
    try:
        assert L.ddpm_unet_temb_layout(h, 0, None, None, None, None, None, None, None, None) != 0
        assert b"no plan" in L.ddpm_last_error()
        assert L.ddpm_unet_temb_forward(h, None, 0, None, None, None, None, None) != 0
        assert b"null t" in L.ddpm_last_error()
        assert L.ddpm_unet_temb_forward(h, FAKE, 2, None, None, None, None, None) != 0
        assert b"uniform must be 0 or 1" in L.ddpm_last_error()
        assert L.ddpm_unet_temb_backward(h, None, None, None, None) != 0
        assert b"null dTP" in L.ddpm_last_error()
        # a dry plan gives a layout but no device buffers: both probes refuse it
        assert L.ddpm_unet_workspace_bytes(h, 3, 16, 16, 1) > 0
        assert L.ddpm_unet_temb_layout(h, 0, None, None, None, None, None, None, None, None) == 8
        assert L.ddpm_unet_temb_forward(h, FAKE, 0, None, None, None, None, None) != 0
        assert b"has not been called" in L.ddpm_last_error()
        assert L.ddpm_unet_temb_backward(h, FAKE, None, None, None) != 0
        assert b"has not been called" in L.ddpm_last_error()
    finally:
        L.ddpm_unet_destroy(h)


def test_no_gpu_means_the_probes_refuse(L):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = _handle(L, R.TINY_CFG)
    try:
        assert L.ddpm_unet_plan(h, 3, 16, 16, 1, FAKE, FAKE, FAKE, 1 << 30) != 0
        assert L.ddpm_unet_temb_forward(h, FAKE, 0, None, None, None, None, None) != 0
        assert L.ddpm_unet_temb_backward(h, FAKE, None, None, None) != 0
    finally:
        L.ddpm_unet_destroy(h)
