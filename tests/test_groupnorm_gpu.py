"""GroupNorm(32, C, eps=1e-6) [+ SiLU] [+ dropout] and the bias column sums, kernel by kernel, against fp64 torch on the same bf16
inputs, through the C ABI operators that launch exactly what the engine's plans launch (same kernels, same grids).

Every route the planner takes is run on every shape that it accepts, so the routes are also compared with each other:
  1  k_gn_stats + k_gn_apply        2  k_gn_small (HW <= 64)
  3  k_gn_apply from quad statistics (C % 128 == 0)        4  k_gn_prep (K only, C % 128 == 0)
Shapes are the norm sites of the tiny / small64 / CIFAR-10 / CelebA-HQ configs, the CIFAR net at 40 x 40 (HW 1600/400/100/25),
groups that straddle the two concat sources in both orders, and B = 128 at 32 x 32 (the benchmarked plan).

Outputs are filled with NaN (or a known pattern where the kernel accumulates) before each call, so that an element that was
never written fails.  Each test prints its worst error-to-bound ratio under -s."""
import ctypes as ct

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
U8 = 2.0 ** -8          # one bf16 rounding (8-bit significand, round to nearest)
# sigmoid_fast is 0.5 * tanh.approx.f32(y / 2) + 0.5; the PTX ISA gives tanh.approx a maximum relative error of 2^-10.987,
# so |error of silu(z)| <= |z| * 0.5 * 2^-10.987
SILU_APPROX = 0.5 * 2.0 ** -10.987


def L():
    from ddpm_torch_b200 import _lib
    return _lib.lib()


def _check(rc):
    from ddpm_torch_b200 import _lib
    _lib.check(rc, "groupnorm operator")


def _stream():
    from ddpm_torch_b200 import _lib
    return _lib.stream_ptr()


def _p(t):
    return t.data_ptr() if t is not None else None


def _flag_ok():
    assert L().ddpm_device_error_flag() == 0


# ------------------------------------------------------------------------------------------------ operators
def quad_stats(x):
    """what a producer's statistics epilogue delivers: per (image, 4-channel quad) {sum, sum of squares} in fp64"""
    B, HW, Cs = x.shape
    xd = x.double().view(B, HW, Cs // 4, 4)
    return torch.stack([xd.sum((1, 3)), (xd * xd).sum((1, 3))], -1).contiguous()


def gn_forward(route, x0, x1, gamma, beta, silu=1, drop_p=0.0, seed=0, layer=1):
    from ddpm_torch_b200 import _lib
    B, HW, C0 = x0.shape
    C1 = x1.shape[2] if x1 is not None else 0
    Ch = C0 + C1
    y = torch.full((B, HW, Ch), float("nan"), dtype=torch.bfloat16, device=DEV)
    K = torch.full((B, 4, Ch), float("nan"), device=DEV)
    mask = torch.full((B, HW, Ch // 8), 0x5A, dtype=torch.uint8, device=DEV)
    scratch = torch.zeros(L().ddpm_gn_scratch_bytes(B, Ch), dtype=torch.uint8, device=DEV)
    qs0 = quad_stats(x0) if route >= 3 else None
    qs1 = quad_stats(x1) if route >= 3 and x1 is not None else None
    d = _lib.GnDesc()
    d.route, d.B, d.HW, d.C0, d.C1 = route, B, HW, C0, C1
    d.x0, d.x1, d.gamma, d.beta = _p(x0), _p(x1), _p(gamma), _p(beta)
    d.silu, d.drop_p, d.seed, d.layer, d.mask = silu, drop_p, seed, layer, _p(mask)
    d.qs0, d.qs1, d.y, d.K, d.scratch = _p(qs0), _p(qs1), _p(y), _p(K), _p(scratch)
    _check(L().ddpm_groupnorm_fwd_run(ct.byref(d), _stream()))
    torch.cuda.synchronize()
    return y, K, mask


def gn_backward(x0, x1, dy, K, gamma, dgamma, dbeta, dx0, dx1, *, silu, drop_p=0.0, mask=None, dn_inplace=0, acc0=0, acc1=0,
                addend=None, cs_per_img=None, cs_total=None, cs_total2=None):
    from ddpm_torch_b200 import _lib
    B, HW, C0 = x0.shape
    C1 = x1.shape[2] if x1 is not None else 0
    scratch = torch.zeros(L().ddpm_gn_scratch_bytes(B, C0 + C1), dtype=torch.uint8, device=DEV)
    d = _lib.GnBwdDesc()
    d.B, d.HW, d.C0, d.C1 = B, HW, C0, C1
    d.x0, d.x1, d.dy, d.K, d.gamma, d.dgamma, d.dbeta = _p(x0), _p(x1), _p(dy), _p(K), _p(gamma), _p(dgamma), _p(dbeta)
    d.dx0, d.dx1, d.acc0, d.acc1, d.addend = _p(dx0), _p(dx1), acc0, acc1, _p(addend)
    d.silu, d.drop_p, d.mask, d.dn_inplace = silu, drop_p, _p(mask), dn_inplace
    d.cs_per_img, d.cs_ld = _p(cs_per_img), (cs_per_img.shape[1] if cs_per_img is not None else 0)
    d.cs_total, d.cs_total2, d.scratch = _p(cs_total), _p(cs_total2), _p(scratch)
    _check(L().ddpm_groupnorm_bwd_run(ct.byref(d), _stream()))
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ fp64 reference
def unpack_mask(m, Ch):
    """bit e of byte (b, pixel, octet o) <-> channel 8*o + e"""
    bits = (m.unsqueeze(-1) >> torch.arange(8, device=m.device, dtype=torch.uint8)) & 1
    return bits.reshape(*m.shape[:-1], Ch).double()


def ref_stats(x):
    """per (image, channel) mean and rstd of the channel's group, fp64; x [B, HW, C] fp64"""
    B, HW, Ch = x.shape
    cg = Ch // 32
    xg = x.view(B, HW, 32, cg)
    mean = xg.mean((1, 3))
    var = ((xg - mean[:, None, :, None]) ** 2).mean((1, 3))
    rstd = (var + 1e-6).rsqrt()
    return mean.repeat_interleave(cg, 1), rstd.repeat_interleave(cg, 1)


def ref_forward(x, gamma, beta, silu, keep, ks):
    z = F.group_norm(x.permute(0, 2, 1), 32, gamma, beta, eps=1e-6).permute(0, 2, 1)
    a = F.silu(z) if silu else z
    return z, a * keep * ks


def inputs(B, HW, C0, C1, seed, mu=0.0):
    """x = mu + z (z ~ N(0, 1)) in bf16, gamma ~ 1 + 0.2 N, beta ~ 0.2 N"""
    g = torch.Generator(DEV).manual_seed(seed)
    x0 = (mu + torch.randn(B, HW, C0, device=DEV, generator=g)).to(torch.bfloat16)
    x1 = (mu + torch.randn(B, HW, C1, device=DEV, generator=g)).to(torch.bfloat16) if C1 else None
    Ch = C0 + C1
    gamma = 1 + 0.2 * torch.randn(Ch, device=DEV, generator=g)
    beta = 0.2 * torch.randn(Ch, device=DEV, generator=g)
    return x0, x1, gamma, beta


def cat64(x0, x1):
    return (torch.cat([x0, x1], 2) if x1 is not None else x0).double()


# ------------------------------------------------------------------------------------------------ forward
def check_forward(route, x0, x1, gamma, beta, *, silu=1, drop_p=0.0, seed=0, layer=1, tol_k=1e-5):
    """Runs one route and checks K and y.  Returns (K ratio, y ratio, mask, y, K): worst error-to-bound ratios (<= 1 passes).

    K per (image, channel), each error in units of what it scales: rstd and sc = rstd*gamma relative; mean*rstd in units of
    (|mean*rstd| + 1), i.e. the mean error in units of sigma; sh = beta - mean*sc in units of |beta| + |gamma|(|mean*rstd| + 1).
    y element-wise: |y - ref| <= 2^-8 |ref| (the bf16 rounding) + keep/(1-p) * (1 + 2^-8) * (silu approximation
    SILU_APPROX * |z| + 1.1 * (statistics term + fp32 term)), 1.1 bounding silu'.  The statistics term propagates the kernel's
    own K error, |gamma| (|xhat| |rstd error| / rstd + |mean error| * rstd); the fp32 term is 2^-20 of the magnitudes in
    x * sc + sh.  Where a keep bit is clear the bound is 0: y must be exactly 0."""
    x = cat64(x0, x1)
    B, HW, Ch = x.shape
    y, K, mask = gn_forward(route, x0, x1, gamma, beta, silu=silu, drop_p=drop_p, seed=seed, layer=layer)
    mean, rstd = ref_stats(x)
    g64, b64 = gamma.double()[None], beta.double()[None]
    mr = mean * rstd
    Kd = K.double()
    assert torch.isfinite(Kd).all(), f"route {route}: K not written everywhere"
    e_r = (Kd[:, 2] - rstd) / rstd
    e_sc = (Kd[:, 0] - rstd * g64).abs() / (rstd * g64.abs())
    e_mr = (Kd[:, 3] - mr).abs() / (mr.abs() + 1)
    e_sh = (Kd[:, 1] - (b64 - mr * g64)).abs() / (b64.abs() + g64.abs() * (mr.abs() + 1))
    rk = max(e_r.abs().max().item(), e_sc.max().item(), e_mr.max().item(), e_sh.max().item()) / tol_k
    if route == 4:
        assert torch.isnan(y.float()).all(), "route 4 writes K only"
        return rk, 0.0, None, None, K
    assert torch.isfinite(y.float()).all(), f"route {route}: y not written everywhere"
    keep = unpack_mask(mask, Ch) if drop_p > 0 else torch.ones_like(x)
    ks = 1.0 / (1.0 - drop_p) if drop_p > 0 else 1.0
    z, ref = ref_forward(x, g64[0], b64[0], silu, keep, ks)
    mean_k = Kd[:, 3] / Kd[:, 2]
    xhat = (x - mean[:, None]) * rstd[:, None]
    stat = g64.abs()[:, None] * (xhat.abs() * e_r.abs()[:, None] + ((mean_k - mean) * rstd).abs()[:, None])
    fp32 = 2.0 ** -20 * (x.abs() * (g64.abs() * rstd)[:, None] + b64.abs()[:, None] + (g64.abs() * mr.abs())[:, None] + z.abs())
    dz = (1.1 if silu else 1.0) * (stat + fp32)
    sil = SILU_APPROX * z.abs() if silu else 0.0
    tol = U8 * ref.abs() + keep * ks * (1 + U8) * (sil + dz)
    err = (y.double() - ref).abs()
    assert (err[tol == 0] == 0).all(), f"route {route}: dropped elements are not exactly 0"
    ry = (err / tol.clamp_min(1e-300)).max().item()
    return rk, ry, mask, y, K


FWD_SHAPES = [   # (B, HW, C0, C1)
    (3, 256, 32, 0), (3, 64, 64, 0), (3, 64, 64, 32), (3, 256, 128, 64), (3, 16, 64, 32),                # tiny / small64
    (3, 1024, 128, 0), (3, 256, 256, 0), (3, 64, 256, 0), (3, 16, 256, 0),                                 # CIFAR-10
    (3, 1024, 256, 128), (3, 1024, 128, 256), (3, 256, 256, 256), (3, 16, 256, 128), (3, 16, 256, 256),
    (1, 65536, 128, 0), (2, 64, 512, 256), (2, 256, 512, 256), (2, 256, 512, 512), (2, 64, 512, 512),     # CelebA-HQ
    (2, 16, 1024, 1024),                                                                                   # 256 octets
    (3, 1600, 128, 0), (3, 400, 256, 128), (3, 100, 256, 256), (3, 25, 256, 128), (3, 25, 128, 0),        # 40 x 40
    (128, 1024, 128, 0), (128, 64, 256, 0),                                                                # benchmarked plan
]


def routes_for(HW, Ch):
    return [1] + ([2] if HW <= 64 else []) + ([3, 4] if Ch % 128 == 0 else [])


@pytest.mark.parametrize("silu", [1, 0])
def test_forward_every_route_vs_fp64(silu):
    worst_k, worst_y = (0.0, None), (0.0, None)
    for i, (B, HW, C0, C1) in enumerate(FWD_SHAPES):
        x0, x1, gamma, beta = inputs(B, HW, C0, C1, seed=100 + i)
        ys = {}
        for r in routes_for(HW, C0 + C1):
            rk, ry, _, y, _ = check_forward(r, x0, x1, gamma, beta, silu=silu)
            tag = (B, HW, C0, C1, r)
            assert rk <= 1 and ry <= 1, (tag, rk, ry)
            worst_k = max(worst_k, (rk, tag), key=lambda t: t[0])
            worst_y = max(worst_y, (ry, tag), key=lambda t: t[0])
            if y is not None:
                ys[r] = y.float()
        # the routes differ only in how the statistics are summed: their outputs agree to a few bf16 ulps
        for r, y in ys.items():
            d = ((y - ys[1]).abs() / (ys[1].abs() + 1e-2)).max().item()
            assert d < 4 * U8, ((B, HW, C0, C1), r, d)
    print(f"\n[groupnorm fwd silu={silu}] worst K error / 1e-5: {worst_k[0]:.3f} at {worst_k[1]}; "
          f"worst y error / bound: {worst_y[0]:.3f} at {worst_y[1]}  (B, HW, C0, C1, route)")
    _flag_ok()


@pytest.mark.parametrize("mu", [0.0, 8.0, 32.0])
def test_offset_data_rstd_within_half_a_bf16_ulp(mu):
    """x = mu + sigma * z with mu / sigma in {0, 8, 32}: k_gn_small forms E[x^2] - m^2 in fp32, the other routes reduce fp32 partial
    sums into fp64.  Every route must keep the rstd (and the other K entries, in the units of check_forward) within 2^-9, half a
    bf16 ulp, up to 64 channels per group; y keeps its element-wise bound."""
    worst = (0.0, None)
    for i, (B, HW, C0, C1) in enumerate([(3, 64, 1024, 1024), (3, 16, 1024, 1024), (3, 64, 256, 128), (3, 25, 256, 0),
                                         (3, 1024, 128, 0), (2, 256, 512, 512)]):
        x0, x1, gamma, beta = inputs(B, HW, C0, C1, seed=200 + i, mu=mu)
        for r in routes_for(HW, C0 + C1):
            rk, ry, *_ = check_forward(r, x0, x1, gamma, beta, tol_k=2.0 ** -9)
            tag = (B, HW, C0, C1, r)
            assert rk <= 1 and ry <= 1, (tag, rk, ry)
            worst = max(worst, (rk, tag), key=lambda t: t[0])
    print(f"\n[groupnorm offset mu/sigma={mu:g}] worst K error / 2^-9: {worst[0]:.4f} at {worst[1]}")
    _flag_ok()


@pytest.mark.parametrize("B,HW,C0,C1", [(3, 64, 128, 128), (2, 1024, 256, 128)])
def test_dropout_mask_is_route_independent(B, HW, C0, C1):
    """p = 0.1: y is exactly 0 where a keep bit is clear and ref / (1 - p) elsewhere (check_forward); the kept fraction is within
    5 sigma of 1 - 6553/65536; the same (seed, layer) gives bit-identical masks on every route (the Philox counter is the element
    index, not the launch geometry); masks differ between images and between layers."""
    p, seed, layer = 0.1, 0x1234_5678_9ABC, 7
    x0, x1, gamma, beta = inputs(B, HW, C0, C1, seed=300)
    masks, worst = {}, 0.0
    for r in [1, 2, 3]:
        if r == 2 and HW > 64:
            continue
        rk, ry, m, y, _ = check_forward(r, x0, x1, gamma, beta, drop_p=p, seed=seed, layer=layer)
        assert rk <= 1 and ry <= 1, (r, rk, ry)
        worst = max(worst, ry)
        masks[r] = m
    for r, m in masks.items():
        assert torch.equal(m, masks[1]), f"route {r} drew a different mask"
    keep = unpack_mask(masks[1], C0 + C1)
    n = keep.numel()
    q = 1 - 6553 / 65536
    frac = keep.mean().item()
    assert abs(frac - q) < 5 * (q * (1 - q) / n) ** 0.5, (frac, q)
    # two independent masks differ in ~79 % of their bytes (a byte is all-kept with probability 0.9^8)
    assert (masks[1][0] != masks[1][1]).float().mean().item() > 0.5, "images share a dropout mask"
    _, _, m2 = gn_forward(1, x0, x1, gamma, beta, drop_p=p, seed=seed, layer=layer + 1)
    assert (m2 != masks[1]).float().mean().item() > 0.5, "layers share a dropout mask"
    _, _, m3 = gn_forward(1, x0, x1, gamma, beta, drop_p=p, seed=seed + 1, layer=layer)
    assert (m3 != masks[1]).float().mean().item() > 0.5, "seeds share a dropout mask"
    print(f"\n[groupnorm dropout {B}x{HW}x({C0}+{C1})] kept {frac:.5f} (expected {q:.5f}); worst y error / bound {worst:.3f}")
    _flag_ok()


# ------------------------------------------------------------------------------------------------ backward
BWD_SHAPES = [(3, 1024, 256, 128), (3, 1024, 128, 256), (1, 65536, 128, 0), (128, 1024, 128, 0), (3, 16, 1024, 1024),
              (3, 25, 64, 32), (2, 400, 256, 0), (3, 64, 256, 256)]
# silu, dropout p, dn_inplace, (acc0, acc1), addend, column sums
VARIANTS = {
    "exact": (0, 0.0, 0, (0, 0), False, True),
    "silu_drop_inplace_acc0_addend": (1, 0.1, 1, (1, 0), True, True),
    "silu_acc1": (1, 0.0, 0, (0, 1), False, False),
    "plain_inplace_acc_both": (0, 0.0, 1, (1, 1), True, True),
}
# Sums (dgamma, dbeta, the column sums) against fp64, in units of the L1 norm of their summands.  With silu and dropout off the
# kernels' arithmetic is exactly specified (bf16 inputs, fp32 sums): 1e-5.  With silu on, each summand also carries dn's
# bf16 rounding when dn is written back in place (<= 2^-9 of |sc * dn|) and the approximate sigmoid in silu'(y) (<= 2^-11 of
# |dn| for the |y| of normalised data), so 2^-9 + 2^-11 of L1 bounds the sum even if every summand errs the same way.
SUM_TOL = {0: 1e-5, 1: 2.0 ** -9 + 2.0 ** -11}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_backward_vs_fp64_autograd(variant):
    """dx per (image, group) rel-L2 <= 5e-3 (a single wrong group cannot hide in a global norm); dgamma, dbeta (accumulated onto
    a known pattern) and the three column sums of dx (per image with a padded row, total, total2) against fp64 autograd of
    the same forward with the kernel's own dropout mask."""
    silu, p, inplace, (acc0, acc1), use_addend, use_cs = VARIANTS[variant]
    worst = {"dx": (0.0, None), "sums": (0.0, None), "dn": (0.0, None)}
    for i, (B, HW, C0, C1) in enumerate(BWD_SHAPES):
        Ch = C0 + C1
        x0, x1, gamma, beta = inputs(B, HW, C0, C1, seed=400 + i)
        seed = 99 if p > 0 else 0
        _, K, mask = gn_forward(1, x0, x1, gamma, beta, silu=silu, drop_p=p, seed=seed, layer=3)
        keep = unpack_mask(mask, Ch) if p > 0 else torch.ones(B, HW, Ch, dtype=torch.float64, device=DEV)
        ks = 1.0 / (1.0 - p) if p > 0 else 1.0
        g = torch.Generator(DEV).manual_seed(500 + i)
        dy = torch.randn(B, HW, Ch, device=DEV, generator=g).to(torch.bfloat16)
        prev0 = torch.randn(B, HW, C0, device=DEV, generator=g).to(torch.bfloat16)
        prev1 = torch.randn(B, HW, C1, device=DEV, generator=g).to(torch.bfloat16) if C1 else None
        addend = torch.randn(B, HW, Ch, device=DEV, generator=g).to(torch.bfloat16) if use_addend else None
        pat_g, pat_b = torch.randn(Ch, device=DEV, generator=g), torch.randn(Ch, device=DEV, generator=g)
        # fp64 reference
        x = cat64(x0, x1).requires_grad_(True)
        g64 = gamma.double().requires_grad_(True)
        b64 = beta.double().requires_grad_(True)
        z, out = ref_forward(x, g64, b64, silu, keep, ks)
        (out * dy.double()).sum().backward()
        with torch.no_grad():
            z = z.detach()
            sg = torch.sigmoid(z)
            dn = dy.double() * keep * ks * (sg * (1 + z * (1 - sg)) if silu else 1.0)
            mean, rstd = ref_stats(x.detach())
            xhat = (x.detach() - mean[:, None]) * rstd[:, None]
            sc_dn = dn * (rstd * gamma.double()[None])[:, None]
            dx_ref = x.grad
            extra = torch.zeros_like(dx_ref)
            if acc0:
                extra[..., :C0] += prev0.double()
            if acc1 and C1:
                extra[..., C0:] += prev1.double()
            if use_addend:
                extra += addend.double()
            want = dx_ref + extra
            l1_cs = (sc_dn.abs() + (dx_ref - sc_dn).abs() + extra.abs()).sum(1)          # [B, C]
        # kernel
        dx0 = prev0.clone() if acc0 else torch.full((B, HW, C0), float("nan"), dtype=torch.bfloat16, device=DEV)
        dx1 = None
        if C1:
            dx1 = prev1.clone() if acc1 else torch.full((B, HW, C1), float("nan"), dtype=torch.bfloat16, device=DEV)
        dgamma, dbeta = pat_g.clone(), pat_b.clone()
        cs_img = torch.full((B, Ch + 32), 3.0, device=DEV) if use_cs else None
        cs_tot = pat_g.clone() if use_cs else None
        cs_tot2 = pat_b.clone() if use_cs else None
        dyk = dy.clone()
        gn_backward(x0, x1, dyk, K, gamma, dgamma, dbeta, dx0, dx1, silu=silu, drop_p=p, mask=mask if p > 0 else None,
                    dn_inplace=inplace, acc0=acc0, acc1=acc1, addend=addend, cs_per_img=cs_img, cs_total=cs_tot, cs_total2=cs_tot2)
        tag = (B, HW, C0, C1)
        got = cat64(dx0, dx1)
        assert torch.isfinite(got).all(), (tag, "dx not written everywhere")
        cg = Ch // 32
        num = (got - want).view(B, HW, 32, cg).pow(2).sum((1, 3)).sqrt()
        den = want.view(B, HW, 32, cg).pow(2).sum((1, 3)).sqrt()
        rdx = (num / den).max().item() / 5e-3
        tol = SUM_TOL[silu]
        rs = [((dbeta.double() - pat_b.double() - b64.grad).abs() / (tol * dn.abs().sum((0, 1)))).max().item(),
              ((dgamma.double() - pat_g.double() - g64.grad).abs() / (tol * (dn * xhat).abs().sum((0, 1)))).max().item()]
        if use_cs:
            cs_want = want.sum(1)
            rs.append(((cs_img[:, :Ch].double() - 3.0 - cs_want).abs() / (tol * l1_cs)).max().item())
            assert (cs_img[:, Ch:] == 3.0).all(), (tag, "column sums written past C")
            for t, pat in ((cs_tot, pat_g), (cs_tot2, pat_b)):
                rs.append(((t.double() - pat.double() - cs_want.sum(0)).abs() / (tol * l1_cs.sum(0))).max().item())
        if inplace:   # dy now holds bf16(dn): one bf16 rounding + silu' approximation; exact zeros where dropped
            dnk = dyk.double()
            assert (dnk[keep == 0] == 0).all(), tag
            rdn = ((dnk - dn).norm() / dn.norm()).item() / 5e-3
        else:
            assert torch.equal(dyk, dy), (tag, "dy modified without dn_inplace")
            rdn = 0.0
        rsum = max(rs)
        assert rdx <= 1 and rsum <= 1 and rdn <= 1, (tag, rdx, rs, rdn)
        for k, v in (("dx", rdx), ("sums", rsum), ("dn", rdn)):
            worst[k] = max(worst[k], (v, tag), key=lambda t: t[0])
    print(f"\n[groupnorm bwd {variant}] worst dx per-group rel-L2 / 5e-3: {worst['dx'][0]:.3f} at {worst['dx'][1]}; "
          f"worst sum error / ({SUM_TOL[silu]:.3g} L1): {worst['sums'][0]:.3f} at {worst['sums'][1]}"
          + (f"; in-place dn rel-L2 / 5e-3: {worst['dn'][0]:.3f}" if inplace else ""))
    _flag_ok()


# ------------------------------------------------------------------------------------------------ column sums
def test_colsum_vs_fp64():
    """k_colsum (bias gradients): per-image and total column sums at C up to 3 * 1024 (attention project_in at the 1024-channel
    level, wider than one block's 2048 channels), against fp64 at 1e-5 of the L1 norm of the summands; columns at or past
    C_valid stay untouched."""
    worst = (0.0, None)
    for i, (B, HW, Ch, Cv) in enumerate([(3, 1024, 128, 128), (128, 1024, 128, 128), (3, 256, 256, 256), (2, 1024, 768, 768),
                                         (3, 100, 1536, 1536), (2, 64, 3072, 3072), (3, 16, 3072, 3000), (1, 65536, 128, 120)]):
        g = torch.Generator(DEV).manual_seed(600 + i)
        dy = torch.randn(B, HW, Ch, device=DEV, generator=g).to(torch.bfloat16)
        ld = Ch + 16
        per = torch.full((B, ld), 5.0, device=DEV)
        tot = torch.randn(Ch, device=DEV, generator=g)
        tot2 = torch.randn(Ch, device=DEV, generator=g)
        t0, t20 = tot.clone(), tot2.clone()
        _check(L().ddpm_colsum_run(dy.data_ptr(), per.data_ptr(), ld, tot.data_ptr(), tot2.data_ptr(), B, HW, Ch, Cv, _stream()))
        torch.cuda.synchronize()
        ref = dy.double().sum(1)
        l1 = dy.double().abs().sum(1)
        r = [((per[:, :Cv].double() - 5.0 - ref[:, :Cv]).abs() / (1e-5 * l1[:, :Cv])).max().item(),
             ((tot[:Cv].double() - t0[:Cv].double() - ref[:, :Cv].sum(0)).abs() / (1e-5 * l1[:, :Cv].sum(0))).max().item(),
             ((tot2[:Cv].double() - t20[:Cv].double() - ref[:, :Cv].sum(0)).abs() / (1e-5 * l1[:, :Cv].sum(0))).max().item()]
        tag = (B, HW, Ch, Cv)
        assert max(r) <= 1, (tag, r)
        assert (per[:, Cv:] == 5.0).all() and torch.equal(tot[Cv:], t0[Cv:]) and torch.equal(tot2[Cv:], t20[Cv:]), (tag, "wrote past C_valid")
        worst = max(worst, (max(r), tag), key=lambda t: t[0])
    print(f"\n[colsum] worst error / (1e-5 L1): {worst[0]:.3f} at {worst[1]}  (B, HW, C, C_valid)")
    _flag_ok()
