"""Oracle of the ``resample_with_conv=False`` UNet — test infrastructure, not product code.

The reference's constructor option (unet.py:106,164-170,199-202) replaces the resample convs by ``nn.AvgPool2d(2)`` on the
way down and a bare ``nn.Upsample(scale_factor=2, mode="nearest")`` on the way up, and drops their parameters from the
``state_dict``.  This module restates that variant on top of the pieces of ``oracle/ddpm_ref.py`` (whose conv-resample
restatement every other test relies on and which is used unchanged here), in plain fp32 PyTorch so that it runs where the
reference does not exist.  ``tests/test_noresample_cpu.py`` pins it against the unmodified reference
(``tests/golden/unet_noresample.pt``, written by ``tools/gen_golden_noresample.py``).
"""
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle import ddpm_ref as R


def normalize_cfg(cfg: dict) -> dict:
    """R.normalize_cfg, with ``resample_with_conv`` forced to False."""
    c = R.normalize_cfg(dict(cfg, resample_with_conv=True))
    c["resample_with_conv"] = False
    return c


def _conv_cfg(cfg: dict) -> dict:
    c = dict(cfg)
    c.pop("resample_with_conv", None)
    return c


def resample_keys(cfg: dict) -> List[str]:
    """state_dict keys of the resample convs, which the variant does not have."""
    c = normalize_cfg(cfg)
    L, nrb = len(c["ch_multipliers"]), c["num_res_blocks"]
    keys = []
    for i in range(L - 1):
        keys += [f"downsamples.level_{i}.{nrb}.1.weight", f"downsamples.level_{i}.{nrb}.1.bias"]
    for i in range(1, L):
        keys += [f"upsamples.level_{i}.{nrb + 1}.1.weight", f"upsamples.level_{i}.{nrb + 1}.1.bias"]
    return keys


def param_shapes(cfg: dict) -> "Dict[str, tuple]":
    """Ordered {state_dict key: shape} of the reference's UNet(..., resample_with_conv=False)."""
    drop = set(resample_keys(cfg))
    return {k: v for k, v in R.param_shapes(_conv_cfg(cfg)).items() if k not in drop}


def make_state_dict(cfg: dict, seed: int, scale: float = 1.0) -> "Dict[str, torch.Tensor]":
    """R.fill_params over this variant's inventory (the weights tools/gen_golden_noresample.py loads into the reference)."""
    return R.fill_params(param_shapes(cfg), seed, scale)


def unet_forward(sd, cfg, x, t, keep_masks: Optional[List[torch.Tensor]] = None):
    """unet.py:205-233 with AvgPool2d(2) down (unet.py:168-169) and nearest x2 alone up (unet.py:199-202)."""
    c = normalize_cfg(cfg)
    ch, mult, nrb = c["hid_channels"], c["ch_multipliers"], c["num_res_blocks"]
    L, aa, dr = len(mult), c["apply_attn"], c["drop_rate"]
    masks = list(keep_masks) if keep_masks is not None else None
    temb = R.timestep_embedding(t, ch)
    temb = F.linear(temb, sd["embed.0.weight"], sd["embed.0.bias"])
    temb = F.linear(F.silu(temb), sd["embed.2.weight"], sd["embed.2.bias"])
    hs = [R._conv(sd, "in_conv", x, padding=1)]
    for i in range(L):
        p = f"downsamples.level_{i}"
        for j in range(nrb):
            hs.append(R._block(sd, f"{p}.{j}", hs[-1], temb, aa[i], masks, dr))
        if i != L - 1:
            hs.append(F.avg_pool2d(hs[-1], 2))
    h = hs[-1]
    h = R.res_block(sd, "middle.0", h, temb, masks.pop(0) if masks is not None else None, dr)
    h = R.attn_block(sd, "middle.1", h)
    h = R.res_block(sd, "middle.2", h, temb, masks.pop(0) if masks is not None else None, dr)
    for i in range(L - 1, -1, -1):
        p = f"upsamples.level_{i}"
        for j in range(nrb + 1):
            h = R._block(sd, f"{p}.{j}", torch.cat([h, hs.pop()], dim=1), temb, aa[i], masks, dr)
        if i != 0:
            h = F.interpolate(h, scale_factor=2, mode="nearest")
    h = F.silu(R._gn(sd, "out_conv.0", h))
    return R._conv(sd, "out_conv.2", h, padding=1)


def fwd_flops_per_image(cfg, H, W) -> float:
    """R.fwd_flops_per_image less the resample convs: a 3x3 C -> C conv at 1/2^(i+1) resolution per down level i < L-1 and
    at 1/2^(i-1) resolution per up level i > 0 (pooling and upsampling count no FLOPs)."""
    c = normalize_cfg(cfg)
    chs = [c["hid_channels"] * m for m in c["ch_multipliers"]]
    L = len(chs)
    fl = R.fwd_flops_per_image(_conv_cfg(cfg), H, W)
    for i in range(L - 1):
        fl -= 2.0 * chs[i] * chs[i] * 9 * (H >> (i + 1)) * (W >> (i + 1))
    for i in range(1, L):
        fl -= 2.0 * chs[i] * chs[i] * 9 * (H >> (i - 1)) * (W >> (i - 1))
    return fl


# cases of tests/golden/unet_noresample.pt: (name, cfg, B, H/W, seed)
TINY_CFG = dict(R.TINY_CFG, resample_with_conv=False)
SMALL64_CFG = dict(R.SMALL64_CFG, resample_with_conv=False)
CIFAR10_CFG = dict(R.CIFAR10_CFG, resample_with_conv=False)
CASES = [("tiny", TINY_CFG, 2, 16, 51), ("small64", SMALL64_CFG, 2, 32, 52), ("cifar10", CIFAR10_CFG, 2, 32, 53)]
BPD_CASE = "small64"
BPD_T = 20
