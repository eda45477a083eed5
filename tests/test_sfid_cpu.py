"""sFID's spatial features without a GPU: the torch route against an independent restatement with torchvision's own modules, the
flatten order, the CPU statistics, refusals in Python and through the ABI, exports and the gather kernel's SASS.  Seeded weights
(inception.seeded_state_dict); nothing reaches the network."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import inception as I
from ddpm_torch_b200 import metrics as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "ddpm_torch_b200", "libddpm_b200.so")
U = 2.0 ** -53


@pytest.fixture
def offline(monkeypatch, tmp_path):
    def refuse(*a, **k):
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    os.makedirs(os.path.dirname(I.weights_path()))
    torch.save(I.seeded_state_dict(0), I.weights_path())


def restated(net, x):
    """torchvision's Mixed_6d.branch1x1 (BasicConv2d: conv, BatchNorm, ReLU) on the Mixed_6c output, channels 0..6 in NHWC order."""
    x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
    for m in [*net.blocks[0], *net.blocks[1], *list(net.blocks[2])[:6]]:      # up to Mixed_6c
        x = m(x)
    b = net.blocks[2][6].branch1x1(x)
    return b[:, :7].permute(0, 2, 3, 1).reshape(x.shape[0], -1)


@pytest.mark.parametrize("blocks", [[3], [2], [0, 2, 3]])
def test_torch_route_features_are_branch1x1_of_mixed_6d(offline, blocks):
    net = I.InceptionV3(blocks).eval()
    x = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(1))
    with torch.inference_mode():
        out, sp = net(x, spatial=True)
        plain = net(x)
        want = restated(net, x)
    assert sp.shape == (2, 2023) == want.shape and sp.dtype == torch.float32
    assert torch.equal(sp, want)
    assert len(out) == len(plain) and all(torch.equal(a, b) for a, b in zip(out, plain))
    assert (sp >= 0).all() and (sp > 0).any()


def test_flatten_order_is_tf_nhwc():
    N, Cc, h, w = 2, 768, 5, 3                          # h != w: a transposed flatten would move values
    t = torch.arange(N * Cc * h * w, dtype=torch.float32).reshape(N, Cc, h, w)
    sp = I.spatial_features(t)
    assert sp.shape == (N, h * w * 7)
    for n in range(N):
        for y in range(h):
            for xx in range(w):
                for c in range(7):
                    assert sp[n, (y * w + xx) * 7 + c] == t[n, c, y, xx]
    assert M.SPATIAL_DIM == 2023 == 17 * 17 * 7


def test_cpu_statistics(offline):
    g = torch.Generator().manual_seed(4)
    imgs = torch.rand(9, 3, 32, 32, generator=g) * 2 - 1
    sizes = [4, 2, 3]
    sp = M.InceptionStatistics(spatial=True)
    plain = M.InceptionStatistics()
    feats = []
    for b in imgs.split(sizes):
        sp(b)
        plain(b)
        with torch.inference_mode():
            feats.append(sp.model(b)[1])
    assert sp.count == plain.count == 9
    for a, b in zip(sp.get_statistics(), plain.get_statistics()):
        assert np.array_equal(a, b)
    assert np.array_equal(sp.running_var, plain.running_var)
    m, c = sp.get_spatial_statistics()
    assert m.shape == (2023,) and c.shape == (2023, 2023) and m.dtype == c.dtype == np.float64
    x = torch.cat(feats).double().numpy()
    rm, rc = x.mean(0), np.cov(x, rowvar=False)
    # both sides sum exact fp64 products of fp32 features in different orders (see test_fid_gpu.py)
    a = np.abs(x).max(0) + np.abs(rm)
    assert np.all(np.abs(c - rc) <= 8 * 9 * U * np.outer(a, a) / 8)
    assert np.all(np.abs(m - rm) <= 4 * 9 * U * a)
    sp.reset()
    assert sp.count == 0
    assert not sp._moments[1][0].any() and not sp._moments[1][1].any() and not sp.running_var.any()
    with pytest.raises(RuntimeError, match="spatial=True"):
        plain.get_spatial_statistics()


@pytest.mark.parametrize("dim", [64, 192])
def test_blocks_before_mixed_6d_refuse_spatial(offline, dim):
    with pytest.raises(ValueError, match="Mixed_6d"):
        M.InceptionStatistics(activation_dim=dim, spatial=True)
    net = I.InceptionV3([I.InceptionV3.BLOCK_INDEX_BY_DIM[dim]]).eval()
    with pytest.raises(ValueError, match="Mixed_6d"):
        net(torch.rand(1, 3, 32, 32), spatial=True)


def test_abi_refusals():
    L = _lib.lib()
    buf = (C.c_uint8 * 8192)()
    p = C.addressof(buf) + (-C.addressof(buf)) % 256
    outs = (C.c_void_p * 4)()
    fwd = L.ddpm_inception_forward_ex
    for blk in (0, 1):
        assert fwd(p, p, 1, 32, 32, 1, 0, blk, C.byref(outs), None, p, p, 1 << 40, None) < 0
        assert b"spatial" in L.ddpm_last_error() and b"last_block >= 2" in L.ddpm_last_error()
    assert fwd(p, p, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p + 2, p, 1 << 40, None) < 0             # misaligned
    assert b"spatial" in L.ddpm_last_error()
    # accepted spatial buffers (null at any block, aligned from block 2) reach the workspace check, which refuses 16 bytes
    for blk, s in ((0, None), (1, None), (2, None), (2, p + 4), (3, p)):
        assert fwd(p, p, 1, 32, 32, 1, 0, blk, C.byref(outs), None, s, p, 16, None) < 0
        err = L.ddpm_last_error()
        assert b"ddpm_inception_forward_ex" in err and b"workspace" in err and b"spatial" not in err, err
    # the other checks are the forward's own
    assert fwd(None, p, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p, p, 1 << 40, None) < 0
    assert fwd(p, p, 1, 32, 32, 1, 2, 3, C.byref(outs), None, p, p, 1 << 40, None) < 0
    assert fwd(p, p, 1, 32, 32, 0, 0, 3, C.byref(outs), None, p, p, 1 << 40, None) < 0 and b"too small" in L.ddpm_last_error()
    assert L.ddpm_inception_forward(p, p, 1, 32, 32, 1, 0, 3, C.byref(outs), None, p, 16, None) < 0
    assert b"ddpm_inception_forward:" in L.ddpm_last_error()


def test_exports_match_header():
    hdr = open(os.path.join(ROOT, "include", "ddpm_b200.h")).read()
    name = "ddpm_inception_forward_ex"
    assert name in _lib.EXPORTS
    getattr(_lib.lib(), name)
    m = re.search(r"\bint " + name + r"\(([^)]*)\);", hdr)
    assert m
    params = [a.strip() for a in m.group(1).split(",")]
    assert len(params) == len(_lib.lib().ddpm_inception_forward_ex.argtypes) == 14
    assert params[10] == "float* spatial"


def test_gather_kernel_sass_and_spills():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    per, cur = {}, None
    for ln in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1); per[cur] = set(); continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", ln)
        if m and cur:
            per[cur].add(m.group(1))
    hits = [ops for fn, ops in per.items() if "k_sfid_gather" in fn]
    assert len(hits) == 1
    assert not any(o.startswith(("ATOM", "RED", "HGMMA", "HMMA", "STL", "LDL")) for o in hits[0])
    log = os.path.join(ROOT, "ddpm_torch_b200", "csrc", "build.log")
    if not os.path.exists(log):
        pytest.skip("no build log (-Xptxas -v) next to the sources")
    lines = open(log).read().splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and "k_sfid_gather" in ln:
            seen += 1
            spill = next(x for x in lines[i + 1:i + 5] if "bytes spill stores" in x)
            assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", spill), spill
    assert seen == 1
