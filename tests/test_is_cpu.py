"""The Inception Score without a GPU: the CPU formula against the TensorFlow code's loop, a CPU ``InceptionScore`` end to end with
seeded weights, the C ABI's refusals and sizes, the logits kernel's SASS, and the public names.  Nothing reaches the network."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import inception as I
from ddpm_torch_b200 import metrics as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "ddpm_torch_b200", "libddpm_b200.so")
NAMES = ("ddpm_is_fc_packed_bytes", "ddpm_is_fc_pack", "ddpm_is_logits_workspace_bytes", "ddpm_is_logits",
         "ddpm_is_score_scratch_bytes", "ddpm_is_score")


@pytest.fixture
def offline(monkeypatch, tmp_path):
    def refuse(*a, **k):
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    os.makedirs(os.path.dirname(I.weights_path()))
    torch.save(I.seeded_state_dict(0), I.weights_path())


def tf_inception_score(logits, splits):
    """improved-gan/inception_score.py's loop, verbatim, on a softmax of the logits (fp64 here, fp32 in the TF graph)."""
    z = np.asarray(logits, dtype=np.float64)
    e = np.exp(z - z.max(axis=1, keepdims=True))
    preds = e / e.sum(axis=1, keepdims=True)
    scores = []
    for i in range(splits):
        part = preds[(i * preds.shape[0] // splits):((i + 1) * preds.shape[0] // splits), :]
        kl = part * (np.log(part) - np.log(np.expand_dims(np.mean(part, 0), 0)))
        kl = np.mean(np.sum(kl, 1))
        scores.append(np.exp(kl))
    return np.mean(scores), np.std(scores)


@pytest.mark.parametrize("N,splits", [(1000, 10), (1003, 10), (37, 1), (50, 7)])
def test_cpu_formula_is_the_tf_loop(N, splits):
    rng = np.random.default_rng(N + splits)
    logits = (rng.standard_normal((N, 1008)) * 3 + rng.standard_normal((1, 1008))).astype(np.float32)
    want = tf_inception_score(logits, splits)
    for arg in (logits, torch.from_numpy(logits)):
        got = M.calc_is(arg, splits, device="cpu")
        assert isinstance(got[0], float) and isinstance(got[1], float)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


def test_cpu_formula_refusals():
    z = np.zeros((5, 1008), dtype=np.float32)
    with pytest.raises(ValueError):
        M.calc_is(z, 6, device="cpu")
    with pytest.raises(ValueError):
        M.calc_is(z, 0, device="cpu")
    with pytest.raises(ValueError):
        M.calc_is(z[0], 1, device="cpu")
    z[3, 7] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        M.calc_is(z, 2, device="cpu")


def test_cpu_formula_saturated_rows_stay_finite():
    z = np.zeros((8, 1008), dtype=np.float32)
    z[np.arange(8), np.arange(8) * 3] = 80.0           # one-hot-like: the fp32 softmax underflows to exact zeros
    z[4:, :] = -80.0
    z[4:, 5] = 80.0
    mean, std = M.calc_is(z, 2, device="cpu")
    assert np.isfinite(mean) and np.isfinite(std)
    # part 0: four distinct one-hot rows -> KL = log 4; part 1: four identical rows -> KL = 0
    np.testing.assert_allclose([mean, std], [(4 + 1) / 2, (4 - 1) / 2], rtol=1e-12)


def test_cpu_inception_score_end_to_end(offline):
    g = torch.Generator().manual_seed(3)
    x = torch.rand(4, 3, 40, 40, generator=g) * 2 - 1
    ist = M.InceptionScore(splits=2)
    ist(x[:3])
    ist(x[3:])
    assert ist.count == 4
    got = ist.get_score()
    net = I.InceptionV3([3]).eval()
    with torch.inference_mode():                        # batch by batch, as ist saw them: CPU kernels may differ with the batch
        w = I.seeded_state_dict(0)["fc.weight"]
        logits = torch.cat([net(b)[0].flatten(1) @ w.T for b in (x[:3], x[3:])])
    assert got == M.calc_is(logits, 2, device="cpu")
    np.testing.assert_allclose(got, tf_inception_score(logits.numpy(), 2), rtol=1e-10, atol=1e-12)
    ist.reset()
    assert ist.count == 0
    with pytest.raises(ValueError):
        ist.get_score()


def test_names_and_state_dict_keys(offline):
    assert "InceptionScore" in M.__all__ and "calc_is" in M.__all__
    full = I.fid_inception_v3().state_dict()
    want = set()
    for k in full:
        if k.startswith("fc."):
            continue
        mod, rest = k.split(".", 1)
        want.add(f"{I._ENGINE_BLOCK[mod]}.{rest}")
    net = I.InceptionV3()
    assert set(net.state_dict()) == want
    assert torch.equal(net.fc_weight, full["fc.weight"])


def test_exports_and_sizes():
    hdr = open(os.path.join(ROOT, "include", "ddpm_b200.h")).read()
    for name in NAMES:
        assert name in _lib.EXPORTS
        getattr(_lib.lib(), name)
        assert re.search(r"\b" + name + r"\(", hdr)
    L = _lib.lib()
    assert L.ddpm_is_fc_packed_bytes() == 1024 * 6144 * 4
    for n in (1, 7, 512, 50000):
        assert L.ddpm_is_logits_workspace_bytes(n) == -(-n * 6144 * 4 // 256) * 256
    al = lambda b: -(-b // 256) * 256                     # noqa: E731
    for n, c, s, chunks in ((1003, 1008, 10, 1), (50000, 1008, 10, 32), (1000, 5, 1, 7), (7, 1, 7, 1)):
        assert L.ddpm_is_score_scratch_bytes(n, c, s) == 256 + 2 * al(n * 8) + al(s * chunks * c * 8)


def test_refusals_without_a_device():
    L = _lib.lib()
    p = 1 << 20                                         # a well-aligned non-null address that is never dereferenced
    assert L.ddpm_is_fc_pack(None, p, None) < 0
    assert L.ddpm_is_fc_pack(p + 2, p, None) < 0
    assert L.ddpm_is_fc_pack(p, p + 16, None) < 0
    assert L.ddpm_is_logits_workspace_bytes(0) < 0
    ws = L.ddpm_is_logits_workspace_bytes(8)
    good = dict(packed=p, feats=p, N=8, ld=2048, logits=p, ws=p, ws_bytes=ws)
    bad = [dict(packed=None), dict(packed=p + 16), dict(feats=None), dict(feats=p + 2), dict(N=0), dict(N=-1), dict(ld=2047),
           dict(logits=None), dict(logits=p + 4), dict(ws=None), dict(ws=p + 16), dict(ws_bytes=ws - 1)]
    for b in bad:
        a = {**good, **b}
        rc = L.ddpm_is_logits(a["packed"], a["feats"], a["N"], a["ld"], a["logits"], a["ws"], a["ws_bytes"], None)
        assert rc < 0 and b"ddpm_is_logits" in L.ddpm_last_error(), b
    for n, c, s in ((9, 1008, 10), (10, 1008, 0), (10, 1008, -1), (10, 0, 1), (0, 1008, 1)):
        assert L.ddpm_is_score_scratch_bytes(n, c, s) < 0
    sb = L.ddpm_is_score_scratch_bytes(100, 1008, 10)
    good = dict(z=p, N=100, C=1008, ld=1008, splits=10, out=p, scratch=p, bytes=sb)
    bad = [dict(z=None), dict(z=p + 2), dict(N=9), dict(splits=0), dict(splits=101), dict(C=0), dict(ld=1007), dict(out=None),
           dict(out=p + 4), dict(scratch=None), dict(scratch=p + 8), dict(bytes=sb - 1)]
    for b in bad:
        a = {**good, **b}
        rc = L.ddpm_is_score(a["z"], a["N"], a["C"], a["ld"], a["splits"], a["out"], a["scratch"], a["bytes"], None)
        assert rc < 0 and b"ddpm_is_score" in L.ddpm_last_error(), b


def test_logits_kernel_sass_and_spills():
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
    gemm = [ops for fn, ops in per.items() if "is_logits_tf32_kernel" in fn]
    assert len(gemm) == 1
    assert any(o.startswith("HGMMA") for o in gemm[0]) and not any(o.startswith(("HMMA", "IMMA")) for o in gemm[0])
    simt = {fn: ops for fn, ops in per.items() if re.search(r"k_is_(pack|split|rows|cols|final)", fn)}
    assert len(simt) == 5 and not any(o.startswith(("HGMMA", "HMMA", "IMMA")) for ops in simt.values() for o in ops)
    log = os.path.join(ROOT, "ddpm_torch_b200", "csrc", "build.log")
    if not os.path.exists(log):
        pytest.skip("no build log (-Xptxas -v) next to the sources")
    lines = open(log).read().splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and ("is_logits_tf32_kernel" in ln or re.search(r"k_is_(pack|split|rows|cols|final)", ln)):
            seen += 1
            spill = next(x for x in lines[i + 1:i + 5] if "bytes spill stores" in x)
            assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", spill), (ln, spill)
    assert seen == 6
