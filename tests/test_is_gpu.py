"""The Inception Score on an H100 (csrc/inception_score.cuh), with seeded weights (no network).

Bounds, derived here rather than tuned:

* Logits (``ddpm_is_logits``).  Each logit is z = sum_k f_k w_k over K = 2048 fp32 features f and fc weights w.  The kernel forms
  f_hi w_hi + f_lo w_hi + f_hi w_lo with f_hi = tf32(f), f_lo = tf32(f - f_hi), w_hi = tf32(w), w_lo = tf32(w - w_hi) (TF32 rounding
  to nearest, u = 2^-11).  Then f = f_hi + f_lo + e_f with |e_f| <= u |f - f_hi| <= u^2 |f|, likewise for w, and the dropped term
  (f - f_hi)(w - w_hi) is at most u^2 |f| |w|, so each product's representation error is at most 3 u^2 |f| |w| (+ higher order).
  The 3K TF32 products are exact in fp32; the tensor core's fp32 accumulation is not specified as round-to-nearest, so each of its
  3K additions is allowed the truncation error 2^-23 of a partial sum bounded by (1 + 2u) S, S = sum |f| |w|, and the output is a
  stored fp32.  Hence |z - z_ref| <= (3 u^2 + (3K + 1) 2^-23 (1 + 2u)) S.  In practice the accumulation error is a random walk
  far below that; the test checks the bound and reports the ratio.
  Against single TF32 on the same data (tf32(f) . tf32(w)^T, the error the issue rules out): the random mode also requires the
  error to stay below a quarter of that product's error, which a kernel that drops or duplicates a lo block cannot meet.
  Exact mode: integer features in [-8, 8] and integer weights in [-8, 8]: every operand is its own w_hi with w_lo = 0, every
  partial sum is an integer below 2^24, so the result equals the fp64 product bit for bit.
  Split mode (exact, with every lo block in play): on 256 of the 2048 columns f = a + b 2^-12 and w = c + d 2^-12 with
  a, c in +-{1, 2, 3} and b, d in {-1, 0, 1}, elsewhere f = 0.  Half a TF32 ulp of |a| >= 1 is at least 2^-11 > 2^-12, so
  f_hi = a, f_lo = b 2^-12 and likewise for w, all TF32 values.  The kernel's sum a c + (b c + a d) 2^-12 has every partial sum a
  multiple of 2^-12 below 256 (9 + 2^-9) < 2^12 in magnitude, hence exact in fp32, and must equal that fp64 value bit for bit;
  single TF32 (a c alone) and the full product (which adds b d 2^-24) both differ from it.
* Score (``ddpm_is_score``) against numpy fp64 on the same fp32 logits.  Both compute log p = z - lse in fp64 and fixed sums; they
  differ only in summation order.  Each IS_i = exp(KL_i) with KL_i a difference of two sums of at most N C terms of size at most
  max |log p| + log C; with fp64 rounding the relative error of IS_i is below 1e-12 for the sizes here (N C < 2^21,
  |log p| < 200: N C 2^-53 200 < 5e-8 in the worst case, and a random-walk estimate of 1e-13).  The tests use 1e-9 relative.
* End to end (``InceptionScore``) against the torch modules in fp64 (features, logits and score), per part: each IS_i's relative
  error is at most twice that of cuDNN with TF32 (fp32 fc matmul, fp64 formula) wherever cuDNN's exceeds 1e-4 -- the criterion
  the Inception test uses for its features -- and at most 1e-4 elsewhere.
"""
import copy
import os

import numpy as np
import pytest
import torch

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M
from ddpm_torch_b200.inception import seeded_state_dict, weights_path

pytestmark = pytest.mark.gpu

U = 2.0 ** -11
DEV = torch.device("cuda", 0)


@pytest.fixture
def offline(monkeypatch, tmp_path):
    def refuse(*a, **k):
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    os.makedirs(os.path.dirname(weights_path()))
    torch.save(seeded_state_dict(0), weights_path())
    yield tmp_path


def numpy_score(z, splits):
    z = np.asarray(z, dtype=np.float64)
    lse = z.max(1, keepdims=True) + np.log(np.exp(z - z.max(1, keepdims=True)).sum(1, keepdims=True))
    logp = z - lse
    p = np.exp(logp)
    n = z.shape[0]
    out = []
    for i in range(splits):
        b, e = i * n // splits, (i + 1) * n // splits
        pbar = p[b:e].mean(0)
        nz = pbar > 0
        out.append(np.exp(np.sum(p[b:e] * logp[b:e]) / (e - b) - np.sum(pbar[nz] * np.log(pbar[nz]))))
    return np.array(out)


def native_splits(z, splits):
    return np.array(M._is_native(z, splits, DEV))


def tf32(x):
    """fp32 -> TF32 rounded to nearest, ties away from zero (cvt.rna.tf32.f32) for finite x."""
    return ((x.contiguous().view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


def _split_operand(rows, g, mask=None):
    hi = torch.randint(1, 4, (rows, 2048), device="cuda", generator=g) * (torch.randint(0, 2, (rows, 2048), device="cuda", generator=g) * 2 - 1)
    lo = torch.randint(-1, 2, (rows, 2048), device="cuda", generator=g)
    if mask is not None:
        hi, lo = hi * mask, lo * mask
    return hi.double(), lo.double()


@pytest.mark.parametrize("N", [1, 300, 1003])
def test_logits_split_exact(N):
    g = torch.Generator(device="cuda").manual_seed(100 + N)
    k = torch.arange(2048, device="cuda")
    mask = ((k[None, :] + torch.arange(N, device="cuda")[:, None]) % 8 == 0).long()     # 256 columns per row
    a, b = _split_operand(N, g, mask)
    c, d = _split_operand(1008, g)
    f = (a + b * 2.0 ** -12).float()
    w = (c + d * 2.0 ** -12).float()
    assert torch.equal(tf32(f).double(), a) and torch.equal(tf32(w).double(), c)
    got, _ = M._is_logits(M._is_pack(w, DEV), f, DEV)
    want = a @ c.T + (b @ c.T + a @ d.T) * 2.0 ** -12
    assert torch.equal(got.double(), want)
    assert not torch.equal(a @ c.T, want)                         # single TF32 gives a c alone
    assert not torch.equal(f.double() @ w.double().T, want)       # the full product has the b d 2^-24 terms


@pytest.mark.parametrize("mode,N", [("exact", 1), ("exact", 300), ("random", 7), ("random", 513), ("random", 1003)])
def test_logits_against_fp64(mode, N):
    g = torch.Generator(device="cuda").manual_seed(N)
    if mode == "exact":
        f = torch.randint(-8, 9, (N, 2048), device="cuda", generator=g).float()
        w = torch.randint(-8, 9, (1008, 2048), device="cuda", generator=g).float()
    else:
        f = torch.relu(torch.randn(N, 2048, device="cuda", generator=g)) * 0.5       # pool3-like: non-negative
        w = torch.randn(1008, 2048, device="cuda", generator=g) * (2.0 / 2048) ** 0.5 * 4
    packed = M._is_pack(w, DEV)
    # a row pitch above 2048 as well: the features are read with a stride
    fs = torch.zeros(N, 2048 + 64, device="cuda")
    fs[:, :2048] = f
    for feats in (f, fs[:, :2048]):
        got, _ = M._is_logits(packed, feats, DEV)
        torch.cuda.synchronize()
        want = f.double() @ w.double().T
        if mode == "exact":
            assert torch.equal(got.double(), want)
            continue
        S = f.double().abs() @ w.double().abs().T
        K = 2048
        bound = (3 * U * U + (3 * K + 1) * 2.0 ** -23 * (1 + 2 * U)) * S
        err = (got.double() - want).abs()
        assert torch.all(err <= bound), (err / bound).max().item()
        single = (tf32(f).double() @ tf32(w).double().T - want).abs().max().item()
        assert err.max().item() < single / 4, (err.max().item(), single)
        print("logits", N, "max err / bound", (err / bound).max().item(), "max abs err", err.max().item(),
              "single TF32 max abs err", single, "max |z|", want.abs().max().item())


@pytest.mark.parametrize("N,splits", [(1000, 10), (1003, 10), (10, 10), (333, 1), (517, 7)])
def test_score_against_numpy(N, splits):
    g = torch.Generator(device="cuda").manual_seed(N * 31 + splits)
    z = (torch.randn(N, 1008, device="cuda", generator=g) * 3 + torch.randn(1, 1008, device="cuda", generator=g) * 2)
    got = native_splits(z, splits)
    want = numpy_score(z.cpu().numpy(), splits)
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=0)
    mean, std = M.calc_is(z, splits)
    np.testing.assert_allclose([mean, std], [np.mean(want), np.std(want)], rtol=1e-9, atol=1e-12)
    assert (mean, std) == M.calc_is(z, splits)                 # the same bits on a second call
    zs = torch.zeros(N, 1008 + 16, device="cuda")               # a row pitch above C
    zs[:, :1008] = z
    assert np.array_equal(native_splits(zs[:, :1008], splits), got)


def test_adversarial_rows_stay_finite():
    N = 40
    z = torch.zeros(N, 1008)
    z[:10] = -80.0
    z[torch.arange(10), torch.arange(10) * 7] = 80.0            # one-hot-like: an fp32 softmax underflows to zeros
    z[10:20] = 80.0                                             # ties: ten rows of a flat 80
    z[20:30, :3] = 80.0                                         # three-way ties at +80, the rest -80
    z[20:30, 3:] = -80.0
    g = torch.Generator().manual_seed(5)
    z[30:] = torch.randn(10, 1008, generator=g) * 40             # huge spread
    # what the TF code does: np.log of an fp32 softmax, with -inf * 0 for the underflowed classes
    p32 = torch.softmax(z, 1).numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        tf = np.sum(p32 * (np.log(p32) - np.log(p32.mean(0, keepdims=True))), 1)
    assert not np.isfinite(tf).all()
    for splits in (1, 4, 7):
        got = native_splits(z.cuda(), splits)
        want = numpy_score(z.numpy(), splits)
        assert np.isfinite(got).all()
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=0)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_logit_raises(bad):
    z = torch.randn(50, 1008, device="cuda")
    z[37, 500] = bad
    with pytest.raises(ValueError, match="non-finite"):
        M.calc_is(z, 5)
    z[37, 500] = 0.0
    M.calc_is(z, 5)                                             # the status is reset on the next call


def test_batch_invariance(offline):
    g = torch.Generator().manual_seed(21)
    x = torch.rand(500, 3, 32, 32, generator=g).cuda() * 2 - 1
    ist = M.InceptionScore(splits=10, device=DEV)
    scores = []
    for bs in (7, 64, 500):
        ist.reset()
        for b in x.split(bs):
            ist(b)
        assert ist.count == 500
        scores.append(ist.get_score())
    assert scores[0] == scores[1] == scores[2], scores
    assert np.isfinite(scores[0]).all()


def test_end_to_end_against_fp64(offline):
    g = torch.Generator().manual_seed(13)
    x = torch.rand(200, 3, 32, 32, generator=g).cuda() * 2 - 1
    splits = 4
    native = M.InceptionScore(splits=splits, device=DEV)
    net = native.model._module
    for b in x.split(64):
        native(b)
    got = native.get_score()
    w = net.fc_weight
    ref = copy.deepcopy(net).double()
    ref.use_engine = False
    with torch.inference_mode():
        f64 = torch.cat([ref(b.double())[0].flatten(1) for b in x.split(50)])
    want = M.calc_is((f64 @ w.to(f64).T).cpu().numpy(), splits, device="cpu")
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    net.use_engine = False
    try:
        with torch.inference_mode():
            f32 = torch.cat([net(b)[0].flatten(1) for b in x.split(64)])
    finally:
        torch.backends.cudnn.allow_tf32 = prev
        net.use_engine = True
    cud = M.calc_is((f32 @ w.to(f32).T).cpu().numpy(), splits, device="cpu")
    # per part: the seeded network maps every image to similar features, so the IS_i sit close to 1 and their spread (the std) is
    # tiny; the criterion is applied to each IS_i, of which the mean and std are functions
    got_i = np.array(M._is_native(native._logits[0], splits, DEV))
    want_i = np.array(M._is_numpy((f64 @ w.to(f64).T).cpu().numpy(), splits))
    cud_i = np.array(M._is_numpy((f32 @ w.to(f32).T).cpu().numpy(), splits))
    err, err_c = np.abs(got_i - want_i) / want_i, np.abs(cud_i - want_i) / want_i
    print("IS native", got, "fp64", want, "cudnn tf32", cud, "per-part rel err", err, "cudnn", err_c)
    assert np.isfinite(got).all() and got == (float(np.mean(got_i)), float(np.std(got_i)))
    assert np.all(err <= np.maximum(2 * err_c, 1e-4)), (err, err_c)
    # the same errors relative to KL_i = log IS_i (about 1e-3 here, so the 1e-4 floor above is loose): within the Inception
    # test's per-image feature bound of 5e-3, a first-order estimate for a KL computed from those features
    kl_err = np.abs(np.log(got_i) - np.log(want_i)) / np.log(want_i)
    print("per-part KL rel err", kl_err, "cudnn", np.abs(np.log(cud_i) - np.log(want_i)) / np.log(want_i))
    assert np.all(kl_err <= 5e-3), kl_err


def test_device_list_runs_torch_then_the_native_score(offline, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)        # the torch forward gives the same features twice
    g = torch.Generator().manual_seed(4)
    x = torch.rand(40, 3, 32, 32, generator=g).cuda() * 2 - 1
    a = M.InceptionScore(splits=4, device=[DEV])
    b = M.InceptionScore(splits=4, device=DEV)
    assert isinstance(a.model, torch.nn.DataParallel)
    a(x)
    b(x)
    # a's logits: the torch (DataParallel) features through the native 3xTF32 GEMM, within the logits bound of those features
    with torch.inference_mode():
        f = a.model(x).flatten(1).double()
    w = a.model.module._module.fc_weight.to(f)
    want = f @ w.T
    bound = (3 * U * U + (3 * 2048 + 1) * 2.0 ** -23 * (1 + 2 * U)) * (f.abs() @ w.abs().T)
    assert torch.all((a._logits[0].double() - want).abs() <= bound)
    # b's logits come from the engine's features: the same images to the Inception test's per-image feature tolerance
    rel = (b._logits[0].double() - want).norm(dim=1) / want.norm(dim=1)
    assert torch.all(rel <= 5e-3), rel.max().item()
    # and the score is the one of the kept logits, computed on the first device
    sa = a.get_score()
    np.testing.assert_allclose(np.array(M._is_native(a._logits[0], 4, DEV)), M._is_numpy(a._logits[0].cpu().numpy(), 4),
                               rtol=1e-9, atol=0)
    assert sa == M.calc_is(a._logits[0], 4)


def test_no_device_error():
    assert _lib.lib().ddpm_device_error_flag() == 0
