"""The Kernel Inception Distance on an H100 (csrc/kid.cuh), with seeded weights where Inception runs (no network).

Bounds, derived here rather than tuned (u = 2^-53, fp64 round to nearest):

* Random features, native ``ddpm_kid`` against numpy fp64 (``_kid_numpy``) on the same fp32 features and the same subsets.  For one
  kernel entry with Gram value g = a . b over d columns, both routes form the d products exactly (fp32 x fp32 fits in fp64) and sum
  them in some order, so |g_hat - g| <= d u A with A = sum_k |a_k| |b_k|.  The base b = gamma g + c0 adds at most 2 u (gamma A + |c0|)
  (one multiply, one add, or one FMA), so e_b = gamma (d + 2) u A + 2 u |c0|; raising to the power p (p - 1 multiplications here,
  ``pow`` in numpy) gives |k_hat - k| <= p |b|^(p-1) e_b + (p + 1) u |k| to first order.  Summing n <= m^2 terms in any order adds
  at most n u sum |k|.  So each of the three kernel sums is off by at most E = sum_entries (p |b|^(p-1) e_b + (p + 1) u |k|) + m^2 u
  sum |k|, and mmd2_s, a combination with weights 1 / (m (m - 1)) and 2 / m^2 followed by two divisions and a subtraction, by at most
  w_xx E_xx + w_yy E_yy + w_xy E_xy + 4 u (w_xx (|K_xx| + |K_yy|) + w_xy |K_xy|) + u |mmd2_s|.  The two routes each satisfy this, so
  their difference is below twice it; 1 % is added for the second-order terms.  The bound is relative to the kernel sums, not to the
  small mmd2_s: the m^2 u term dominates (~1e-9 at m = 1000 against kernel means ~1), and the measured differences are far below.
* Integer mode (bit-exact): features in {-2..2}, d = 256, gamma = 1, c0 = 1, degree 3.  Every Gram entry is an integer with
  |g| <= 4 d = 1024, every kernel value (g + 1)^3 is an integer of magnitude below 1025^3 < 1.1e9, and every partial or total sum
  is an integer of magnitude below m^2 1.1e9 <= 1.1e15 < 2^53, so all of it is exact in fp64 in any order.  The native mmd2_s must
  then equal the exact integers pushed through the same two fp64 divisions and one subtraction -- in Python, int / int is the
  correctly rounded quotient -- bit for bit.  A dropped, duplicated or un-doubled tile, or a wrong diagonal or padding mask, moves
  a sum by at least one kernel value and breaks the equality.
* Batch invariance and repeatability: bit-identical, since the result depends on the drawn feature rows only and every sum runs in
  a fixed order.
* End to end: ``KernelInceptionDistance`` on the engine against ``calc_kid(..., device="cpu")`` on the same features, within the
  random-mode bound.
"""
import os

import numpy as np
import pytest
import torch

from ddpm_torch_b200 import metrics as M
from ddpm_torch_b200.inception import seeded_state_dict, weights_path

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
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


def bound(x, y, idx, degree, gamma, coef0):
    """Per subset, the bound of the module docstring on |native - numpy fp64|."""
    x = torch.as_tensor(x).to(DEV, torch.float64)
    y = torch.as_tensor(y).to(DEV, torch.float64)
    m, d = idx.shape[2], x.shape[1]
    out = []
    for s in range(idx.shape[0]):
        a, b = x[torch.as_tensor(idx[s, 0]).long()], y[torch.as_tensor(idx[s, 1]).long()]
        tot, mags = 0.0, []
        for p_, q_, w, diag in ((a, a, 1 / (m * (m - 1)), True), (b, b, 1 / (m * (m - 1)), True), (b, a, 2 / (m * m), False)):
            base = gamma * (p_ @ q_.T) + coef0
            A = p_.abs() @ q_.abs().T
            k = base ** degree
            eb = gamma * (d + 2) * U * A + 2 * U * abs(coef0)
            e = degree * base.abs() ** (degree - 1) * eb + (degree + 1) * U * k.abs()
            if diag:
                keep = ~torch.eye(m, dtype=torch.bool, device=DEV)
                e, k = e[keep], k[keep]
            tot += w * (e.sum().item() + m * m * U * k.abs().sum().item())
            mags.append(w * abs(k.sum().item()))
        mmd = mags[0] + mags[1] + mags[2]
        out.append(2 * 1.01 * (tot + 4 * U * mmd + U * mmd))
    return np.array(out)


def gaussian(n1, n2, d, seed, shift=0.1, pitch=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n1, d, device="cuda", generator=g)
    y = torch.randn(n2, d, device="cuda", generator=g) + shift
    if pitch is not None:                               # read with a row pitch above d
        xs = torch.zeros(n1, pitch, device="cuda")
        xs[:, :d] = x
        x = xs[:, :d]
    return x, y


@pytest.mark.parametrize("m", [1000, 777])
def test_random_against_numpy_fp64(m):
    n1, n2, d, S = 3000, 2500, 2048, 10
    x, y = gaussian(n1, n2, d, m, pitch=d + 64)
    assert x.stride(0) == d + 64
    idx = M._kid_indices(n1, n2, S, m, 1234)
    gamma = 1.0 / d
    got, status = M._kid_native(x, y, idx, 3, gamma, 1.0, DEV)
    assert status == 0
    want = M._kid_numpy(x.cpu().numpy(), y.cpu().numpy(), idx, 3, gamma, 1.0)
    bd = bound(x, y, idx, 3, gamma, 1.0)
    err = np.abs(got - want)
    print(f"m = {m}: max |native - numpy| = {err.max():.3e}, max ratio to bound {np.max(err / bd):.3e}, "
          f"mmd2 in [{want.min():.3e}, {want.max():.3e}], bound {bd.max():.3e}")
    assert (err <= bd).all(), (err, bd)
    assert (want > 0).all()                              # the mean shift is visible: a sanity check on the data, not the kernel
    mean, std = M.calc_kid(x, y, S, m)
    np.testing.assert_allclose([mean, std], [np.mean(want), np.std(want)], rtol=0, atol=2 * bd.max())
    assert M.calc_kid(x, y, S, m) == (mean, std)         # two runs: the same bits


def exact_mmd2(x, y, idx):
    """Integer mode: exact kernel sums as Python ints, then the two fp64 divisions and the subtraction."""
    xd, yd = x.double(), y.double()
    m = idx.shape[2]
    out = []
    for s in range(idx.shape[0]):
        a, b = xd[torch.as_tensor(idx[s, 0]).long()], yd[torch.as_tensor(idx[s, 1]).long()]
        sums = []
        for p_, q_, diag in ((a, a, True), (b, b, True), (a, b, False)):
            g = (p_ @ q_.T).long()                       # |g| <= 1024: exact in fp64
            k = (g + 1) ** 3
            sums.append(int(k.sum().item()) - (int(k.diagonal().sum().item()) if diag else 0))
        kxx, kyy, kxy = sums
        out.append((kxx + kyy) / (m * (m - 1)) - 2 * kxy / (m * m))
    return np.array(out)


@pytest.mark.parametrize("m", [1000, 777, 64, 2])
def test_integer_mode_bit_exact(m):
    n1, n2, d, S = 3000, 2500, 256, 10
    g = torch.Generator(device="cuda").manual_seed(7 + m)
    x = torch.randint(-2, 3, (n1, d), device="cuda", generator=g).float()
    y = torch.randint(-2, 3, (n2, d), device="cuda", generator=g).float()
    idx = M._kid_indices(n1, n2, S, m, m)
    got, status = M._kid_native(x, y, idx, 3, 1.0, 1.0, DEV)
    assert status == 0
    want = exact_mmd2(x, y, idx)
    assert np.array_equal(got, want), np.abs(got - want).max()
    mean, std = M.calc_kid(x, y, S, m, gamma=1.0, seed=m)
    # the mean and std are fp64 sums of S values in another order than numpy's: S^2 u of the largest
    np.testing.assert_allclose([mean, std], [np.mean(want), np.std(want)], rtol=0, atol=S * S * U * np.abs(want).max())


def test_nonfinite_refusal():
    x, y = gaussian(300, 200, 64, 3)
    idx = M._kid_indices(300, 200, 4, 100, 1234)
    x[int(idx[2, 0, 17]), 5] = float("nan")             # one drawn row of one subset
    with pytest.raises(ValueError, match="non-finite"):
        M.calc_kid(x, y, 4, 100)
    _, status = M._kid_native(x, y, idx, 3, 1 / 64, 1.0, DEV)
    assert status == 1
    x2, _ = gaussian(300, 200, 64, 3)
    y[:, 0] = float("inf")
    with pytest.raises(ValueError, match="non-finite"):
        M.calc_kid(x2, y, 4, 100)


def test_batch_invariance_and_end_to_end(offline):
    g = torch.Generator(device="cuda").manual_seed(11)
    imgs = torch.rand(600, 3, 32, 32, device="cuda", generator=g) * 2 - 1
    other = torch.relu(torch.randn(700, 2048, device="cuda", generator=g)) * 0.5
    kid = M.KernelInceptionDistance(num_subsets=6, subset_size=300, device=DEV)
    kid(imgs)
    ref_feats = kid.features.clone()
    assert ref_feats.shape == (600, 2048) and ref_feats.is_cuda and ref_feats.dtype == torch.float32
    ref = kid.get_kid(other)
    assert kid.get_kid(other) == ref                    # two runs: the same bits
    for bs in (7, 64, 500):
        kid.reset()
        for b in imgs.split(bs):
            kid(b)
        assert kid.count == 600
        assert torch.equal(kid.features, ref_feats), bs
        assert kid.get_kid(other) == ref, bs
    # end to end: against numpy fp64 on the same features, within the random-mode bound
    cpu = M.calc_kid(ref_feats, other, 6, 300, device="cpu")
    idx = M._kid_indices(600, 700, 6, 300, 1234)
    bd = bound(ref_feats, other, idx, 3, 1 / 2048, 1.0)
    print(f"end to end: native {ref}, numpy {cpu}, bound {bd.max():.3e}")
    assert abs(ref[0] - cpu[0]) <= bd.max() and abs(ref[1] - cpu[1]) <= 2 * bd.max()
    # another KernelInceptionDistance as the second set: its features, the subsets' iy drawn from it
    twin = M.KernelInceptionDistance(num_subsets=6, subset_size=300, device=DEV)
    twin._feats = [other]
    assert kid.get_kid(twin) == ref
