"""sFID on the engine: the spatial tap of the Inception forward (``ddpm_inception_forward_ex``, k_sfid_gather in
csrc/inception.cuh) and ``InceptionStatistics(spatial=True)``, on an H100 with seeded weights (no network).

Bounds:
* Features, per image against the torch module in fp64: relative L2 <= 5e-3 and cosine >= 0.9999, and the engine's error at most
  twice cuDNN's (TF32 allowed) wherever cuDNN's exceeds 1e-4: the gates of the Inception forward's own end-to-end test
  (test_inception_native_gpu.py), since the gather copies Mixed_6d's fp32 output as it is.
* Statistics: the bound of test_fid_gpu.py.  Every product of two fp32 features is exact in fp64, and the native state and the
  reference's per-batch np.cov with its merge differ in the order of O(n) fp64 additions, so per element
  |cov_ij - ref_ij| <= B_ij = 8 n u a_i a_j / (n - 1), a_i = max_r |x_ri| + |mean_i|, u = 2^-53.
* sFID of 2000 images against a second set: within 1e-2 of the fp64 route, the FID row's bound (2000 images give rank-deficient
  2023 x 2023 covariances, where the TF32 feature error moves tr sqrt(S1 S2) by a few 1e-3; see test_fid_level).
"""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ddpm_torch_b200 import _lib
from ddpm_torch_b200 import metrics as M
from ddpm_torch_b200.inception import InceptionV3, _block_hw, seeded_state_dict, spatial_features, weights_path

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


def _offline(monkeypatch, tmp_path, sd):
    def refuse(*a, **k):
        raise AssertionError("network reached")
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    os.makedirs(os.path.dirname(weights_path()), exist_ok=True)
    torch.save(sd, weights_path())


@pytest.fixture
def offline(monkeypatch, tmp_path):
    _offline(monkeypatch, tmp_path, seeded_state_dict(0))


def _model(blocks=(3,), resize=True, normalize=False):
    return InceptionV3(list(blocks), resize_input=resize, normalize_input=normalize).eval().cuda()


def _torch_route(model, x):
    """The torch modules' (out, spatial) for a module that would otherwise run on the engine."""
    prev = model.use_engine
    model.use_engine = False
    try:
        return model(x, spatial=True)
    finally:
        model.use_engine = prev


def _raw_forward(model, x, last, spatial, pooled=None, outs=None, pad=0):
    """ddpm_inception_forward_ex on x; returns the NaN-prefilled spatial buffer with `pad` extra floats at its end."""
    L = _lib.lib()
    model._repack_if_needed(x.device)
    N, _, H, W = x.shape
    need = L.ddpm_inception_workspace_bytes(N, H, W, int(model.resize_input), last)
    assert need > 0, L.ddpm_last_error()
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    h, w = _block_hw(H, W, model.resize_input, 2)
    sp = torch.full((N * h * w * 7 + pad,), float("nan"), device="cuda") if spatial else None
    o = (C.c_void_p * 4)(*[None if t is None else t.data_ptr() for t in (outs or [None] * 4)])
    _lib.check(L.ddpm_inception_forward_ex(model._packed.data_ptr(), x.data_ptr(), N, H, W, int(model.resize_input),
                                           int(model.normalize_input), last, C.byref(o), None if pooled is None else pooled.data_ptr(),
                                           None if sp is None else sp.data_ptr(), ws.data_ptr(), need, _lib.stream_ptr()), "forward_ex")
    torch.cuda.synchronize()
    return sp


CASES = [(32, 1, True, False), (32, 3, True, True), (32, 64, True, False), (64, 3, False, True), (64, 1, True, True),
         (256, 3, False, False), (256, 1, True, True), (299, 3, False, True), (299, 1, True, False), (299, 64, False, False)]


@pytest.mark.parametrize("size,N,resize,normalize", CASES)
def test_features_against_fp64(offline, size, N, resize, normalize, record_property):
    blocks = (2,) if (size == 64 and not resize) else (3,)
    model = _model(blocks, resize, normalize)
    ref = copy.deepcopy(model).double()
    g = torch.Generator(device="cuda").manual_seed(size + N)
    x = torch.rand(N, 3, size, size, device="cuda", generator=g)
    with torch.inference_mode():
        out, got = model(x, spatial=True)
    h, w = _block_hw(size, size, resize, 2)
    assert got.shape == (N, h * w * 7) and got.dtype == torch.float32
    n_ref = min(N, 8)
    with torch.inference_mode():
        want = ref(x[:n_ref].double(), spatial=True)[1]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        with torch.inference_mode():
            cud = _torch_route(model, x[:n_ref])[1]
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    gd, wd, cd = got[:n_ref].double(), want, cud.double()
    rel = (gd - wd).norm(dim=1) / wd.norm(dim=1)
    rel_c = (cd - wd).norm(dim=1) / wd.norm(dim=1)
    cos = (gd * wd).sum(1) / (gd.norm(dim=1) * wd.norm(dim=1))
    worst = (rel.max().item(), cos.min().item(), rel_c.max().item())
    record_property("worst", worst)
    print("sfid features", size, N, resize, normalize, "rel %.3e cos %.8f cudnn-tf32 rel %.3e" % worst)
    assert torch.all(rel <= 5e-3) and torch.all(cos >= 0.9999), worst
    big = rel_c > 1e-4
    assert torch.all(rel[big] <= 2 * rel_c[big]), worst


@pytest.mark.parametrize("size,resize,last", [(32, True, 3), (64, False, 2), (299, False, 3)])
def test_outputs_fully_written_and_nothing_else(offline, size, resize, last):
    model = _model((last,), resize)
    x = torch.rand(3, 3, size, size, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    with torch.inference_mode():
        sp = _raw_forward(model, x, last, True, pad=33)
        want = model(x, spatial=True)[1]
    n = want.numel()
    assert not torch.isnan(sp[:n]).any() and torch.isnan(sp[n:]).all()
    assert torch.equal(sp[:n].view_as(want), want)


def test_batch_independence_repeat_and_graph(offline):
    model = _model()
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.rand(64, 3, 32, 32, device="cuda", generator=g)
    with torch.inference_mode():
        a = model(x, spatial=True)[1]
        b = model(x, spatial=True)[1]
        assert torch.equal(a, b)
        for i in (0, 17, 63):
            assert torch.equal(model(x[i:i + 1], spatial=True)[1][0], a[i])
        xs = x[:8].clone()
        eager = model.forward_native(xs, pooled=True, spatial=True)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model.forward_native(xs, pooled=True, spatial=True)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cap = model.forward_native(xs, pooled=True, spatial=True)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(cap[0], eager[0]) and torch.equal(cap[1], eager[1])
    assert torch.equal(eager[1], a[:8])


@pytest.mark.parametrize("size,resize", [(32, True), (299, False)])
def test_tap_changes_no_other_output(offline, size, resize):
    model = _model((0, 1, 2, 3), resize)
    x = torch.rand(5, 3, size, size, device="cuda", generator=torch.Generator(device="cuda").manual_seed(size))
    with torch.inference_mode():
        plain = model.forward_native(x)
        outs, sp = model.forward_native(x, spatial=True)
        pooled = model.forward_native(x, pooled=True)
        pooled_sp, sp2 = model.forward_native(x, pooled=True, spatial=True)
    assert all(torch.equal(a, b) for a, b in zip(plain, outs))
    assert torch.equal(pooled, pooled_sp) and torch.equal(sp, sp2)


def _mixed_6d_torch(model, x):
    """Mixed_6d's NCHW output from the torch modules of a copy of ``model`` cut right after Mixed_6d."""
    sub = copy.deepcopy(model)
    sub.blocks = sub.blocks[:3]
    sub.blocks[2] = torch.nn.Sequential(*list(sub.blocks[2])[:7])
    sub.output_blocks, sub.last_needed_block = [2], 2
    sub.use_engine = False
    with torch.inference_mode():
        return sub(x)[0]


def chan_recipe(batches):
    """fid_score.py:116-142 in numpy: per-batch np.cov (ddof 0) merged, then rescaled to ddof 1."""
    m = v = None
    cnt = 0
    for x in batches:
        x = np.asarray(x, dtype=np.float32)
        mean = np.mean(x, axis=0, dtype=np.float64)
        var = np.cov(x, rowvar=False, ddof=0, dtype=np.float64).reshape(x.shape[1], x.shape[1])
        k = x.shape[0]
        a = k / (cnt + k)
        if cnt == 0:
            m, v = mean.copy(), var.copy()
        else:
            d = mean - m
            m += a * d
            v += a * (var - v)
            v += a * (1 - a) * np.outer(d, d)
        cnt += k
    return m, v * cnt / (cnt - 1)


def test_statistics_on_cuda(offline):
    g = torch.Generator().manual_seed(2)
    imgs = torch.rand(300, 3, 32, 32, generator=g) * 2 - 1
    sizes = [128, 1, 100, 71]
    sp = M.InceptionStatistics(device=torch.device("cuda"), spatial=True)
    plain = M.InceptionStatistics(device=torch.device("cuda"))
    net = sp.model._module
    batches = []
    for b in imgs.split(sizes):
        sp(b.cuda())
        plain(b.cuda())
        with torch.inference_mode():
            batches.append(net.forward_native(b.cuda(), pooled=True, spatial=True)[1].cpu().numpy())
    assert sp.count == plain.count == 300
    for a, b in zip(sp.get_statistics(), plain.get_statistics()):
        assert np.array_equal(a, b)
    assert np.array_equal(sp.running_var, plain.running_var)
    m, c = sp.get_spatial_statistics()
    rm, rc = chan_recipe(batches)
    x = np.concatenate(batches)
    n = x.shape[0]
    a = np.abs(x).max(0).astype(np.float64) + np.abs(rm)
    B = 8 * n * U * np.outer(a, a) / (n - 1)
    ratio = float(np.max(np.abs(c - rc) / np.where(B > 0, B, 1)))
    print(f"spatial stats 300 x 2023: err/bound {ratio:.3e}")
    assert np.all(np.abs(c - rc) <= B), ratio
    assert np.all(np.abs(m - rm) <= 4 * n * U * a)
    sp.reset()
    assert sp.count == 0 and not any(s.any() for s in sp._states)


def test_torch_routes_return_the_features(offline, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    g = torch.Generator().manual_seed(3)
    xc = (torch.rand(4, 3, 32, 32, generator=g)).cuda()
    model = _model()
    want = spatial_features(_mixed_6d_torch(model, xc))
    # a device list: DataParallel over the torch modules
    dl = M.InceptionStatistics(device=[0], spatial=True)
    with torch.inference_mode():
        act, sp = dl.model(xc)
        assert torch.equal(sp, want)
        dl(xc)
        dl(xc)
    assert dl.count == 8 and dl.get_spatial_statistics()[1].shape == (2023, 2023)
    # gradients wanted
    m = InceptionV3([3], requires_grad=True).eval().cuda()
    out, sp = m(xc, spatial=True)
    assert sp.requires_grad and torch.equal(sp.detach(), want)
    # training-mode BatchNorm (torch path, batch statistics): the same slice of Mixed_6d
    m = _model().train()
    with torch.no_grad():
        out, sp = m(xc, spatial=True)
    sub_want = spatial_features(_mixed_6d_torch(m, xc))
    assert sp.shape == (4, 2023) and torch.equal(sp, sub_want)


def _stats_fp64(net, imgs):
    ref = copy.deepcopy(net).double()
    feats = []
    with torch.inference_mode():
        for b in imgs.split(100):
            feats.append(ref(b.cuda().double(), spatial=True)[1].cpu())
    f = torch.cat(feats).numpy()
    return f.mean(0), np.cov(f, rowvar=False)


def test_sfid_level(offline, record_property):
    g = torch.Generator().manual_seed(11)
    imgs1 = torch.rand(2000, 3, 32, 32, generator=g)
    imgs2 = torch.rand(2000, 3, 32, 32, generator=g) ** 2
    native = M.InceptionStatistics(device=torch.device("cuda"), spatial=True)
    for b in imgs1.split(500):
        native(b.cuda())
    net = native.model._module
    r1m, r1s = _stats_fp64(net, imgs1)
    r2m, r2s = _stats_fp64(net, imgs2)
    sfid_native = M.calc_fd(*native.get_spatial_statistics(), r2m, r2s)
    sfid_ref = M.calc_fd(r1m, r1s, r2m, r2s)
    rel = abs(sfid_native - sfid_ref) / abs(sfid_ref)
    record_property("sfid", (float(sfid_native), float(sfid_ref), float(rel)))
    print(f"sfid native {sfid_native:.6f} fp64 {sfid_ref:.6f} rel {rel:.3e}")
    assert rel <= 1e-2


def test_dead_features_give_a_finite_sfid(monkeypatch, tmp_path):
    """Channels 2 and 5 of Mixed_6d.branch1x1 pushed far below zero before the ReLU: 578 features are 0 on every image, and
    their rows and columns of both covariances are exactly zero."""
    sd = seeded_state_dict(0)
    sd["Mixed_6d.branch1x1.bn.bias"][[2, 5]] = -1e3
    _offline(monkeypatch, tmp_path, sd)
    g = torch.Generator().manual_seed(5)
    stats = []
    for k in range(2):
        ist = M.InceptionStatistics(device=torch.device("cuda"), spatial=True)
        for b in (torch.rand(300, 3, 32, 32, generator=g) ** (k + 1)).split(150):
            ist(b.cuda())
        stats.append(ist.get_spatial_statistics())
    dead = np.zeros(2023, dtype=bool)
    dead[2::7] = dead[5::7] = True
    for m, c in stats:
        assert not m[dead].any() and not c[dead].any() and not c[:, dead].any()
        assert (m[~dead] > 0).any()
    fd, info = M.frechet_distance_native(*stats[0], *stats[1], "cuda")
    live = [(m[~dead], c[~dead][:, ~dead]) for m, c in stats]
    fd_live, _ = M.frechet_distance_native(*live[0], *live[1], "cuda")
    s1, s2 = stats[0][1], stats[1][1]
    floor = 2023 * np.sqrt(U * np.linalg.eigvalsh(s1).max() * np.linalg.eigvalsh(s2).max())
    print(f"dead features: sfid {fd:.6f}, live-only {fd_live:.6f}, min ratios {info['min_ratio']}")
    assert np.isfinite(fd) and info["status"] == 0
    assert abs(fd - fd_live) <= 1e-10 * (np.trace(s1) + np.trace(s2)) + floor


def test_no_device_error():
    assert _lib.lib().ddpm_device_error_flag() == 0
