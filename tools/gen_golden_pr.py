"""Generate tests/golden/pr.pt by running the UNMODIFIED reference ``ddpm_torch/metrics/precision_recall.py`` on the CPU
(build container only, where the reference checkout exists):

    python tools/gen_golden_pr.py [OUT_DIR]          # default OUT_DIR: tests/golden

The module is loaded by file path: ``ddpm_torch/metrics/__init__.py`` would pull in ``fid_score`` (torchvision, requests).
``ManifoldBuilder(features=...)`` raises upstream because only the extraction branch sets ``op_device``; the class attribute
``ManifoldBuilder.op_device`` is set before constructing instead of editing the reference.

Recorded:
  * feature pairs (real, fake), VGG-like (relu of a rank-16 projection, the fake latents shifted and widened), quantised to
    multiples of 1/16 so that they are stored as uint8 codes (``real_q`` / ``fake_q``; features = code * ``scale``, exact in
    fp16) and the file stays small: 600 x 64 (with duplicated rows), 150 x 512 and 32 x 4096; for nhood_size in {1, 3, 7}:
    both manifolds' kth and calc_pr's (precision, recall), with the
    row / column batch sizes used (the CPU mirror must use the same ones to match bit for bit);
  * the data paths of the extraction branch through an identity feature extractor (the flattened uint8 images as floats):
    a uint8 tensor (which upstream routes through its dataset branch: a tensor has __getitem__ and __len__) and a map-style
    dataset, each larger than max_sample_size (so a subset is drawn), and ``model.sample_x``
    through ``to_uint8``; their features, kth and the subset indices;
  * ``to_uint8`` of a fixed tensor.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402


def load_pr():
    r = ref_loader.root()
    if r is None:
        raise SystemExit("reference not available")
    path = os.path.join(r, "ddpm_torch", "metrics", "precision_recall.py")
    spec = importlib.util.spec_from_file_location("ref_precision_recall", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


SCALE = 1.0 / 16


def vgg_like(n, W, shift, g):
    """uint8 codes of relu of a rank-16 projection (a low intrinsic dimension, like VGG features) in steps of SCALE;
    shift > 0 moves and widens the latent."""
    z = torch.randn(n, W.shape[0], generator=g) * (1 + shift) + shift
    return (torch.relu(z @ W / 4) / SCALE).round().clamp(0, 255).to(torch.uint8)


class Identity(torch.nn.Module):
    """Stands in for VGG16: the flattened images as fp32 features."""
    def forward(self, x):
        return x.flatten(1).float()


class Images(torch.utils.data.Dataset):
    def __init__(self, x):
        self.x = x

    def __getitem__(self, i):
        return self.x[i], 0

    def __len__(self):
        return len(self.x)


class Sampler:
    """model.sample_x stand-in: n images in [-1.2, 1.2] from a fixed sequence."""
    def __init__(self):
        self.g = torch.Generator().manual_seed(7)

    def sample_x(self, n):
        return torch.rand(n, 3, 4, 4, generator=self.g) * 2.4 - 1.2


def main(out_dir):
    pr = load_pr()
    pr.ManifoldBuilder.op_device = torch.device("cpu")
    g = torch.Generator().manual_seed(2024)
    fx = dict(cases=[], nhoods=(1, 3, 7))
    # batch sizes: upstream's CPU cdist has no fp16 kernel for blocks of <= 25 rows AND <= 25 columns
    for n, d, rb, cb in ((600, 64, 256, 200), (150, 512, 100, 128), (32, 4096, 32, 32)):
        W = torch.randn(16, d, generator=g)
        real_q, fake_q = vgg_like(n, W, 0.0, g), vgg_like(n, W, 0.15, g)
        if d == 64:                      # duplicated rows: exact zero distances beside the self-distance
            real_q[1::50] = real_q[0::50][: len(real_q[1::50])]
            fake_q[5:15] = real_q[5:15]
        real, fake = real_q.half() * SCALE, fake_q.half() * SCALE
        case = dict(real_q=real_q, fake_q=fake_q, scale=SCALE, row_batch_size=rb, col_batch_size=cb, results={})
        for k in fx["nhoods"]:
            mr = pr.ManifoldBuilder(features=real, nhood_size=k, row_batch_size=rb, col_batch_size=cb)
            mf = pr.ManifoldBuilder(features=fake, nhood_size=k, row_batch_size=rb, col_batch_size=cb)
            p, r = pr.calc_pr(mf.manifold, mr.manifold, row_batch_size=rb, col_batch_size=cb, device="cpu")
            case["results"][k] = dict(kth_real=mr.kth, kth_fake=mf.kth, precision=p, recall=r)
            print(f"{n}x{d} nhood {k}: precision {p.item():.5f} recall {r.item():.5f}")
        fx["cases"].append(case)

    # extraction branch, identity extractor
    pr.VGGFeatureExtractor = Identity
    imgs = torch.randint(0, 256, (300, 3, 4, 4), generator=g, dtype=torch.uint8)
    data = {}
    kw = dict(extr_batch_size=64, max_sample_size=200, nhood_size=3, row_batch_size=128, col_batch_size=100, random_state=1234)
    for name, src in (("tensor", dict(data=imgs)), ("dataset", dict(data=Images(imgs))), ("model", dict(model=Sampler()))):
        m = pr.ManifoldBuilder(**kw, **src)
        entry = dict(features=m.features, kth=m.kth)
        if name != "model":              # which images were drawn, in order (the images are distinct)
            flat = imgs.flatten(1).half()
            entry["inds"] = torch.tensor([int(torch.nonzero((flat == row).all(1))[0]) for row in m.features])
        data[name] = entry
    np.random.seed(1234)
    assert torch.equal(data["tensor"]["inds"], torch.as_tensor(np.random.choice(300, size=200, replace=False)))
    fx["data"] = dict(images=imgs, kwargs=kw, results=data)
    x = torch.linspace(-1.3, 1.3, 1001)
    fx["to_uint8"] = dict(x=x, y=pr.to_uint8(x))
    os.makedirs(out_dir, exist_ok=True)
    torch.save(fx, os.path.join(out_dir, "pr.pt"))
    print("pr.pt written to", out_dir)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
