"""Generate tests/golden/fid.pt by running the UNMODIFIED reference ``ddpm_torch/metrics/{inception,fid_score}.py`` on the CPU
(build container only, where the reference checkout exists):

    python tools/gen_golden_fid.py [OUT_DIR]          # default OUT_DIR: tests/golden

The environment is patched, never the reference: ``load_state_dict_from_url`` returns ``seeded_state_dict(SEED)``
(ddpm_torch_b200/inception.py, the rule the tests apply too), and ``scipy.linalg.sqrtm`` accepts and drops the ``disp`` keyword
that SciPy has removed (returning ``(sqrtm(A), None)`` when it is given, as old SciPy did).

Recorded:
  * InceptionV3 features of three 3 x 32 x 32 images in [-1, 1] for every block index: block 3 in full, blocks 0-2 as a seeded
    subset of elements (``idx{b}`` / ``val{b}``);
  * InceptionStatistics running values (population) and get_statistics() after batches of sizes 1, 1, 5, 2, 9, 3 of D = 64
    features fed straight to the statistics (the extractor replaced by the identity on [B, D, 1, 1] and the running arrays
    sized for D);
  * calc_fd values and inputs at D in {8, 64, 192}: full rank (D = 8, 64), rank-deficient (D = 64), identical inputs (D = 192), and a non-PSD input on which
    the reference raises ValueError (recorded as ``None``).
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from ddpm_torch_b200.inception import seeded_state_dict  # noqa: E402

SEED = 0
STAT_SIZES = [1, 1, 5, 2, 9, 3]


class AsMaps(torch.nn.Module):
    """Stands in for Inception in the statistics: [B, D] features as [B, D, 1, 1] maps."""
    def forward(self, t):
        return t[:, :, None, None]


def patch_env():
    import scipy.linalg
    orig = scipy.linalg.sqrtm

    def sqrtm(A, disp=None, **kw):
        r = orig(A, **kw)
        return (r, None) if disp is False else r
    scipy.linalg.sqrtm = sqrtm
    import torch.utils.model_zoo
    import torch.hub
    sd = seeded_state_dict(SEED)
    torch.hub.load_state_dict_from_url = torch.utils.model_zoo.load_url = lambda *a, **k: {k2: v.clone() for k2, v in sd.items()}


def load_ref():
    r = ref_loader.root()
    if r is None:
        raise SystemExit("reference not available")
    ref_loader.load()
    return importlib.import_module("ddpm_torch.metrics.inception"), importlib.import_module("ddpm_torch.metrics.fid_score")


def fd_inputs(D, n1, n2, seed, psd=True):
    g = np.random.default_rng(seed)
    W = g.standard_normal((D, D)) / np.sqrt(D)
    x1 = np.maximum(g.standard_normal((n1, D)) @ W, 0)
    x2 = np.maximum((g.standard_normal((n2, D)) * 1.2 + 0.1) @ W, 0)
    s2 = np.cov(x2, rowvar=False)
    if not psd:
        s2 = s2 - 0.5 * np.linalg.eigvalsh(s2).max() * np.eye(D)
    return x1.mean(0), np.cov(x1, rowvar=False), x2.mean(0), s2


def main(out_dir):
    patch_env()
    inc, fid = load_ref()
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)
    imgs = torch.rand(3, 3, 32, 32, generator=g) * 2 - 1
    net = inc.InceptionV3([0, 1, 2, 3]).eval()
    with torch.inference_mode():
        feats = net(imgs)
    out = {"seed": SEED, "images": imgs, "block3": feats[3].clone()}
    for b in range(3):
        f = feats[b].flatten()
        idx = torch.randperm(f.numel(), generator=g)[:4000]
        out[f"idx{b}"], out[f"val{b}"] = idx.to(torch.int32).clone(), f[idx].clone()

    istats = fid.InceptionStatistics(activation_dim=2048)
    x = torch.as_tensor(np.maximum(np.random.default_rng(2).standard_normal((sum(STAT_SIZES), 64)), 0) * 3, dtype=torch.float32)
    istats.model = AsMaps()
    istats.running_mean, istats.running_var = np.zeros(64), np.zeros((64, 64))
    for b in x.split(STAT_SIZES):
        istats(b)
    m, v = istats.get_statistics()
    out["stats"] = {"features": x, "sizes": STAT_SIZES, "running_mean": istats.running_mean.copy(),
                    "running_var": istats.running_var.copy(), "mean": m, "cov": v}

    cases = []
    for i, (D, n1, n2, psd, same) in enumerate([(8, 200, 300, True, False), (64, 2000, 1500, True, False),
                                                (64, 40, 50, True, False), (192, 3000, 3000, True, True),
                                                (8, 200, 300, False, False)]):
        mu1, s1, mu2, s2 = fd_inputs(D, n1, n2, 10 + i, psd)
        if same:
            mu2, s2 = mu1, s1
        try:
            val = float(fid.calc_fd(mu1, s1, mu2, s2))
        except ValueError:
            val = None
        cases.append({"D": D, "mu1": mu1, "sigma1": s1, "mu2": mu2, "sigma2": s2, "fd": val, "psd": psd})
    out["fd"] = cases
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "fid.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
