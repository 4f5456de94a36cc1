"""Generate tests/golden/field.npz FROM THE REFERENCE ITSELF: the density of the field at Gaussians off any ray.

Run with a checkout of the reference (MIPNERF_REFERENCE=<path>):

    python tests/golden/make_golden_field.py

It imports the unmodified hjxwhy/mipnerf_pl `models.mip.integrated_pos_enc` and `models.mip_nerf.MLP`, runs them on
CPU (fp32) on deterministic points with zero, isotropic and anisotropic covariances, for xavier and trained_like
weights and one narrow encoding (max_deg_point=10, deg_view=2), and stores inputs and the raw density MLP.forward
returns.  Nothing from the reference's source is copied; only its numerical outputs are recorded.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
REF = os.environ.get("MIPNERF_REFERENCE", "")
sys.path.insert(0, REF)
sys.path.insert(1, ROOT)

from models import mip as ref_mip  # noqa: E402  (reference)
from models.mip_nerf import MipNerf as RefMipNerf  # noqa: E402  (reference)

from mipnerf_pl_b200.weights import make_state_dict  # noqa: E402  (ours: weight generator only)

torch.set_num_threads(8)

# (tag, seed, weights kind, max_deg_point, deg_view)
CASES = (("xavier", 0, "xavier", 16, 4), ("trained_like", 1, "trained_like", 16, 4),
         ("deg10_view2", 6, "trained_like", 10, 2))
NUM_POINTS = 512


def points(seed):
    """Means in [-1.5, 1.5]^3 and three covariance sets: zero, isotropic, anisotropic (log-uniform 1e-6 .. 1e-1)."""
    g = torch.Generator().manual_seed(100 + seed)
    means = 3.0 * torch.rand(NUM_POINTS, 3, generator=g) - 1.5
    iso = (10 ** (-6 + 5 * torch.rand(NUM_POINTS, 1, generator=g))).expand(NUM_POINTS, 3).contiguous()
    aniso = 10 ** (-6 + 5 * torch.rand(NUM_POINTS, 3, generator=g))
    return means, {"zero": torch.zeros(NUM_POINTS, 3), "iso": iso, "aniso": aniso}


def main():
    out = {}
    for tag, seed, kind, max_deg, deg_view in CASES:
        model = RefMipNerf(max_deg_point=max_deg, deg_view=deg_view)
        model.load_state_dict(make_state_dict(seed=seed, kind=kind, xyz_dim=6 * max_deg, view_dim=6 * deg_view + 3))
        model.eval()
        means, covs = points(seed)
        out[f"{tag}_means"] = means.numpy()
        out[f"{tag}_meta"] = np.array([seed, max_deg, deg_view], dtype=np.int64)
        for cname, cov in covs.items():
            with torch.no_grad():
                enc = ref_mip.integrated_pos_enc((means[None], cov[None]), 0, max_deg)
                # the colour branch needs a view input; the raw density does not read it
                _, raw_density = model.mlp(enc, torch.zeros(1, 6 * deg_view + 3))
            out[f"{tag}_covs_{cname}"] = cov.numpy()
            out[f"{tag}_raw_{cname}"] = raw_density[0, :, 0].numpy()
    path = os.path.join(HERE, "field.npz")
    np.savez_compressed(path, **out)
    print(f"field.npz: {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()
