"""Generate tests/golden/radiance.npz FROM THE REFERENCE ITSELF: the radiance of the field at Gaussians, each point seen
from its own direction.

Run with a checkout of the reference (MIPNERF_REFERENCE=<path>):

    python tests/golden/make_golden_radiance.py

It imports the unmodified hjxwhy/mipnerf_pl `models.mip.integrated_pos_enc`, `models.mip.pos_enc` and
`models.mip_nerf.MLP`, and runs `MLP.forward(x [P,1,xyz_dim], pos_enc(viewdirs) [P,view_dim])` on CPU (fp32) at the
points and covariances of field.npz (make_golden_field.points), with random unit directions, for the same three weight
cases.  It stores the directions and the raw rgb / raw density MLP.forward returns.  Nothing from the reference's source
is copied; only its numerical outputs are recorded.
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
sys.path.insert(2, HERE)

from models import mip as ref_mip  # noqa: E402  (reference)
from models.mip_nerf import MipNerf as RefMipNerf  # noqa: E402  (reference)

from make_golden_field import CASES, NUM_POINTS, points  # noqa: E402  (the points of field.npz)
from mipnerf_pl_b200.weights import make_state_dict  # noqa: E402  (ours: weight generator only)

torch.set_num_threads(8)


def directions(seed):
    """NUM_POINTS random unit directions."""
    g = torch.Generator().manual_seed(200 + seed)
    d = torch.randn(NUM_POINTS, 3, generator=g)
    return d / d.norm(dim=-1, keepdim=True)


def main():
    out = {}
    for tag, seed, kind, max_deg, deg_view in CASES:
        model = RefMipNerf(max_deg_point=max_deg, deg_view=deg_view)
        model.load_state_dict(make_state_dict(seed=seed, kind=kind, xyz_dim=6 * max_deg, view_dim=6 * deg_view + 3))
        model.eval()
        means, covs = points(seed)
        dirs = directions(seed)
        out[f"{tag}_means"] = means.numpy()
        out[f"{tag}_viewdirs"] = dirs.numpy()
        out[f"{tag}_meta"] = np.array([seed, max_deg, deg_view], dtype=np.int64)
        for cname, cov in covs.items():
            with torch.no_grad():
                enc = ref_mip.integrated_pos_enc((means[:, None], cov[:, None]), 0, max_deg)  # [P,1,xyz_dim]
                venc = ref_mip.pos_enc(dirs, 0, deg_view, True)                               # [P,view_dim]
                raw_rgb, raw_density = model.mlp(enc, venc)
            out[f"{tag}_covs_{cname}"] = cov.numpy()
            out[f"{tag}_raw_rgb_{cname}"] = raw_rgb[:, 0].numpy()
            out[f"{tag}_raw_density_{cname}"] = raw_density[:, 0, 0].numpy()
    path = os.path.join(HERE, "radiance.npz")
    np.savez_compressed(path, **out)
    print(f"radiance.npz: {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()
