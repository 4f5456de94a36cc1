"""Radiance-query throughput: MipNerf.query_radiance alternated with MipNerf.query_density on the same points, with
device events; plus a coloured mesh extraction split into its stages.

    python tools/bench_radiance.py [--sizes 22 24] [--precisions bf16 fp16x3 fp32] [--repeats 3] [--mesh-res 512]
                                   [--out f.json]

The points are the anti-aliased Gaussians of a lattice over the default bounds (2^k points, variance step^2 / 12 per
axis, as density_grid queries them), each with a random unit direction.  Reports ms per query, points/s and TFLOP/s
(FLOP_PER_POINT for the radiance, bench_field's trunk count for the density), and the card name, power limit and SM
clock of the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200.field import lattice_axes  # noqa: E402
from tools.bench_field import FLOP_PER_POINT as DENSITY_FLOP_PER_POINT, card, timed  # noqa: E402

# multiply-adds per point: the trunk and density head (bench_field), extra_layer 256x256, view layer 283x128, colour
# head 128x3
MACS_PER_POINT = 96 * 256 + 6 * 256 * 256 + 352 * 256 + 256 + 256 * 256 + 283 * 128 + 128 * 3
FLOP_PER_POINT = 2 * MACS_PER_POINT
assert FLOP_PER_POINT == 2 * 610_304


def lattice_points(log2, dev, seed=0):
    """2^log2 lattice Gaussians (nx = 2 ny = 2 nz or a cube) with random unit directions."""
    e = [log2 // 3 + (1 if log2 % 3 > i else 0) for i in range(3)]
    res = tuple(1 << k for k in e)
    (xs, ys, zs), step = lattice_axes(res, mp.field.DEFAULT_BOUNDS, dev)
    z, y, x = torch.meshgrid(zs, ys, xs, indexing="ij")
    means = torch.stack([x, y, z], -1).reshape(-1, 3)
    covs = torch.tensor(step ** 2 / np.float32(12), device=dev).expand(means.shape[0], 3).contiguous()
    g = torch.Generator(device=dev).manual_seed(seed)
    dirs = torch.randn(means.shape[0], 3, device=dev, generator=g)
    return means, covs, torch.nn.functional.normalize(dirs, dim=-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[22, 24], help="log2 of the point counts")
    ap.add_argument("--precisions", nargs="+", default=["bf16", "fp16x3", "fp32"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--mesh-res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = mp.make_state_dict(seed=0, kind="trained_like")
    rows = []
    for log2 in args.sizes:
        means, covs, dirs = lattice_points(log2, dev)
        pts = means.shape[0]
        for precision in args.precisions:
            model = mp.MipNerf(precision=precision)
            model.load_state_dict(sd)
            model = model.to(dev).eval()
            rad = lambda: model.query_radiance(means, covs, dirs)  # noqa: E731
            dens = lambda: model.query_density(means, covs)  # noqa: E731
            rgb, d_rad = rad()                               # warm-up of both, and their densities compared
            d_only = dens()
            same_density = bool(torch.equal(d_rad, d_only))
            del rgb, d_rad, d_only
            t_rad, t_dens = [], []
            for _ in range(args.repeats):                    # alternated
                t_rad += timed(rad, 1)
                t_dens += timed(dens, 1)
            for name, ts, flop in (("query_radiance", t_rad, FLOP_PER_POINT),
                                   ("query_density", t_dens, DENSITY_FLOP_PER_POINT)):
                ms = float(np.median(ts))
                rows.append(dict(precision=precision, points=pts, method=name, ms=ms, ms_all=ts,
                                 points_per_s=pts / (ms * 1e-3), tflops=pts * flop / (ms * 1e-3) / 1e12,
                                 density_equal_to_query_density=same_density))
                print(json.dumps(rows[-1]), flush=True)
        del means, covs, dirs
    # coloured mesh at mesh_res^3 (bf16), by stage: density grid, isosurface + normals, colours
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    res = args.mesh_res
    grid = mp.density_grid(model, res)
    thr = float(torch.quantile(grid.flatten()[::97].float(), 0.9))
    verts, faces, normals = mp.isosurface(grid, thr, normals=True)
    var = mp.voxel_variance(res)
    mp.mesh_colors(model, verts, normals, var)
    stages = {"grid": [], "isosurface": [], "isosurface+normals": [], "colors": []}
    for _ in range(args.repeats):
        stages["grid"] += timed(lambda: mp.density_grid(model, res), 1)
        stages["isosurface"] += timed(lambda: mp.isosurface(grid, thr), 1)
        stages["isosurface+normals"] += timed(lambda: mp.isosurface(grid, thr, normals=True), 1)
        stages["colors"] += timed(lambda: mp.mesh_colors(model, verts, normals, var), 1)
    mesh = dict(resolution=res, threshold=thr, vertices=len(verts), faces=len(faces),
                **{f"{k}_ms": float(np.median(v)) for k, v in stages.items()},
                normals_ms=float(np.median(stages["isosurface+normals"]) - np.median(stages["isosurface"])))
    print(json.dumps(mesh), flush=True)
    result = dict(card=card(), flop_per_point=FLOP_PER_POINT, rows=rows, mesh=mesh)
    print(json.dumps(result["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
