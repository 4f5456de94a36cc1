"""Extract the density isosurface of a trained MipNeRFSystem checkpoint as a binary PLY.

    python tools/extract_mesh.py --ckpt last.ckpt --threshold 50 --out mesh.ply \
        [--resolution 256] [--bounds -1.5 -1.5 -1.5 1.5 1.5 1.5] [--precision bf16] [--point-sampled] [--colors] [--sh DEGREE]

The density is queried on a resolution^3 lattice over the bounds (each lattice point the Gaussian of its voxel unless
--point-sampled), and the surface density > threshold is extracted with marching tetrahedra on the GPU.  With
--colors the PLY also carries vertex normals (from the grid's gradient) and colours: the field's radiance at each
vertex's Gaussian, seen along the inward normal.  With --sh DEGREE the view-dependent colour of each vertex's Gaussian
is also baked into real spherical harmonics of that degree (0..3, `mp.mesh_sh`) and written as `coeffs` [V, K, 3]
float32 to OUT-without-extension.sh.npz, with `degree` and `convention`; the PLY is the same as without --sh.
"""
import argparse
import os
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402

SH_CONVENTION = ("real SH, eval_sh convention (C0 = 0.28209479177387814, Y1..3 = -C1 y, C1 z, -C1 x, ...); "
                 "colour(dir) = sum_k Y_k(dir) coeffs[v, k, :] (mipnerf_pl_b200.eval_sh)")


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--ckpt", required=True, help="MipNeRFSystem checkpoint (PL layout: state_dict + hyper_parameters)")
    ap.add_argument("--threshold", type=float, required=True, help="density level of the surface")
    ap.add_argument("--resolution", type=int, nargs="+", default=[256], help="n, or nx ny nz")
    ap.add_argument("--bounds", type=float, nargs=6, default=[-1.5, -1.5, -1.5, 1.5, 1.5, 1.5],
                    metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"))
    ap.add_argument("--precision", default="bf16", choices=sorted(mp._cabi.PRECISIONS))
    ap.add_argument("--point-sampled", action="store_true", help="zero covariance instead of the voxel's")
    ap.add_argument("--colors", action="store_true", help="add vertex normals and colours (query_radiance)")
    ap.add_argument("--sh", type=int, default=None, metavar="DEGREE",
                    help="also bake spherical-harmonic colour coefficients of this degree (0..3) into OUT.sh.npz")
    ap.add_argument("--out", required=True)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args(argv)
    system = mp.MipNeRFSystem.load_from_checkpoint(args.ckpt, map_location="cpu", precision=args.precision)
    model = system.mip_nerf.to(args.device).eval()
    res = args.resolution[0] if len(args.resolution) == 1 else tuple(args.resolution)
    bounds = (tuple(args.bounds[:3]), tuple(args.bounds[3:]))
    t0 = time.perf_counter()
    grid = mp.density_grid(model, res, bounds, variance=0.0 if args.point_sampled else None)
    normals = colors = None
    if args.colors:
        verts, faces, normals = mp.isosurface(grid, args.threshold, bounds, normals=True)
        colors = mp.mesh_colors(model, verts, normals, 0.0 if args.point_sampled else mp.voxel_variance(res, bounds))
    else:
        verts, faces = mp.isosurface(grid, args.threshold, bounds)
    coeffs = None
    if args.sh is not None:
        coeffs = mp.mesh_sh(model, verts, 0.0 if args.point_sampled else mp.voxel_variance(res, bounds), args.sh)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    mp.write_ply(args.out, verts, faces, colors=colors, normals=normals)
    if coeffs is not None:
        sh_path = os.path.splitext(args.out)[0] + ".sh.npz"
        np.savez(sh_path, coeffs=coeffs.cpu().numpy(), degree=np.int32(args.sh), convention=np.str_(SH_CONVENTION))
        print(f"{sh_path}: SH coefficients {tuple(coeffs.shape)}")
    print(f"{args.out}: {len(verts)} vertices, {len(faces)} faces (grid {tuple(grid.shape[::-1])}, density "
          f"{float(grid.min()):.3g}..{float(grid.max()):.3g}, {t1 - t0:.2f} s on the GPU)")


if __name__ == "__main__":
    main()
