"""Radiance under a shared direction set: MipNerf.query_radiance_dirs on 2^20 anti-aliased lattice Gaussians with D
directions, its two stages apart, query_radiance on the expanded P * D pairs (alternated with the new query in the same
run), and a degree-2 spherical-harmonic bake of a 512^3 bf16 mesh's vertices.

    python tools/bench_radiance_dirs.py [--log2 20] [--dirs 16 64 256] [--precisions bf16 fp16x3 fp32] [--repeats 3]
                                        [--mesh-res 512] [--out f.json]

Reports, per precision and D: ms per call, G pairs/s and points/s; the level kernel's ms and TFLOP/s (LEVEL_FLOP_PER_POINT,
the MLP up to the view layer's bottleneck GEMM) and the pair kernel's ms and pairs/s, from the library's per-kernel
event timing in a separate pass; at D = 16 the expanded query_radiance.  Reads the card name, power limit and SM clock
in the same run.
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
from mipnerf_pl_b200 import _cabi  # noqa: E402
from tools.bench_field import card, timed  # noqa: E402
from tools.bench_radiance import lattice_points  # noqa: E402

# multiply-adds per point of the view-accumulator launch: layer 0 (96 -> 256), layers 1-7 (layer 5 with the 96 skip
# columns), the density head, extra_layer and the view layer's 256 bottleneck columns
LEVEL_MACS_PER_POINT = 96 * 256 + 6 * 256 * 256 + 352 * 256 + 256 + 256 * 256 + 256 * 128
LEVEL_FLOP_PER_POINT = 2 * LEVEL_MACS_PER_POINT
assert LEVEL_FLOP_PER_POINT == 2 * 606_464


def kernel_ms(fn, names):
    """Per-kernel ms of one call of fn, from the library's event timing."""
    _cabi.lib().mipnerf_b200_profile_enable(1)
    _cabi.profile_snapshot(reset=True)
    fn()
    torch.cuda.synchronize()
    snap = _cabi.profile_snapshot(reset=True)
    _cabi.lib().mipnerf_b200_profile_enable(0)
    return {n: snap[n][1] for n in names}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2", type=int, default=20)
    ap.add_argument("--dirs", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--precisions", nargs="+", default=["bf16", "fp16x3", "fp32"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--mesh-res", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = mp.make_state_dict(seed=0, kind="trained_like")
    means, covs, _ = lattice_points(args.log2, dev)
    pts = means.shape[0]
    rows = []
    for precision in args.precisions:
        model = mp.MipNerf(precision=precision)
        model.load_state_dict(sd)
        model = model.to(dev).eval()
        for nd in args.dirs:
            g = torch.Generator(device=dev).manual_seed(nd)
            dirs = torch.nn.functional.normalize(torch.randn(nd, 3, device=dev, generator=g), dim=-1)
            new = lambda: model.query_radiance_dirs(means, covs, dirs)  # noqa: E731
            new()
            expand = None
            if nd == 16:
                def expand():
                    for d in range(nd):
                        model.query_radiance(means, covs, dirs[d].expand(pts, 3))
                expand()
            t_new, t_exp = [], []
            for _ in range(args.repeats):  # alternated
                t_new += timed(new, 1)
                if expand is not None:
                    t_exp += timed(expand, 1)
            ks = kernel_ms(new, ["radiance_dirs_tc", "radiance_pairs", "linear_f32"])
            ms = float(np.median(t_new))
            pairs = pts * nd
            row = dict(precision=precision, points=pts, dirs=nd, ms=ms, ms_all=t_new, gpairs_per_s=pairs / ms / 1e6,
                       points_per_s=pts / (ms * 1e-3), kernel_ms=ks,
                       pair_kernel_gpairs_per_s=pairs / ks["radiance_pairs"] / 1e6 if ks["radiance_pairs"] else None)
            if precision != "fp32" and ks["radiance_dirs_tc"]:
                row["level_tflops"] = pts * LEVEL_FLOP_PER_POINT / (ks["radiance_dirs_tc"] * 1e-3) / 1e12
            if t_exp:
                e = float(np.median(t_exp))
                row.update(expanded_query_radiance_ms=e, expanded_ms_all=t_exp, speedup_vs_expanded=e / ms)
            rows.append(row)
            print(json.dumps(row), flush=True)
    del means, covs
    # degree-2 SH bake of the vertices of a mesh_res^3 bf16 mesh (128 quadrature directions)
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    res = args.mesh_res
    grid = mp.density_grid(model, res)
    thr = float(torch.quantile(grid.flatten()[::97].float(), 0.9))
    verts, faces = mp.isosurface(grid, thr)
    del grid
    var = mp.voxel_variance(res)
    mp.mesh_sh(model, verts, var, 2)
    t_sh = []
    for _ in range(args.repeats):
        t_sh += timed(lambda: mp.mesh_sh(model, verts, var, 2), 1)
    mesh = dict(resolution=res, vertices=len(verts), degree=2, directions=128, sh_ms=float(np.median(t_sh)),
                sh_ms_all=t_sh)
    print(json.dumps(mesh), flush=True)
    result = dict(card=card(), level_flop_per_point=LEVEL_FLOP_PER_POINT, rows=rows, mesh=mesh)
    print(json.dumps(result["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
