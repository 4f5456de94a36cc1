"""Sparse brick cells for baked grids (`BakedGrid.sparsify`) against the dense cells, on two scenes.

(a) The setting of tools/bench_baked.py: trained-like weights in bf16, seed 0, a 257^3 bake at degree 2 and its 0.7
    density quantile as threshold, at 1 and 3 levels.  The scene fills nearly the whole box.
(b) A model-free surface scene: three concentric spherical shells (`shell_grid`, through `grid_structure`) with seeded
    random SH rows, at 257^3, 513^3 and 1025^3, 1 and 3 levels, degree 2.  Most of the box is empty.

Per grid: kept points, stored bricks against table entries per level, cell MiB and grid MiB dense against sparse,
the sparse .npz size and `sparsify` time (synchronised wall clock), and 800x800 `render_baked_frame` time with the two
layouts alternated in one process (medians of --rounds rounds), with the `grid_render` / `grid_render_bricks` kernel
time from the library's per-launch events (a separate set of rounds).  Each timed frame pair is checked for bit
equality in the run.  Card name, power limit and SM clock are read in the same run.

    python tools/bench_baked_sparse.py [--rounds 5] [--levels 1 3] [--shells 257 513 1025] [--out result.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402
from tools.bench_baked import card, timed  # noqa: E402

DEV = "cuda:0"
SHELL_RADII = (0.5, 0.9, 1.3)
SHELL_HALF_WIDTH = 0.01
SHELL_DENSITY = 40.0


@torch.no_grad()
def shell_grid(resolution, levels, degree=2, seed=0, device=DEV, bounds=mp.field.DEFAULT_BOUNDS):
    """Three concentric spherical shells of density SHELL_DENSITY around radii SHELL_RADII, baked with
    `grid_structure` (threshold half the density) at every level's own lattice, and seeded random SH rows (N(0,
    0.8^2)).  A shell is SHELL_HALF_WIDTH thick on each side, or 0.9 of the level's largest voxel edge where that is
    more, so that no coarse level samples it with holes."""
    dens = []
    for nx, ny, nz in mp.baked.level_resolutions(resolution, levels):
        (xs, ys, zs), step = mp.field.lattice_axes((nx, ny, nz), bounds, device)
        half = max(SHELL_HALF_WIDTH, 0.9 * float(step.max()))
        r = torch.sqrt(zs[:, None, None] ** 2 + ys[None, :, None] ** 2 + xs[None, None, :] ** 2)
        near = torch.zeros_like(r, dtype=torch.bool)
        for radius in SHELL_RADII:
            near |= (r - radius).abs() <= half
        del r
        dens.append(torch.where(near, torch.tensor(SHELL_DENSITY, device=device), torch.tensor(0.0, device=device)))
        del near
    baked, idx, occ = mp.grid_structure(dens, 0.5 * SHELL_DENSITY)
    del dens
    g = torch.Generator(device=device).manual_seed(seed)
    nc = (degree + 1) ** 2
    sh = [0.8 * torch.randn(int((i >= 0).sum()), nc, 3, generator=g, device=device) for i in idx]
    return mp.BakedGrid(baked, idx, sh, occ, bounds, degree)


def npz_bytes(grid, tmp):
    path = os.path.join(tmp, "grid.npz")
    grid.save(path)
    size = os.path.getsize(path)
    os.remove(path)
    return size


def cell_bytes(grid):
    cells = [t for pair in grid.bricks for t in pair] if grid.sparse else grid.cells
    return sum(t.numel() * t.element_size() for t in cells)


def sparsify_timed(grid):
    grid.sparsify()  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = grid.sparsify()
    torch.cuda.synchronize()
    return s, (time.perf_counter() - t0) * 1e3


def frame_times(pair, c2w, rounds):
    """(wall medians, all walls, kernel ms per launch, bit-equal) of 800x800 frames of (dense, sparse), alternated
    every round."""
    first = [mp.render_baked_frame(g, c2w, 800, 800) for g in pair]
    equal = all(torch.equal(a, b) for a, b in zip(*first))
    walls = ([], [])
    for _ in range(rounds):
        frames = []
        for i, g in enumerate(pair):
            dt, out = timed(lambda: mp.render_baked_frame(g, c2w, 800, 800))
            walls[i].append(dt * 1e3)
            frames.append(out)
        equal = equal and all(torch.equal(a, b) for a, b in zip(*frames))
    lib = _cabi.lib()
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    for _ in range(rounds):
        for g in pair:
            mp.render_baked_frame(g, c2w, 800, 800)
    torch.cuda.synchronize()
    lib.mipnerf_b200_profile_enable(0)
    prof = _cabi.profile_snapshot(reset=True)
    kern = [prof[k][1] / max(prof[k][2], 1) for k in ("grid_render", "grid_render_bricks")]
    return [float(np.median(w)) for w in walls], walls, kern, equal


def compare(grid, c2w, rounds, tmp):
    s, ms = sparsify_timed(grid)
    walls, all_walls, kern, equal = frame_times((grid, s), c2w, rounds)
    r = {"kept": grid.kept,
         "stored_bricks / table entries": [[int(p.shape[0]), t.numel()] for t, p in s.bricks],
         "sparsify_ms": round(ms, 1), "frames_bit_equal": equal}
    for i, (name, g) in enumerate((("dense", grid), ("sparse", s))):
        r[name] = {"cells_MiB": round(cell_bytes(g) / 2 ** 20, 1), "grid_MiB": round(g.nbytes / 2 ** 20, 1),
                   "frame_ms_800_median": round(walls[i], 3), "frame_ms_800_all": [round(t, 3) for t in all_walls[i]],
                   "kernel_ms_800": round(kern[i], 3)}
    r["sparse"]["npz_bytes"] = npz_bytes(s, tmp)
    del s
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--levels", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--resolution", type=int, default=257, help="scene (a)'s bake resolution")
    ap.add_argument("--shells", type=int, nargs="+", default=[257, 513, 1025], help="scene (b)'s resolutions")
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args(argv)
    c2w = mp.spheric_path(48)[1::2][3]  # tools/bench_baked_quantize.py's first held-out pose
    res = {"card (name, power limit, SM clock, max SM clock)": card(), "degree": 2}
    with tempfile.TemporaryDirectory() as tmp:
        model = mp.MipNerf(precision="bf16")
        model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
        model = model.to(DEV).eval()
        threshold = float(torch.quantile(mp.density_grid(model, 65).flatten()[::7], 0.7))  # as bench_baked.py
        res["a_trained_like"] = {"precision": "bf16", "weights": "trained_like seed 0", "threshold": threshold,
                                 "resolution": args.resolution}
        for levels in args.levels:
            grid = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
            r = compare(grid, c2w, args.rounds, tmp)
            res["a_trained_like"][f"L{levels}"] = r
            print(json.dumps({f"a_L{levels}": r}), flush=True)
            del grid
            torch.cuda.empty_cache()
        del model
        res["b_shells"] = {"radii": SHELL_RADII, "half_width": SHELL_HALF_WIDTH, "density": SHELL_DENSITY}
        for n in args.shells:
            for levels in args.levels:
                grid = shell_grid(n, levels)
                torch.cuda.empty_cache()
                r = compare(grid, c2w, args.rounds, tmp)
                res["b_shells"][f"{n}_L{levels}"] = r
                print(json.dumps({f"b_{n}_L{levels}": r}), flush=True)
                del grid
                torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
