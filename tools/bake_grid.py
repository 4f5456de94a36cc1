"""Bake a trained MipNeRFSystem checkpoint into a mip-mapped grid of density and SH colour (one .npz), and optionally
render the spheric video path from the grid.

    python tools/bake_grid.py --ckpt last.ckpt --out GRID.npz [--resolution 257] [--levels 1] [--threshold 0.01]
        [--degree 2] [--bounds -1.5 -1.5 -1.5 1.5 1.5 1.5] [--precision bf16] [--prune DATA_DIR]
        [--weight-threshold 1e-5] [--quantize] [--sparse] [--stream-points 16777216] [--frames DIR] [--size 800]

Level l has (n - 1) / 2^l + 1 points per axis (n - 1 divisible by 2^(levels - 1)).  Lattice points farther than one
point from any point of density > threshold are dropped (density 0).  With --prune, the kept points that no pixel of
the Blender scene's train split sees (largest blending weight times colour coefficient <= --weight-threshold over
every training ray, `mp.prune_grid`) are dropped as well, before the grid is saved.  With --quantize, the SH rows are
stored as uint8 with a per-level, per-coefficient affine code (`BakedGrid.quantize`, after any pruning; the .npz is
then format 2).  With --sparse, each level's cells keep only their non-empty bricks of 8^3 points (lossless; the .npz
is then format 3).  Without --prune, --sparse bakes straight into bricks (`mp.bake_grid(sparse=True)`, with
`quantize=True` under --quantize), in z-slabs of about --stream-points lattice points, so that no level's whole
lattice is ever held: the saved arrays are the same as the dense bake's.  With --prune, which needs the dense grid,
the grid is baked dense, pruned, quantized and sparsified last (`BakedGrid.sparsify`).  With --frames, the 120 poses of
`metrics.spheric_path()` are rendered from the grid with `render_baked_frame` and written with `save_images`
(<idx>_rgb.png, _dist.png, _acc.png).  A saved grid renders without the checkpoint: `mp.BakedGrid.load(path)`.
"""
import argparse
import os
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--ckpt", required=True, help="MipNeRFSystem checkpoint (PL layout: state_dict + hyper_parameters)")
    ap.add_argument("--out", required=True, help="the baked grid, .npz")
    ap.add_argument("--resolution", type=int, nargs="+", default=[257], help="n, or nx ny nz (finest level)")
    ap.add_argument("--levels", type=int, default=1, help="mip levels, 1..4")
    ap.add_argument("--threshold", type=float, default=mp.baked.DEFAULT_THRESHOLD)
    ap.add_argument("--degree", type=int, default=2, help="SH degree, 0..3")
    ap.add_argument("--bounds", type=float, nargs=6, default=[-1.5, -1.5, -1.5, 1.5, 1.5, 1.5],
                    metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"))
    ap.add_argument("--precision", default="bf16", choices=sorted(mp._cabi.PRECISIONS))
    ap.add_argument("--prune", default=None, metavar="DATA_DIR",
                    help="prune by visibility from the train split of this Blender scene")
    ap.add_argument("--weight-threshold", type=float, default=mp.baked.DEFAULT_WEIGHT_THRESHOLD)
    ap.add_argument("--quantize", action="store_true", help="store the SH rows in 8 bits (after --prune)")
    ap.add_argument("--sparse", action="store_true", help="keep only the non-empty 8^3 bricks of the cells (last)")
    ap.add_argument("--stream-points", type=int, default=1 << 24,
                    help="lattice points per z-slab of the streamed bake (--sparse without --prune)")
    ap.add_argument("--frames", default=None, metavar="DIR", help="render the spheric path from the grid into DIR")
    ap.add_argument("--size", type=int, default=800, help="frame height and width for --frames")
    ap.add_argument("--device", default="cuda:0")
    return ap.parse_args(argv)


def streamed(args) -> bool:
    """Whether the grid is baked straight into bricks: --sparse without --prune (pruning needs the dense grid)."""
    return bool(args.sparse and not args.prune)


def main(argv=None):
    args = parse_args(argv)
    system = mp.MipNeRFSystem.load_from_checkpoint(args.ckpt, map_location="cpu", precision=args.precision)
    model = system.mip_nerf.to(args.device).eval()
    res = args.resolution[0] if len(args.resolution) == 1 else tuple(args.resolution)
    bounds = (tuple(args.bounds[:3]), tuple(args.bounds[3:]))
    t0 = time.perf_counter()
    stream = streamed(args)
    grid = mp.bake_grid(model, res, levels=args.levels, threshold=args.threshold, degree=args.degree, bounds=bounds,
                        sparse=stream, quantize=stream and args.quantize, stream_points=args.stream_points)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    summary = lambda g: (f"kept points {g.kept}, occupied macro cells {int(g.occupancy.sum())}/"  # noqa: E731
                         f"{g.occupancy.numel()}, {g.nbytes / 2 ** 20:.1f} MiB")
    how = "straight into 8^3 bricks" + (", SH rows in 8 bits" if args.quantize else "") if stream else "dense"
    print(f"baked ({how}): levels {grid.resolutions}, {summary(grid)}, in {t1 - t0:.2f} s, peak "
          f"{torch.cuda.max_memory_allocated(args.device) / 2 ** 20:.0f} MiB allocated")
    if args.prune:
        bank = mp.DeviceRayBank(mp.load_blender_scene(args.prune, "train", white_bkgd=True), args.device)
        t0 = time.perf_counter()
        grid = mp.prune_grid(grid, bank, args.weight_threshold)
        torch.cuda.synchronize()
        print(f"pruned over {bank.num_pixels} training rays at weight threshold {args.weight_threshold:g}: "
              f"{summary(grid)}, in {time.perf_counter() - t0:.2f} s")
    if args.quantize and not stream:
        t0 = time.perf_counter()
        grid = grid.quantize()
        torch.cuda.synchronize()
        print(f"quantized the SH rows to 8 bits: {summary(grid)}, in {time.perf_counter() - t0:.2f} s")
    if args.sparse and not stream:
        print(f"before sparsify: {summary(grid)}")
        t0 = time.perf_counter()
        grid = grid.sparsify()
        torch.cuda.synchronize()
        stored = [f"{int(p.shape[0])}/{t.numel()}" for t, p in grid.bricks]
        print(f"sparsified the cells into 8^3 bricks (stored / table entries per level {stored}): {summary(grid)}, in "
              f"{time.perf_counter() - t0:.2f} s")
    grid.save(args.out)
    print(f"{args.out}: written")
    if args.frames:
        times = []
        for idx, c2w in enumerate(mp.spheric_path()):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rgb, dist, acc = mp.render_baked_frame(grid, c2w, args.size, args.size)
            e1.record()
            mp.save_images(rgb, dist, acc, args.frames, idx)
            times.append(e0.elapsed_time(e1))
        print(f"{args.frames}: {len(times)} frames, median {sorted(times)[len(times) // 2]:.2f} ms per frame")


if __name__ == "__main__":
    main()
