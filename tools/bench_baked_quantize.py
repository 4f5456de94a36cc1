"""8-bit SH rows for baked grids (`BakedGrid.quantize`) on trained-like weights in bf16, in the setting of
tools/bench_baked_prune.py: a 257^3 bake at 1 and 3 levels, degree 2, a training bank of MLP renders at 24 spheric-path
poses (200x200) and 2 held-out poses between them.  Per level count, three fp32 grids: unpruned, pruned at the 1e-5
default (`prune_grid`), and that grid after --steps `finetune_grid` steps; each against its quantized copy: grid MiB and
.npz bytes, quantize time (synchronised wall clock), 800x800 `render_baked_frame` time with the two storage types
alternated in one process (medians of --rounds rounds) and the `grid_render` / `grid_render_u8` kernel time from the
library's per-launch events (a separate set of rounds), held-out PSNR / SSIM against the MLP at 800x800 and 200x200,
and the PSNR of the u8 frames against the fp32 grid's own frames.  Card name, power limit and SM clock are read in the
same run.

    python tools/bench_baked_quantize.py [--steps 1000] [--rounds 5] [--levels 1 3] [--out result.json]
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
from tools.bench_baked_finetune import distill_scene, quality  # noqa: E402

DEV = "cuda:0"


def npz_bytes(grid, tmp):
    path = os.path.join(tmp, "grid.npz")
    grid.save(path)
    size = os.path.getsize(path)
    os.remove(path)
    return size


def quantize_timed(grid):
    grid.quantize()  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    q = grid.quantize()
    torch.cuda.synchronize()
    return q, (time.perf_counter() - t0) * 1e3


def frame_times(pair, c2w, rounds):
    """(wall medians, all walls, kernel ms per launch) of 800x800 frames of (fp32, u8), alternated every round."""
    for g in pair:
        mp.render_baked_frame(g, c2w, 800, 800)
    walls = ([], [])
    for _ in range(rounds):
        for i, g in enumerate(pair):
            walls[i].append(timed(lambda: mp.render_baked_frame(g, c2w, 800, 800))[0] * 1e3)
    lib = _cabi.lib()
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    for _ in range(rounds):
        for g in pair:
            mp.render_baked_frame(g, c2w, 800, 800)
    torch.cuda.synchronize()
    lib.mipnerf_b200_profile_enable(0)
    prof = _cabi.profile_snapshot(reset=True)
    kern = [prof[k][1] / max(prof[k][2], 1) for k in ("grid_render", "grid_render_u8")]
    return [float(np.median(w)) for w in walls], walls, kern


def self_psnr(pair, poses, size):
    """Mean PSNR of the u8 grid's frames against the fp32 grid's own frames (inf where they are identical)."""
    vals = []
    for c2w in poses:
        a = mp.render_baked_frame(pair[0], c2w, size, size)[0]
        b = mp.render_baked_frame(pair[1], c2w, size, size)[0]
        mse = float(((a - b) ** 2).mean())
        vals.append(float("inf") if mse == 0 else -10 * np.log10(mse))
    return round(float(np.mean(vals)), 2)


def compare(model, grid, held, rounds, tmp):
    q, qms = quantize_timed(grid)
    walls, all_walls, kern = frame_times((grid, q), held[0], rounds)
    r = {"kept": grid.kept, "quantize_ms": round(qms, 2)}
    for i, (name, g) in enumerate((("fp32", grid), ("u8", q))):
        r[name] = {"MiB": round(g.nbytes / 2 ** 20, 1), "npz_bytes": npz_bytes(g, tmp),
                   "frame_ms_800_median": round(walls[i], 3), "frame_ms_800_all": [round(t, 3) for t in all_walls[i]],
                   "kernel_ms_800": round(kern[i], 3),
                   "psnr_ssim_800": quality(model, g, held, 800), "psnr_ssim_200": quality(model, g, held, 200)}
    r["u8_vs_fp32_frame_psnr_800"] = self_psnr((grid, q), held, 800)
    del q
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--resolution", type=int, default=257)
    ap.add_argument("--train-poses", type=int, default=24)
    ap.add_argument("--train-size", type=int, default=200)
    ap.add_argument("--levels", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args(argv)
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    threshold = float(torch.quantile(mp.density_grid(model, 65).flatten()[::7], 0.7))  # as bench_baked.py
    path = mp.spheric_path(2 * args.train_poses)
    train, held = path[0::2], path[1::2][[3, 11]]  # held-out poses lie between training poses
    bank = mp.DeviceRayBank(distill_scene(model, train, args.train_size), DEV)
    res = {"card (name, power limit, SM clock, max SM clock)": card(), "precision": "bf16",
           "weights": "trained_like seed 0", "threshold": threshold, "resolution": args.resolution, "degree": 2,
           "scene": f"{args.train_poses} training poses at {args.train_size}x{args.train_size} "
                    f"({bank.num_pixels} rays), 2 held-out poses", "steps": args.steps, "batch": args.batch}
    with tempfile.TemporaryDirectory() as tmp:
        for levels in args.levels:
            grid = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
            r = {"unpruned": compare(model, grid, held, args.rounds, tmp)}
            pruned = mp.prune_grid(grid, bank)
            del grid
            torch.cuda.empty_cache()
            r["pruned_1e-5"] = compare(model, pruned, held, args.rounds, tmp)
            gen = torch.Generator(device=DEV).manual_seed(0)
            mp.finetune_grid(pruned, bank, args.steps, args.batch, generator=gen)
            pruned.requires_grad_(False)
            torch.cuda.empty_cache()
            r[f"pruned_1e-5_finetuned_{args.steps}"] = compare(model, pruned, held, args.rounds, tmp)
            res[f"L{levels}"] = r
            print(json.dumps({f"L{levels}": r}), flush=True)
            del pruned
            torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
