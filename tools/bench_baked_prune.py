"""Pruning baked grids by visibility (`prune_grid`) on trained-like weights in bf16, in the setting of
tools/bench_baked_finetune.py: a 257^3 bake at 1 and 3 levels, degree 2, and a training bank of MLP renders at 24
spheric-path poses (200x200) with 2 held-out poses between them.  Per grid: the visibility pass over every pixel of
the bank (synchronised wall clock, and kernel time from the library's per-launch events); then per weight threshold of
the sweep the kept points per level, grid memory, occupied macro cells, the 800x800 `render_baked_frame` time against
the unpruned grid (alternated rounds, medians) and held-out PSNR / SSIM against the MLP at 200x200 and 800x800; then
a `finetune_grid` of --steps steps of the unpruned grid and of every pruned one: step time split into forward,
backward and Adam, gradient and Adam-state memory, held-out quality after.  Card name, power limit and SM clock are
read in the same run.

    python tools/bench_baked_prune.py [--steps 1000] [--rounds 5] [--levels 1 3] [--out result.json]
"""
import argparse
import json
import os
import sys
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
SWEEP = (0.0, 1e-5, 1e-4, 3e-4, 1e-3, 1e-2, 1e-1)


def grid_stats(grid):
    return {"kept": grid.kept, "MiB": round(grid.nbytes / 2 ** 20, 1),
            "occupied_macro_cells": f"{int(grid.occupancy.sum())} / {grid.occupancy.numel()}"}


def visibility_pass(grid, bank, batch):
    """prune_grid's scores over the whole bank: (scores, wall ms, kernel ms, launches)."""
    lib = _cabi.lib()
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    scores = [torch.zeros(m, device=DEV) for m in grid.kept]
    for s in range(0, bank.num_pixels, batch):
        rays, _ = bank.rays(torch.arange(s, min(s + batch, bank.num_pixels), device=DEV))
        grid.visibility(rays, out=scores)
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    lib.mipnerf_b200_profile_enable(0)
    n, ms, _ = _cabi.profile_snapshot(reset=True)["grid_visibility"]
    return scores, wall, ms, n


def finetune(grid, bank, steps, batch):
    """One finetune_grid call: wall ms per step, per-step kernel split, memory of gradients and Adam state."""
    lib = _cabi.lib()
    gen = torch.Generator(device=DEV).manual_seed(0)
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    losses = mp.finetune_grid(grid, bank, steps, batch, generator=gen)
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / steps
    lib.mipnerf_b200_profile_enable(0)
    prof = _cabi.profile_snapshot(reset=True)
    nparam = sum(p.numel() for p in grid.parameters())
    return {"step_ms_wall": round(wall, 3),
            "kernel_ms_per_step": {k: round(prof[k][1] / steps, 3) for k in ("grid_render", "grid_render_backward",
                                                                              "adam")},
            "loss_first_last_50": [round(float(np.mean(losses[:50])), 6), round(float(np.mean(losses[-50:])), 6)],
            "grad_MiB": round(nparam * 4 / 2 ** 20, 1), "adam_state_MiB": round(2 * nparam * 4 / 2 ** 20, 1)}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--resolution", type=int, default=257)
    ap.add_argument("--train-poses", type=int, default=24)
    ap.add_argument("--train-size", type=int, default=200)
    ap.add_argument("--levels", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--vis-batch", type=int, default=1 << 20, help="rays per visibility call")
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
    for levels in args.levels:
        grid = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
        r = {"unpruned": grid_stats(grid)}
        visibility_pass(grid, bank, args.vis_batch)  # warm-up
        scores, wall, kern, n = visibility_pass(grid, bank, args.vis_batch)
        r["visibility"] = {"wall_ms": round(wall, 3), "kernel_ms": round(kern, 3), "launches": n,
                           "rays_per_s_M": round(bank.num_pixels / (wall * 1e-3) / 1e6, 1)}
        grids = {"unpruned": grid}
        for t in SWEEP:
            grids[f"t={t:g}"] = grid.prune(scores, t)
            r[f"t={t:g}"] = grid_stats(grids[f"t={t:g}"])
        del scores
        for name, g in grids.items():
            for size in (200, 800):
                r[name][f"psnr_ssim_{size}"] = quality(model, g, held, size)
        # 800x800 frames at the first held-out pose, every grid once per round
        for g in grids.values():
            mp.render_baked_frame(g, held[0], 800, 800)
        times = {name: [] for name in grids}
        for _ in range(args.rounds):
            for name, g in grids.items():
                times[name].append(timed(lambda: mp.render_baked_frame(g, held[0], 800, 800))[0] * 1e3)
        for name in grids:
            r[name]["frame_ms_800_median"] = round(float(np.median(times[name])), 3)
            r[name]["frame_ms_800_all"] = [round(t, 3) for t in times[name]]
        # fine-tuning: warm up every shape on a throwaway copy, then one call per grid (each is tuned in place)
        warm = grid.prune([torch.ones(m, device=DEV) for m in grid.kept], 0.0)
        mp.finetune_grid(warm, bank, 20, args.batch)
        del warm
        for name in list(grids):
            g = grids.pop(name)
            r[name]["finetune"] = finetune(g, bank, args.steps, args.batch)
            for size in (200, 800):
                r[name]["finetune"][f"psnr_ssim_{size}_after"] = quality(model, g, held, size)
            del g
            torch.cuda.empty_cache()
        res[f"L{levels}"] = r
        del grid
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
