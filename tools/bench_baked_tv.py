"""The total-variation prior in fine-tuning baked grids (`finetune_grid(tv_density=, tv_sh=)`) on trained-like weights
in bf16, in the setting of tools/bench_baked_prune.py: a 257^3 bake, degree 2, a training bank of MLP renders at 24
spheric-path poses (200x200) and 2 held-out poses between them.  Each level count of --levels is run on the unpruned
grid and on the grid pruned at 1e-5 (`prune_grid`).  On the first level count every weight pair of the --tv-density x
--tv-sh sweep (0/0 included) fine-tunes a copy of each grid; then the best pair by held-out 200x200 SSIM also runs
with lr_sh = 0.03 (against 0/0 at that rate), and on the other level counts 0/0 and the best pair run.  Per run:
held-out PSNR / SSIM at 200x200 and 800x800 against the MLP's fine frames, the synchronised wall clock per step, its
split into forward, backward, TV kernel and Adam (the library's per-launch events, on during the call) and the sync
(CUDA events, timed alone), and the peak memory the fine-tune adds over the grid.  The TV kernel alone is timed by CUDA
events per launch in both of its modes (terms; gradient), with its bytes counted here.  Card name, power limit and SM
clock are read in the same run.

    python tools/bench_baked_tv.py [--steps 500] [--levels 1 3] [--out result.json]
"""
import argparse
import itertools
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
from mipnerf_pl_b200 import _cabi, baked  # noqa: E402
from tools.bench_baked import card  # noqa: E402
from tools.bench_baked_finetune import distill_scene  # noqa: E402

DEV = "cuda:0"
PRUNE_THRESHOLD = 1e-5
KERNELS = ("grid_render", "grid_render_backward", "grid_tv", "adam")


def copy(grid):
    """A fresh, non-trainable copy of a dense fp32 grid."""
    return grid.prune([torch.ones(m, device=DEV) for m in grid.kept], 0.0)


def quality(grid, refs):
    """{size: [PSNR, SSIM]}: means over the held-out poses against the MLP's fine frames `refs[size]`."""
    out = {}
    for size, frames in refs.items():
        vals = [[float(v) for v in mp.eval_errors(mp.render_baked_frame(grid, c2w, size, size)[0], fine)]
                for c2w, fine in frames]
        out[size] = [round(float(np.mean([v[0] for v in vals])), 2), round(float(np.mean([v[1] for v in vals])), 4)]
    return out


def stencil_points(grid, offsets):
    """Lattice points the TV kernel reads a word of: the kept points shifted by each of `offsets` ((dz, dy, dx)),
    inside the lattice, with the kept points themselves."""
    total = 0
    for lvl in range(grid.levels):
        keep = grid.index(lvl) >= 0
        seen = keep.clone()
        n = keep.shape
        for o in offsets:
            dst = tuple(slice(max(0, d), n[a] + min(0, d)) for a, d in enumerate(o))
            src = tuple(slice(max(0, -d), n[a] - max(0, d)) for a, d in enumerate(o))
            seen[dst] |= keep[src]
        total += int(seen.sum())
    return total


def tv_bytes(grid):
    """Bytes each mode of mipnerf_b200_grid_tv must move, every array element it reads or writes counted once: the
    positions (8 B a row), the 8-byte words of the points its stencil reads, the SH rows (12 nc B), and the outputs
    (terms: 2 x 4 B a row; gradient: 4 B + 12 nc B a row)."""
    m, nc = sum(grid.kept), (grid.degree + 1) ** 2
    fwd = [(0, 0, 1), (0, 1, 0), (1, 0, 0)]
    back = [tuple(-v for v in o) for o in fwd]
    diag = [tuple(b + f for b, f in zip(bo, fo)) for bo in back for fo in fwd if tuple(-v for v in bo) != fo]
    rows = 12 * nc * m
    return {"terms": 8 * m + 8 * stencil_points(grid, fwd) + rows + 8 * m,
            "gradient": 8 * m + 8 * stencil_points(grid, fwd + back + diag) + rows + 4 * m + rows}


def time_tv(grid, reps=20):
    """Median ms per launch of each mode of the TV kernel on a trainable grid, by CUDA events around the launch."""
    pos = grid._kept_pos
    terms = ([torch.empty(p.numel(), device=DEV) for p in pos], [torch.empty(p.numel(), device=DEV) for p in pos])
    grads = [torch.empty_like(p) for p in grid.parameters()]
    weights = torch.ones(2, device=DEV)
    out = {}
    for mode, kw in (("terms", {"terms": terms}), ("gradient", {"weights": weights, "grads": grads})):
        ts = []
        for rep in range(reps + 2):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            baked._tv_launch(grid, pos, **kw)
            ev[1].record()
            torch.cuda.synchronize()
            if rep >= 2:  # the first two are warm-up
                ts.append(ev[0].elapsed_time(ev[1]))
        out[mode] = float(np.median(ts))
    return out


def finetune(grid, bank, steps, batch, refs, lr_sh, tv_d, tv_sh):
    """One finetune_grid call on `grid`: quality after, step time and its split, the added peak memory."""
    lib = _cabi.lib()
    gen = torch.Generator(device=DEV).manual_seed(0)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    t0 = time.perf_counter()
    losses = mp.finetune_grid(grid, bank, steps, batch, lr_sh=lr_sh, generator=gen, tv_density=tv_d, tv_sh=tv_sh)
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / steps
    lib.mipnerf_b200_profile_enable(0)
    prof = _cabi.profile_snapshot(reset=True)
    r = {"tv_density": tv_d, "tv_sh": tv_sh, "lr_sh": lr_sh, "step_ms_wall": round(wall, 3),
         "kernel_ms_per_step": {k: round(prof[k][1] / steps, 3) for k in KERNELS},
         "launches_per_step": {k: prof[k][0] / steps for k in KERNELS},
         "added_peak_MiB": round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1),
         "mse_first_last_50": [round(float(np.mean(losses[:50])), 6), round(float(np.mean(losses[-50:])), 6)]}
    with torch.no_grad():
        r["tv_after"] = [round(float(t), 6) for t in grid.total_variation()]
    q = quality(grid, refs)
    r["psnr_ssim_200"], r["psnr_ssim_800"] = q[200], q[800]
    return r


def sync_ms(grid, reps=10):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ts = []
    for _ in range(reps):
        with torch.no_grad():
            grid.kept_density[0].add_(0.0)  # a version bump: the next read syncs
        ev[0].record()
        grid.density(0)
        ev[1].record()
        torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]))
    return round(float(np.median(ts)), 3)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--resolution", type=int, default=257)
    ap.add_argument("--train-poses", type=int, default=24)
    ap.add_argument("--train-size", type=int, default=200)
    ap.add_argument("--levels", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--tv-density", type=float, nargs="+", default=[0.0, 0.01, 0.1])
    ap.add_argument("--tv-sh", type=float, nargs="+", default=[0.0, 0.01, 0.1, 1.0])
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args(argv)
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    threshold = float(torch.quantile(mp.density_grid(model, 65).flatten()[::7], 0.7))  # as bench_baked.py
    path = mp.spheric_path(2 * args.train_poses)
    train, held = path[0::2], path[1::2][[3, 11]]  # held-out poses lie between training poses
    bank = mp.DeviceRayBank(distill_scene(model, train, args.train_size), DEV)
    refs = {size: [(c2w, mp.render_frame(model, c2w, size, size)[1]) for c2w in held] for size in (200, 800)}
    res = {"card (name, power limit, SM clock, max SM clock)": card(), "precision": "bf16",
           "weights": "trained_like seed 0", "threshold": threshold, "resolution": args.resolution, "degree": 2,
           "scene": f"{args.train_poses} training poses at {args.train_size}x{args.train_size} "
                    f"({bank.num_pixels} rays), 2 held-out poses", "steps": args.steps, "batch": args.batch,
           "lr_density": baked.FINETUNE_LR_DENSITY, "lr_sh": baked.FINETUNE_LR_SH, "tv_eps": baked.TV_EPS}
    best = None
    for li, levels in enumerate(args.levels):
        unpruned = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
        grids = {"unpruned": unpruned, f"pruned_{PRUNE_THRESHOLD:g}": mp.prune_grid(unpruned, bank, PRUNE_THRESHOLD)}
        warm = copy(unpruned)  # every shape warmed up, the TV path included
        mp.finetune_grid(warm, bank, 20, args.batch, tv_density=0.01, tv_sh=0.01)
        del warm
        r = {}
        for name, grid in grids.items():
            g = {"kept": grid.kept, "before": quality(grid, refs), "tv_before": [round(float(t), 6)
                                                                                  for t in grid.total_variation()]}
            t = copy(grid).requires_grad_()
            nbytes = tv_bytes(t)
            ms = time_tv(t)
            g["tv_kernel"] = {mode: {"ms": round(ms[mode], 3), "bytes_counted": nbytes[mode],
                                     "GB_per_s": round(nbytes[mode] / (ms[mode] * 1e-3) / 1e9, 1)} for mode in ms}
            g["sync_ms_median"] = sync_ms(t)
            del t
            pairs = list(itertools.product(args.tv_density, args.tv_sh)) if li == 0 else \
                [(0.0, 0.0)] + ([best] if best and best != (0.0, 0.0) else [])
            runs = []
            for tv_d, tv_sh in pairs:
                runs.append(finetune(copy(grid), bank, args.steps, args.batch, refs, baked.FINETUNE_LR_SH, tv_d, tv_sh))
                torch.cuda.empty_cache()
            if li == 0 and name == "unpruned":
                top = max(runs, key=lambda x: (x["psnr_ssim_200"][1], x["psnr_ssim_200"][0]))
                best = (top["tv_density"], top["tv_sh"])
            if li == 0:
                for tv_d, tv_sh in [(0.0, 0.0)] + ([best] if best != (0.0, 0.0) else []):
                    runs.append(finetune(copy(grid), bank, args.steps, args.batch, refs, 0.03, tv_d, tv_sh))
                    torch.cuda.empty_cache()
            g["runs"] = runs
            r[name] = g
            print(json.dumps({f"L{levels}": {name: g}}), flush=True)
        res[f"L{levels}"] = r
        res["best_by_ssim_200_unpruned_L1"] = best
        del grids, unpruned
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
