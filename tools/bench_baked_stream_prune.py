"""Pruning inside the bake (`bake_grid(sparse=True, prune=bank)`) against the dense bake, `prune_grid` and `sparsify()`,
on trained-like weights in bf16 (seed 0), degree 2, 1 level, with the training bank of tools/bench_baked_prune.py:
MLP renders at 24 spheric-path poses, 200x200 (960,000 rays), pruned at the default weight threshold (1e-5).  The
density threshold is 7.88 at 257^3 (bench_baked_prune.py's) and the 0.9999 density quantile of a 65^3 grid from
513^3 up (bench_baked_stream.py's), so that the kept set is sparse.

(a) At --compare sizes (default 257^3 and 513^3): the two paths, (a) dense -> prune_grid -> sparsify() and (b) the
    pruned streamed bake, alternated in one process for --rounds rounds.  Per path the median wall time (synchronised
    host clock); from one instrumented round that synchronises around every density and SH query, the time inside the
    queries and the rest; the visibility kernel's time (the library's per-launch events: grid_visibility on dense
    cells, grid_visibility_bricks on bricks); the peak allocated memory beyond what was allocated before; kept points
    before and after the prune, grid MiB, and whether (a) and (b) are equal in every array.
(b) At --stream sizes (default 1025^3 and 2049^3): the pruned streamed bake only.  At the first size the same
    numbers; at the others one uninstrumented run (wall time, peak memory, kept points, grid MiB).  A size whose bake
    runs out of device memory is reported as not fitting.

Card name, power limit and SM clock are read in the same run.

    python tools/bench_baked_stream_prune.py [--rounds 3] [--compare 257 513] [--stream 1025 2049] [--out result.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402
from tools.bench_baked import card  # noqa: E402
from tools.bench_baked_finetune import distill_scene  # noqa: E402
from tools.bench_baked_stream import DEGREE, DEV, QUANTILE, QueryClock, run, same  # noqa: E402

THRESHOLD_257 = 7.88


def profiled(fn):
    """(result, seconds, {kernel: (launches, ms)} of the visibility kernels) of one run with per-launch timing."""
    lib = _cabi.lib()
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    out, sec, _ = run(fn)
    lib.mipnerf_b200_profile_enable(0)
    prof = _cabi.profile_snapshot(reset=True)
    return out, sec, {k: (prof[k][0], round(prof[k][1], 3)) for k in ("grid_visibility", "grid_visibility_bricks")}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--compare", type=int, nargs="*", default=[257, 513])
    ap.add_argument("--stream", type=int, nargs="*", default=[1025, 2049])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    quantile = float(torch.quantile(mp.density_grid(model, 65).flatten(), QUANTILE))
    bank = mp.DeviceRayBank(distill_scene(model, mp.spheric_path(48)[0::2], 200), DEV)
    result = {"card (name, power limit, SM clock, max SM clock)": card(), "precision": "bf16", "degree": DEGREE,
              "bank_rays": bank.num_pixels, "weight_threshold": mp.baked.DEFAULT_WEIGHT_THRESHOLD,
              "compare": [], "stream": []}
    print(f"card: {result['card (name, power limit, SM clock, max SM clock)']}; {bank.num_pixels} bank rays")

    def threshold(n):
        return THRESHOLD_257 if n == 257 else quantile

    bakes = {"dense_prune_sparsify": lambda n: mp.prune_grid(mp.bake_grid(model, n, 1, threshold(n), DEGREE),
                                                             bank).sparsify(),
             "stream_prune": lambda n: mp.bake_grid(model, n, 1, threshold(n), DEGREE, sparse=True, prune=bank)}
    for name in bakes:  # load modules and size the query workspace
        bakes[name](65)

    def row_for(names, n, rounds, instrumented=True):
        times = {k: [] for k in names}
        peaks, grids = {}, {}
        for _ in range(rounds):
            for name in names:
                grids[name] = None
                grids[name], sec, peak = run(lambda: bakes[name](n))
                times[name].append(sec)
                peaks[name] = max(peaks.get(name, 0), peak)
        g = grids[names[-1]]
        row = {"n": n, "threshold": threshold(n), "kept_after": g.kept[0],
               "bricks_after": int(g.bricks[0][1].shape[0]), "grid_mib": round(g.nbytes / 2 ** 20, 1)}
        if len(names) == 2:
            row["equal"] = same(grids[names[0]], grids[names[1]])
        grids.clear()
        for name in names:
            wall = sorted(times[name])[len(times[name]) // 2]
            row[name] = {"wall_s": round(wall, 3), "wall_all_s": [round(t, 3) for t in times[name]],
                         "peak_mib": round(peaks[name] / 2 ** 20, 1)}
            if instrumented:
                with QueryClock() as clock:
                    _, sec, _ = run(lambda: bakes[name](n))
                _, _, vis = profiled(lambda: bakes[name](n))
                row[name].update({"instrumented_s": round(sec, 3), "query_s": round(clock.seconds, 3),
                                  "rest_s": round(sec - clock.seconds, 3),
                                  "query_share": round(clock.seconds / sec, 3), "visibility_kernel": vis})
        return row

    for n in args.compare:
        before = mp.bake_grid(model, n, 1, threshold(n), DEGREE, sparse=True)
        kept_before = before.kept[0]
        del before
        row = row_for(list(bakes), n, args.rounds)
        row["kept_before"] = kept_before
        result["compare"].append(row)
        print(json.dumps(row))
    for i, n in enumerate(args.stream):
        torch.cuda.empty_cache()
        try:
            row = row_for(["stream_prune"], n, args.rounds if i == 0 else 1, instrumented=i == 0)
            row["fits"] = True
        except torch.cuda.OutOfMemoryError as e:
            row = {"n": n, "fits": False, "error": str(e).splitlines()[0]}
        torch.cuda.empty_cache()
        result["stream"].append(row)
        print(json.dumps(row))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
