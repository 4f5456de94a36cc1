"""The streamed sparse bake (`bake_grid(sparse=True)`) against the dense bake then `sparsify()`, on trained-like
weights in bf16 (seed 0), degree 2, with the 0.9999 density quantile of a 65^3 grid as threshold so that the kept set
is sparse.

(a) At --compare sizes (default 257^3 and 513^3), 1 level: the two paths alternated in one process for --rounds rounds.
    Per path the median wall time (synchronised host clock), the time inside the density and SH queries and the glue
    (the rest: masks, numbering, bricks, occupancy, in torch on the device) from a separate instrumented round that
    synchronises around every query, the peak allocated memory beyond what was allocated before, and whether the
    streamed grid equals the dense one in every array.
(b) At --stream sizes (default 1025^3 and 2049^3), 1 level: the streamed bake only, once: kept points, stored bricks,
    grid MiB, bake time, glue share, peak memory, and the median 800x800 `render_baked_frame` time over --frames poses.

Card name, power limit and SM clock are read in the same run.

    python tools/bench_baked_stream.py [--rounds 3] [--compare 257 513] [--stream 1025 2049] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import baked  # noqa: E402
from tools.bench_baked import card  # noqa: E402

DEV = "cuda:0"
DEGREE = 2
QUANTILE = 0.9999


class QueryClock:
    """Wraps the bake's density and SH queries with synchronised host clocks, summing their time."""

    def __init__(self):
        self.seconds = 0.0
        self._orig = (baked.density_grid, baked.bake_sh)

    def _wrap(self, fn):
        def timed(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize()
            self.seconds += time.perf_counter() - t0
            return out
        return timed

    def __enter__(self):
        baked.density_grid, baked.bake_sh = (self._wrap(f) for f in self._orig)
        return self

    def __exit__(self, *exc):
        baked.density_grid, baked.bake_sh = self._orig


def run(fn):
    """(result, seconds, peak bytes allocated beyond the memory allocated before)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated(DEV) - base


def same(a, b) -> bool:
    arrays = lambda g: [t for pair in g.bricks for t in pair] + g.sh + [g.occupancy]  # noqa: E731
    return (a.kept == b.kept and a.resolutions == b.resolutions
            and all(x.dtype == y.dtype and torch.equal(x, y) for x, y in zip(arrays(a), arrays(b))))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--compare", type=int, nargs="*", default=[257, 513])
    ap.add_argument("--stream", type=int, nargs="*", default=[1025, 2049])
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    threshold = float(torch.quantile(mp.density_grid(model, 65).flatten(), QUANTILE))
    result = {"card": card(), "precision": "bf16", "degree": DEGREE, "threshold": threshold, "quantile": QUANTILE,
              "compare": [], "stream": []}
    print(f"card: {result['card']}; threshold {threshold:.4g} (the {QUANTILE} density quantile)")
    bakes = {"dense": lambda n: mp.bake_grid(model, n, 1, threshold, DEGREE).sparsify(),
             "stream": lambda n: mp.bake_grid(model, n, 1, threshold, DEGREE, sparse=True)}
    mp.bake_grid(model, 65, 1, threshold, DEGREE, sparse=True)  # load modules and size the query workspace
    for n in args.compare:
        times = {k: [] for k in bakes}
        peaks, grids = {}, {}
        for _ in range(args.rounds):
            for name, bake in bakes.items():
                grids[name] = None
                grids[name], sec, peak = run(lambda: bake(n))
                times[name].append(sec)
                peaks[name] = max(peaks.get(name, 0), peak)
        equal = same(grids["stream"], grids["dense"])
        row = {"n": n, "kept": grids["stream"].kept[0], "bricks": int(grids["stream"].bricks[0][1].shape[0]),
               "grid_mib": grids["stream"].nbytes / 2 ** 20, "equal": equal}
        grids.clear()
        for name, bake in bakes.items():
            with QueryClock() as clock:
                _, sec, _ = run(lambda: bake(n))
            wall = sorted(times[name])[len(times[name]) // 2]
            row[name] = {"wall_s": wall, "instrumented_s": sec, "query_s": clock.seconds,
                         "glue_s": sec - clock.seconds, "glue_share": (sec - clock.seconds) / sec,
                         "peak_mib": peaks[name] / 2 ** 20}
        result["compare"].append(row)
        print(json.dumps(row))
    poses = mp.spheric_path(args.frames)
    for n in args.stream:
        grid, sec, peak = run(lambda: bakes["stream"](n))
        mp.render_baked_frame(grid, poses[0], 800, 800)
        frame_ms = []
        for c2w in poses:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            mp.render_baked_frame(grid, c2w, 800, 800)
            e1.record()
            torch.cuda.synchronize()
            frame_ms.append(e0.elapsed_time(e1))
        row = {"n": n, "kept": grid.kept[0], "bricks": int(grid.bricks[0][1].shape[0]),
               "table_entries": grid.bricks[0][0].numel(), "grid_mib": grid.nbytes / 2 ** 20, "bake_s": sec,
               "peak_mib": peak / 2 ** 20, "frame_ms": sorted(frame_ms)[len(frame_ms) // 2]}
        del grid
        with QueryClock() as clock:
            _, isec, _ = run(lambda: bakes["stream"](n))
        row.update({"instrumented_s": isec, "query_s": clock.seconds, "glue_share": (isec - clock.seconds) / isec})
        result["stream"].append(row)
        print(json.dumps(row))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
