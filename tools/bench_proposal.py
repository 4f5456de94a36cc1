"""Proposal sampling from a baked grid (`render_proposed_frame`) on trained-like weights in bf16 and fp16x3: per
precision, bakes at 257^3 with 1 and 3 levels (degree 2, `bench_baked.py`'s threshold), dense and sparse; 800x800
frame time of `render_frame`, `render_proposed_frame` and `render_baked_frame` at spheric poses (alternated rounds,
medians), per-kernel times from the library's profiler in a separate pass, and PSNR / SSIM of the proposed frame and
of the baked frame against the MLP's fine frame.  Card name, power limit and SM clocks are read in the same run.

    python tools/bench_proposal.py [--rounds 5] [--poses 7 60] [--out result.json]
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
from tools.bench_baked import card, timed  # noqa: E402


def kernel_ms(fn):
    """{kernel: (launches, ms)} of one call of fn, from the library's launch accounting (events on every launch)."""
    lib = _cabi.lib()
    torch.cuda.synchronize()
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    fn()
    torch.cuda.synchronize()
    lib.mipnerf_b200_profile_enable(0)
    return {k: [n, round(ms, 3)] for k, (n, ms, _) in _cabi.profile_snapshot(reset=True).items() if n}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--resolution", type=int, default=257)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--precisions", nargs="+", default=["bf16", "fp16x3"])
    ap.add_argument("--poses", type=int, nargs="+", default=[7, 60], help="indices into metrics.spheric_path(120)")
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args(argv)
    dev = "cuda:0"
    hw = args.size
    path = mp.spheric_path(120)
    poses = [path[i] for i in args.poses]
    res = {"card (name, power limit, SM clock, max SM clock)": card(), "weights": "trained_like seed 0",
           "resolution": args.resolution, "degree": 2, "frame": f"{hw}x{hw}", "poses": args.poses}
    for precision in args.precisions:
        model = mp.MipNerf(precision=precision)
        model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
        model = model.to(dev).eval()
        threshold = float(torch.quantile(mp.density_grid(model, 65).flatten()[::7], 0.7))
        grids = {}
        for levels in (1, 3):
            dense = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
            grids[f"L{levels}_dense"], grids[f"L{levels}_sparse"] = dense, dense.sparsify()
        out = {"threshold": threshold, "grid_MB": {k: round(g.nbytes / 2 ** 20, 1) for k, g in grids.items()}}
        frames = {"mlp": lambda c2w: mp.render_frame(model, c2w, hw, hw)}
        for k, g in grids.items():
            frames[f"proposed_{k}"] = lambda c2w, g=g: mp.render_proposed_frame(model, g, c2w, hw, hw)
            frames[f"baked_{k}"] = lambda c2w, g=g: mp.render_baked_frame(g, c2w, hw, hw)
        for fn in frames.values():  # warm up every shape the timed rounds use
            fn(poses[0])
        times = {k: [] for k in frames}
        for _ in range(args.rounds):  # alternated
            for k, fn in frames.items():
                times[k].append(timed(lambda: fn(poses[0]))[0] * 1e3)
        med = {k: float(np.median(v)) for k, v in times.items()}
        out["frame_ms_median"] = {k: round(v, 2) for k, v in med.items()}
        out["frame_ms_all"] = {k: [round(t, 2) for t in v] for k, v in times.items()}
        out["frame_time_vs_mlp"] = {k: round(v / med["mlp"], 3) for k, v in med.items() if k != "mlp"}
        out["kernel_ms"] = {k: kernel_ms(lambda: fn(poses[0])) for k, fn in frames.items()
                            if k == "mlp" or k.endswith("_dense") or k == "proposed_L1_sparse"}
        quality = {}
        for i, c2w in zip(args.poses, poses):
            fine = mp.render_frame(model, c2w, hw, hw)[1]
            for k, g in grids.items():
                for kind, rgb in (("proposed", mp.render_proposed_frame(model, g, c2w, hw, hw)[0]),
                                  ("baked", mp.render_baked_frame(g, c2w, hw, hw)[0])):
                    psnr, ssim = mp.eval_errors(rgb, fine)
                    quality.setdefault(f"{kind}_{k}", {})[f"pose {i}"] = [round(float(psnr), 2), round(float(ssim), 4)]
        out["psnr_ssim_vs_mlp_fine"] = quality
        res[precision] = out
        del grids
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
