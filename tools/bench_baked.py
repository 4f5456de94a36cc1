"""Baked grids on trained-like weights in bf16: bake time at 257^3 (1 and 3 levels, degree 2), grid memory and kept
points, 800x800 frame time of `render_baked_frame` against `render_frame` at the same spheric pose (alternated rounds,
medians), nominal sample-lattice samples per second, and PSNR / SSIM of the baked frames against the MLP frame at
full and 1/4 resolution.  Card name, power limit and SM clock are read in the same run.

    python tools/bench_baked.py [--rounds 5] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def lattice_samples(grid, c2w, h, w, step):
    """sum over the frame's rays of K = max(1, ceil((far - near) |d| / step)) (fp32, as the kernel forms it)."""
    rays = mp.generate_rays(c2w, h, w, device="cuda")
    d = rays.directions
    dn = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    k = torch.ceil((rays.far[:, 0] - rays.near[:, 0]) * dn / torch.tensor(step, dtype=torch.float32, device="cuda"))
    return int(k.clamp(min=1).sum())


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--resolution", type=int, default=257)
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args(argv)
    dev = "cuda:0"
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
    model = model.to(dev).eval()
    # a threshold that keeps part of the lattice: the 70th percentile of a 65^3 density grid
    threshold = float(torch.quantile(mp.density_grid(model, 65).flatten()[::7], 0.7))
    res = {"card (name, power limit, SM clock, max SM clock)": card(), "precision": "bf16",
           "weights": "trained_like seed 0", "threshold": threshold, "resolution": args.resolution, "degree": 2}
    grids = {}
    for levels in (1, 3):
        ts = []
        for _ in range(2):
            t, g = timed(lambda: mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2))
            ts.append(t)
        grids[levels] = g
        res[f"bake_s_L{levels}"] = [round(t, 3) for t in ts]
        res[f"grid_MB_L{levels}"] = round(g.nbytes / 2 ** 20, 1)
        res[f"kept_L{levels}"] = g.kept
        res[f"occupied_macro_cells_L{levels}"] = f"{int(g.occupancy.sum())} / {g.occupancy.numel()}"
    c2w = mp.spheric_path(120)[7]
    h = w = 800
    # warm up every shape the timed rounds use
    mp.render_frame(model, c2w, h, w)
    for g in grids.values():
        mp.render_baked_frame(g, c2w, h, w)
    times = {"mlp": [], "L1": [], "L3": []}
    for _ in range(args.rounds):  # alternated
        times["mlp"].append(timed(lambda: mp.render_frame(model, c2w, h, w))[0])
        times["L1"].append(timed(lambda: mp.render_baked_frame(grids[1], c2w, h, w))[0])
        times["L3"].append(timed(lambda: mp.render_baked_frame(grids[3], c2w, h, w))[0])
    med = {k: float(np.median(v)) * 1e3 for k, v in times.items()}
    res["frame_ms_800_median"] = {k: round(v, 3) for k, v in med.items()}
    res["frame_ms_800_all"] = {k: [round(t * 1e3, 3) for t in v] for k, v in times.items()}
    res["speedup_vs_mlp"] = {k: round(med["mlp"] / med[k], 1) for k in ("L1", "L3")}
    step = grids[1].default_step()
    n = lattice_samples(grids[1], c2w, h, w, step)
    res["lattice_samples_per_frame"] = n
    res["lattice_samples_per_s_G"] = {k: round(n / (med[k] * 1e-3) / 1e9, 2) for k in ("L1", "L3")}
    # quality against the MLP frame at full and 1/4 resolution
    for name, hh in (("full", 800), ("quarter", 200)):
        _, fine, _ = mp.render_frame(model, c2w, hh, hh)
        for levels, g in grids.items():
            rgb = mp.render_baked_frame(g, c2w, hh, hh)[0]
            psnr, ssim = mp.eval_errors(rgb, fine)
            res[f"psnr_ssim_{name}_L{levels}"] = [round(float(psnr), 2), round(float(ssim), 4)]
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
