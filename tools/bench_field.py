"""Density-grid throughput: the density query (MipNerf.query_density) against today's composition of public calls
(integrated_pos_enc + MLP.forward in MLP-only mode with a dummy view encoding, then softplus), alternated, with device
events; plus isosurface extraction.

    python tools/bench_field.py [--resolutions 256 512] [--precisions bf16 fp16x3 fp32] [--repeats 3] [--out f.json]

Both methods query the same lattice (anti-aliased Gaussians, variance step^2 / 12) in the same z-slabs of at most
2^22 points.  Reports ms per grid, points/s and trunk TFLOP/s from FLOP_PER_POINT, and the card name, power limit and
SM clock of the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200.field import lattice_axes  # noqa: E402

# multiply-adds per point: layer 0 96x256, layers 1-4, 6, 7 256x256, layer 5 352x256, density head 256x1
MACS_PER_POINT = 96 * 256 + 6 * 256 * 256 + 352 * 256 + 256
FLOP_PER_POINT = 2 * MACS_PER_POINT
assert FLOP_PER_POINT == 1_016_320
SLAB_POINTS = 1 << 22


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa: BLE001  (reported, not hidden)
        return {"error": repr(e)}


def composed_density(model, precision):
    """Today's route: the IPE stage kernel, then MLP.forward (MLP-only mode) on groups of 128 points."""
    def fn(means, covs):
        p = means.shape[0]
        pad = (-p) % 128
        if pad:
            means = torch.cat([means, means.new_zeros(pad, 3)])
            covs = torch.cat([covs, covs.new_zeros(pad, 3)])
        enc = mp.integrated_pos_enc((means, covs), 0, 16).view(-1, 128, 96)
        _, raw = model.mlp(enc, torch.zeros(enc.shape[0], 27, device=means.device), precision=precision)
        return torch.nn.functional.softplus(raw.reshape(-1)[:p] - 1.0)
    return fn


def grid_run(fn, res, dev):
    (xs, ys, zs), step = lattice_axes(res, mp.field.DEFAULT_BOUNDS, dev)
    covs_row = torch.tensor(step ** 2 / np.float32(12), device=dev)
    out = torch.empty(res, res, res, device=dev)
    slab = max(1, SLAB_POINTS // (res * res))
    yy, xx = torch.meshgrid(ys, xs, indexing="ij")
    for z0 in range(0, res, slab):
        z = zs[z0:z0 + slab]
        k = len(z)
        means = torch.stack([xx.expand(k, res, res), yy.expand(k, res, res), z[:, None, None].expand(k, res, res)], -1)
        out[z0:z0 + k] = fn(means.reshape(-1, 3), covs_row.expand(k * res * res, 3)).view(k, res, res)
    return out


def timed(f, repeats):
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        f()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolutions", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--precisions", nargs="+", default=["bf16", "fp16x3", "fp32"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = mp.make_state_dict(seed=0, kind="trained_like")
    rows = []
    for precision in args.precisions:
        model = mp.MipNerf(precision=precision)
        model.load_state_dict(sd)
        model = model.to(dev).eval()
        query = lambda m, c: model.query_density(m, c)  # noqa: E731
        compose = composed_density(model, precision)
        for res in args.resolutions:
            pts = res ** 3
            g_new = grid_run(query, res, dev)        # warm-up of both, and the outputs compared
            g_old = grid_run(compose, res, dev)
            rel = float(((g_new - g_old).abs() / g_old.abs().clamp(min=1.0)).max())
            del g_new, g_old
            t_new, t_old = [], []
            for _ in range(args.repeats):            # alternated
                t_new += timed(lambda: grid_run(query, res, dev), 1)
                t_old += timed(lambda: grid_run(compose, res, dev), 1)
            for name, ts in (("query_density", t_new), ("ipe+mlp_only", t_old)):
                ms = float(np.median(ts))
                rows.append(dict(precision=precision, resolution=res, method=name, ms=ms, ms_all=ts,
                                 points_per_s=pts / (ms * 1e-3), trunk_tflops=pts * FLOP_PER_POINT / (ms * 1e-3) / 1e12,
                                 max_rel_diff_vs_other=rel))
                print(json.dumps(rows[-1]), flush=True)
    # isosurface extraction at 512^3 on the bf16 density grid of the same model
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    res = max(args.resolutions)
    grid = mp.density_grid(model, res)
    thr = float(torch.quantile(grid.flatten()[::97].float(), 0.9))
    mp.isosurface(grid, thr)
    verts, faces = mp.isosurface(grid, thr)
    ts = timed(lambda: mp.isosurface(grid, thr), args.repeats)
    iso = dict(resolution=res, threshold=thr, ms=float(np.median(ts)), ms_all=ts, vertices=len(verts),
               faces=len(faces))
    print(json.dumps(iso), flush=True)
    result = dict(card=card(), flop_per_point=FLOP_PER_POINT, rows=rows, isosurface=iso)
    print(json.dumps(result["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
