"""Cost of differentiating a field query: the forward query alone against forward + backward (gradients of
<cot, outputs> with respect to the MLP tensors, mipnerf_b200_query_backward), for query_density and query_radiance,
alternated, with device events.

    python tools/bench_query_grad.py [--sizes 22 24] [--precisions bf16 fp32] [--repeats 3] [--out f.json]

The points are bench_radiance's: 2^k anti-aliased lattice Gaussians over the default bounds with random unit
directions, `trained_like` weights, random cotangents on the activated outputs.  Reports the median ms of each call
and the backward's share, and the card name, power limit and SM clock read in the same run.
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
from tools.bench_field import card, timed  # noqa: E402
from tools.bench_radiance import lattice_points  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[22, 24], help="log2 of the point counts")
    ap.add_argument("--precisions", nargs="+", default=["bf16", "fp32"])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    sd = mp.make_state_dict(seed=0, kind="trained_like")
    rows = []
    for log2 in args.sizes:
        means, covs, dirs = lattice_points(log2, dev)
        pts = means.shape[0]
        g = torch.Generator(device=dev).manual_seed(1)
        cot_rgb = torch.randn(pts, 3, device=dev, generator=g) / pts
        cot_dens = torch.randn(pts, device=dev, generator=g) / pts
        for precision in args.precisions:
            model = mp.MipNerf(precision=precision, autograd=True)
            model.load_state_dict(sd)
            model = model.to(dev)

            def dens_fwd():
                with torch.no_grad():
                    model.query_density(means, covs)

            def dens_fwd_bwd():
                model.query_density(means, covs).backward(cot_dens)

            def rad_fwd():
                with torch.no_grad():
                    model.query_radiance(means, covs, dirs)

            def rad_fwd_bwd():
                torch.autograd.backward(model.query_radiance(means, covs, dirs), (cot_rgb, cot_dens))

            calls = {"query_density": dens_fwd, "query_density+backward": dens_fwd_bwd,
                     "query_radiance": rad_fwd, "query_radiance+backward": rad_fwd_bwd}
            for f in calls.values():  # warm-up of every call
                f()
            times = {k: [] for k in calls}
            for _ in range(args.repeats):  # alternated
                for k, f in calls.items():
                    times[k] += timed(f, 1)
            for k, ts in times.items():
                ms = float(np.median(ts))
                rows.append(dict(precision=precision, points=pts, call=k, ms=ms, ms_all=ts,
                                 points_per_s=pts / (ms * 1e-3)))
                print(json.dumps(rows[-1]), flush=True)
            del model
        del means, covs, dirs, cot_rgb, cot_dens
    result = dict(card=card(), rows=rows)
    print(json.dumps(result["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
