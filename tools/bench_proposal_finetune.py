"""Fine-tuning a baked grid as the MLP's proposal (`finetune_proposal`, mip-NeRF 360's interlevel loss) on trained-like
weights in bf16 and fp16x3: per precision, dense bakes at 257^3 with 1 and 3 levels (degree 2, `bench_proposal.py`'s
threshold), tuned against the distillation scene of `bench_baked_finetune.py` (the model's own renders at training
poses).  Reported before and after: the interlevel loss on a held-out batch (the rays of two held-out poses, no
noise), PSNR / SSIM of the proposed frame (`render_proposed_frame`) and of the grid's own baked frame against the MLP's
fine frame at spheric poses.  Also the median time of a one-step `finetune_proposal` call (its optimizer construction
included) and the per-launch times of `grid_proposal_backward` and `interlevel_loss` from the library's profiler.  Card
name, power limit and SM clocks are read in the same run.

    python tools/bench_proposal_finetune.py [--steps 200] [--batch 8192] [--poses 7 60] [--out result.json]
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
from tools.bench_baked import card, timed  # noqa: E402
from tools.bench_baked_finetune import distill_scene  # noqa: E402
from tools.bench_proposal import kernel_ms  # noqa: E402

DEV = "cuda:0"


def held_out_loss(model, grid, rays):
    """The interlevel loss of `grid`'s proposal against `model`'s fine weights on `rays`, without noise."""
    with torch.no_grad():
        t_hat, rng, u_jitter, normals = model._proposal_fenceposts(rays, False, None, None, None)
        w_hat = grid.proposal(rays, t_hat)
        fine = model._forward_from(rays, t_hat, w_hat, False, True, rng, u_jitter, normals, False)[-1]
        return float(mp.interlevel_loss(fine[4], fine[3], t_hat, w_hat))


def quality(model, grid, poses, names, hw):
    """{frame kind: {pose: [PSNR, SSIM]}} of the proposed and the baked frame against the MLP's fine frame."""
    out = {}
    for name, c2w in zip(names, poses):
        fine = mp.render_frame(model, c2w, hw, hw)[1]
        with torch.no_grad():
            frames = (("proposed", mp.render_proposed_frame(model, grid, c2w, hw, hw)[0]),
                      ("baked", mp.render_baked_frame(grid, c2w, hw, hw)[0]))
        for kind, rgb in frames:
            psnr, ssim = mp.eval_errors(rgb, fine)
            out.setdefault(kind, {})[f"pose {name}"] = [round(float(psnr), 2), round(float(ssim), 4)]
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--resolution", type=int, default=257)
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--train-poses", type=int, default=24)
    ap.add_argument("--train-size", type=int, default=200)
    ap.add_argument("--timing-calls", type=int, default=21)
    ap.add_argument("--precisions", nargs="+", default=["bf16", "fp16x3"])
    ap.add_argument("--poses", type=int, nargs="+", default=[7, 60], help="indices into metrics.spheric_path(120)")
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args(argv)
    hw = args.size
    spheric = mp.spheric_path(120)
    poses = [spheric[i] for i in args.poses]
    path = mp.spheric_path(2 * args.train_poses)
    train, held = path[0::2], path[1::2][[3, 11]]  # held-out poses lie between training poses
    res = {"card (name, power limit, SM clock, max SM clock)": card(), "weights": "trained_like seed 0",
           "resolution": args.resolution, "degree": 2, "frame": f"{hw}x{hw}", "poses": args.poses,
           "scene": f"{args.train_poses} training poses at {args.train_size}x{args.train_size}",
           "held-out batch": f"2 held-out poses at {args.train_size}x{args.train_size}", "steps": args.steps,
           "batch": args.batch}
    for precision in args.precisions:
        model = mp.MipNerf(precision=precision)
        model.load_state_dict(mp.make_state_dict(seed=0, kind="trained_like"))
        model = model.to(DEV).eval()
        threshold = float(torch.quantile(mp.density_grid(model, 65).flatten()[::7], 0.7))
        bank = mp.DeviceRayBank(distill_scene(model, train, args.train_size), DEV)
        held_rays = mp.generate_rays(held[0], args.train_size, args.train_size, device=DEV)
        held_rays = mp.Rays(*[torch.cat([a, b]) for a, b in zip(
            held_rays, mp.generate_rays(held[1], args.train_size, args.train_size, device=DEV))])
        out = {"threshold": threshold}
        for levels in (1, 3):
            grid = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
            r = {"kept": grid.kept, "held_out_loss_before": held_out_loss(model, grid, held_rays),
                 "quality_before": quality(model, grid, poses, args.poses, hw)}
            gen = torch.Generator(device=DEV).manual_seed(0)
            secs, losses = timed(lambda: mp.finetune_proposal(grid, model, bank, args.steps, args.batch,
                                                              generator=gen))
            r["run_s"] = round(secs, 3)
            r["loss_first_last_10"] = [float(np.mean(losses[:10])), float(np.mean(losses[-10:]))]
            r["held_out_loss_after"] = held_out_loss(model, grid, held_rays)
            r["quality_after"] = quality(model, grid, poses, args.poses, hw)
            # timing after the measured run: each call is one step with a fresh optimizer, so it moves the grid on
            calls = [timed(lambda: mp.finetune_proposal(grid, model, bank, 1, args.batch, generator=gen))[0] * 1e3
                     for _ in range(args.timing_calls)]
            r["step_ms_median"] = round(float(np.median(calls[1:])), 3)
            k = kernel_ms(lambda: mp.finetune_proposal(grid, model, bank, 1, args.batch, generator=gen))
            r["kernel_ms_per_launch"] = {name: round(k[name][1] / k[name][0], 4)
                                         for name in ("grid_proposal_backward", "interlevel_loss", "grid_proposal",
                                                      "mlp_level_tc")
                                         if name in k}
            r["kernel_launches_per_step"] = {name: k[name][0] for name in k}
            out[f"L{levels}_dense"] = r
            del grid
            torch.cuda.empty_cache()
        res[precision] = out
        print(json.dumps({precision: out}), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
