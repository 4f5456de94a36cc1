"""Fine-tuning baked grids (`finetune_grid`) on trained-like weights in bf16, in the setting of tools/bench_baked.py:
a 257^3 bake at 1 and 3 levels, degree 2, fine-tuned against a distillation scene of MLP renders at training poses
of the spheric path.  One finetune_grid call of --steps steps per grid (after warm-up on a throwaway bake) gives the
step time (synchronised wall clock) and its split per step into forward (grid_render), backward kernel
(grid_render_backward) and Adam (the library's per-launch events, on during that call); the sync is timed by CUDA
events.  Also: forward and backward kernel times and backward samples per second at two batch sizes, gradient and
optimiser-state memory, and PSNR / SSIM against the MLP frame at held-out poses before and after, at 200x200 and
800x800.  `--sweep` first compares learning rates on the 1-level grid.  Card name,
power limit and SM clock are read in the same run.

    python tools/bench_baked_finetune.py [--steps 2000] [--batch 8192] [--sweep] [--out result.json]
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
from mipnerf_pl_b200 import _cabi, baked  # noqa: E402
from tools.bench_baked import card  # noqa: E402

DEV = "cuda:0"


def distill_scene(model, poses, size):
    """A Scene whose images are the model's fine renders at `poses` (size x size, the default camera)."""
    focal = float(np.float32(0.5 * size / np.tan(0.5 * mp.rays.BLENDER_CAMERA_ANGLE_X)))
    k_inv = np.array([[1 / focal, 0, -0.5 * size / focal], [0, -1 / focal, 0.5 * size / focal], [0, 0, -1]], np.float32)
    images = [mp.render_frame(model, c2w, size, size)[1].cpu().numpy() for c2w in poses]
    return mp.Scene(images, np.broadcast_to(k_inv, (len(poses), 3, 3)), np.stack(poses), 1.0, 2.0, 6.0)


def quality(model, grid, poses, size):
    """Mean (PSNR, SSIM) of the baked frames against the MLP's fine frames."""
    vals = []
    for c2w in poses:
        fine = mp.render_frame(model, c2w, size, size)[1]
        vals.append([float(v) for v in mp.eval_errors(mp.render_baked_frame(grid, c2w, size, size)[0], fine)])
    return [round(float(np.mean([v[0] for v in vals])), 2), round(float(np.mean([v[1] for v in vals])), 4)]


def batch_samples(bank, batch, step):
    """Mean over 8 batches of the nominal lattice samples K = max(1, ceil((far - near) |d| / step)) per batch."""
    g = torch.Generator(device=DEV).manual_seed(1)
    tot = 0
    for _ in range(8):
        rays, _ = bank.sample(batch, g)
        d = rays.directions
        dn = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        k = torch.ceil((rays.far[:, 0] - rays.near[:, 0]) * dn / torch.tensor(step, device=DEV))
        tot += int(k.clamp(min=1).sum())
    return tot / 8


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--resolution", type=int, default=257)
    ap.add_argument("--train-poses", type=int, default=24)
    ap.add_argument("--train-size", type=int, default=200)
    ap.add_argument("--lr-density", type=float, default=baked.FINETUNE_LR_DENSITY)
    ap.add_argument("--lr-sh", type=float, default=baked.FINETUNE_LR_SH)
    ap.add_argument("--sweep", action="store_true")
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
           "scene": f"{args.train_poses} training poses at {args.train_size}x{args.train_size}, 2 held-out poses",
           "steps": args.steps, "batch": args.batch}
    lib = _cabi.lib()
    if args.sweep:
        sweep = {}
        for lr_d in (0.03, 0.1, 0.3):
            for lr_sh in (0.003, 0.01, 0.03):
                grid = mp.bake_grid(model, args.resolution, levels=1, threshold=threshold, degree=2)
                gen = torch.Generator(device=DEV).manual_seed(0)
                losses = mp.finetune_grid(grid, bank, args.steps // 4, args.batch, lr_d, lr_sh, generator=gen)
                sweep[f"lr_density={lr_d} lr_sh={lr_sh}"] = {"final_loss": round(float(np.mean(losses[-50:])), 6),
                                                             "psnr_ssim_200": quality(model, grid, held, 200)}
                del grid
                torch.cuda.empty_cache()
        res[f"sweep_L1_{args.steps // 4}_steps"] = sweep
    res["lr_density"], res["lr_sh"] = args.lr_density, args.lr_sh
    for levels in (1, 3):
        # warm up every shape on a throwaway bake, so that the measured grid sees exactly `steps` steps of one optimiser
        warm = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
        mp.finetune_grid(warm, bank, 20, args.batch, args.lr_density, args.lr_sh)
        del warm
        torch.cuda.empty_cache()
        grid = mp.bake_grid(model, args.resolution, levels=levels, threshold=threshold, degree=2)
        r = {"kept": grid.kept}
        for size in (200, 800):
            r[f"psnr_ssim_{size}_before"] = quality(model, grid, held, size)
        # one finetune_grid call: a synchronised wall clock around it and the library's per-launch events inside it
        gen = torch.Generator(device=DEV).manual_seed(0)
        _cabi.profile_snapshot(reset=True)
        lib.mipnerf_b200_profile_enable(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        losses = mp.finetune_grid(grid, bank, args.steps, args.batch, args.lr_density, args.lr_sh, generator=gen)
        torch.cuda.synchronize()
        r["step_ms_wall"] = round((time.perf_counter() - t0) * 1e3 / args.steps, 3)
        lib.mipnerf_b200_profile_enable(0)
        prof = _cabi.profile_snapshot(reset=True)
        names = ("grid_render", "grid_render_backward", "adam")
        r["kernel_ms_per_step"] = {k: round(prof[k][1] / args.steps, 3) for k in names}
        r["launches_per_step"] = {k: prof[k][0] / args.steps for k in names}
        r["loss_first_last_50"] = [round(float(np.mean(losses[:50])), 6), round(float(np.mean(losses[-50:])), 6)]
        nparam = sum(p.numel() for p in grid.parameters())
        r["grad_MiB"] = round(nparam * 4 / 2 ** 20, 1)
        r["adam_state_MiB"] = round(2 * nparam * 4 / 2 ** 20, 1)
        for size in (200, 800):
            r[f"psnr_ssim_{size}_after"] = quality(model, grid, held, size)
        # the sync (projection, scatter, occupancy rebuild) by CUDA events
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ts = []
        for _ in range(10):
            with torch.no_grad():
                grid.kept_density[0].add_(0.0)  # a version bump: the next read syncs
            ev[0].record()
            grid.density(0)
            ev[1].record()
            torch.cuda.synchronize()
            ts.append(ev[0].elapsed_time(ev[1]))
        r["sync_ms_median"] = round(float(np.median(ts)), 3)
        # forward and backward kernels alone at two batch sizes (an rgb cotangent, as the MSE gives)
        scaling = {}
        for batch in (args.batch, 8 * args.batch):
            rays, _ = bank.sample(batch, torch.Generator(device=DEV).manual_seed(2))
            d_rgb = torch.ones(batch, 3, device=DEV)
            for rep in range(11):
                if rep == 1:  # the first is warm-up
                    _cabi.profile_snapshot(reset=True)
                    lib.mipnerf_b200_profile_enable(1)
                rgb, _, _ = grid.render(rays, True)
                torch.autograd.grad(rgb, grid.parameters(), d_rgb, allow_unused=True)
            torch.cuda.synchronize()
            lib.mipnerf_b200_profile_enable(0)
            prof = _cabi.profile_snapshot(reset=True)
            n = batch_samples(bank, batch, grid.default_step())
            ms = {k: prof[k][1] / max(prof[k][2], 1) for k in ("grid_render", "grid_render_backward")}
            scaling[batch] = {"lattice_samples": round(n), "forward_ms": round(ms["grid_render"], 3),
                              "backward_ms": round(ms["grid_render_backward"], 3),
                              "backward_lattice_samples_per_s_G": round(n / (ms["grid_render_backward"] * 1e-3) / 1e9, 2)}
        r["kernels_by_batch"] = scaling
        res[f"L{levels}"] = r
        del grid
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
