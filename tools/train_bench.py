"""Time the fp32 training step (forward + backward + Adam) on one GPU: ms per step for a 4096-ray batch of
BASELINE configs[1] shape, with the per-kernel breakdown from the library's launch accounting.

    python tools/train_bench.py [--rays 4096] [--steps 5]
    python tools/train_bench.py --autograd [--rounds 5]

--autograd times MipNerf(autograd=True): forward -> the reference loss written in torch (masked MSE per level +
0.01 distloss, coarse multiplier 0.1) -> loss.backward() -> FusedAdam, alternating it with the fused step
(`forward_backward` + FusedAdam) on the same rays in the same process, fp32 and bf16, and prints one JSON line per
precision with the median ms of each and the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402

FLOP_PER_RAY_FWD = 312_475_648


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16", "fp16", "bf16x3"])
    ap.add_argument("--autograd", action="store_true", help="time the autograd step against the fused step")
    ap.add_argument("--rounds", type=int, default=5, help="--autograd: alternations of the two steps")
    args = ap.parse_args()
    if args.autograd:
        return autograd_vs_fused(args)
    dev = torch.device("cuda", 0)
    model = mp.MipNerf(precision=args.precision)
    model.load_state_dict(mp.make_state_dict(seed=0, kind="xavier"))
    model = model.to(dev)
    opt = mp.FusedAdam(model.parameters(), lr=5e-4)
    rays = mp.namedtuple_map(lambda t: t.to(dev), mp.random_ray_batch(args.rays, seed=0, multiscale=True))
    rgbs = torch.rand(args.rays, 3, device=dev)

    def step():
        out = mp.forward_backward(model, rays, rgbs, True, True)
        opt.step()
        return out

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    lib = _cabi.lib()
    # the step time: CUDA events around `steps` un-instrumented steps ...
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    # ... and the per-kernel breakdown from a second pass with an event pair around every launch (which itself
    # costs a few microseconds per launch, so its sum is not the step time)
    _cabi.profile_snapshot(reset=True)
    lib.mipnerf_b200_profile_enable(1)
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
    lib.mipnerf_b200_profile_enable(0)
    prof = _cabi.profile_snapshot(reset=True)
    flops = 3 * args.rays * FLOP_PER_RAY_FWD          # forward + dgrad + wgrad (dgrad of layer 0 is not needed)
    print(json.dumps({"what": f"{args.precision} training step (forward + backward + Adam), randomized, 128+128 samples",
                      "rays": args.rays, "ms_per_step": ms, "rays_per_s": args.rays / (ms * 1e-3),
                      "approx_tflops": flops / (ms * 1e-3) / 1e12, "loss": float(out["loss"]),
                      "kernel_ms_per_step": {k: round(v[1] / args.steps, 3) for k, v in prof.items() if v[2]},
                      "launches_per_step": {k: v[0] / args.steps for k, v in prof.items() if v[0]}}))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def reference_loss(ret, rays, rgbs):
    """models/nerf_system.py:95-111 as the reference writes it."""
    mask = rays.lossmult
    losses, dls = [], []
    for (rgb, _, _, weights, t_samples) in ret:
        losses.append((mask * (rgb - rgbs[..., :3]) ** 2).sum() / mask.sum())
        dls.append(mp.distloss(weights, t_samples))
    return 0.1 * (losses[0] + 0.01 * dls[0]) + losses[-1] + 0.01 * dls[-1]


def autograd_vs_fused(args):
    dev = torch.device("cuda", 0)
    card = _card()
    rays = mp.namedtuple_map(lambda t: t.to(dev), mp.random_ray_batch(args.rays, seed=0, multiscale=True))
    rgbs = torch.rand(args.rays, 3, device=dev)
    for precision in ("fp32", "bf16"):
        models = {}
        for kind in ("fused", "autograd"):
            m = mp.MipNerf(precision=precision, autograd=kind == "autograd")
            m.load_state_dict(mp.make_state_dict(seed=0, kind="xavier"))
            m = m.to(dev)
            models[kind] = (m, mp.FusedAdam(m.parameters(), lr=5e-4))

        def fused():
            m, opt = models["fused"]
            mp.forward_backward(m, rays, rgbs, True, True)
            opt.step()

        def autograd():
            m, opt = models["autograd"]
            opt.zero_grad()
            reference_loss(m(rays, True, True), rays, rgbs).backward()
            opt.step()

        steps = {"fused": fused, "autograd": autograd}
        for fn in steps.values():                # warm-up: modules loaded, workspaces and caches allocated
            for _ in range(2):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in steps}
        for _ in range(args.rounds):             # alternate the two so that drift of the shared host hits both
            for k, fn in steps.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / args.steps)
        print(json.dumps({"what": f"{precision} training step, {args.rays} rays, randomized, 128+128 samples: "
                                  "forward_backward + FusedAdam vs MipNerf(autograd=True) forward -> reference loss "
                                  "in torch -> backward -> FusedAdam",
                          "card": card, "rays": args.rays, "steps_per_round": args.steps, "rounds": args.rounds,
                          "fused_ms_median": statistics.median(times["fused"]),
                          "autograd_ms_median": statistics.median(times["autograd"]),
                          "fused_ms": [round(x, 3) for x in times["fused"]],
                          "autograd_ms": [round(x, 3) for x in times["autograd"]]}), flush=True)


if __name__ == "__main__":
    main()
