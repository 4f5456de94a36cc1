"""Forward cost at 128 and 256 samples per level on the tensor cores (and the fp32 path at 256 for comparison).

bench.py's protocol on one GPU: a 4096-ray batch resident on the device, device events around every step, the L2
flushed (untimed) before each step, warm-up first; the cases are alternated round by round within one run so that
clock drift hits them alike.  Then one eager pass per case with the library's per-kernel CUDA events gives the level
kernel's time, from which its achieved TFLOP/s follows: 2 * 610304 FLOPs per sample of the MLP (SURVEY.md §8d),
N samples per level, one level per launch.  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_samples.py [--rays 4096] [--steps 20] [--warmup 5] [--rounds 3]

Prints one JSON line per case and a summary line; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, ROOT)

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402

FLOP_PER_SAMPLE = 2 * 610304
CASES = [(128, "bf16"), (256, "bf16"), (128, "fp16x3"), (256, "fp16x3"), (256, "fp32")]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, plim, sm, sm_max = (s.strip() for s in out.stdout.strip().splitlines()[0].split(","))
        return {"name": name, "power_limit": plim, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, with the reason the card is unknown
        return {"name": torch.cuda.get_device_name(), "error": repr(e)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_samples.py needs a CUDA device")
    dev = torch.device("cuda:0")
    lib = _cabi.lib()
    rays = mp.namedtuple_map(lambda t: t.to(dev), mp.random_ray_batch(args.rays, seed=0))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)       # > 50 MB L2

    models = {}
    for n, prec in CASES:
        m = mp.MipNerf(num_samples=n, precision=prec)
        m.load_state_dict(mp.make_state_dict(seed=0, kind="xavier"))
        models[(n, prec)] = m.to(dev).eval()

    def step(key):
        return models[key](rays, False, True)

    def timed(key, steps):
        starts = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        stops = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        torch.cuda.synchronize()
        for i in range(steps):
            flush.zero_()
            starts[i].record()
            step(key)
            stops[i].record()
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in zip(starts, stops)) / steps

    with torch.no_grad():
        for key in models:
            for _ in range(args.warmup):
                step(key)
        torch.cuda.synchronize()
        before = card()
        ms = {key: [] for key in models}
        for _ in range(args.rounds):                     # alternate the cases within the run
            for key in models:
                ms[key].append(timed(key, args.steps))
        after = card()
        kernel = {}
        for key in models:                               # per-kernel device events: the level kernel's time
            _cabi.profile_snapshot(reset=True)
            lib.mipnerf_b200_profile_enable(1)
            timed(key, args.steps)
            lib.mipnerf_b200_profile_enable(0)
            kernel[key] = _cabi.profile_snapshot(reset=True)

    rows = {}
    for (n, prec), runs in ms.items():
        best = min(runs)
        row = {"num_samples": n, "precision": prec, "rays": args.rays, "ms_per_step": best,
               "ms_per_step_runs": runs, "rays_per_s": args.rays / (best * 1e-3),
               "samples_per_s": args.rays * n * 2 / (best * 1e-3)}
        prof = kernel[(n, prec)]
        if "mlp_level_tc" in prof and prof["mlp_level_tc"][2] > 0:
            _, k_ms, k_timed = prof["mlp_level_tc"]
            per_launch = k_ms / k_timed
            row["level_kernel_ms_per_launch"] = per_launch
            row["level_kernel_tflops"] = args.rays * n * FLOP_PER_SAMPLE / (per_launch * 1e-3) / 1e12
        rows[(n, prec)] = row
        print(json.dumps(row), flush=True)

    summary = {"card_before": before, "card_after": after,
               "flops": "2 * 610304 per sample, N samples per level, one level per launch; library kernel events"}
    for prec in ("bf16", "fp16x3"):
        a, b = rows[(128, prec)], rows[(256, prec)]
        if "level_kernel_tflops" in a and "level_kernel_tflops" in b:
            summary[f"{prec}_tflops_ratio_256_over_128"] = b["level_kernel_tflops"] / a["level_kernel_tflops"]
        summary[f"{prec}_per_sample_cost_ratio_256_over_128"] = a["samples_per_s"] / b["samples_per_s"]
        summary[f"{prec}_speedup_over_fp32_at_256"] = rows[(256, "fp32")]["ms_per_step"] / b["ms_per_step"]
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
