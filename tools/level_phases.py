"""Where the time of the fused level kernel goes, measured inside the kernel.

Builds the `phases` variant of the library (-DMIPNERF_LEVEL_PHASES: clock64 phase accounting in mlp_level_kernel), runs
the benchmark's forward (4096 rays, xavier weights) in bf16 and fp16x3, and prints, per level launch and per role, the
share of each phase in the role's cycles, averaged over CTAs, next to the GPU's name and power limit.  Phases a role
never enters are left out: in bf16 / fp16 the consumers' layer loop has no barrier, so their `barrier` counts only the
wait for a free raw-heads buffer; the helpers' `barrier` is their own named barrier (prologue -> features, the
compositing scans).

    python tools/level_phases.py [--rays 4096] [--reps 20] [--precisions bf16,fp16x3] [--json OUT]
    python tools/level_phases.py --query 4194304 ...   # query_radiance and query_density on that many points instead

In query mode the helpers' `prologue` is the radiance mode's per-point view-direction terms and `composite` the
writing of the outputs; both query modes charge slot `level0`.

With MIPNERF_B200_LIB set, that (instrumented) library is used instead of building one.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
PHASES = ["prologue", "ipe", "w_full_wait", "mma", "epilogue", "composite", "barrier", "w_empty_wait", "issue",
          "feat_full_wait", "feat_empty_wait", "heads_full_wait"]
ROLES = ["consumer_wg0", "consumer_wg1", "producer", "helpers"]
LEVELS = ["level0", "level1"]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rays", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--precisions", default="bf16,fp16x3")
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    ap.add_argument("--query", type=int, default=0, help="points of a query_radiance / query_density run instead")
    args = ap.parse_args()

    if not os.environ.get("MIPNERF_B200_LIB"):  # a prebuilt instrumented library may be passed in
        os.environ["MIPNERF_B200_LIB"] = subprocess.run(
            [sys.executable, "-m", "mipnerf_pl_b200.build", "--variant", "phases", "-DMIPNERF_LEVEL_PHASES"], cwd=ROOT,
            check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1]
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import mipnerf_pl_b200 as mp
    from mipnerf_pl_b200 import _cabi

    lib = _cabi.lib()
    read = lib.mipnerf_b200_level_phases
    read.restype = C.c_int
    dev = torch.device("cuda", 0)
    rays = mp.namedtuple_map(lambda t: t.to(dev), mp.random_ray_batch(args.rays, seed=0))
    sd = mp.make_state_dict(seed=0, kind="xavier")
    max_ctas = C.c_int(0)
    buf = np.zeros(2 * 1024 * len(ROLES) * (len(PHASES) + 1), dtype=np.uint64)  # [slot][cta][role][phase + total]
    result = {"gpu": gpu_info(), "rays": args.rays, "reps": args.reps, "runs": {}}
    if args.query:
        g = torch.Generator().manual_seed(0)
        q_means = (3.0 * torch.rand(args.query, 3, generator=g) - 1.5).to(dev)
        q_covs = (10 ** (-6 + 5 * torch.rand(args.query, 3, generator=g))).to(dev)
        q_dirs = torch.nn.functional.normalize(torch.randn(args.query, 3, generator=g), dim=-1).to(dev)
    for precision, what in [(p, w) for p in args.precisions.split(",")
                            for w in (("radiance", "density") if args.query else ("forward",))]:
        model = mp.MipNerf(precision=precision)
        model.load_state_dict(sd)
        model = model.to(dev).eval()
        call = {"forward": lambda: model(rays, False, True),
                "radiance": lambda: model.query_radiance(q_means, q_covs, q_dirs),
                "density": lambda: model.query_density(q_means, q_covs)}[what]
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        read(buf.ctypes.data_as(C.POINTER(C.c_ulonglong)), C.byref(max_ctas))  # reset
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.reps):
            call()
        stop.record()
        torch.cuda.synchronize()
        nph = read(buf.ctypes.data_as(C.POINTER(C.c_ulonglong)), C.byref(max_ctas))
        assert nph == len(PHASES) + 1, nph
        data = buf.reshape(2, max_ctas.value, len(ROLES), nph).astype(np.float64)
        run = {f"{what}_ms": start.elapsed_time(stop) / args.reps}
        for s, level in enumerate(LEVELS[:1] if args.query else LEVELS):
            d = data[s]
            ctas = d[:, 0, -1] > 0
            row = {"ctas": int(ctas.sum()),
                   "cycles_per_launch": float(d[ctas, 0, -1].mean() / args.reps)}
            for r, role in enumerate(ROLES):
                tot = d[ctas, r, -1]
                row[role] = {ph: round(float((d[ctas, r, i] / tot).mean()), 4) for i, ph in enumerate(PHASES)
                             if d[ctas, r, i].any()}
            run[level] = row
        result["runs"][precision if what == "forward" else f"{precision}_{what}"] = run
    print(json.dumps(result, indent=1))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
