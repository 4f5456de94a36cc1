"""Build libmipnerf_b200.so in-tree with nvcc for sm_90a (no GPU needed to compile)."""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
OUT = os.path.join(HERE, "libmipnerf_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]
SOURCES = ["api.cu", "ray_kernels.cu", "linear_f32.cu", "mlp_tc.cu", "profile.cu", "tc_selftest.cu", "train_kernels.cu", "linear_tc.cu", "metrics.cu", "train_t16.cu", "isosurface.cu", "grid_render.cu",
           "grid_tv.cu"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, variant: str = "", defines=()) -> str:
    """variant != "": an experiment build `libmipnerf_b200.<variant>.so` compiled with extra -D flags
    (selected at run time with MIPNERF_B200_LIB=<path>)."""
    global OBJ, OUT
    if variant:
        OBJ = os.path.join(HERE, "build", variant)
        OUT = os.path.join(HERE, f"libmipnerf_b200.{variant}.so")
        force = True
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(HERE, "..", "include", "mipnerf_b200.h"))
    nvcc = _nvcc()
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + headers):
            jobs.append([nvcc] + FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else []) +
                        ["-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stderr

    with cf.ThreadPoolExecutor(max_workers=4) as ex:
        for log in ex.map(run, jobs):
            if verbose and log:
                print(log, file=sys.stderr)
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(OUT, objs):
        run([nvcc, "-shared"] + ARCH + ["-o", OUT] + objs)
    return OUT


if __name__ == "__main__":
    var = ""
    defs = [a[2:] for a in sys.argv[1:] if a.startswith("-D")]
    if "--variant" in sys.argv:
        var = sys.argv[sys.argv.index("--variant") + 1]
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=var, defines=defs))
