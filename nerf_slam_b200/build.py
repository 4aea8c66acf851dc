"""Build libnslam_sm90a.so (the C-ABI library with every hand-written sm_90a kernel) in-tree.

    python -m nerf_slam_b200.build [--force]

Plain nvcc, no torch headers in any kernel translation unit (seconds per file).  The shared
object lands next to this file so it travels to the GPU box with the repo snapshot.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libnslam_sm90a.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
# NB: no --use_fast_math: frame_distance / corr lookup reproduce the reference's IEEE arithmetic.
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
         "--expt-relaxed-constexpr", "-diag-suppress", "550"]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    inc = os.path.join(os.path.dirname(HERE), "include")
    headers += [os.path.join(inc, f) for f in os.listdir(inc)] if os.path.isdir(inc) else []
    objs, jobs = [], []
    for src in sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src[:-3] + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [NVCC] + ARCH + FLAGS + ["-I", inc, "-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(o + ".log", "w") as f:
            f.write(log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{log}")
        return s, log

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for s, log in ex.map(compile_one, jobs):
                if verbose:
                    print(f"[nvcc] {os.path.basename(s)}")
                    print("\n".join(l for l in log.splitlines() if "registers" in l or "spill" in l.lower() and "0 bytes spill" not in l))
    if jobs or force or _stale(LIB, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose=True)
    print(path)
