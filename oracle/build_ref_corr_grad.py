"""ORACLE build recipe (test infrastructure only) for the reference's correlation BACKWARD kernels.

Compiles src/correlation_kernels.cu + src/altcorr_kernel.cu of the reference (same `.type()` -> `.scalar_type()`
patch as oracle/build_ref.py, in a temp dir outside the repo) with oracle/ref_glue_corr_grad.cpp into
oracle/_ref/nslam_ref_corr_grad.so, which binds corr_index_backward and altcorr_backward.  A module of its own, so
that a nslam_ref_corr.so built before these bindings existed is never taken for one that has them.
Used by tests/test_gpu_corr_grad.py and tools/corr_grad_bench.py (both skip the reference when it is absent).
"""
import os
import shutil
import sys
import tempfile

from oracle import build_ref

NAME = "nslam_ref_corr_grad"


def build(force=False):
    if not os.path.isdir(os.path.join(build_ref.REF, "src")):
        return False  # no reference tree here: an oracle/_ref/ built beforehand is used as it is
    if not force and os.path.exists(os.path.join(build_ref.OUT, NAME + ".so")):
        return True
    tmp = tempfile.mkdtemp(prefix="nslam_ref_grad_")
    srcs = []
    for f in ("correlation_kernels.cu", "altcorr_kernel.cu"):
        txt = open(os.path.join(build_ref.REF, "src", f)).read().replace(".type()", ".scalar_type()")
        p = os.path.join(tmp, f)
        open(p, "w").write(txt)
        srcs.append(p)
    build_ref._build(NAME, srcs + [os.path.join(build_ref.HERE, "ref_glue_corr_grad.cpp")], tmp)
    shutil.rmtree(tmp, ignore_errors=True)
    return True


def load():
    return build_ref.load(NAME)


if __name__ == "__main__":
    print("built" if build(force="--force" in sys.argv) else "reference sources not found; nothing built")
