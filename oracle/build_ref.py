"""ORACLE build recipe (test infrastructure only).

Compiles the reference's OWN CUDA kernels for sm_90a, from the sources where they lie under
/root/reference, into oracle/_ref/*.so (git-ignored, but shipped to the GPU box by gpurun):

  nslam_ref_corr.so   src/correlation_kernels.cu + src/altcorr_kernel.cu, with the 3-token
                      torch-2.x patch `.type()` -> `.scalar_type()` (SURVEY.md §0.8)
  nslam_ref_droid.so  src/droid_kernels.cu minus the Eigen-dependent host code (Eigen is an
                      empty submodule): lines 15-20 (includes/typedefs), 1240-1346 (SparseBlock),
                      1349-1438 (schur_block), 1441-1568 (ba_cuda), 1678-1768
                      (reduced_camera_matrix_cuda), plus oracle/ref_glue_droid.cu which redoes
                      that host orchestration with dense fp64 torch tensors.

Patched intermediates go to a temp dir outside the repo; no reference source is copied into the
tree.  Used to (a) pin the CPU oracle and the CUDA product path against the reference kernels on
the GPU (tests/test_gpu_vs_reference.py), (b) generate tests/golden/*.npz, (c) time the
reference's CUDA build next to ours (bench.py --impl reference-cuda).
"""
import os
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = os.environ.get("NSLAM_REFERENCE", "/root/reference")
STRIP = [(15, 20), (1240, 1346), (1349, 1438), (1441, 1568), (1678, 1768)]


def _build(name, sources, tmp):
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "10.0")
    from torch.utils import cpp_extension
    bdir = os.path.join(tmp, name)
    os.makedirs(bdir, exist_ok=True)
    cpp_extension.load(name=name, sources=sources, build_directory=bdir, verbose=False,
                       extra_cuda_cflags=["-O3", "-gencode", "arch=compute_90a,code=sm_90a"],
                       is_python_module=False)
    os.makedirs(OUT, exist_ok=True)
    shutil.copy(os.path.join(bdir, name + ".so"), os.path.join(OUT, name + ".so"))


def build(force=False):
    if not os.path.isdir(os.path.join(REF, "src")):
        return False  # GPU box: only the prebuilt .so files exist
    want = [os.path.join(OUT, n) for n in ("nslam_ref_corr.so", "nslam_ref_droid.so")]
    if not force and all(os.path.exists(w) for w in want):
        return True
    tmp = tempfile.mkdtemp(prefix="nslam_ref_")
    # --- correlation kernels
    srcs = []
    for f in ("correlation_kernels.cu", "altcorr_kernel.cu"):
        txt = open(os.path.join(REF, "src", f)).read().replace(".type()", ".scalar_type()")
        p = os.path.join(tmp, f)
        open(p, "w").write(txt)
        srcs.append(p)
    _build("nslam_ref_corr", srcs + [os.path.join(HERE, "ref_glue_corr.cpp")], tmp)
    # --- droid kernels
    lines = open(os.path.join(REF, "src", "droid_kernels.cu")).read().split("\n")
    keep = [l for n, l in enumerate(lines, 1) if not any(a <= n <= b for a, b in STRIP)]
    p = os.path.join(tmp, "droid_kernels_ref.cu")
    open(p, "w").write("\n".join(keep) + "\n" + open(os.path.join(HERE, "ref_glue_droid.cu")).read())
    _build("nslam_ref_droid", [p], tmp)
    shutil.rmtree(tmp, ignore_errors=True)
    return True


def load(name):
    """import oracle/_ref/<name>.so as a python module (needs torch loaded first)"""
    import importlib.util
    import torch  # noqa: F401
    path = os.path.join(OUT, name + ".so")
    if not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    ok = build(force="--force" in sys.argv)
    print("built" if ok else "reference sources not found; nothing built", os.listdir(OUT) if os.path.isdir(OUT) else [])
