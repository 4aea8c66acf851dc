"""The C-ABI shared library loads on a CPU-only box and exports every symbol the headers declare."""
import os
import re

from nerf_slam_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    names = set()
    inc = os.path.join(ROOT, "include")
    for f in os.listdir(inc):
        txt = open(os.path.join(inc, f)).read()
        names |= set(re.findall(r"^int\s+(nslam_\w+)\s*\(", txt, flags=re.M))
    return names


def test_library_loads_and_exports_all_declared_symbols(lib):
    declared = _declared()
    assert declared, "no declarations found"
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/ but not exported"
    # and the python binding table covers exactly the declared set
    assert set(_lib.exported_symbols()) == declared


def test_ops_fail_loudly_without_cuda():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from nerf_slam_b200 import droid_backends
    with pytest.raises(RuntimeError):
        droid_backends.frame_distance(torch.zeros(2, 7), torch.zeros(2, 4, 4), torch.zeros(4),
                                      torch.zeros(1, dtype=torch.long), torch.ones(1, dtype=torch.long), 0.3)


def test_product_code_never_touches_the_oracle():
    """oracle/ is test infrastructure: the package must not import, load or reference it"""
    import re
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nerf_slam_b200")
    pat = re.compile(r"^\s*(from\s+oracle|import\s+oracle|from\s+\.\.?oracle)|oracle/_ref|oracle\._ref|build_ref", re.M)
    bad = []
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):                      # (CUDA sources only mention the oracle in comments)
                txt = open(os.path.join(root, f), errors="ignore").read()
                if pat.search(txt):
                    bad.append(os.path.join(root, f))
    assert not bad, bad


def _mutable_device_globals(txt):
    """namespace-scope `__device__` / `__managed__` variables that are not const: device memory no caller owns, shared
    by every user of the library in the process (the `__constant__` tables of tsdf_mesh.cu are read-only and allowed)"""
    code = re.sub(r"//[^\n]*|/\*.*?\*/", "", txt, flags=re.S)
    found, blocks = [], []            # blocks: True for a namespace / extern "C" block (its contents stay at namespace scope)
    for piece in re.split(r"(?<=[;{}])", code):
        stmt = " ".join(piece.split())
        if stmt.endswith("}"):                                       # the end of a block or of a braced initialiser row
            if blocks:
                blocks.pop()
            continue
        words = stmt.rstrip(";{").replace("(", " ( ").split()
        if all(blocks) and ("__device__" in words or "__managed__" in words) and "(" not in words \
                and not {"const", "constexpr", "__constant__"} & set(words):
            found.append(stmt)
        if stmt.endswith("{"):
            blocks.append(bool(re.search(r"\bnamespace\b[\w\s]*\{$|extern \"C\" \{$", stmt)))
    return found


def test_mutable_device_global_scan_finds_what_it_should():
    src = ("namespace ngp {\n__device__ float g_partials[2 * 592];\n__device__ __forceinline__ float f(float x) { return x; }\n"
           "__constant__ int c_tab[4] = {1, 2, 3, 4};\n__device__ const float k_half = 0.5f;\nstatic __device__ int counter = 0;\n"
           "__global__ void k(float* o) { __shared__ float s[32]; o[0] = s[0]; }\n}  // namespace ngp\n"
           "extern \"C\" {\n__managed__ int m_flag;\n}\n// __device__ float in_a_comment;\n")
    assert _mutable_device_globals(src) == ["__device__ float g_partials[2 * 592];", "static __device__ int counter = 0;",
                                            "__managed__ int m_flag;"]


def test_library_keeps_no_hidden_device_state():
    """the caller owns all device memory and the library never synchronises: no allocation, free or synchronous memset
    in csrc/, no mutable namespace-scope device variable (two callers on two streams would race on it), and the
    per-device dynamic shared-memory attribute is set only through ensure_dyn_smem"""
    csrc = os.path.join(ROOT, "nerf_slam_b200", "csrc")
    src = {f: open(os.path.join(csrc, f)).read() for f in sorted(os.listdir(csrc)) if f.endswith((".cu", ".cuh"))}
    for f, txt in src.items():
        assert not re.search(r"\bcuda(Malloc|Free)\w*\s*\(", txt), f
        assert not re.search(r"\bcudaMemset(2D|3D)?\s*\(", txt), f
        assert "static bool configured" not in txt, f
        assert not _mutable_device_globals(txt), (f, _mutable_device_globals(txt))
    helper = re.search(r"cudaError_t ensure_dyn_smem\(.*?\n}\n", src["common.cuh"], flags=re.S)
    assert helper and helper.group(0).count("cudaFuncSetAttribute(") == 1
    assert sum(txt.count("cudaFuncSetAttribute") for txt in src.values()) == 1
