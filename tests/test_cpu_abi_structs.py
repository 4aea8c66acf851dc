"""ABI drift guard: the ctypes mirrors in the Python host code must have exactly the size and field offsets of
the C structs in include/*.h (compiled here with gcc: the headers are plain C)."""
import ctypes
import os
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

C_SRC = r"""
#include <stdio.h>
#include <stddef.h>
#include "nslam.h"
#include "nslam_ba.h"
#include "nslam_nn.h"
#include "nslam_ngp.h"
#define SZ(T) printf("size " #T " %zu\n", sizeof(T))
#define OFF(T, f) printf("off " #T "." #f " %zu\n", offsetof(T, f))
int main(void) {
  SZ(nslam_ba_graph); OFF(nslam_ba_graph, NVC); OFF(nslam_ba_graph, ii); OFF(nslam_ba_graph, vc_idx);
  SZ(nslam_ba_buffers); OFF(nslam_ba_buffers, sblk); OFF(nslam_ba_buffers, ht); OFF(nslam_ba_buffers, T);
  SZ(nslam_update_ctx); OFF(nslam_update_ctx, ep); OFF(nslam_update_ctx, net); OFF(nslam_update_ctx, upmask);
  OFF(nslam_update_ctx, wp); OFF(nslam_update_ctx, bias); OFF(nslam_update_ctx, glo_w); OFF(nslam_update_ctx, e16);
  SZ(nslam_ngp_model); OFF(nslam_ngp_model, aabb_scale); OFF(nslam_ngp_model, scale); OFF(nslam_ngp_model, n_grid);
  OFF(nslam_ngp_model, grid_grad_fx); OFF(nslam_ngp_model, mlp_grad_part); OFF(nslam_ngp_model, part_rows);
  OFF(nslam_ngp_model, density_partials);
  printf("define NSLAM_NGP_DENSITY_BLOCKS %d\n", (int)NSLAM_NGP_DENSITY_BLOCKS);
  SZ(nslam_ngp_images); OFF(nslam_ngp_images, n_active); OFF(nslam_ngp_images, W);
  SZ(nslam_ngp_batch); OFF(nslam_ngp_batch, max_rays); OFF(nslam_ngp_batch, enc); OFF(nslam_ngp_batch, denc);
  OFF(nslam_ngp_batch, loss_fx);
  printf("enum NSLAM_W_COUNT %d\n", (int)NSLAM_W_COUNT);
  return 0;
}
"""


@pytest.fixture(scope="module")
def c_layout():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "abi.c"), os.path.join(d, "abi")
        open(src, "w").write(C_SRC)
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        out = subprocess.check_output([exe]).decode()
    lay = {}
    for line in out.splitlines():
        kind, name, val = line.split()
        lay[(kind, name)] = int(val)
    return lay


def test_ctypes_mirrors_match_c_structs(c_layout):
    sys.path.insert(0, ROOT)
    from nerf_slam_b200 import _lib, pyngp
    mirrors = {"nslam_ba_graph": _lib.BAGraph, "nslam_ba_buffers": _lib.BABuffers, "nslam_update_ctx": _lib.UpdateCtx,
               "nslam_ngp_model": pyngp.NgpModel, "nslam_ngp_images": pyngp.NgpImages, "nslam_ngp_batch": pyngp.NgpBatch}
    for (kind, name), val in c_layout.items():
        if kind == "size":
            assert ctypes.sizeof(mirrors[name]) == val, (name, ctypes.sizeof(mirrors[name]), val)
        elif kind == "off":
            st, field = name.split(".")
            assert getattr(mirrors[st], field).offset == val, (name, getattr(mirrors[st], field).offset, val)
    assert c_layout[("enum", "NSLAM_W_COUNT")] == _lib.N_UPDATE_WEIGHTS
    assert c_layout[("define", "NSLAM_NGP_DENSITY_BLOCKS")] == pyngp.DENSITY_BLOCKS
    from nerf_slam_b200.conv import UpdateOperatorTC
    assert len(UpdateOperatorTC.W_ORDER) == _lib.N_UPDATE_WEIGHTS


def test_headers_are_plain_c(c_layout):
    """compiling with gcc -std=c99 above already proves it; every exported symbol is declared (test_cpu_lib)"""
    assert c_layout
