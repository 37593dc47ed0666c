"""CPU-only: every __global__ kernel of csrc/rpn.cu, csrc/roi.cu and csrc/project.cu has a row in the decision-kernel table of
tests/test_gpu_decision_kernels.py (mlp_tail_kernel and mask_select_kernel: in the CUDA-core table of
tests/test_gpu_simt_accuracy.py), no row names a kernel that is gone, every proposal route has a row, and the route boundary
rows follow the constants of rpn.cu."""
import os
import re

from conftest import ROOT
from test_gpu_decision_kernels import MAX_FUSED, REDUCE_CAP, ROUTES, ROWS, SORT_CAP, _reduce_bytes
from test_gpu_simt_accuracy import ROWS as SIMT_ROWS

CSRC = os.path.join(ROOT, "3d-sis_b200", "csrc")
SIMT_OWNED = {"mlp_tail_kernel", "mask_select_kernel"}


def source_kernels():
    found = set()
    for f in ("rpn.cu", "roi.cu", "project.cu"):
        found |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", open(os.path.join(CSRC, f)).read()))
    return found


def test_every_decision_kernel_has_a_row():
    found = source_kernels()
    owned = found - SIMT_OWNED
    assert len(owned) == 19, f"parsed {len(owned)} kernels: {sorted(owned)}"
    covered = {k for r in ROWS for k in r["kernels"]}
    assert not sorted(owned - covered), f"kernels without a row: {sorted(owned - covered)}"
    assert not sorted(covered - found), f"rows naming kernels that are gone: {sorted(covered - found)}"
    simt = {k for r in SIMT_ROWS for k in r["kernels"]}
    assert SIMT_OWNED <= simt and SIMT_OWNED <= found


def test_every_route_has_a_row():
    routes = {r["route"] for r in ROWS}
    assert ROUTES <= routes, f"routes without a row: {sorted(ROUTES - routes)}"


def test_boundary_rows_follow_the_constants():
    assert SORT_CAP > 0
    assert _reduce_bytes(MAX_FUSED) <= REDUCE_CAP < _reduce_bytes(MAX_FUSED + 1)
    pres = {r["pre"] for r in ROWS if r["fam"] == "rpn"}
    assert {MAX_FUSED, MAX_FUSED + 1} <= pres
    scores = {r["score"] for r in ROWS if r["fam"] == "rpn"}
    assert {f"top{SORT_CAP}", f"top{SORT_CAP + 1}"} <= scores
    fused = [r for r in ROWS if r["fam"] == "rpn" and r["pre"] == MAX_FUSED and not r["unfused_env"]]
    unfused = [r for r in ROWS if r["fam"] == "rpn" and r["pre"] == MAX_FUSED + 1]
    assert fused[0]["launches"] == 5 and unfused[0]["launches"] == 6


def test_row_ids_are_unique():
    ids = [r["id"] for r in ROWS]
    assert len(ids) == len(set(ids))
