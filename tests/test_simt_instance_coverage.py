"""CPU-only: every instance of the fp32 CUDA-core kernels -- conv3d_igemm_f32<BN, TM> (conv_simt.cu), sparse_gemm_kernel<COUT>
(sparse.cu) and SIS3D_ENET_GO(BN, VEC, TM) (enet2d/enet2d.cu) -- has a row in the per-element accuracy table of
tests/test_gpu_simt_accuracy.py, and no row names an instance the sources no longer launch."""
import os
import re

from conftest import ROOT
from test_gpu_simt_accuracy import ROWS

CSRC = os.path.join(ROOT, "3d-sis_b200", "csrc")


def _src(name):
    return open(os.path.join(CSRC, name)).read()


def source_instances():
    found = {f"conv3d_igemm_f32<{a},{b}>" for a, b in re.findall(r"conv3d_igemm_f32<(\d+),\s*(\d+)><<<", _src("conv_simt.cu"))}
    found |= {f"sparse_gemm_kernel<{a}>" for a in re.findall(r"sparse_gemm_kernel<(\d+)><<<", _src("sparse.cu"))}
    found |= {f"enet_conv2d_kernel<{a},{b},{c}>"
              for a, b, c in re.findall(r"SIS3D_ENET_GO\((\d+),\s*(true|false),\s*(\d+)\)", _src(os.path.join("enet2d", "enet2d.cu")))}
    return found


def test_every_simt_instance_has_a_case():
    found = source_instances()
    assert len(found) == 14, f"parsed {len(found)} instances: {sorted(found)}"
    covered = {k for r in ROWS for k in r["kernels"] if "<" in k}
    missing = sorted(found - covered)
    assert not missing, f"kernel instances without a row in tests/test_gpu_simt_accuracy.py: {missing}"
    stale = sorted(covered - found)
    assert not stale, f"rows naming instances the sources no longer launch: {stale}"


def test_case_ids_are_unique():
    ids = [r["id"] for r in ROWS]
    assert len(ids) == len(set(ids))
