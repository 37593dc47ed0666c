"""CPU-only: every launch_tc<...> instance of 3d-sis_b200/csrc/conv_tc.cu has a row in the per-element accuracy table of
tests/test_gpu_tc_accuracy.py, so a kernel change that adds an instance also adds the case that checks it."""
import os
import re

from conftest import ROOT
from test_gpu_tc_accuracy import CLUSTER_ROWS, ROWS, parse_inst


def source_instances():
    src = open(os.path.join(ROOT, "3d-sis_b200", "csrc", "conv_tc.cu")).read()
    return {parse_inst(a) for a in re.findall(r"launch_tc<([^<>]*)>\(", src)}


def test_every_tensor_core_instance_has_a_case():
    found = source_instances()
    assert len(found) >= 60, f"parsed only {len(found)} launch_tc<...> instances"
    covered = {r["inst"] for r in ROWS + CLUSTER_ROWS}
    missing = sorted(found - covered, key=str)
    assert not missing, f"launch_tc instances without a row in tests/test_gpu_tc_accuracy.py: {missing}"
    stale = sorted(covered - found, key=str)
    assert not stale, f"rows naming instances conv_tc.cu no longer has: {stale}"


def test_case_ids_are_unique():
    ids = [r["id"] for r in ROWS + CLUSTER_ROWS]
    assert len(ids) == len(set(ids))
