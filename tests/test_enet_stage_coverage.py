"""CPU: the launch-by-launch ENet check (tests/test_gpu_enet_stage.py) covers what it claims -- every op kind of the
folded program has a check, every broken-encoder model applies to at least one row, and the kernel instances its rows
reach under sis3d_enet_conv2d's launch rule, with those of the `enet` kernel rows of tests/test_gpu_simt_accuracy.py,
are exactly the enet_conv2d_kernel instances enet2d.cu launches."""
import os
import re

import torch

from conftest import ROOT, load_golden
from lib.nets.enet_program import compile_enet
from test_gpu_enet_stage import CHECKS, MODELS, ROWS, _roles, encoder_launches, instances_reached
from test_gpu_simt_accuracy import ENET_ROWS


def _golden_params():
    g = load_golden("enet_encoder.npz")
    return [torch.from_numpy(g[k]) for k in sorted(k for k in g if k.startswith("p"))]


def test_every_program_op_kind_has_a_check():
    assert {op[0] for op in compile_enet(_golden_params())} == set(CHECKS)


def test_every_model_applies_to_a_row():
    for name, applies in MODELS.items():
        assert any(applies(r) for r in ROWS), name


def test_rows_reach_every_enet_conv_instance():
    src = open(os.path.join(ROOT, "3d-sis_b200", "csrc", "enet2d", "enet2d.cu")).read()
    listed = {f"enet_conv2d_kernel<{a},{b},{c}>"
              for a, b, c in re.findall(r"SIS3D_ENET_GO\((\d+),\s*(true|false),\s*(\d+)\)", src)}
    assert len(listed) == 10
    stage = instances_reached()
    assert stage | {k for r in ENET_ROWS for k in r["kernels"]} == listed
    # the view counts straddle every half- / full-height switch: both tile heights of each narrow N tile at 256 x 328
    assert {"enet_conv2d_kernel<16,false,2>", "enet_conv2d_kernel<16,false,4>", "enet_conv2d_kernel<16,true,2>",
            "enet_conv2d_kernel<16,true,4>", "enet_conv2d_kernel<32,true,2>", "enet_conv2d_kernel<32,true,4>",
            "enet_conv2d_kernel<64,true,4>"} == stage


def test_rows_hit_the_odd_pooled_skips():
    """250 x 328 pools a 125-row skip at the first down-sampling bottleneck; 244 x 328 a 61-row and 256 x 324 an 81-column
    one at the second."""
    def odd_skips(r):
        return [(L["res"][1], L["res"][2]) for L in encoder_launches(r["n"], r["H"], r["W"])
                if L["res"] and L["res"][0] == "pool" and (L["res"][1] % 2 or L["res"][2] % 2)]
    got = {(r["H"], r["W"]): odd_skips(r) for r in ROWS if odd_skips(r)}
    assert got == {(250, 328): [(125, 164)], (244, 328): [(61, 82)], (256, 324): [(64, 81)]}


def test_structure_matches_the_parameter_list():
    params = _golden_params()
    assert len(_roles()) == len(params) == 429
    convs = [op for op in compile_enet(params) if op[0] == "conv"]
    launches = encoder_launches(1, 256, 328)
    assert len(convs) == len(launches)
    for op, L in zip(convs, launches):
        cout, cin, kh, kw = op[1].shape
        assert (cout, cin, kh, kw, op[3], op[4], op[5]) == (L["cout"], L["cin"], L["kh"], L["kw"], L["stride"], L["pad"],
                                                             L["dil"])
