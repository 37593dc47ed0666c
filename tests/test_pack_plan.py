"""CPU: the weight packs `Network._ensure_packed` makes in each conv math mode (Network.pack_plan, a function of the layers'
weight shapes and the mode) -- the forms the mode reads, every pack the kernel routes of tests/golden/conv_routes.json read
(captured on the GPU by tools/capture_routes.py), and less memory than packing every layer into every form."""
import json
import os
import re

import pytest
import torch

import sis3d_synth as synth
from conftest import GOLDEN
from lib.nets.network import Network

# mode -> weight forms: the CUDA-core fp32 form, the static-stage form, its fallbacks and the mask-stage form
FORMS = {"exact": {"fp32", "f16x3", "fp16"}, "f16x3": {"fp32", "f16x3", "tf32"}, "tf32x3": {"fp32", "tf32x3", "tf32"},
         "mixed": {"fp32", "tf32", "fp16"}, "tf32": {"fp32", "tf32"}, "fp16": {"fp32", "fp16", "tf32"}, "fp32": {"fp32"}}
ALL_FORMS = ("fp32", "tf32", "tf32x3", "f16x3", "fp16")
CONFIGS = {"cfg2": ("scannet", None), "cfg5": ("suncg", None), "gt_rois": ("scannet", True)}
# timing name of a route -> the form of the pack it reads (of the layer in brackets; of its conv2 and conv3 for a fused tail)
ROUTE_FORM = {"conv": "fp32", "linear": "fp32", "conv_tc16": "fp16", "conv_tc": "tf32", "conv_tc_x3": "tf32x3",
              "conv_tc_h3": "f16x3", "conv_tc_h3_split": "f16x3", "linear_tc": "tf32", "linear_tc_x3": "tf32x3",
              "linear_tc_h3": "f16x3"}
FUSED_FORM = {"conv_tc_fused": "tf32", "conv_tc_fused_x3": "tf32x3", "conv_tc_fused_h3": "f16x3", "conv_tc_fused_h3_split": "f16x3"}
NO_WEIGHTS = {"project_map", "maxpool3", "cast_f16", "rpn_proposals", "roi_pool_levels", "detect_decode"}
MLP_TAIL = ("classifier.2", "classifier.4", "classifier_cls_score_net", "classifier_bbox_pred_net")


def routes():
    with open(os.path.join(GOLDEN, "conv_routes.json")) as f:
        return json.load(f)


_SHAPES = {}


def shapes_of(config):
    if config not in _SHAPES:
        cfgname, gt_rois = CONFIGS[config]
        net, _ = synth.make_net(dict(cfgname=cfgname, use_images=True, use_mask=True), keep_debug=False, gt_rois=gt_rois)
        _SHAPES[config] = {k: tuple(w.shape) for k, (w, _) in net._layer_weights().items()}
    return _SHAPES[config]


def packs_read(case):
    """{(form, layer)} the recorded route of one forward reads."""
    out = set()
    for name in case["routes"]:
        m = re.fullmatch(r"(\w+)\[(.+)\]", name)
        kind, layer = m.groups() if m else (name, None)
        if m and kind in ROUTE_FORM:
            out.add((ROUTE_FORM[kind], layer))
        elif m and kind in FUSED_FORM:
            out |= {(FUSED_FORM[kind], layer + ".conv2"), (FUSED_FORM[kind], layer + ".conv3")}
        elif name == "backproject_conv_k2s2":
            out.add(("fp32", "color.0"))
        elif name == "mlp_tail":
            out |= {("fp32", k) for k in MLP_TAIL}
        elif name == "mask_stage":
            inst = case["mask_tc_instances"]
            form = "fp32" if not inst else {2: "fp16", 4: "tf32"}[inst[0][2]]  # element bytes of the 64->64 layers' operands
            out |= {("fp32", "mask_backbone.geometry.0"), ("fp32", "mask_backbone.geometry.10")}
            out |= {(form, f"mask_backbone.geometry.{i}") for i in (2, 4, 6, 8)}
        else:
            assert name in NO_WEIGHTS, f"route name {name!r} not understood"
    return out


def nbytes(layout):
    return 0 if layout == () else torch.Size(layout[0]).numel() * torch.empty(0, dtype=layout[1]).element_size()


def test_fixture_covers_every_mode_and_config():
    assert set(routes()) == {f"{c}/{m}" for c in CONFIGS for m in Network.MATH_MODES}


@pytest.mark.parametrize("mode", list(Network.MATH_MODES))
@pytest.mark.parametrize("config", list(CONFIGS))
def test_plan_holds_every_pack_the_routes_read(config, mode):
    shapes = shapes_of(config)
    plan = Network.pack_plan(shapes, mode)
    assert set(plan) == FORMS[mode] == set(Network.mode_forms(mode))
    assert set(plan["fp32"]) == set(shapes)  # every layer keeps its CUDA-core pack
    read = packs_read(routes()[f"{config}/{mode}"])
    missing = sorted(p for p in read if p[1] not in plan.get(p[0], {}))
    assert not missing, f"{config}/{mode}: routes read packs that are not planned: {missing}"
    planned = sum(nbytes(lay) for layers in plan.values() for lay in layers.values())
    every_form = sum(nbytes(Network.pack_layout(f, s) or ()) for f in ALL_FORMS for s in shapes.values())
    print(f"{config}/{mode}: {planned / 2**20:.1f} MiB planned, {every_form / 2**20:.1f} MiB in every form")
    assert planned < every_form

