"""CPU-only: the per-layer table of the static stage (tests/test_gpu_static_stage.py) is complete.

  - every route name recorded in tests/golden/conv_routes.json (all cases, all modes) has a check in the table, or is listed
    as out of scope with the file that checks it; no entry of either list goes unused;
  - every math mode has a promise;
  - every conv and linear layer of both backbone programs (ScanNet with and without colour, SUNCG), the RPN hidden and
    merged head layers and classifier.0 is reached by at least one row;
  - row ids are unique, and every scene runs every math mode."""
import json
import os

from conftest import GOLDEN
from lib.nets.network import Network
from test_gpu_static_stage import (CYCLE, OUT_OF_SCOPE, PROMISE, ROUTE_CHECKS, ROWS, SCENES, active_levels,
                                   stage_layers)
import sis3d_synth as synth

# route names of paths no golden case records: the dense colour path (one row runs it with the sparse path off) and the
# forward from raw images through the 2-D encoder (USE_IMAGES_GT = False)
UNRECORDED = ("backproject_max", "enet_encoder")
# parameters of the static stage's model that no static-stage layer reads as such: the MLP tail and its heads (mlp_tail),
# the mask head (mask_stage); the two RPN heads run as one merged layer per level
NOT_STATIC = ("classifier.2", "classifier.4", "classifier_cls_score_net", "classifier_bbox_pred_net", "mask_backbone.",
              "rpn_cls_score_net_level", "rpn_bbox_pred_net_level")


def golden_families():
    with open(os.path.join(GOLDEN, "conv_routes.json")) as f:
        routes = json.load(f)
    return {n.split("[")[0] for case in routes.values() for n in case["routes"]}


def test_every_recorded_route_has_a_check():
    fams = golden_families()
    missing = fams - set(ROUTE_CHECKS) - set(OUT_OF_SCOPE)
    assert not missing, f"routes with neither a check nor an out-of-scope entry: {sorted(missing)}"
    assert not set(ROUTE_CHECKS) & set(OUT_OF_SCOPE)
    unused = (set(ROUTE_CHECKS) | set(OUT_OF_SCOPE)) - fams - set(UNRECORDED)
    assert not unused, f"table entries no recorded route uses: {sorted(unused)}"
    for name, where in OUT_OF_SCOPE.items():
        for f in where.split(",")[0].split():
            assert os.path.exists(os.path.join(os.path.dirname(GOLDEN), os.path.basename(f))), f"{name}: {f} does not exist"


def test_every_mode_has_a_promise():
    assert set(PROMISE) == set(Network.MATH_MODES)
    assert set(CYCLE) == set(Network.MATH_MODES)
    assert set(PROMISE.values()) <= {"h3", "tf32", "fmaf"}
    for mode, (static, _) in Network.MATH_MODES.items():  # a compensated static form promises the compensated bound
        assert (PROMISE[mode] == "h3") == (static in ("f16x3", "tf32x3")), mode
        assert (PROMISE[mode] == "fmaf") == (static == "fp32"), mode


def _net(scene):
    net, cfg = synth.make_net(SCENES[scene], keep_debug=False, math="exact")
    return net, cfg


def test_every_layer_is_reached_by_a_row():
    programs = {}  # (backbone, colour) -> (layers of the model, layers the rows reach)
    for scene in dict.fromkeys(r["scene"] for r in ROWS):
        net, cfg = _net(scene)
        key = (cfg.NET, bool(cfg.USE_IMAGES))
        params = {k[:-len(".weight")] for k in net.state_dict() if k.endswith(".weight")}
        params = {p for p in params if not p.startswith(NOT_STATIC)}
        params |= {f"rpn_heads_level{lvl}" for lvl in active_levels()}
        reached = set(stage_layers(net.SPEC, cfg.USE_IMAGES, active_levels()))
        have, got = programs.get(key, (set(), set()))
        programs[key] = (have | params, got | reached)
    assert set(programs) == {("ScanNet_Backbone", True), ("ScanNet_Backbone", False), ("SUNCG_Backbone", True)}
    for key, (params, reached) in programs.items():
        assert params - reached == set(), f"{key}: layers no row reaches: {sorted(params - reached)}"
        assert reached - params == set(), f"{key}: rows name layers the model does not have: {sorted(reached - params)}"


def test_rows():
    ids = [r["id"] for r in ROWS]
    assert len(set(ids)) == len(ids)
    for scene in ("cfg2", "cfg5", "odd_45x27x41", "cfg1_32"):
        modes = [r["mode"] for r in ROWS if r["scene"] == scene and not r["updated"]]
        assert modes == list(CYCLE), scene
        assert any(r["updated"] for r in ROWS if r["scene"] == scene)
    assert {r["mode"] for r in ROWS if r["scene"] == "cfg3"} == {"exact", "fp16"}
    assert any(not r["sparse"] and r["scene"] == "cfg2" and r["mode"] == "exact" for r in ROWS)
