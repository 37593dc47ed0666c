"""CPU-only: the tables of the detection-head test (tests/test_gpu_head_stage.py) are complete.

  - every `_rec` name the forward records between the merged RPN heads and the mask stage, other than classifier.0 (a
    static-stage layer), has a check in HEAD_CHECKS, in every case and mode of tests/golden/conv_routes.json, and the
    static-stage table sends each of them to the head test;
  - every wiring model names a step the head test checks, and every step with a model has one;
  - row ids are unique, the bench scenes run every math mode, and the special rows are there."""
import json
import os

from conftest import GOLDEN
from lib.nets.network import Network
from test_gpu_head_stage import EMPTY_D, HEAD_CHECKS, MUTANTS, ROWS, SCENES, STEPS
from test_gpu_static_stage import CYCLE, OUT_OF_SCOPE


def head_names():
    with open(os.path.join(GOLDEN, "conv_routes.json")) as f:
        routes = json.load(f)
    out = set()
    for case in routes.values():
        names = [n.split("[")[0] for n in case["routes"]]
        heads = [i for i, n in enumerate(case["routes"]) if "[rpn_heads_level" in n]
        if not heads:  # ground-truth RoIs: no proposal head
            continue
        last_head = heads[-1]
        for n, full in zip(names[last_head + 1:], case["routes"][last_head + 1:]):
            if n == "mask_stage":
                break
            if not full.endswith("[classifier.0]"):
                out.add(n)
    return out


def test_every_head_route_has_a_check():
    names = head_names()
    assert names == set(HEAD_CHECKS), f"head routes {sorted(names)}, checks {sorted(HEAD_CHECKS)}"
    assert set(HEAD_CHECKS.values()) <= set(STEPS)
    for name in HEAD_CHECKS:
        assert "tests/test_gpu_head_stage.py" in OUT_OF_SCOPE[name], f"{name}: the static-stage table does not point at the head test"


def test_every_model_names_a_step():
    assert set(MUTANTS.values()) <= set(STEPS), sorted(set(MUTANTS.values()) - set(STEPS))
    assert set(HEAD_CHECKS.values()) <= set(MUTANTS.values()), "a checked step without a wiring model"


def test_rows():
    ids = [r["id"] for r in ROWS]
    assert len(set(ids)) == len(ids)
    for scene in ("cfg2", "cfg5", "odd_45x27x41", "suncg_40x24x40"):
        modes = [r["mode"] for r in ROWS if r["scene"] == scene and r["kind"] == "cycle"]
        assert modes == list(CYCLE), scene
        assert set(CYCLE) == set(Network.MATH_MODES)
        assert any(r["kind"] == "updated" for r in ROWS if r["scene"] == scene)
    assert {r["mode"] for r in ROWS if r["scene"] == "cfg3"} == {"exact", "fp16"}
    assert {r["mode"] for r in ROWS if r["scene"] == "cfg1_32"} == {"exact", "fp32"}
    assert not SCENES["cfg1_32"]["use_mask"]
    kinds = {r["kind"] for r in ROWS}
    assert kinds == {"cycle", "updated", "pre_nms_6000", "post_nms_7", "thresh_exact", "thresh_one", "empty"}
    assert [r["scene"] for r in ROWS if r["kind"] == "pre_nms_6000"] == ["cfg3"]


def test_empty_volume_is_the_largest_without_an_inside_anchor():
    from oracle import port
    from lib.utils.config import cfg
    import sis3d_synth as synth
    synth.make_net(SCENES["empty"], keep_debug=False, math="exact")
    tables = [cfg["ANCHORS_TYPE_LEVEL%d" % lvl] for lvl in (1, 2) if cfg["NUM_ANCHORS_LEVEL%d" % lvl]]

    def inside(d):
        g = ((d // 2) // 2,) * 3
        return sum(int(port.inside_mask(port.generate_anchors(g, port.read_anchor_table(t), 4), (d, d, d)).sum()) for t in tables)

    assert SCENES["empty"]["dims"] == (EMPTY_D,) * 3
    assert inside(EMPTY_D) == 0 and inside(EMPTY_D + 1) > 0, EMPTY_D
