"""CPU-only: the per-element table of the ragged mask stage (tests/test_gpu_mask_stage.py) is complete, and its checker has
the power it claims on this machine.

  - every mask-stage math of Network.MATH_MODES maps to a route the table has rows for;
  - every edge class has a row on every route;
  - CPU torch models of the three correct routes -- fp32 accumulation (route 0), TF32-truncated tensor-core operands (route 1),
    fp16-stored activations with fp16 tensor-core operands (route 2) -- pass the fp64 bound on the table's small rows, and the
    model of each broken composition (a)-(e) that applies to a row misses it by POWER somewhere."""
import pytest
import torch

from lib.nets.network import Network
from test_gpu_mask_stage import (CANVAS, EDGE_CLASSES, MASK_MATH_ROUTE, POWER, ROUTES, ROWS, applicable, check_stage,
                                 cls_per_voxel, det_of, mask_weights, model_stage, reference_packed, scene_of)

SMALL = [r for r in ROWS if len(r["crops"]) <= 8]


def test_every_mask_math_has_a_route_with_rows():
    for mode, (_, mask_math) in Network.MATH_MODES.items():
        route = MASK_MATH_ROUTE[mask_math]
        assert any(route in r["routes"] for r in ROWS), f"{mode}: mask route {route} has no row"
    for route, mode in ROUTES.items():  # the mode each route's rows run in reaches that route
        assert MASK_MATH_ROUTE[Network.MATH_MODES[mode][1]] == route


def test_every_edge_class_has_a_row_on_every_route():
    for cls in EDGE_CLASSES:
        for route in ROUTES:
            assert any(cls in r["tags"] and route in r["routes"] for r in ROWS), f"edge class {cls}: no row on route {route}"
    unknown = set().union(*(r["tags"] for r in ROWS)) - set(EDGE_CLASSES)
    assert not unknown, f"rows tagged with classes the coverage list does not name: {sorted(unknown)}"
    assert len({r["id"] for r in ROWS}) == len(ROWS)
    by_id = {r["id"]: r for r in ROWS}
    assert len(by_id["bench_200"]["crops"]) == 200 and len(by_id["one_voxel_4100"]["crops"]) == 4100


def test_every_broken_model_applies_somewhere_on_every_route():
    for route in ROUTES:
        seen = set().union(*(applicable(r, route) for r in ROWS))
        want = {"scene_pad", "skip", "twice", "nbr_class", "gt"} | ({"no_slab", "unclipped"} if route in CANVAS else set())
        assert seen == want, f"route {route}: broken models with rows {sorted(seen)}"


CPU_ROWS = [(r, route) for r in SMALL for route in r["routes"]]


@pytest.mark.parametrize("r,route", CPU_ROWS, ids=[f"{r['id']}-route{route}" for r, route in CPU_ROWS])
def test_checker_on_cpu_route_models(r, route):
    torch.set_num_threads(max(1, torch.get_num_threads()))
    scene = scene_of(r)
    det = det_of(r)
    W32 = mask_weights(r["ncls"], r["weights"])
    ref, bound, zero, _ = reference_packed(scene.double(), r["crops"], [w.double() for w in W32], route)
    cv = cls_per_voxel(det, "cpu")
    got, bits = model_stage(scene, det, W32, route, "route")
    k = check_stage(ref, bound, zero, cv, got, bits)
    assert max(k) <= 1.0, f"the CPU model of route {route} misses the bound: masks {k[0]:.3g}, bits {k[1]:.3g}"
    for b in sorted(applicable(r, route, det)):
        got, bits = model_stage(scene, det, W32, route, "route", broken=b)
        m = max(check_stage(ref, bound, zero, cv, got, bits))
        assert m >= POWER, f"broken model {b} on route {route}: err/bound only {m:.3g} (correct model: {max(k):.3g})"
