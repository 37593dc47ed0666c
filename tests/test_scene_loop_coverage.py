"""CPU-only: the row table of tests/test_gpu_scene_loop.py covers every workload bench.py times (shape, view count, config,
default math), every conv math mode, graph-cache eviction and the scene counts around the loop's depth, and every row's
sequence is one in which a mix-up between scenes would show."""
import sys

import pytest

from conftest import ROOT
from lib.nets.network import Network
from test_gpu_scene_loop import ROWS, loop_depth

sys.path.insert(0, ROOT)
import bench  # noqa: E402


class _Slots:
    """Duck-typed `self` for Network._scene_loop that only records which stream slots it asks for."""

    def __init__(self):
        self.slots = set()

    def _slot(self, i):
        self.slots.add(i)
        return i

    def _stage_inputs(self, blobs, killing_inds, slot):
        return dict(scene=blobs)

    def _run_static(self, h):
        return h

    def _launch_ragged(self, h):
        return h

    def _finalize(self, h):
        return h


def measured_depth(monkeypatch, static, depth):
    for env, v in (("SIS3D_PIPE_STATIC", static), ("SIS3D_PIPE_DEPTH", depth)):
        if v is None:
            monkeypatch.delenv(env, raising=False)
        else:
            monkeypatch.setenv(env, str(v))
    rec = _Slots()
    assert len(list(Network._scene_loop(rec, iter(range(64))))) == 64
    return len(rec.slots)


def _shapes(r):
    return {(c[0], c[1]) for c in r["seq"]}


@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg3s", "cfg4", "cfg5", "cfg2-enet"])
def test_every_bench_workload_has_a_row(name):
    enet = name.endswith("-enet")
    wl = bench.workload(name.split("-")[0], 0, 1)
    shapes = {(d, n) for _, d, n in wl["scenes"]}
    rows = [r for r in ROWS if r["bench"] == name.split("-")[0] and r["enet"] == enet and r["cfgname"] == wl["cfgname"]
            and r["math"] == wl["math_default"] and _shapes(r) <= shapes]
    if name == "cfg4":
        rows = [r for r in rows if len(_shapes(r)) >= 3]
    else:
        rows = [r for r in rows if _shapes(r) == shapes]
    assert rows, f"no scene-loop row runs the {name} workload"


def test_cfg2_rows_cover_every_input_form():
    assert {r["inputs"] for r in ROWS if r["bench"] == "cfg2" and not r["enet"]} == {"device", "pinned", "pageable"}


def test_every_math_mode_has_a_row():
    for m in Network.MATH_MODES:
        assert any(r["math"] == m and len(_shapes(r)) >= 2 for r in ROWS if r["mech"] is None and r["bench"] is None), \
            f"no mixed-shape row in {m}"


def test_some_rows_evict_graphs():
    evict = [r for r in ROWS if r["graph_cache"] is not None and r["graph_cache"] < len(_shapes(r))]
    assert {r["graph_cache"] for r in evict} >= {1, 2}
    assert {r["graph_after"] for r in evict} >= {1, 3}


def test_loop_depth_follows_the_scene_loop(monkeypatch):
    knobs = {(r["static"], r["depth"]) for r in ROWS} | {(None, None), (1, None), (6, None), (2, 6), (3, 2)}
    for static, depth in knobs:
        assert loop_depth(static, depth) == measured_depth(monkeypatch, static, depth), (static, depth)


def test_scene_counts_around_the_depth(monkeypatch):
    d = measured_depth(monkeypatch, None, None)
    plain = {len(r["seq"]) for r in ROWS if r["static"] is None and r["depth"] is None and r["mech"] is None
             and r["bench"] is None and r["oracle"] is None}
    assert {1, d - 1, d, d + 1} <= plain, f"depth {d}: plain rows have scene counts {sorted(plain)}"
    statics = {r["static"] for r in ROWS}
    assert {1, 4, 6} <= statics and any(r["depth"] is not None for r in ROWS)
    for r in ROWS:
        if r["static"] is not None or r["depth"] is not None:
            assert len(r["seq"]) > 2 * loop_depth(r["static"], r["depth"]), f"{r['id']}: slots are not reused twice"


def test_loop_mechanics_rows():
    assert {r["mech"] for r in ROWS} >= {"home_stream", "break", "reload", "set_math", "edges"}
    families = {(r["cfgname"], r["enet"]) for r in ROWS if r["oracle"] and r["math"] == "fp32"}
    assert families == {("scannet", False), ("suncg", False), ("scannet", True)}, families


@pytest.mark.parametrize("r", [r for r in ROWS if r["mech"] != "edges"], ids=lambda r: r["id"])
def test_sequences_can_show_a_mix_up(r):
    """Consecutive scenes and any two scenes on one slot are different contents (the GPU test checks that their references
    differ as well); the edge row's order is chosen from its references and checked there."""
    seq, depth = r["seq"], loop_depth(r["static"], r["depth"])
    for i in range(len(seq)):
        for j in [i + 1] + list(range(i + depth, len(seq), depth)):
            if j < len(seq):
                assert seq[i] != seq[j], (r["id"], i, j)


def test_row_ids_are_unique():
    ids = [r["id"] for r in ROWS]
    assert len(ids) == len(set(ids))
