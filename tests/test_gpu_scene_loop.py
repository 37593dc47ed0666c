"""GPU: the pipelined scene loop (Network.forward_pipelined / _scene_loop), the code bench.py times, bit for bit against the
synchronous forward of a separate Network run eagerly (no CUDA graph), on every bench workload, every math mode, every input
form (pageable host, pinned host, device-resident as bench.py builds them), the loop's knobs (static stages in flight, slot
count, graph cache size, capture threshold) and scene edges (killed views, single view, no kept mask, a mask-heavy scene after
a light one on the same slot).

The loop keeps several scenes in flight on stream slots, each with captured graphs, static input buffers, a two-entry result
ring and a grow-only arena.  A stale static buffer, a ring entry handed out twice, a graph replayed under the wrong key, a
pinned staging buffer overwritten before its copy ran or a missing stream wait returns another scene's bits or a torn mix of
two scenes.  Every row is built so that such a mix-up cannot go unnoticed: consecutive scenes, and any two scenes on the same
slot, have different references (asserted on the references themselves).  `test_comparison_rejects_a_pairing_shift` shows
that the comparison fails when predictions are paired with the next scene's blobs."""
import functools
import gc
import os
import pickle
import sys

import numpy as np
import pytest
import torch

import sis3d_synth as synth
from conftest import ROOT

sys.path.insert(0, ROOT)
import bench  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMALL, SMALL2 = (45, 27, 41), (40, 24, 36)


# ------------------------------------------------------------------------------------------------ the row table
def sc(dims, n_views, seed, edge=None):
    """One scene's content: volume shape, view count, seed of make_scene / make_views, and an edge:
    None | 'kill1' (view 1 sees nothing: depth 9.0) | 'killall' (every view killed) | 'case:<tag>' (synth.build_case)."""
    return (tuple(dims), int(n_views), int(seed), edge)


def _distinct(dims, n_views, seed0, count):
    return [sc(dims, n_views, seed0 + j) for j in range(count)]


def _cycle(contents, count):
    return [contents[i % len(contents)] for i in range(count)]


def _mixed(seed0):
    """Short mixed-shape sequence: two shapes with different view counts, both repeated (so they are captured)."""
    a, b = _distinct(SMALL, 3, seed0, 3), _distinct(SMALL2, 2, seed0 + 50, 2)
    return [a[0], b[0], a[1], b[1], a[2], a[0], b[0], a[1], b[1]]


def loop_depth(static=None, depth=None):
    """Scenes in flight (= stream slots) of _scene_loop for SIS3D_PIPE_STATIC / SIS3D_PIPE_DEPTH (None: unset).
    tests/test_scene_loop_coverage.py checks this against the loop itself."""
    n_static = max(1, static if static is not None else 4)
    return max(n_static + 2, depth if depth is not None else n_static + 3)


def _cfg4_seq(n_classes=3, uses=4, depth=loop_depth()):
    """cfg4-style sequence: the first n_classes shape classes of bench.CFG4_SHAPES, three contents each.  Slot s sees the
    classes pattern[(u + s) % 4] on its u-th use (A, B, A, C): with a graph cache of 1 every use evicts and A is captured
    again after its eviction; with 2 the second A hits and C evicts B.  Contents are picked so that consecutive scenes and
    scenes on the same slot differ."""
    classes = bench.CFG4_SHAPES[:n_classes]
    pattern = [0, 1, 0, 2]
    seq = []
    for i in range(uses * depth):
        s, u = i % depth, i // depth
        k = pattern[(u + s) % len(pattern)]
        dims, nv = classes[k]
        for v in range(3):
            cand = sc(dims, nv, 4000 + 10 * k + v)
            if (not seq or seq[-1] != cand) and all(seq[j] != cand for j in range(s, i, depth)):
                break
        seq.append(cand)
    return seq


ROWS = []


def _row(id, seq, **kw):
    r = dict(id=id, seq=seq, cfgname="scannet", enet=False, math="exact", inputs="pageable", static=None, depth=None,
             graph_cache=None, graph_after=None, mech=None, bench=None, oracle=None)
    assert set(kw) <= set(r) | {"math2"}, set(kw) - set(r)
    r.update(kw)
    ROWS.append(r)
    return r


# bench workloads (shapes, view counts, math and input forms of bench.workload / bench.main)
CFG2 = _distinct((96, 48, 96), 5, 1000, 3 * loop_depth() + 1)  # every slot replays its graph three times: the ring wraps
for _inp in ("device", "pinned", "pageable"):
    _row(f"cfg2-{_inp}", CFG2, inputs=_inp, bench="cfg2")
_row("cfg3s", _cycle(_distinct((88, 44, 88), 40, 3000, 3), 10), inputs="pinned", bench="cfg3s")
_row("cfg3", _cycle(_distinct((208, 48, 160), 40, 3100, 3), 9), inputs="device", bench="cfg3")
_row("cfg4-cache1-after1", _cfg4_seq(), inputs="pinned", graph_cache=1, graph_after=1, bench="cfg4")
_row("cfg4-cache2-after3", _cfg4_seq(), inputs="device", graph_cache=2, graph_after=3, bench="cfg4")
_row("cfg5", _distinct((96, 48, 96), 3, 5000, 9), cfgname="suncg", math="fp16", inputs="pinned", bench="cfg5")
_row("cfg2-enet", _distinct((96, 48, 96), 5, 1100, 9), enet=True, inputs="pinned", bench="cfg2")
# every math mode over a short mixed-shape sequence
for _m in ("exact", "f16x3", "tf32x3", "mixed", "tf32", "fp16", "fp32"):
    _row(f"math-{_m}", _mixed(200), math=_m)
# scene edges interleaved in one sequence (the order is chosen from the references, see _edge_order)
_row("edges", _distinct(SMALL, 3, 600, 5) + [sc(SMALL, 3, 610, "kill1"), sc(SMALL, 3, 611, "killall"), sc(SMALL, 1, 612)],
     mech="edges")
# loop mechanics
for _s in (1, 4, 6):
    _row(f"static{_s}", _distinct(SMALL, 3, 700 + 30 * _s, 2 * loop_depth(_s) + 1), static=_s)
_row("static2-depth6", _distinct(SMALL, 3, 900, 2 * loop_depth(2, 6) + 1), static=2, depth=6)
for _n in sorted({1, loop_depth() - 1, loop_depth(), loop_depth() + 1}):
    _row(f"count{_n}", _distinct(SMALL, 3, 950, _n))
_row("home-stream", _mixed(230), mech="home_stream", inputs="pinned")
_row("break", _mixed(240), mech="break")
_row("reload", _mixed(250), mech="reload")
_row("set-math", _mixed(260), mech="set_math", math="exact", math2="tf32")
# one row per config family whose first scene is an oracle case: the fp32 reference's integer outputs against the CPU oracle
_row("oracle-scannet", [sc(SMALL, 3, 202, "case:odd_45x27x41")] + _distinct(SMALL, 3, 800, 7), math="fp32",
     oracle="odd_45x27x41")
_row("oracle-suncg", [sc((40, 24, 40), 3, 404, "case:suncg_40x24x40")] + _distinct((40, 24, 40), 3, 810, 7), cfgname="suncg",
     math="fp32", oracle="suncg_40x24x40")
_row("oracle-enet", [sc(SMALL, 3, 202, "case:odd_45x27x41")] + _distinct(SMALL, 3, 820, 7), enet=True, math="fp32",
     oracle="odd_45x27x41")


# ------------------------------------------------------------------------------------------------ scenes and inputs
_PORT = {}  # the CPU oracle module, for contents that are oracle cases


@functools.lru_cache(maxsize=None)
def _content(content, cfgname, enet):
    """(data, views) of a content, numpy; views["feats"] are RGB frames [n,3,256,328] when enet (bench.py --enet)."""
    dims, n, seed, edge = content
    if edge and edge.startswith("case:"):
        c = synth.CASES[edge[5:]]
        assert c["dims"] == dims and c["n_img"] == n and c["seed"] == seed and c["cfgname"] == cfgname
        _, _, data, views = synth.build_case(_PORT["port"], c)
    else:
        data, boxes = synth.make_scene(seed, dims)
        views = synth.make_views(seed, dims, n, boxes)
    if edge == "kill1":
        views["depths"][1][:] = 9.0
    elif edge == "killall":
        views["depths"][:] = 9.0
    if enet:
        views["feats"] = np.random.default_rng(seed + 7).standard_normal((n, 3, 256, 328)).astype(np.float32)
    return data, views


def _blobs(content, row, form):
    data, views = _content(content, row["cfgname"], row["enet"])
    hb = synth.make_blobs(None, data, views, pin=(form != "pageable"))
    if form != "device":
        return hb
    ni = hb["nearest_images"]  # exactly bench.py's dev_in
    return {"data": hb["data"].to(DEV), "id": hb["id"],
            "nearest_images": {"images": [ni["images"][0].to(DEV)], "depths": [ni["depths"][0].to(DEV)],
                               "poses": ni["poses"], "world2grid": ni["world2grid"]}}


def _inputs(row, seq, form=None):
    """One blobs dict per position (own identity), sharing the tensors of a content like bench.py's rotating inputs."""
    per = {}
    for c in seq:
        if c not in per:
            per[c] = _blobs(c, row, form or row["inputs"])
    return [dict(per[c]) for c in seq]


# ------------------------------------------------------------------------------------------------ nets and weights
def _make_net(row, math, weights="w0", eager=False):
    c = dict(cfgname=row["cfgname"], use_images=True, use_mask=True)
    net, cfg = synth.make_net(c, keep_debug=False, math=math, enet=row["enet"])
    if weights != "w0":
        net.load_state_dict(_weights(net, weights))
    if eager:
        net._use_graph = False
    return net, cfg


def _weights(net, tag):
    """'w1': every parameter scaled by its own factor in [0.75, 1.25] (another model of the same shape);
    'cls0.05': class scores scaled down so that confidences spread below 1 and a class threshold separates scenes."""
    sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    if tag == "w1":
        rng = np.random.default_rng(11)
        for k, v in sd.items():
            if v.is_floating_point() and k in dict(net.named_parameters()):
                sd[k] = v * torch.from_numpy(rng.uniform(0.75, 1.25, tuple(v.shape)).astype(np.float32))
    elif tag == "cls0.05":
        for k in ("classifier_cls_score_net.weight", "classifier_cls_score_net.bias"):
            sd[k] = sd[k] * 0.05
    else:
        raise ValueError(tag)
    return sd


# ------------------------------------------------------------------------------------------------ snapshots and comparison
def _snap(P, bits="mask_bits_host"):
    """Copies of everything a scene's predictions carry, made on the current (consumer) stream at yield time: the yielded
    dict and its tensors live in slot-owned buffers that the loop reuses."""
    s = {k: P[k][0].clone() for k in ("rois", "roi_scores", "level_inds")}
    s.update({k: P[k].clone() for k in ("cls_score", "cls_prob", "cls_pred", "bbox_pred")})
    s["detections_host"] = P["detections_host"].copy()
    masks = list(P["mask_pred"][0])  # every crop through the public [1, ncls, w, h, l] views
    s["mask_shapes"] = np.array([tuple(m.shape) for m in masks], dtype=np.int64).reshape(-1, 5)
    s["mask_pred"] = torch.cat([m.reshape(-1) for m in masks]) if masks else torch.zeros(0)
    if bits == "mask_bits_host":
        s["mask_bits"] = P["mask_bits_host"].copy() if "mask_bits_host" in P else None
    else:
        s["mask_bits"] = P["mask_bits"].clone() if "mask_bits" in P else None
    return s


def _host(s):
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in s.items()}


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _diff(got, want):
    return [k for k in want if not _same(got[k], want[k])]


def _compare(row_id, seq_blobs, refs, got, check_identity=True):
    """got = [(yielded blobs, host snapshot)] of a loop over seq_blobs; refs[k] = host snapshot of the reference for the scene
    at position k.  The scene a yielded prediction is checked against is the one its yielded blobs name."""
    assert len(got) == len(seq_blobs), f"{row_id}: {len(got)} scenes yielded for {len(seq_blobs)}"
    where = {id(b): k for k, b in enumerate(seq_blobs)}
    for k, (b, s) in enumerate(got):
        if check_identity:
            assert b is seq_blobs[k], f"{row_id}: position {k} yielded the blobs of position {where.get(id(b))}"
        j = where[id(b)]
        bad = _diff(s, refs[j])
        assert not bad, f"{row_id}: scene {k} differs from its reference in {bad}"


def _assert_power(row_id, refs, depth):
    """Consecutive scenes, and any two scenes on the same slot (1 + i % depth), have different references."""
    for i in range(len(refs)):
        for j in [i + 1] + list(range(i + depth, len(refs), depth)):
            if j < len(refs):
                assert _diff(refs[i], refs[j]), f"{row_id}: scenes {i} and {j} have identical references"


_REF = {}  # (cfgname, enet, math, weights, class threshold, content) -> host snapshot of the eager synchronous forward


def _references(row, seq, math, weights="w0", thresh=None, net=None):
    from lib.utils.config import cfg
    todo = [c for c in dict.fromkeys(seq) if (row["cfgname"], row["enet"], math, weights, thresh, c) not in _REF]
    if todo:
        own = net is None
        if own:
            net, cfg = _make_net(row, math, weights, eager=True)
        assert not net._use_graph
        if thresh is not None:
            cfg.CLASS_THRESH = thresh
        for c in todo:
            P = net.forward(_blobs(c, row, "pageable"), "TEST", None)
            _REF[(row["cfgname"], row["enet"], math, weights, thresh, c)] = _host(_snap(P, bits="mask_bits"))
        torch.cuda.synchronize()
        if own:
            del net
            _free()
    return [_REF[(row["cfgname"], row["enet"], math, weights, thresh, c)] for c in seq]


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _loop(net, blobs, stop=None, stream=None):
    got = []
    ctx = torch.cuda.stream(stream) if stream is not None else torch.cuda.stream(torch.cuda.current_stream())
    with ctx:
        for k, (b, P) in enumerate(net.forward_pipelined(iter(blobs))):
            got.append((b, _snap(P)))
            if stop is not None and k + 1 == stop:
                break
        torch.cuda.current_stream().synchronize()  # the consumer's copies; scenes left in flight by a break are not waited for
    return [(b, _host(s)) for b, s in got]


def _knobs(row, monkeypatch, net):
    for env, key in (("SIS3D_PIPE_STATIC", "static"), ("SIS3D_PIPE_DEPTH", "depth")):
        if row[key] is None:
            monkeypatch.delenv(env, raising=False)
        else:
            monkeypatch.setenv(env, str(row[key]))
    if row["graph_cache"] is not None:
        net._graph_cache = row["graph_cache"]
    if row["graph_after"] is not None:
        net._graph_after = row["graph_after"]


# ------------------------------------------------------------------------------------------------ the rows
def _edge_order(refs_by_content):
    """Order of the edge row: the lightest scene that keeps a mask first, a scene that keeps none in the middle, the heaviest
    last, so that position 7 (= depth) puts the heaviest scene on the slot of the lightest one and the mask arena of that slot
    (canvas, pinned tables, pinned bits) grows in the middle of the loop."""
    vox = {c: int(len(r["mask_bits"])) if r["mask_bits"] is not None else 0 for c, r in refs_by_content.items()}
    contents = list(refs_by_content)
    empty = [c for c in contents if vox[c] == 0]
    masky = sorted((c for c in contents if vox[c] > 0), key=lambda c: vox[c])
    assert empty, f"no scene without a kept mask: kept voxels {list(vox.values())}"
    assert len(masky) >= 2, f"fewer than two scenes keep masks: {list(vox.values())}"
    light, heavy, none = masky[0], masky[-1], empty[0]
    assert vox[heavy] > 1.5 * vox[light] + 1024, f"heaviest scene ({vox[heavy]} voxels) does not outgrow the lightest ({vox[light]})"
    rest = [c for c in contents if c not in (light, heavy, none)]
    order = [light] + rest[:2] + [none] + rest[2:] + [heavy]
    assert len(order) == 8 == loop_depth() + 1
    return [order[i % len(order)] for i in range(2 * len(order))], vox, light, heavy


@pytest.mark.parametrize("row", ROWS, ids=[r["id"] for r in ROWS])
def test_scene_loop_equals_synchronous_forward(row, oracle, monkeypatch, record_property):
    _PORT["port"] = oracle
    _free()
    rid, math, seq = row["id"], row["math"], list(row["seq"])
    thresh, weights = None, "w0"
    depth = loop_depth(row["static"], row["depth"])
    if row["mech"] == "edges":
        weights = "cls0.05"
        ref_net, cfg = _make_net(row, math, weights, eager=True)
        probe = _references(row, seq, math, weights, None, ref_net)
        best = []
        for r in probe:  # best confidence among decodable detections
            det = r["detections_host"]
            ok = (det[:, 9:12] < det[:, 12:15]).all(1)
            best.append(float(det[ok, 6].max()) if ok.any() else 0.0)
        lo = sorted(set(best))[:2]
        assert len(lo) == 2, f"no confidence gap between scenes: {best}"
        thresh = (lo[0] + lo[1]) / 2
        by_content = dict(zip(seq, _references(row, seq, math, weights, thresh, ref_net)))
        del ref_net
        _free()
        seq, vox, light, heavy = _edge_order(by_content)
        assert {c[3] for c in seq} >= {None, "kill1", "killall"} and {c[1] for c in seq} == {1, 3}
    refs = _references(row, seq, math, weights, thresh)
    _assert_power(rid, refs, depth)
    if row["oracle"]:
        _check_oracle(row, refs[0])

    net, cfg = _make_net(row, math, weights)
    if thresh is not None:
        cfg.CLASS_THRESH = thresh  # read by every static stage (make_net resets the config)
    _knobs(row, monkeypatch, net)
    blobs = _inputs(row, seq)
    mech = row["mech"]
    if mech == "home_stream":
        s = torch.cuda.Stream()
        _compare(rid, blobs, refs, _loop(net, blobs, stream=s))
    elif mech == "break":
        k = 3
        _compare(rid, blobs[:k], refs[:k], _loop(net, blobs, stop=k))
        _compare(rid + " (second loop)", blobs, refs, _loop(net, blobs))
        for rnd in range(2):  # eager first sight, then captured, on the forward's own slot
            for c, b, r in zip(seq, blobs, refs):
                got = _host(_snap(net.forward(b, "TEST", None)))
                torch.cuda.synchronize()
                assert not _diff(got, r), f"{rid}: synchronous forward after the loops differs ({_diff(got, r)})"
    elif mech == "reload":
        _compare(rid, blobs, refs, _loop(net, blobs))
        refs1 = _references(row, seq, math, "w1")
        assert all(_diff(a, b) for a, b in zip(refs, refs1)), "the second weights do not change every scene"
        _assert_power(rid, refs1, depth)
        net.load_state_dict(_weights(net, "w1"))
        _compare(rid + " (after load_state_dict)", blobs, refs1, _loop(net, blobs))
    elif mech == "set_math":
        _compare(rid, blobs, refs, _loop(net, blobs))
        refs2 = _references(row, seq, row["math2"])
        assert all(_diff(a, b) for a, b in zip(refs, refs2)), f"{math} and {row['math2']} agree bit for bit on some scene"
        _assert_power(rid, refs2, depth)
        net.set_conv_math(row["math2"])
        _compare(rid + f" (after set_conv_math {row['math2']})", blobs, refs2, _loop(net, blobs))
    else:
        _compare(rid, blobs, refs, _loop(net, blobs))
    if mech == "edges":  # the mask arena of the heaviest scene's slot was sized by the lightest one, then grew
        pos = seq.index(heavy)
        assert seq[pos - depth] == light and pos >= depth
        bits = net._slots[1 + pos % depth]["arena"]["bits_host"]
        assert bits.numel() == int(vox[heavy] * 1.5) + 1024, (bits.numel(), vox[heavy], vox[light])
    slots = len(net._slots) - 1
    assert slots == min(depth, len(seq)), f"{rid}: {slots} stream slots used, expected {min(depth, len(seq))}"
    keys = {(c[0], c[1]) for c in seq}
    if max(sum(1 for c in seq if (c[0], c[1]) == k) for k in keys) >= net._graph_after:
        assert net._replayed_kernels > 0, f"{rid}: no shape was captured"
    if row["graph_cache"] is not None and row["graph_cache"] < len(keys):
        assert all(len(sl["graphs"]) <= row["graph_cache"] for sl in net._slots)
    record_property("scenes", len(seq))
    record_property("replayed_kernels", int(net._replayed_kernels))
    del net
    _free()


def _check_oracle(row, ref):
    """The eager fp32 reference's integer outputs for an oracle case equal the CPU oracle's (fma_mode=1): proposal count,
    level ids, class argmax, mask-keep flags and crop bounds."""
    port = _PORT["port"]
    assert row["math"] == "fp32"
    c = synth.CASES[row["oracle"]]
    ocfg, w, data, views = synth.build_case(port, c)
    if row["enet"]:
        net, _ = _make_net(row, "fp32")
        sd = dict(net.named_parameters())
        sd.update(dict(net.named_buffers()))
        params = [sd[n].detach().cpu() for n in net._enet_names]
        del net
        images = _content(row["seq"][0], row["cfgname"], True)[1]["feats"]
        with torch.no_grad():
            views = dict(views, feats=port.enet_encoder(params, torch.from_numpy(images)).numpy())
    want = port.forward(ocfg, w, data, views, fma_mode=1)
    assert ref["rois"].shape == tuple(want["rois"].shape)
    np.testing.assert_allclose(ref["rois"], want["rois"].numpy(), atol=2e-3)
    assert np.array_equal(ref["level_inds"].reshape(-1), want["level_inds"].numpy().reshape(-1))
    assert np.array_equal(ref["cls_pred"], want["cls_pred"].numpy())
    det = ref["detections_host"]
    assert np.array_equal(det[:, 8] > 0.5, want["mask_keep"])
    assert np.array_equal(det[:, 9:15].astype(np.int64), want["mask_crops"])
    assert len(ref["mask_shapes"]) == len(want["mask_pred"])


# ------------------------------------------------------------------------------------------------ the comparison's power
def _held(P):
    """A private copy of a yielded prediction dict in its own format (cloned tensors, copied arrays)."""
    from lib.nets.network import _MaskList
    out = {}
    for k, v in P.items():
        if torch.is_tensor(v):
            out[k] = v.clone()
        elif isinstance(v, np.ndarray):
            out[k] = v.copy()
        elif isinstance(v, list) and v and isinstance(v[0], _MaskList):
            m = v[0]
            out[k] = [_MaskList(m.packed.clone(), m.offs, m.sizes, m.ncls)]
        elif isinstance(v, list):
            out[k] = [x.clone() if torch.is_tensor(x) else x for x in v]
        else:
            out[k] = v
    return out


def test_comparison_rejects_a_pairing_shift(oracle, monkeypatch):
    """A host-side mutant of _scene_loop yields scene k's predictions with scene k+1's blobs (the last scene is dropped;
    nothing is replayed on a mismatched shape).  The comparison must reject it, by the yielded order and by content."""
    from lib.nets.network import Network
    _PORT["port"] = oracle
    _free()
    row = next(r for r in ROWS if r["id"] == "math-exact")
    seq = row["seq"]
    refs = _references(row, seq, "exact")
    real = Network._scene_loop

    def shifted(self, blobs_iter):
        prev = None
        for b, P in real(self, blobs_iter):
            if prev is not None:
                yield b, prev
            prev = _held(P)

    net, _ = _make_net(row, "exact")
    blobs = _inputs(row, seq)
    _compare("unmodified", blobs, refs, _loop(net, blobs))
    monkeypatch.setattr(Network, "_scene_loop", shifted)
    got = _loop(net, blobs)
    assert len(got) == len(seq) - 1
    with pytest.raises(AssertionError):
        _compare("mutant", blobs, refs, got)
    # the content check alone rejects it too: each yielded blobs dict is compared with its own scene's reference
    with pytest.raises(AssertionError, match="differs from its reference"):
        _compare("mutant", blobs[1:], refs[1:], got, check_identity=False)
    del net
    _free()


# ------------------------------------------------------------------------------------------------ the inference driver
def test_run_scenes_pipelined_files_equal_synchronous(tmp_path):
    """lib.model.trainval.run_scenes over .chunk files of three shapes: the pipelined loop fed by the prefetcher with device
    chunk decode writes exactly the bytes the synchronous path (eager forward, host decode) writes."""
    from lib.datasets.dataset import Dataset, collate_fn
    from lib.datasets.prefetch import Prefetcher
    from lib.datasets.scene_io import write_scene
    from lib.model.trainval import run_scenes, scene_key
    _free()
    kinds = [(SMALL, 3), (SMALL2, 2), ((48, 28, 44), 4)]
    paths, provs = [], {}
    for k in range(9):
        dims, n = kinds[k % 3]
        data, boxes = synth.make_scene(1200 + k, dims)
        views = synth.make_views(1200 + k, dims, n, boxes)
        sdf = np.where(data[0, 1] > 0.5, data[0, 0], -data[0, 0]).astype(np.float32)
        sdf[(data[0, 1] < 0.5) & (data[0, 0] < 1.0)] = -1.0
        p = str(tmp_path / f"scene{k:04d}_00__0.chunk")
        write_scene(p, sdf, world2grid=views["world2grid"], frame_ids=list(range(0, 20 * n, 20)))
        paths.append(p)
        provs[p] = views
    provider = lambda p, ids, w2g, dims: {"images": provs[p]["feats"], "depths": provs[p]["depths"], "poses": provs[p]["poses"],
                                          "world2grid": provs[p]["world2grid"]}
    row = dict(cfgname="scannet", enet=False)
    sync_net, _ = _make_net(row, "exact", eager=True)
    out_a, out_b = str(tmp_path / "sync"), str(tmp_path / "pipe")
    host = Dataset(paths, "test", view_provider=provider)
    assert run_scenes(sync_net, (collate_fn([host[i]]) for i in range(len(paths))), out_a, pipelined=False) == len(paths)
    del sync_net
    _free()
    net, _ = _make_net(row, "exact")
    devd = Dataset(paths, "test", view_provider=provider, device_decode=True)
    loader = (collate_fn([item]) for item in Prefetcher((devd[i] for i in range(len(paths))), depth=3))
    assert run_scenes(net, loader, out_b, pipelined=True) == len(paths)
    assert net._replayed_kernels > 0, "no shape was captured"
    kept = 0
    for p in paths:
        da, db = os.path.join(out_a, scene_key(p)), os.path.join(out_b, scene_key(p))
        names = sorted(os.listdir(da))
        assert names == sorted(os.listdir(db)) and {"pred_class.npy", "pred_mask", "scene.npy"} <= set(names)
        for f in names:
            with open(os.path.join(da, f), "rb") as fa, open(os.path.join(db, f), "rb") as fb:
                assert fa.read() == fb.read(), (p, f)
        kept += len(pickle.load(open(os.path.join(da, "pred_mask"), "rb")))
    assert kept > 0, "no scene kept a mask"
    del net
    _free()
