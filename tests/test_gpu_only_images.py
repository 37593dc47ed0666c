"""GPU: the image-only ScanNet backbone (ONLY_IMAGES = USE_IMAGES = True) through the C ABI.

- golden parity with the unmodified reference (tests/golden/only_images_reference.npz) in `exact` and `fp32`: integer
  outputs exactly (proposal order and NMS keep list row by row, level ids, class argmax, mask-keep flags, crop bounds),
  features, boxes and probabilities within 1e-4, masks within 1e-3; raw images through the 2-D encoder eager and on graph
  replay;
- every layer of the image-only static stage within the fp64 bound of its route in all seven math modes, by the method of
  tests/test_gpu_static_stage.py (its Row checks on the live parameters, each op on the previous op's output), with the
  wiring of the image-only program and its own models (level 1 half from the previous scene, geometry2.0 reading at
  channel 64, the colour stack's final pool skipped, color.4 truncated to 64 outputs) missing the bound by POWER;
- routes: no geometry1 launch, color.4 on conv_tc_h3 in `exact`, color.6 as three conv_tc_h3 launches, and only
  conv3d_k3_tc_kernel instances the default nets also launch;
- the scene loop: forward_pipelined equals forward bit for bit, graph replay equals eager, the dense colour route gives
  the same integer outputs; run_scenes writes byte-identical files pipelined and synchronously, equal to the reference's
  loops; a default net and an image-only net alternating in one process give what each gives alone."""
import filecmp
import os
import pickle

import numpy as np
import pytest
import torch

import sis3d_synth as synth
from conftest import load_golden
from lib.nets.network import Network
from test_gpu_mask_stage import _launched
from test_gpu_static_stage import ROUTE_CHECKS, Row, active_levels, prev_inputs, run_hooked, same_bits, stage_layers
from test_gpu_tc_accuracy import _conv
from test_only_images import FORWARD, GOLDEN, case_inputs, enet_params, stats_close, step

pytestmark = pytest.mark.gpu
DEV = "cuda"
C = dict(cfgname="scannet", use_images=True, use_mask=True)


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def make_only_net(math="exact", enet=False, keep_debug=False):
    """The image-only product Network with the weights the golden's reference model loaded; enet=True declares the 2-D
    encoder (USE_IMAGES_GT = False) with the parameters of tests/golden/enet_encoder.npz."""
    net, cfg = synth.make_net(C, keep_debug=keep_debug, math=math, only_images=True)
    if not enet:
        return net, cfg
    sd3d = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    del net
    cfg.USE_IMAGES_GT = False
    from lib.nets import backbones
    net = backbones.ScanNet_Backbone()
    net.init_modules()
    sd = net.state_dict()
    for n, p in zip(net._enet_names, enet_params(), strict=True):
        sd[n] = p
    sd.update(sd3d)
    net.load_state_dict(sd, strict=True)
    net._keep_debug = keep_debug
    net.set_conv_math(math)
    return net, cfg


def _sub(vc, step):
    return vc.permute(3, 0, 1, 2).reshape(-1)[::step].cpu().numpy()


def check_golden(P, g, tag, features=True):
    k = tag + "_"
    if features:
        for lvl in (1, 2):
            vc = P[f"level{lvl}_vc"]
            np.testing.assert_allclose(_sub(vc, step(g, "level")), g[k + f"level{lvl}_sub"], atol=1e-4, rtol=1e-4)
            assert stats_close(vc.double().cpu().numpy(), g[k + f"level{lvl}_stats"], 1e-4), f"level {lvl}: whole-tensor moments"
    n = P["rois"][0].shape[0]
    assert n == g[k + "rois"].shape[0]
    # row-by-row box equality in score order == the same top-N order and NMS keep list
    np.testing.assert_allclose(P["rois"][0].cpu().numpy(), g[k + "rois"], atol=2e-3)
    np.testing.assert_allclose(P["roi_scores"][0].cpu().numpy().reshape(-1), g[k + "roi_scores"].reshape(-1), atol=1e-4)
    assert np.array_equal(P["level_inds"][0].cpu().numpy(), g[k + "level_inds"])
    assert np.array_equal(P["cls_pred"].cpu().numpy(), g[k + "cls_pred"])
    np.testing.assert_allclose(P["cls_prob"].cpu().numpy(), g[k + "cls_prob"], atol=1e-4)
    np.testing.assert_allclose(P["bbox_pred"].cpu().numpy(), g[k + "bbox_pred"], atol=1e-4)
    det = P["detections_host"]
    np.testing.assert_allclose(det[:, :6], g[k + "pred_box"], atol=1e-4)
    assert np.array_equal(det[:, 8] > 0.5, g[k + "keep"])
    assert np.array_equal(det[:, 9:15].astype(np.int64), g[k + "crops"])
    masks = P["mask_pred"][0]
    assert len(masks) == int(g[k + "n_masks"])
    pc = g[k + "cls_pred"][g[k + "keep"]]
    for j, m in enumerate(masks):
        m = m[0].cpu().numpy()
        assert float(np.abs(m[pc[j]].reshape(-1)[::step(g, "mask_cls")] - g[k + f"mask_{j}_cls_sub"]).max()) < 1e-3
        assert float(np.abs(m.reshape(-1)[::step(g, "mask_allcls")] - g[k + f"mask_{j}_allcls_sub"]).max()) < 1e-3


@pytest.mark.parametrize("math", ["exact", "fp32"])
@pytest.mark.parametrize("tag", FORWARD)
def test_golden(golden, tag, math):
    g = golden
    enet = int(g[f"{tag}_images_seed"]) >= 0
    c, data, views = case_inputs(g, tag)
    net, _ = make_only_net(math, enet=enet, keep_debug=True)
    blobs = synth.make_blobs(c, data, views)
    check_golden(net.forward(blobs, "TEST", None), g, tag)
    # the default forward: eager on first sight, then captured and replayed (the encoder inside the graph when enet)
    net._keep_debug = False
    for _ in range(3):
        check_golden(net.forward(blobs, "TEST", None), g, tag, features=False)
    assert net._replayed_kernels > 0


# ------------------------------------------------------------------------------------------------ layer by layer
class OnlyImagesRow(Row):
    """Row checks of tests/test_gpu_static_stage.py with the wiring of the image-only program and its own models."""

    def __init__(self, *a):
        super().__init__(*a)
        c6 = [o for o in self.cap.ops if o["kind"] == "bottleneck" and o["name"] == "color.6"]
        assert len(c6) == 1
        self.colour6 = c6[0]["y"]

    def conv_models(self, layer, x, w, b, r, prev_x):
        m = super().conv_models(layer, x, w, b, r, prev_x)
        d = lambda t: t.to(DEV).double()
        lin = lambda a: _conv(d(a), d(w), w.shape[2]) + (d(b) if b is not None else 0)
        if layer in ("geometry2.0", "rpn_net_level1"):
            assert x.shape[-1] == 128
            if prev_x is not None and prev_x.shape == x.shape:
                m["level1_upper_half_of_previous_scene"] = lin(torch.cat([x[..., :64], prev_x[..., 64:]], -1))
            m["colour_final_pool_skipped"] = lin(self.colour6)
        if layer == "geometry2.0":
            flat = x.reshape(-1)
            m["read_at_channel_offset_64"] = lin(torch.cat([flat[64:], flat.new_zeros(64)]).view_as(x))
        if layer == "color.4":
            m["truncated_to_64_outputs"] = lambda ref: torch.cat([ref[..., :64], torch.zeros_like(ref[..., 64:])], -1)
        return m

    def wiring(self):
        rid, spec = self.row["id"], self.net.SPEC
        ops = self.cap.ops
        assert not any((o.get("name") or "").startswith("geometry1") for o in ops), f"{rid}: a geometry1 op ran"
        top = [o for o in ops if o["parent"] is None]
        seq, cur = {"color": [], "geometry2": []}, None
        for o in top:
            if o["kind"] == "pool":
                seq[cur].append(o)
            elif o["kind"] in ("conv", "bottleneck") and o["name"].split(".")[0] in seq:
                cur = o["name"].split(".")[0]
                seq[cur].append(o)
        for stage, got in seq.items():
            want = list(spec[stage])[1 if stage == "color" and self.row["sparse"] else 0:]
            assert len(got) == len(want), f"{rid}: {stage} ran {len(got)} ops, its program has {len(want)}"
            for o, w in zip(got, want):
                assert o["kind"] == {"k2s2": "conv", "k3": "conv", "bneck": "bottleneck", "pool": "pool"}[w[0]]
                if o["kind"] != "pool":
                    assert o["name"] == f"{stage}.{w[1]}", (o["name"], w)
            for a, b in zip(got, got[1:]):
                assert self.follows(a, b), f"{rid} [{b.get('name') or 'maxpool3'}]: input is not the previous op's output"
        bp = [o for o in top if o["kind"] == "backproject"]
        assert len(bp) == 1
        if self.row["sparse"]:
            assert self.follows(bp[0], seq["color"][0]), f"{rid}: color.2 does not read color.0's output"
        else:
            assert same_bits(seq["color"][0]["x"], bp[0]["y"]), f"{rid} [color.0]: input is not the back-projected volume"
        level1 = seq["geometry2"][0]["x"]
        assert level1.shape[-1] == 128 and same_bits(level1, seq["color"][-1]["y"]), f"{rid}: level 1 is not the colour output"
        level2 = seq["geometry2"][-1]["y"]
        rpn = {o["name"]: o for o in top if o["kind"] == "conv" and o["name"].startswith("rpn_")}
        for lvl, feat in ((1, level1), (2, level2)):
            hid, heads = rpn[f"rpn_net_level{lvl}"], rpn[f"rpn_heads_level{lvl}"]
            assert same_bits(hid["x"], feat), f"{rid} [rpn_net_level{lvl}]: input is not level {lvl}"
            assert self.follows(hid, heads), f"{rid} [rpn_heads_level{lvl}]: input is not rpn_net_level{lvl}'s output"


def golden_blobs(g, tag, seed=None):
    """Blobs of a golden case; seed: another scene of the same shape, views and killed views."""
    c, data, views = case_inputs(g, tag)
    if seed is not None:
        data, boxes = synth.make_scene(seed, c["dims"])
        views = synth.make_views(seed, c["dims"], c["n_img"], boxes)
        for k in g[f"{tag}_killed"]:
            views["depths"][int(k)][:] = 9.0
    return c, synth.make_blobs(c, data, views)


@pytest.mark.parametrize("tag", ["cfg2_96x48x96", "killed_45x27x41"])
def test_layers_against_fp64(golden, tag):
    c, blobs = golden_blobs(golden, tag)
    _, prev_blobs = golden_blobs(golden, tag, seed=int(golden[f"{tag}_seed"]) + 1)
    net, _ = make_only_net("exact")
    prev_cap, _ = run_hooked(net, prev_blobs)
    prev = prev_inputs(prev_cap)
    del prev_cap
    scene_vc = blobs["data"][0].permute(1, 2, 3, 0).contiguous().to(DEV)
    rows = [dict(mode=m, sparse=True, id=f"{tag}-{m}", updated=False) for m in Network.MATH_MODES]
    rows.append(dict(mode="exact", sparse=False, id=f"{tag}-exact-dense", updated=False))
    for row in rows:
        net.set_conv_math(row["mode"])
        net._sparse_color = row["sparse"]
        try:
            cap, got = run_hooked(net, blobs)
        finally:
            net._sparse_color = True
        res = OnlyImagesRow(row, net, cap, prev, True, scene_vc).run()
        reached = set()
        for layer, fam, *_ in res:
            block = ROUTE_CHECKS[fam][0] in ("fused", "split_block")
            reached |= {f"{layer}.conv{i}" for i in (1, 2, 3)} if block else {layer}
        assert reached == set(stage_layers(net.SPEC, True, active_levels()))
        worst, weakest = max(res, key=lambda t: t[2]), min(res, key=lambda t: t[3])
        print(f"{row['id']}: worst kernel err/bound {worst[2]:.3g} ({worst[1]}[{worst[0]}]), smallest model ratio "
              f"{weakest[3]:.3g} ({weakest[1]}[{weakest[0]}])")
        if row["mode"] == "exact" and row["sparse"]:
            routes = {n for o in cap.ops for n in o["routes"]} | set(cap.loose)
            assert not any("geometry1" in n for n in routes)
            assert "conv_tc_h3[color.4]" in routes
            c6 = [o for o in cap.ops if o["kind"] == "bottleneck" and o["name"] == "color.6"][0]
            kids = [o for o in cap.ops if o["parent"] == c6["i"]]
            assert c6["routes"] == [] and [o["routes"] for o in kids] == [[f"conv_tc_h3[color.6.conv{i}]"] for i in (1, 2, 3)]
        del cap


def _tc_instances(net, blobs):
    net.forward(blobs, "TEST", None)  # packs, warms up
    found = _launched(lambda: net.forward(blobs, "TEST", None), None, attempts=2)
    assert found is not None
    return set(found[1])


@pytest.mark.parametrize("math", list(Network.MATH_MODES))
def test_tc_instances_are_those_of_the_default_nets(golden, math):
    _, blobs = golden_blobs(golden, "cfg2_96x48x96")
    net, _ = make_only_net(math)
    mine = _tc_instances(net, blobs)
    assert bool(mine) == (math != "fp32"), f"{math}: tensor-core instances {sorted(mine, key=str)}"  # fp32: CUDA cores only
    del net
    theirs = set()
    for use_images in (True, False):
        net, _ = synth.make_net(dict(C, use_images=use_images), keep_debug=False, math=math)
        b = blobs if use_images else synth.make_blobs(dict(use_images=False), blobs["data"].numpy(), None)
        theirs |= _tc_instances(net, b)
        del net
    assert mine <= theirs, f"{math}: instances only the image-only net launches: {sorted(mine - theirs, key=str)}"


# ------------------------------------------------------------------------------------------------ the scene loop
def _snap(P):
    masks = P["mask_pred"][0]
    return dict(det=P["detections_host"].copy(), cls_prob=P["cls_prob"].clone(), rois=P["rois"][0].clone(),
                masks=[m.clone() for m in masks])


def _same(a, b):
    return (np.array_equal(a["det"].view(np.int32), b["det"].view(np.int32)) and torch.equal(a["cls_prob"], b["cls_prob"])
            and torch.equal(a["rois"], b["rois"]) and len(a["masks"]) == len(b["masks"])
            and all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a["masks"], b["masks"])))


def _loop_blobs(k):
    dims, n_img = (40 + 8 * (k % 3), 24 + 4 * (k % 2), 40 + 4 * (k % 4)), 1 + k % 5
    data, boxes = synth.make_scene(800 + k, dims)
    return synth.make_blobs(C, data, synth.make_views(800 + k, dims, n_img, boxes))


def test_pipelined_equals_forward_and_graph_equals_eager():
    blobs = [_loop_blobs(k) for k in range(6)]
    seq = [blobs[i] for i in (0, 1, 2, 3, 4, 5, 1, 0, 3, 2, 5, 4, 0, 1)]
    net, _ = make_only_net()
    net._use_graph = False
    eager = [_snap(net.forward(b, "TEST", None)) for b in seq]
    net._use_graph = True
    sync = [_snap(net.forward(b, "TEST", None)) for b in seq]
    assert net._replayed_kernels > 0
    got = [(b, _snap(P)) for b, P in net.forward_pipelined(iter(seq))]
    assert len(got) == len(seq) and all(a[0] is b for a, b in zip(got, seq))
    for k, (e, s, (_, p)) in enumerate(zip(eager, sync, got)):
        assert _same(e, s), f"scene {k}: graph replay differs from eager"
        assert _same(s, p), f"scene {k}: pipelined differs from forward"
    assert any(len(s["masks"]) for s in sync)


def test_dense_colour_route(golden):
    """SIS3D_SPARSE_COLOR=0: color.0 on the materialised back-projected volume instead of the fused sparse kernel."""
    for tag in ("cfg2_96x48x96", "killed_45x27x41"):
        _, blobs = golden_blobs(golden, tag)
        out = {}
        for sparse in (True, False):
            net, _ = make_only_net()
            net._sparse_color = sparse
            cap, _ = run_hooked(net, blobs)
            level1 = [o for o in cap.ops if o["kind"] == "conv" and o["name"] == "geometry2.0"][0]["x"]
            out[sparse] = (level1, _snap(net.forward(blobs, "TEST", None)))
        (l1s, s), (l1d, d) = out[True], out[False]
        torch.testing.assert_close(l1d, l1s, atol=1e-5, rtol=1e-5)
        assert s["rois"].shape == d["rois"].shape
        torch.testing.assert_close(s["rois"], d["rois"], atol=1e-4, rtol=1e-5)
        for col in (7, 8):
            assert np.array_equal(s["det"][:, col], d["det"][:, col])
        assert np.array_equal(s["det"][:, 9:15], d["det"][:, 9:15])


def test_two_nets_in_one_process():
    """A default ScanNet net and an image-only net, scenes alternating between them (synchronous and pipelined), give bit for
    bit what each gives with its scenes alone: no graph, constant or layout cache is shared."""
    blobs = [_loop_blobs(k) for k in range(4)]
    alone = {}
    for only in (False, True):
        net, _ = synth.make_net(C, keep_debug=False, math="exact", only_images=only)
        alone[only] = [_snap(net.forward(b, "TEST", None)) for b in blobs + blobs]
        del net
    default, _ = synth.make_net(C, keep_debug=False, math="exact")
    only, _ = synth.make_net(C, keep_debug=False, math="exact", only_images=True)
    assert "geometry1" in default.SPEC and "geometry1" not in only.SPEC
    for i, b in enumerate(blobs + blobs):
        assert _same(_snap(default.forward(b, "TEST", None)), alone[False][i]), f"default net, scene {i}"
        assert _same(_snap(only.forward(b, "TEST", None)), alone[True][i]), f"image-only net, scene {i}"
    for net, want in ((default, alone[False]), (only, alone[True])):
        for i, (_, P) in enumerate(net.forward_pipelined(iter(blobs))):
            assert _same(_snap(P), want[i])
    assert not any(_same(a, b) for a, b in zip(alone[False], alone[True]))


def _gt_masks(g, s):
    bits = np.unpackbits(g[f"loop_{s}_gt_bits"])
    out, o = [], 0
    for b in g[f"loop_{s}_gt_box"]:
        ext = tuple(int(v) for v in np.rint(b[3:6]).astype(int) - np.rint(b[0:3]).astype(int))
        n = int(np.prod(ext))
        out.append(bits[o:o + n].reshape(ext).astype(np.uint8))
        o += n
    return out


@pytest.mark.parametrize("mode", ["test", "benchmark"])
def test_run_scenes_matches_the_reference_loops(golden, tmp_path, mode):
    from lib.model.trainval import SceneEvaluator, run_scenes
    g = golden
    dims, n_img = tuple(int(v) for v in g["loop_dims"]), int(g["loop_n_img"])
    scenes = []
    for s in range(int(g["loop_n_scenes"])):
        data, boxes = synth.make_scene(int(g[f"loop_{s}_seed"]), dims)
        b = synth.make_blobs(C, data, synth.make_views(int(g[f"loop_{s}_seed"]), dims, n_img, boxes))
        b["id"], b["gt_box"], b["gt_mask"] = [str(g[f"loop_{s}_id"])], [torch.from_numpy(g[f"loop_{s}_gt_box"])], [_gt_masks(g, s)]
        scenes.append(b)
    for drv in ("pipelined", "sync"):
        net, _ = make_only_net()
        ev = SceneEvaluator() if mode == "test" else None
        assert run_scenes(net, iter(scenes), str(tmp_path / drv), pipelined=drv == "pipelined", evaluator=ev) == len(scenes)
    for s in range(len(scenes)):
        d = {m: tmp_path / m / str(g[f"loop_{s}_id"]) for m in ("pipelined", "sync")}
        names = sorted(os.listdir(d["sync"]))
        assert names == sorted(os.listdir(d["pipelined"]))
        for f in names:
            assert filecmp.cmp(d["sync"] / f, d["pipelined"] / f, shallow=False), f"scene {s}: {f} differs"
        k = f"loop_{mode}_{s}_"
        assert int(g[k + "written"]) == 1
        ld = lambda f: np.load(d["sync"] / (f + ".npy"))
        assert ld("pred_class").dtype == g[k + "pred_class"].dtype and np.array_equal(ld("pred_class"), g[k + "pred_class"])
        np.testing.assert_allclose(ld("pred_conf"), g[k + "pred_conf"], atol=1e-4)
        np.testing.assert_allclose(ld("pred_box"), g[k + "pred_box"], atol=2e-3)
        assert pickle.load(open(d["sync"] / "pred_mask_index", "rb")) == [bool(v) for v in g[k + "pred_mask_index"]]
        pm = pickle.load(open(d["sync"] / "pred_mask", "rb"))
        assert [m.shape for m in pm] == [tuple(v) for v in g[k + "pred_mask_shapes"]]
        if pm:
            got = np.concatenate([m.reshape(-1) != 0 for m in pm])
            want = np.unpackbits(g[k + "pred_mask_bits"])[:got.size].astype(bool)
            assert (got != want).mean() < 1e-3, f"scene {s}: {(got != want).sum()} of {got.size} mask voxels differ"
