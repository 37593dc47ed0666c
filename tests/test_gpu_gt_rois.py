"""GPU: test mode on ground-truth boxes and classes (USE_RPN = USE_CLASS = False, USE_BACKBONE on or off).

- every math mode: crop bounds, keep flags and classes equal the reference (tests/golden/gt_rois_reference.npz) exactly, the
  masks within 1e-3;
- the ragged mask stage on 250 ground-truth boxes in a 208x48x160 scene plus a crop spanning the whole scene, on every mask
  route, within the per-element fp64 bound of tests/test_gpu_mask_stage.py;
- forward_pipelined over scenes of changing shapes and box counts equals forward bit for bit;
- run_scenes writes byte-identical files pipelined and synchronously, equal to the reference's test loop, and the summary is
  the reference's;
- per scene, libsis3d launches only the mask stage: no ENet, backbone, RPN or classifier kernel."""
import filecmp
import os
import pickle

import numpy as np
import pytest
import torch

import sis3d_synth as synth
from conftest import load_golden
from lib import _sis3d as S
from lib.nets.network import Network
from test_gpu_mask_stage import LAUNCHES, check_stage, cls_per_voxel, reference_packed

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = "gt_rois_reference.npz"
FORWARD = ("cfg1_32", "odd_45x27x41", "cfg2_96x48x96", "suncg_40x24x40", "thresh1_45x27x41")


def make_gt_net(cfgname="scannet", use_images=True, backbone=False, math="exact", enet=False, class_thresh=None):
    """The product Network of a released config switched to ground-truth RoIs, with the weights of the oracle's fixture."""
    net, cfg = synth.make_net(dict(cfgname=cfgname, use_images=use_images, use_mask=True), keep_debug=False, math=math,
                              enet=enet, gt_rois=backbone)
    if class_thresh is not None:
        cfg.CLASS_THRESH = class_thresh
    return net, cfg


def golden_blobs(g, tag):
    dims = tuple(int(v) for v in g[f"{tag}_dims"])
    seed, n_img = int(g[f"{tag}_seed"]), int(g[f"{tag}_n_img"])
    c = dict(cfgname=str(g[f"{tag}_cfgname"]), use_images=n_img > 0)
    data, boxes = synth.make_scene(seed, dims)
    views = synth.make_views(seed, dims, n_img, boxes) if n_img else None
    blobs = synth.make_blobs(c, data, views)
    blobs["gt_box"] = [torch.from_numpy(g[f"{tag}_gt_box"])]
    return blobs


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


@pytest.mark.parametrize("math", list(Network.MATH_MODES))
def test_golden_in_every_math_mode(golden, math):
    g = golden
    worst = 0.0
    for tag in FORWARD:
        for backbone in (True, False):
            net, cfg = make_gt_net(str(g[f"{tag}_cfgname"]), int(g[f"{tag}_n_img"]) > 0, backbone, math,
                                   class_thresh=float(g[f"{tag}_class_thresh"]))
            blobs = golden_blobs(g, tag)
            P = net.forward(blobs, "TEST", None)
            torch.cuda.synchronize()
            k = f"{tag}_b{int(backbone)}_"
            gt = g[f"{tag}_gt_box"]
            det = P["detections_host"]
            assert "level_inds" not in P and "cls_score" not in P
            assert np.array_equal(P["rois"][0].numpy(), g[k + "rois"])
            assert np.array_equal(P["roi_scores"][0].numpy(), g[k + "roi_scores"])
            assert P["cls_pred"].dtype == torch.int64 and np.array_equal(P["cls_pred"].numpy(), g[k + "cls_pred"])
            assert np.array_equal(P["cls_prob"].numpy(), g[k + "cls_prob"])
            assert np.array_equal(P["bbox_pred"].numpy(), g[k + "bbox_pred"])
            assert np.array_equal(det[:, 0:6].view(np.int32), g[k + "pred_box"].view(np.int32))
            assert np.array_equal(det[:, 7].astype(np.int64), g[k + "cls_pred"])
            assert np.array_equal(det[:, 8] > 0.5, g[k + "keep"])
            assert np.array_equal(det[:, 9:15].astype(np.int64), g[k + "crops"])
            assert det.shape[0] == len(gt) and det[0, 15] == len(gt)
            masks = P["mask_pred"][0]
            assert len(masks) == int(g[k + "n_masks"])
            pc = g[k + "cls_pred"][g[k + "keep"]]
            for j, m in enumerate(masks):
                m = m[0].cpu().numpy()
                assert m.shape[1:] == tuple(np.diff(g[k + "crops"][g[k + "keep"]][j].reshape(2, 3), axis=0)[0])
                for got, key, step in ((m[pc[j]].reshape(-1)[::7], "cls_sub", 7), (m.reshape(-1)[::97], "allcls_sub", 97)):
                    err = float(np.abs(got - g[f"{tag}_b1_mask_{j}_{key}"]).max())
                    worst = max(worst, err)
                    assert err < 1e-3, f"{tag} backbone={backbone} {math}: mask {j} {key} err {err:.3g}"
    print(f"{math}: worst mask error {worst:.3g}")


def _random_boxes(n, dims, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        size = rng.uniform(2, 28, 3)
        lo = rng.uniform(-4, np.array(dims) - 2)
        lo = np.round(lo * 4) / 4  # quarter-voxel corners: half-integers among them
        out.append(list(lo) + list(lo + np.round(size * 4) / 4) + [int(rng.integers(0, 19))])
    return np.array(out, np.float32).reshape(-1, 7)


@pytest.mark.parametrize("math,route", [("fp32", 0), ("tf32", 1), ("exact", 2)])
def test_mask_stage_on_250_boxes_and_the_whole_scene(math, route):
    dims = (208, 48, 160)
    net, cfg = make_gt_net(math=math)
    data, _ = synth.make_scene(606, dims)
    gt = np.concatenate([_random_boxes(250, dims, 7), np.array([[-2, -1, -3, 210, 50, 161, 4]], np.float32)])
    blobs = synth.make_blobs(dict(use_images=False), data, None)
    blobs["gt_box"] = [torch.from_numpy(gt)]
    P = net.forward(blobs, "TEST", None)
    torch.cuda.synchronize()
    det = P["detections_host"]
    kd = det[det[:, 8] > 0.5]
    crops = [tuple(int(v) for v in d[9:12]) + tuple(int(e) - int(s) for s, e in zip(d[9:12], d[12:15])) for d in kd]
    assert len(crops) > 200 and crops[-1] == (0, 0, 0) + dims, "the whole-scene crop is missing"
    W = [dict(net.named_parameters())[f"mask_backbone.geometry.{i}.weight"].detach().to(DEV).double() for i in (0, 2, 4, 6, 8, 10)]
    ref, bound, zero, _ = reference_packed(torch.from_numpy(data).to(DEV).double(), crops, W, route)
    masks = P["mask_pred"][0]
    kerr, berr = check_stage(ref, bound, zero, cls_per_voxel(det, DEV), masks.packed.view(-1, 19), P["mask_bits"])
    print(f"route {route}: {len(crops)} crops, masks err/bound {kerr:.3g}, bits {berr:.3g}")
    assert kerr <= 1.0 and berr <= 1.0
    assert np.array_equal(P["mask_bits_host"] if "mask_bits_host" in P else P["mask_bits"].cpu().numpy(),
                          P["mask_bits"].cpu().numpy())


def _loop_blobs(dims, n_img, seed, n_boxes):
    data, boxes = synth.make_scene(seed, dims)
    views = synth.make_views(seed, dims, n_img, boxes)
    blobs = synth.make_blobs(dict(use_images=True), data, views)
    blobs["gt_box"] = [torch.from_numpy(_random_boxes(n_boxes, dims, seed))]
    return blobs


def _snap(P):
    masks = P["mask_pred"][0]
    return dict(det=P["detections_host"].copy(), cls_prob=P["cls_prob"].clone(), rois=P["rois"][0].clone(),
                masks=masks.packed.clone() if len(masks) else None, sizes=[tuple(m.shape) for m in masks],
                bits=P["mask_bits_host"].copy() if "mask_bits_host" in P else None)


def test_pipelined_equals_forward():
    pool = [((40 + 4 * k, 24 + 4 * (k % 2), 36 + 8 * (k % 3)), 1 + k % 3, 700 + k, (0, 3, 17, 60, 1, 40)[k % 6])
            for k in range(8)]
    blobs = [_loop_blobs(*p) for p in pool]
    seq = [blobs[i] for i in (0, 1, 2, 3, 4, 5, 6, 7, 1, 0, 3, 2, 5, 4, 7, 6, 2, 1)]
    net_sync, _ = make_gt_net(backbone=True)
    want = [_snap(net_sync.forward(b, "TEST", None)) for b in seq]
    net, _ = make_gt_net(backbone=True)
    got = [(b, _snap(P)) for b, P in net.forward_pipelined(iter(seq))]
    assert len(got) == len(seq) and all(a[0] is b for a, b in zip(got, seq))
    assert any(w["masks"] is None for w in want) and any(w["masks"] is not None for w in want)
    for k, ((_, g), w) in enumerate(zip(got, want)):
        assert np.array_equal(g["det"], w["det"]) and torch.equal(g["cls_prob"], w["cls_prob"]) and torch.equal(g["rois"], w["rois"])
        assert g["sizes"] == w["sizes"], f"scene {k}"
        if w["masks"] is None:
            assert g["masks"] is None and g["bits"] is None
            continue
        assert torch.equal(g["masks"].view(torch.int32), w["masks"].view(torch.int32)), f"scene {k}: masks differ"
        assert np.array_equal(g["bits"], w["bits"]), f"scene {k}: bits differ"
    assert net._replayed_kernels == 0


def test_one_mask_stage_per_scene_and_nothing_else():
    """ENet declared (USE_IMAGES_GT = False) and the backbone switched on: the scene still launches only the seven kernels of
    its mask stage, and none when no box is kept."""
    net, cfg = make_gt_net(backbone=True, enet=True)
    blobs = [_loop_blobs((48, 24, 40), 2, 720 + k, n) for k, n in enumerate((5, 0, 12, 30))]
    net.forward(blobs[0], "TEST", None)  # packs the weights (and builds the ENet encoder) once
    for b in blobs:
        n0 = S.launch_count()
        P = net.forward(b, "TEST", None)
        torch.cuda.synchronize()
        kept = int((P["detections_host"][:, 8] > 0.5).sum())
        assert S.launch_count() - n0 == (LAUNCHES if kept else 0), (kept, S.launch_count() - n0)
    n0 = S.launch_count()
    for _ in net.forward_pipelined(iter(blobs)):
        pass
    assert S.launch_count() - n0 == LAUNCHES * sum(1 for b in blobs if len(b["gt_box"][0]))
    assert net._replayed_kernels == 0


def _gt_masks(g, s):
    bits = np.unpackbits(g[f"loop_{s}_gt_bits"])
    out, o = [], 0
    for b in g[f"loop_{s}_gt_box"]:
        ext = tuple(int(v) for v in np.rint(b[3:6]).astype(int) - np.rint(b[0:3]).astype(int))
        n = int(np.prod(ext))
        out.append(bits[o:o + n].reshape(ext).astype(np.uint8))
        o += n
    return out


def test_run_scenes_matches_the_reference_loop(golden, tmp_path):
    from lib.model.trainval import SceneEvaluator, run_scenes
    g = golden
    dims, n_img = tuple(int(v) for v in g["loop_dims"]), int(g["loop_n_img"])
    scenes = []
    for s in range(int(g["loop_n_scenes"])):
        data, boxes = synth.make_scene(int(g[f"loop_{s}_seed"]), dims)
        views = synth.make_views(int(g[f"loop_{s}_seed"]), dims, n_img, boxes)
        b = synth.make_blobs(dict(use_images=True), data, views)
        b["id"], b["gt_box"], b["gt_mask"] = [str(g[f"loop_{s}_id"])], [torch.from_numpy(g[f"loop_{s}_gt_box"])], [_gt_masks(g, s)]
        scenes.append(b)
    lines = {}
    for mode in ("pipelined", "sync"):
        net, cfg = make_gt_net()
        ev = SceneEvaluator()
        assert run_scenes(net, iter(scenes), str(tmp_path / mode), pipelined=mode == "pipelined", evaluator=ev) == len(scenes)
        lines[mode] = ev.summary()
    assert lines["pipelined"] == lines["sync"] == str(g["loop_test_printed"]).split("\n")
    assert lines["sync"][0].startswith("mAP of mask: ") and not any("CLASSIFICATION" in ln for ln in lines["sync"])
    for s, b in enumerate(scenes):
        d = {m: tmp_path / m / str(g[f"loop_{s}_id"]) for m in ("pipelined", "sync")}
        names = sorted(os.listdir(d["sync"]))
        assert names == sorted(os.listdir(d["pipelined"]))
        assert {"pred_class.npy", "pred_conf.npy", "pred_box.npy", "scene.npy", "pred_mask", "pred_mask_index"} <= set(names)
        for f in names:
            assert filecmp.cmp(d["sync"] / f, d["pipelined"] / f, shallow=False), f"scene {s}: {f} differs"
        assert int(g[f"loop_test_{s}_written"]) == 1
        k = f"loop_test_{s}_"
        ld = lambda f: np.load(d["sync"] / (f + ".npy"))
        for f in ("pred_class", "pred_conf", "pred_box"):
            assert ld(f).dtype == g[k + f].dtype and np.array_equal(ld(f), g[k + f]), f"scene {s}: {f}"
        keep = pickle.load(open(d["sync"] / "pred_mask_index", "rb"))
        assert keep == [bool(v) for v in g[k + "pred_mask_index"]]
        pm = pickle.load(open(d["sync"] / "pred_mask", "rb"))
        assert [m.shape for m in pm] == [tuple(v) for v in g[k + "pred_mask_shapes"]]
        if pm:
            got = np.concatenate([m.reshape(-1) != 0 for m in pm])
            want = np.unpackbits(g[k + "pred_mask_bits"])[:got.size].astype(bool)
            assert (got != want).mean() < 1e-3, f"scene {s}: {(got != want).sum()} of {got.size} mask voxels differ"
