"""oracle/make_golden_gt_rois.py -- TEST INFRASTRUCTURE ONLY; runs ONLY in the build container (needs the reference tree).

Runs the UNMODIFIED reference through oracle/ref_harness.py with ground-truth RoIs (USE_RPN = USE_CLASS = False) and stores
tests/golden/gt_rois_reference.npz, which pins oracle/port_gt_rois.py's forward_gt_rois, the host detection-table builder of
lib/nets/network.py and the GPU mode (tests/test_gt_rois.py, tests/test_gpu_gt_rois.py).

    python oracle/make_golden_gt_rois.py

Forward cases (Network.forward, the reference's own test-mode forward): the four existing forward geometries (32^3
geometry-only, 45x27x41 with 3 views, 96x48x96 with 5 views, SUNCG 40x24x40 with 3 views), each with USE_BACKBONE on and
off, on ground-truth boxes that cross every scene face, have negative corners, an empty rounded extent, half-integer and
fractional corners, class 0, zero or negative width, and lie wholly outside the scene, beside the scene's own boxes; and one
case at CLASS_THRESH = 1.0, where nothing is kept (1.0 > 1.0 is false).

Loop set: the reference's SolverWrapper.test and SolverWrapper.benchmark (lib/model/trainval.py:634-941) on seeded 45x27x41
scenes with 3 views and ground-truth boxes and masks, one of them with no ground-truth box, writing the result files and
printing the summary.

Layout: per forward case t: t_dims, t_seed, t_n_img, t_cfgname, t_class_thresh, t_gt_box [n, 7] (inputs); per USE_BACKBONE
b in (1, 0): t_b{b}_rois, _roi_scores, _cls_pred, _cls_prob, _bbox_pred, _pred_box (the driver's decode), _keep, _crops
(int(round(.)) of pred_box), _mask_{j}_cls_sub (the kept crop j's predicted-class mask, every 7th voxel in C order),
_mask_{j}_cls_on (its voxels >= MASK_THRESH), _mask_{j}_allcls_sub (all classes, every 97th value), _n_masks; the masks
only for b = 1 (those of b = 0 are checked to be identical when the fixture is written).
Loop set: loop_n_scenes, loop_dims, loop_n_img, loop_{s}_seed, loop_{s}_id, loop_{s}_gt_box, loop_{s}_gt_bits
(np.packbits of the GT masks, each C order in its rounded box, back to back); per mode m in (test, benchmark):
loop_{m}_{s}_{pred_class, pred_conf, pred_box, pred_mask_index, pred_mask_bits, pred_mask_shapes} (empty arrays for a
scene the loop skipped: loop_{m}_{s}_written = 0), loop_{m}_printed (the summary lines the loop printed).
"""
from __future__ import annotations

import contextlib
import io
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-sis_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, ROOT)
import sis3d_synth as synth  # noqa: E402
import ref_harness as rh  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "gt_rois_reference.npz")
CASES = [  # tag, yml, dims, n_img, seed, use_images, net, CLASS_THRESH override
    ("cfg1_32", "ScanNet/rpn_class_mask_5.yml", (32, 32, 32), 0, 101, False, "ScanNet_Backbone", None),
    ("odd_45x27x41", "ScanNet/rpn_class_mask_5.yml", (45, 27, 41), 3, 202, True, "ScanNet_Backbone", None),
    ("cfg2_96x48x96", "ScanNet/rpn_class_mask_5.yml", (96, 48, 96), 5, 303, True, "ScanNet_Backbone", None),
    ("suncg_40x24x40", "SUNCG/rpn_class_mask_5.yml", (40, 24, 40), 3, 404, True, "SUNCG_Backbone", None),
    ("thresh1_45x27x41", "ScanNet/rpn_class_mask_5.yml", (45, 27, 41), 3, 202, True, "ScanNet_Backbone", 1.0),
]
LOOP_DIMS, LOOP_N_IMG, LOOP_SEEDS = (45, 27, 41), 3, (211, 212, 213, 214)
LOOP_EMPTY = 2  # the loop scene without ground-truth boxes


def edge_boxes(dims, ncls, seed):
    """Ground-truth boxes at every decision edge of the decode, then the scene's own boxes with random classes."""
    X, Y, Z = dims
    b = [[-3.5, 2, 3, 6.25, 9, 10, 1],            # crosses x = 0 (negative corner)
         [X - 5.5, 1, 2, X + 4, 8, 9, 2],          # crosses x = X
         [4, -2, 5, 10, 6.5, 12, 3],               # crosses y = 0
         [6, Y - 4.5, 2, 12, Y + 3, 8, 4],         # crosses y = Y
         [8, 3, -6, 14, 9, 4.5, 5],                # crosses z = 0
         [2, 5, Z - 3.5, 9, 12, Z + 7, 6],         # crosses z = Z
         [-1, -1.5, -2, X + 1, Y + 0.5, Z + 3, 7],  # every face: the whole scene
         [3.6, 2, 2, 4.4, 8, 8, 8],                # rounded extent empty in x (4, 4)
         [2, 3.5, 2, 8, 4.5, 9, 9],                # rounded extent 4..4 in y: empty (half to even)
         [2.5, 3.5, 4.5, 7.5, 8.5, 9.5, 10],       # half-integer corners (2, 4, 4, 8, 8, 10)
         [1.25, 0.75, 2.125, 6.75, 5.3, 8.9, 11],  # fractional corners
         [10, 4, 6, 16, 10, 14, 0],                # class 0
         [5, 5, 5, 5, 9, 9, 12],                   # zero width
         [9, 2, 2, 5, 6, 6, 13],                   # negative width
         [-10, -10, -10, -2, -3, -4, 14]]          # wholly outside the scene
    rng = np.random.default_rng(seed + 31)
    _, own = synth.make_scene(seed, dims)
    for o in own:
        b.append(list(o) + [int(rng.integers(1, ncls))])
    return np.array(b, np.float32)


def predictions(net, cfg, P, dims, g, key, store_masks):
    """The reference's predictions and its driver's decode (trainval.py:825-858) of one forward -> its masks."""
    from lib.utils.bbox_transform import bbox_transform_inv, clip_boxes
    g[key + "rois"] = P["rois"][0].numpy()
    g[key + "roi_scores"] = P["roi_scores"][0].numpy()
    pc = P["cls_pred"].numpy()
    g[key + "cls_pred"], g[key + "cls_prob"], g[key + "bbox_pred"] = pc, P["cls_prob"].numpy(), P["bbox_pred"].numpy()
    assert "level_inds" not in P
    box_reg = np.zeros((len(pc), 6))
    for i in range(len(pc)):
        box_reg[i] = g[key + "bbox_pred"][i, pc[i] * 6:(pc[i] + 1) * 6]
    pb = clip_boxes(bbox_transform_inv(P["rois"][0], torch.from_numpy(box_reg).float()), list(dims)).numpy()
    conf = np.array([g[key + "cls_prob"][i, pc[i]] for i in range(len(pc))])
    keep = conf > cfg.CLASS_THRESH
    for i, b in enumerate(pb):
        if round(b[0]) >= round(b[3]) or round(b[1]) >= round(b[4]) or round(b[2]) >= round(b[5]):
            keep[i] = False
    g[key + "pred_box"], g[key + "keep"] = pb, keep
    g[key + "crops"] = np.array([[int(round(float(v))) for v in b] for b in pb], np.int64).reshape(-1, 6)
    masks = P["mask_pred"][0]
    assert len(masks) == keep.sum(), (len(masks), keep.sum())
    for j, i in enumerate(np.nonzero(keep)[0] if store_masks else []):
        m = masks[j][0].numpy()
        g[key + f"mask_{j}_cls_sub"] = m[pc[i]].reshape(-1)[::7].copy()
        g[key + f"mask_{j}_cls_on"] = np.array(int((m[pc[i]] >= cfg.MASK_THRESH).sum()))
        g[key + f"mask_{j}_allcls_sub"] = m.reshape(-1)[::97].copy()
    g[key + "n_masks"] = np.array(len(masks))
    return masks


def run_case(g, tag, yml, dims, n_img, seed, use_images, net_name, thresh):
    gt = first = None
    for b in (1, 0):
        over = dict(USE_IMAGES=use_images, USE_IMAGES_GT=True, USE_MASK=True, USE_RPN=False, USE_CLASS=False,
                    USE_BACKBONE=bool(b))
        if thresh is not None:
            over["CLASS_THRESH"] = thresh
        cfg = rh.load_cfg(yml, **over)
        w = synth.make_weights(seed=0, net=cfg.NET, use_images=use_images, num_classes=cfg.NUM_CLASSES, a1=0, a2=0,
                               use_mask=True)
        w = {k: v for k, v in w.items() if not k.startswith("classifier_")}  # no RPN, no classifier heads in this mode
        net = rh.build_net(cfg, w)
        data, boxes = synth.make_scene(seed, dims)
        gt = edge_boxes(dims, cfg.NUM_CLASSES, seed)
        views = synth.make_views(seed, dims, n_img, boxes, intrinsic=np.array(cfg.INTRINSIC, dtype=np.float32)) \
            if use_images else None
        blobs = {"data": torch.from_numpy(data), "id": [f"synthetic_{tag}"], "gt_box": [torch.from_numpy(gt)], "gt_mask": [[]]}
        killing = None
        if use_images:
            from lib.layer_utils.projection import ProjectionHelper
            helper = ProjectionHelper(cfg.INTRINSIC, cfg.PROJ_DEPTH_MIN, cfg.PROJ_DEPTH_MAX, cfg.DEPTH_SHAPE,
                                      blobs["data"].shape[-3:], cfg.VOXEL_SIZE)
            maps = [helper.compute_projection(torch.from_numpy(d), torch.from_numpy(c), torch.from_numpy(views["world2grid"]))
                    for d, c in zip(views["depths"], views["poses"])]
            killing = [i for i, m in enumerate(maps) if m is None]
            real = [m for m in maps if m is not None]
            blobs["proj_ind_3d"] = [torch.stack([m[0] for m in real])]
            blobs["proj_ind_2d"] = [torch.stack([m[1] for m in real])]
            blobs["nearest_images"] = {"images": [torch.from_numpy(views["feats"])]}
        net.forward(blobs, "TEST", killing)
        masks = predictions(net, cfg, net._predictions, dims, g, f"{tag}_b{b}_", store_masks=b == 1)
        if first is None:
            first = masks
        else:  # USE_BACKBONE cannot change a mask: only those of the first run are stored
            assert len(masks) == len(first) and all(torch.equal(a, c) for a, c in zip(masks, first))
        print(f"[golden] {tag} USE_BACKBONE={b}: {len(gt)} boxes, {int(g[f'{tag}_b{b}_n_masks'])} masks")
    g.update({f"{tag}_dims": np.array(dims), f"{tag}_seed": np.array(seed), f"{tag}_n_img": np.array(n_img),
              f"{tag}_cfgname": np.array("suncg" if "SUNCG" in yml else "scannet"), f"{tag}_gt_box": gt,
              f"{tag}_class_thresh": np.float64(cfg.CLASS_THRESH)})


def loop_scene(seed, ncls, empty, w):
    """A seeded scene with ground-truth boxes (corners on the half-voxel grid, inside the scene).  Each GT mask is its box's
    own predicted mask (oracle/port_gt_rois.py, pinned to the reference) thresholded at MASK_THRESH, complemented for every other box:
    IoUs near 1 or 0, so that the summary does not depend on voxels whose mask value sits at the threshold."""
    from oracle import port, port_gt_rois
    data, boxes = synth.make_scene(seed, LOOP_DIMS)
    views = synth.make_views(seed, LOOP_DIMS, LOOP_N_IMG, boxes)
    rng = np.random.default_rng(seed + 7)
    gt = []
    if not empty:
        for b in boxes:
            lo = np.clip(np.round(b[:3] * 2) / 2, 0, LOOP_DIMS)
            hi = np.clip(np.round(b[3:] * 2) / 2, 0, LOOP_DIMS)
            if (np.rint(hi) <= np.rint(lo)).any():
                continue
            gt.append(list(lo) + list(hi) + [int(rng.integers(1, ncls))])
    gt = np.array(gt, np.float32).reshape(-1, 7)
    out = port_gt_rois.forward_gt_rois(port.make_cfg("scannet"), w, data, gt)
    assert out["mask_keep"].all()
    masks = [((m[0, int(c)].numpy() >= 0.5) ^ (j % 2 == 1)).astype(np.uint8)
             for j, (m, c) in enumerate(zip(out["mask_pred"], gt[:, 6]))]
    full = lambda m, c: np.pad(m.astype(bool), [(c[a], LOOP_DIMS[a] - c[a + 3]) for a in range(3)])
    crops = out["mask_crops"]
    for i in range(len(gt)):  # same-class pairs decide the matches: none near MAP_THRESH = 0.25
        p = full(out["mask_pred"][i][0, int(gt[i, 6])].numpy() >= 0.5, crops[i])
        for j in range(len(gt)):
            if gt[i, 6] == gt[j, 6]:
                q = full(masks[j], crops[j])
                iou = (p & q).sum() / max((p | q).sum(), 1)
                assert abs(iou - 0.25) > 0.05, (seed, i, j, iou)
    return data, views, gt, masks


def loop_blobs(data, views, gt, masks, sid):
    return {"data": torch.from_numpy(data), "id": [sid], "gt_box": [torch.from_numpy(gt)], "gt_mask": [masks],
            "nearest_images": {"images": [torch.from_numpy(views["feats"])], "depths": [torch.from_numpy(views["depths"])],
                               "poses": [torch.from_numpy(views["poses"])],
                               "world2grid": [torch.from_numpy(np.repeat(views["world2grid"][None], len(views["depths"]), 0))]}}


def run_loops(g):
    rh.install()
    # imported by the reference's trainval for training and data loading, unused by the two loops (the dataset module pulls
    # in torchvision, which does not import beside the harness's stub modules)
    for name, attrs in (("torchnet.meter", {}), ("torchnet.meter.confusionmeter", dict(ConfusionMeter=object)),
                        ("lib.datasets.dataloader", dict(get_dataloader=None)), ("lib.datasets.dataset", dict(Dataset=None)),
                        ("lib.utils.logger", dict(Logger=None))):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    sys.modules["torchnet"].meter = sys.modules["torchnet.meter"]
    if "int" not in np.__dict__:
        np.int = int  # numpy 2 removed the alias the reference's evaluator casts class ids with (evaluation.py:41-42)
    from lib.model.trainval import SolverWrapper
    cfg = rh.load_cfg("ScanNet/rpn_class_mask_5.yml", USE_IMAGES=True, USE_IMAGES_GT=True, USE_MASK=True, USE_RPN=False,
                      USE_CLASS=False, USE_BACKBONE=False)
    w = synth.make_weights(seed=0, net=cfg.NET, use_images=True, num_classes=cfg.NUM_CLASSES, a1=0, a2=0, use_mask=True)
    net = rh.build_net(cfg, {k: v for k, v in w.items() if not k.startswith("classifier_")})
    scenes = []
    for s, seed in enumerate(LOOP_SEEDS):
        data, views, gt, masks = loop_scene(seed, cfg.NUM_CLASSES, s == LOOP_EMPTY, w)
        sid = f"scene{s:04d}_00"
        scenes.append((data, views, gt, masks, sid))
        bits = np.packbits(np.concatenate([m.reshape(-1) for m in masks])) if masks else np.zeros(0, np.uint8)
        g.update({f"loop_{s}_seed": np.array(seed), f"loop_{s}_id": np.array(sid), f"loop_{s}_gt_box": gt,
                  f"loop_{s}_gt_bits": bits})
    g.update(loop_n_scenes=np.array(len(scenes)), loop_dims=np.array(LOOP_DIMS), loop_n_img=np.array(LOOP_N_IMG))
    for mode in ("test", "benchmark"):
        with tempfile.TemporaryDirectory() as tmp:
            cfg.TEST_SAVE_DIR = tmp
            out = io.StringIO()
            with contextlib.redirect_stdout(out):
                getattr(SolverWrapper, mode)(net, [loop_blobs(*sc) for sc in scenes], None)
            g[f"loop_{mode}_printed"] = np.array("\n".join(ln for ln in out.getvalue().splitlines()
                                                           if ln.startswith(("mAP of ", "class "))))
            for s, sc in enumerate(scenes):
                d = os.path.join(tmp, sc[4])
                key = f"loop_{mode}_{s}_"
                g[key + "written"] = np.array(int(os.path.isdir(d)))
                if not os.path.isdir(d):
                    continue
                for f in ("pred_class", "pred_conf", "pred_box"):
                    g[key + f] = np.load(os.path.join(d, f + ".npy"))
                pm = pickle.load(open(os.path.join(d, "pred_mask"), "rb"))
                g[key + "pred_mask_index"] = np.array(pickle.load(open(os.path.join(d, "pred_mask_index"), "rb")), bool)
                g[key + "pred_mask_shapes"] = np.array([m.shape for m in pm], np.int64).reshape(-1, 3)
                g[key + "pred_mask_bits"] = (np.packbits(np.concatenate([(m.reshape(-1) != 0) for m in pm])) if pm
                                             else np.zeros(0, np.uint8))
            print(f"[golden] loop {mode}: written {[int(g[f'loop_{mode}_{s}_written']) for s in range(len(scenes))]}")
            print(g[f"loop_{mode}_printed"])


def main():
    torch.manual_seed(0)
    g = {}
    which = sys.argv[1:]
    for case in CASES:
        if not which or case[0] in which:
            run_case(g, *case)
    if not which or "loop" in which:
        run_loops(g)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {len(g)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
