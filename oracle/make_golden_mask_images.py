"""oracle/make_golden_mask_images.py -- TEST INFRASTRUCTURE ONLY; runs ONLY in the build container (needs the reference tree).

Runs the UNMODIFIED reference through oracle/ref_harness.py with the colour-aware mask head (MASK_USE_IMAGES, and
MASK_ONLY_IMAGES; lib/nets/backbones.py:236-287, lib/nets/network.py:302-317) and stores tests/golden/mask_images_reference.npz,
which pins the oracle's forward (oracle/port_mask_images.py) and the GPU forward (tests/test_mask_images.py,
tests/test_gpu_mask_images.py).

    python oracle/make_golden_mask_images.py

Forward cases (Network.forward, the reference's own test-mode forward, weights sis3d_synth.make_weights(mask_images=...)),
each on ENet-shaped features (USE_IMAGES_GT) unless it says otherwise:
  use_96x48x96 / only_96x48x96   96x48x96 with 5 views, MASK_USE_IMAGES / MASK_ONLY_IMAGES;
  killed_45x27x41                45x27x41 with 3 views, view 1 sees nothing within PROJ_DEPTH_MAX (killed);
  enet_45x27x41                  45x27x41 with 3 raw 256x328 images through the reference's ENet (USE_IMAGES_GT = False,
                                 encoder parameters of tests/golden/enet_encoder.npz);
  gt_45x27x41                    ground-truth RoIs (USE_RPN = USE_CLASS = False) with USE_BACKBONE off: boxes of
                                 oracle/make_golden_gt_rois.py's edge_boxes (every scene face, the whole scene, extent 1);
  oimg_45x27x41                  the image-only ScanNet backbone (ONLY_IMAGES) with MASK_USE_IMAGES;
  suncg_40x24x40                 SUNCG 40x24x40 with 3 views.
Refusals: MASK_USE_IMAGES with USE_IMAGES = False and MASK_ONLY_IMAGES without MASK_USE_IMAGES; the exception is stored.
Loop set: the reference's SolverWrapper.test and SolverWrapper.benchmark (lib/model/trainval.py:634-941) with
MASK_USE_IMAGES on two seeded 45x27x41 scenes with 3 views, writing the result files.

Layout: step_{imageft, mask_cls, mask_allcls} (the sample strides); per mode m in (use, only): sd_{m}_keys / sd_{m}_shapes
(the reference mask head's state_dict).  Per forward case t: t_dims, t_seed, t_n_img, t_cfgname, t_mask_images ('use' /
'only'), t_only_images_backbone, t_gt (1: ground-truth RoIs, t_gt_box), t_killed, t_images_seed (-1: features),
t_killing_inds; t_imageft_sub / _stats (strided samples, NCDHW C order, [sum, sum |.|, max, min]), t_rois, t_cls_prob,
t_cls_pred, t_bbox_pred, t_pred_box (the driver's decode), t_keep, t_crops, t_mask_{j}_cls_sub (kept crop j's
predicted-class mask, strided), t_mask_{j}_allcls_sub (all classes, strided), t_mask_{j}_cls_on (voxels > 0.5), t_n_masks.
refused_{no_images, only_without_use}: the exception text.  Loop set: as in oracle/make_golden_only_images.py.
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
import make_golden_gt_rois as gtr  # noqa: E402
import make_golden_only_images as oimg  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mask_images_reference.npz")
YML = {"scannet": "ScanNet/rpn_class_mask_5.yml", "suncg": "SUNCG/rpn_class_mask_5.yml"}
CASES = [  # tag, cfg, dims, n_img, seed, killed views, raw-image seed, mask mode, image-only backbone, ground-truth RoIs
    ("use_96x48x96", "scannet", (96, 48, 96), 5, 303, (), None, "use", False, False),
    ("only_96x48x96", "scannet", (96, 48, 96), 5, 303, (), None, "only", False, False),
    ("killed_45x27x41", "scannet", (45, 27, 41), 3, 202, (1,), None, "use", False, False),
    ("enet_45x27x41", "scannet", (45, 27, 41), 3, 202, (), 77, "use", False, False),
    ("gt_45x27x41", "scannet", (45, 27, 41), 3, 202, (), None, "use", False, True),
    ("oimg_45x27x41", "scannet", (45, 27, 41), 3, 202, (), None, "use", True, False),
    ("suncg_40x24x40", "suncg", (40, 24, 40), 3, 404, (), None, "use", False, False),
]
LOOP_DIMS, LOOP_N_IMG, LOOP_SEEDS = (45, 27, 41), 3, (231, 232)
STEPS = dict(imageft=997, mask_cls=29, mask_allcls=389)


def weights(cfg, mask_images, only_images=False, gt=False):
    w = synth.make_weights(seed=0, net=cfg.NET, use_images=True, num_classes=cfg.NUM_CLASSES,
                           a1=0 if gt else cfg.NUM_ANCHORS_LEVEL1, a2=0 if gt else cfg.NUM_ANCHORS_LEVEL2, use_mask=True,
                           only_images=only_images, mask_images=mask_images)
    return {k: v for k, v in w.items() if not (gt and k.startswith("classifier_"))}


def run_case(g, tag, cfgname, dims, n_img, seed, killed, images_seed, mask_images, only_images, gt_rois):
    rh.install()
    from lib.layer_utils.projection import ProjectionHelper
    from lib.utils.bbox_transform import bbox_transform_inv, clip_boxes
    with tempfile.TemporaryDirectory() as tmp:
        over = dict(USE_IMAGES=True, ONLY_IMAGES=only_images, USE_IMAGES_GT=images_seed is None, USE_MASK=True,
                    MASK_USE_IMAGES=True, MASK_ONLY_IMAGES=mask_images == "only")
        over.update(USE_RPN=not gt_rois, USE_CLASS=not gt_rois, USE_BACKBONE=not gt_rois)
        if images_seed is not None:
            over["PRETRAINED_ENET_PATH"] = os.path.join(tmp, "enet.pth")
            cfg = rh.load_cfg(YML[cfgname], **over)
            oimg.enet_checkpoint(over["PRETRAINED_ENET_PATH"], cfg.NUM_2D_CLASSES)
        cfg = rh.load_cfg(YML[cfgname], **over)
        torch.manual_seed(0)
        net = oimg.build(cfg, weights(cfg, mask_images, only_images, gt_rois))
    if tag in ("use_96x48x96", "only_96x48x96"):
        sd = {k: v for k, v in net.state_dict().items() if k.startswith("mask_backbone.")}
        g[f"sd_{mask_images}_keys"] = np.array(list(sd))
        g[f"sd_{mask_images}_shapes"] = np.array([list(v.shape) for v in sd.values()], np.int64)
    data, boxes = synth.make_scene(seed, dims)
    v = synth.make_views(seed, dims, n_img, boxes, intrinsic=np.array(cfg.INTRINSIC, dtype=np.float32))
    for k in killed:
        v["depths"][k][:] = 9.0  # beyond PROJ_DEPTH_MAX: no valid projection
    feats = v["feats"] if images_seed is None else oimg.raw_images(images_seed, n_img)
    gt = gtr.edge_boxes(dims, cfg.NUM_CLASSES, seed) if gt_rois else np.zeros((0, 7), np.float32)
    blobs = {"data": torch.from_numpy(data), "id": [f"synthetic_{tag}"], "gt_box": [torch.from_numpy(gt)], "gt_mask": [[]]}
    helper = ProjectionHelper(cfg.INTRINSIC, cfg.PROJ_DEPTH_MIN, cfg.PROJ_DEPTH_MAX, cfg.DEPTH_SHAPE, blobs["data"].shape[-3:],
                              cfg.VOXEL_SIZE)
    maps = [helper.compute_projection(torch.from_numpy(d), torch.from_numpy(c), torch.from_numpy(v["world2grid"]))
            for d, c in zip(v["depths"], v["poses"])]
    killing = [i for i, m in enumerate(maps) if m is None]
    assert killing == list(killed), (tag, killing)
    real = [m for m in maps if m is not None]
    blobs["proj_ind_3d"] = [torch.stack([m[0] for m in real])]
    blobs["proj_ind_2d"] = [torch.stack([m[1] for m in real])]
    blobs["nearest_images"] = {"images": [torch.from_numpy(feats)]}
    net.forward(blobs, "TEST", killing)
    P = net._predictions
    k = tag + "_"
    g.update({k + "dims": np.array(dims), k + "seed": np.array(seed), k + "n_img": np.array(n_img), k + "cfgname": np.array(cfgname),
              k + "mask_images": np.array(mask_images), k + "only_images_backbone": np.array(int(only_images)),
              k + "gt": np.array(int(gt_rois)), k + "gt_box": gt, k + "killed": np.array(killed, np.int64),
              k + "images_seed": np.array(-1 if images_seed is None else images_seed), k + "killing_inds": np.array(killing, np.int64)})
    g[k + "imageft_sub"], g[k + "imageft_stats"] = oimg.sub(net._imageft, STEPS["imageft"])
    g[k + "rois"] = P["rois"][0].cpu().numpy()
    pc = P["cls_pred"].cpu().numpy()
    g[k + "cls_prob"], g[k + "cls_pred"], g[k + "bbox_pred"] = P["cls_prob"].cpu().numpy(), pc, P["bbox_pred"].cpu().numpy()
    reg = np.stack([g[k + "bbox_pred"][i, pc[i] * 6:(pc[i] + 1) * 6] for i in range(len(pc))]) if len(pc) else np.zeros((0, 6))
    pb = clip_boxes(bbox_transform_inv(P["rois"][0].cpu(), torch.from_numpy(reg).float()), list(dims)).numpy()
    conf = np.array([g[k + "cls_prob"][i, pc[i]] for i in range(len(pc))])
    keep = conf > cfg.CLASS_THRESH
    for i, b in enumerate(pb):
        if round(b[0]) >= round(b[3]) or round(b[1]) >= round(b[4]) or round(b[2]) >= round(b[5]):
            keep[i] = False
    g[k + "pred_box"], g[k + "keep"] = pb, keep
    g[k + "crops"] = np.array([[int(round(float(x))) for x in b] for b in pb], np.int64).reshape(-1, 6)
    masks = P["mask_pred"][0]
    assert len(masks) == keep.sum(), (len(masks), keep.sum())
    for j, i in enumerate(np.nonzero(keep)[0]):
        m = masks[j][0].numpy()
        g[k + f"mask_{j}_cls_sub"] = m[pc[i]].reshape(-1)[::STEPS["mask_cls"]].copy()
        g[k + f"mask_{j}_cls_on"] = np.array(int((m[pc[i]] > 0.5).sum()))
        g[k + f"mask_{j}_allcls_sub"] = m.reshape(-1)[::STEPS["mask_allcls"]].copy()
    g[k + "n_masks"] = np.array(len(masks))
    faces = [int(((c[:3] == 0) | (c[3:] == np.array(dims))).any()) for c in g[k + "crops"][keep]]
    print(f"[golden] {tag}: rois={len(pc)} masks={len(masks)} on a scene face={sum(faces)} killed={killing}")


def refused(g, key, **over):
    """Build the reference model of a switch combination, load the synthetic weights of the model it declares (the mask head
    must keep crops for the forward to reach it: CLASS_THRESH = 0 keeps every RoI) and run one scene through it; store what
    it raised."""
    cfg = rh.load_cfg(YML["scannet"], USE_IMAGES_GT=True, USE_MASK=True, CLASS_THRESH=0.0, **over)
    from lib.nets import backbones
    torch.manual_seed(0)
    try:
        net = getattr(backbones, cfg.NET)()
        net.init_modules()
        w = synth.make_weights(seed=0, net=cfg.NET, use_images=cfg.USE_IMAGES, num_classes=cfg.NUM_CLASSES,
                               a1=cfg.NUM_ANCHORS_LEVEL1, a2=cfg.NUM_ANCHORS_LEVEL2, use_mask=True,
                               mask_images="use" if cfg.MASK_USE_IMAGES else None)
        net.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()}, strict=True)
        net.eval()
        dims, n_img = (45, 27, 41), 3 if cfg.USE_IMAGES else 0
        data, boxes = synth.make_scene(202, dims)
        views = synth.make_views(202, dims, n_img, boxes, intrinsic=np.array(cfg.INTRINSIC, dtype=np.float32)) if n_img else None
        rh.reference_forward(net, cfg, data, views)
    except Exception as e:  # noqa: BLE001 -- the failure is the record
        g[key] = np.array(f"{type(e).__name__}: {e}".splitlines()[0])
        print(f"[golden] {key}: {g[key]}")
        return
    raise SystemExit(f"{key}: the reference ran this combination; support it and pin its outputs instead")


def run_loops(g):
    rh.install()
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
    cfg = rh.load_cfg(YML["scannet"], USE_IMAGES=True, USE_IMAGES_GT=True, USE_MASK=True, ONLY_IMAGES=False, MASK_USE_IMAGES=True,
                      MASK_ONLY_IMAGES=False, USE_RPN=True, USE_CLASS=True, USE_BACKBONE=True)
    torch.manual_seed(0)
    net = oimg.build(cfg, weights(cfg, "use"))
    scenes = []
    rng = np.random.default_rng(5)
    for s, seed in enumerate(LOOP_SEEDS):
        data, boxes = synth.make_scene(seed, LOOP_DIMS)
        views = synth.make_views(seed, LOOP_DIMS, LOOP_N_IMG, boxes)
        gt, masks = [], []
        for b in boxes:  # the scene's own boxes on the half-voxel grid, each GT mask its whole rounded box
            lo, hi = np.clip(np.round(b[:3] * 2) / 2, 0, LOOP_DIMS), np.clip(np.round(b[3:] * 2) / 2, 0, LOOP_DIMS)
            ext = np.rint(hi).astype(int) - np.rint(lo).astype(int)
            if (ext <= 0).any():
                continue
            gt.append(list(lo) + list(hi) + [int(rng.integers(1, cfg.NUM_CLASSES))])
            masks.append(np.ones(ext, np.uint8))
        gt = np.array(gt, np.float32).reshape(-1, 7)
        sid = f"scene{s:04d}_00"
        scenes.append((data, views, gt, masks, sid))
        g.update({f"loop_{s}_seed": np.array(seed), f"loop_{s}_id": np.array(sid), f"loop_{s}_gt_box": gt,
                  f"loop_{s}_gt_bits": np.packbits(np.concatenate([m.reshape(-1) for m in masks]))})
    g.update(loop_n_scenes=np.array(len(scenes)), loop_dims=np.array(LOOP_DIMS), loop_n_img=np.array(LOOP_N_IMG))
    # the loops hand mask_backbone `[]` for the image features (trainval.py:744, 890): a colour-aware head fails there
    with tempfile.TemporaryDirectory() as tmp:
        cfg.TEST_SAVE_DIR = tmp
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                SolverWrapper.test(net, [gtr.loop_blobs(*scenes[0])], None)
        except Exception as e:  # noqa: BLE001 -- the failure is the record
            g["loop_refused"] = np.array(f"{type(e).__name__}: {e}".splitlines()[0])
            print(f"[golden] loop_refused: {g['loop_refused']}")
        else:
            raise SystemExit("the reference's test loop ran the colour-aware head; pin its own outputs instead")
    # the loop set is written with the crop of the forward's own back-projected volume at the loop's box (network.py:302-317
    # crops it so): the crop's origin is the scene view's storage offset in blobs['data'] [1, 2, X, Y, Z]
    head = net.mask_backbone.forward

    def with_imageft(scene, imageft):
        if isinstance(imageft, list):
            _, _, Xs, Ys, Zs = net._scene.shape
            o = scene.storage_offset()
            x0, y0, z0 = o // (Ys * Zs), (o // Zs) % Ys, o % Zs
            w, h, l = scene.shape[2:]
            imageft = net._imageft[:, :, x0:x0 + w, y0:y0 + h, z0:z0 + l]
        return head(scene, imageft)

    net.mask_backbone.forward = with_imageft
    for mode in ("test", "benchmark"):
        with tempfile.TemporaryDirectory() as tmp:
            cfg.TEST_SAVE_DIR = tmp
            out = io.StringIO()
            with contextlib.redirect_stdout(out):
                getattr(SolverWrapper, mode)(net, [gtr.loop_blobs(*sc) for sc in scenes], None)
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


def main():
    g = {f"step_{k}": np.array(v) for k, v in STEPS.items()}
    for case in CASES:
        run_case(g, *case)
    run_loops(g)
    refused(g, "refused_no_images", USE_IMAGES=False, MASK_USE_IMAGES=True, MASK_ONLY_IMAGES=False)
    refused(g, "refused_only_without_use", USE_IMAGES=True, MASK_USE_IMAGES=False, MASK_ONLY_IMAGES=True)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {len(g)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
