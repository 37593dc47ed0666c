"""Seeded synthetic inputs for the 3D-SIS dense-voxel inference hot path.

Nothing here is part of the product path: these generators feed the parity
tests, the golden-vector script and bench.py (there is no network access for
ScanNet/SUNCG, so shapes follow the reference's data contract and values are
synthetic).  numpy's PCG64 generator is used everywhere so a seed means the
same bytes in every process/torch version.

Data contract being mimicked (reference file:line):
  * voxel grid  data[1,2,X,Y,Z]: ch0 = |clip(sdf,-3,3)|, ch1 = sdf > -1
                                  (lib/datasets/dataset.py:50-68)
  * ENet-shaped 2D features [n,128,32,41] (lib/nets/network.py:199-205)
  * depth [n,32,41] metres, camera_to_world poses [n,4,4], world2grid [4,4]
    (lib/datasets/dataset.py:135-187), intrinsics
    (experiments/cfgs/ScanNet/rpn_class_mask_5.yml:99-102)
  * state_dict key names / shapes (lib/nets/backbones.py:171-231,236-287,
    lib/nets/network.py:35-64)
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np

VOXEL_SIZE = 0.046875
INTRINSIC_SCANNET = np.array([[37.01983, 0, 20, 0],
                              [0, 38.52470, 15.5, 0],
                              [0, 0, 1, 0],
                              [0, 0, 0, 1]], dtype=np.float32)
DEPTH_W, DEPTH_H = 41, 32

_ANCHOR_SIZES = np.array([[8, 9, 8], [14, 11, 14], [14, 20, 14], [21, 38, 7], [7, 39, 21],
                          [32, 18, 15], [15, 17, 31], [53, 22, 24], [24, 22, 53], [28, 22, 4],
                          [4, 22, 28], [18, 8, 46], [46, 8, 18], [9, 35, 9]], dtype=np.float64)


def _scene_boxes(rng, dims):
    X, Y, Z = dims
    k = int(rng.integers(4, 13))
    boxes = []
    for _ in range(k):
        size = _ANCHOR_SIZES[int(rng.integers(0, len(_ANCHOR_SIZES)))] * rng.uniform(0.7, 1.3, 3)
        size = np.minimum(size, np.array([X, Y, Z]) * 0.8)
        lo_x = rng.uniform(0, X - size[0])
        lo_z = rng.uniform(0, Z - size[2])
        boxes.append([lo_x, 0.0, lo_z, lo_x + size[0], size[1], lo_z + size[2]])
    return np.asarray(boxes, dtype=np.float64)


def make_scene(seed: int, dims=(96, 48, 96)):
    """Return (data[1,2,X,Y,Z] float32, boxes[k,6] float64 in voxel units)."""
    rng = np.random.default_rng(seed)
    X, Y, Z = dims
    boxes = _scene_boxes(rng, dims)
    gx, gy, gz = np.meshgrid(np.arange(X) + 0.5, np.arange(Y) + 0.5, np.arange(Z) + 0.5, indexing="ij")
    sdf = np.minimum.reduce([gy, gx, X - gx, gz, Z - gz])  # floor + four walls
    for b in boxes:
        dx = np.maximum(b[0] - gx, gx - b[3])
        dy = np.maximum(b[1] - gy, gy - b[4])
        dz = np.maximum(b[2] - gz, gz - b[5])
        outside = np.sqrt(np.maximum(dx, 0) ** 2 + np.maximum(dy, 0) ** 2 + np.maximum(dz, 0) ** 2)
        inside = np.minimum(np.maximum.reduce([dx, dy, dz]), 0)
        sdf = np.minimum(sdf, outside + inside)
    sdf = sdf + rng.normal(0.0, 0.05, sdf.shape)
    sdf = sdf.astype(np.float32)
    ch0 = np.abs(np.clip(sdf, -3.0, 3.0))
    ch1 = (sdf > -1).astype(np.float32)
    data = np.stack([ch0, ch1], 0)[None].astype(np.float32)
    return np.ascontiguousarray(data), boxes


def _ray_box(o, d, lo, hi):
    """Slab test; o[3], d[...,3]; returns entry distance (inf when missed)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t0 = (lo - o) * inv
        t1 = (hi - o) * inv
    tmin = np.minimum(t0, t1).max(-1)
    tmax = np.maximum(t0, t1).min(-1)
    hit = (tmax >= np.maximum(tmin, 0.0))
    return np.where(hit, np.where(tmin > 0, tmin, np.inf), np.inf)


def make_views(seed: int, dims=(96, 48, 96), n_img=5, boxes=None, feat_channels=128,
               intrinsic=INTRINSIC_SCANNET):
    """Return dict(feats[n,C,32,41], depths[n,32,41], poses[n,4,4], world2grid[4,4])."""
    rng = np.random.default_rng(seed + 1_000_003)
    X, Y, Z = dims
    vs = VOXEL_SIZE
    world2grid = np.diag([1.0 / vs, 1.0 / vs, 1.0 / vs, 1.0]).astype(np.float32)
    cam_pos = np.array([X * vs * 0.5, min(1.5, Y * vs * 0.66), Z * vs * 0.5])
    poses, depths = [], []
    u, v = np.meshgrid(np.arange(DEPTH_W), np.arange(DEPTH_H), indexing="xy")
    for i in range(n_img):
        yaw = 2.0 * math.pi * i / n_img + 0.1
        pitch = math.radians(12.0)
        zc = np.array([math.sin(yaw) * math.cos(pitch), -math.sin(pitch), math.cos(yaw) * math.cos(pitch)])
        xc = np.cross(np.array([0.0, -1.0, 0.0]), zc)
        xc /= np.linalg.norm(xc)
        yc = np.cross(zc, xc)
        pose = np.eye(4)
        pose[:3, 0], pose[:3, 1], pose[:3, 2], pose[:3, 3] = xc, yc, zc, cam_pos
        # ray directions with unit camera-z so that t == depth
        dirs_c = np.stack([(u - intrinsic[0, 2]) / intrinsic[0, 0],
                           (v - intrinsic[1, 2]) / intrinsic[1, 1],
                           np.ones_like(u, dtype=np.float64)], -1)
        dirs_w = dirs_c @ pose[:3, :3].T
        room_lo, room_hi = np.zeros(3), np.array([X, Y, Z]) * vs
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / dirs_w
            t_exit = np.maximum((room_lo - cam_pos) * inv, (room_hi - cam_pos) * inv).min(-1)
        depth = t_exit
        if boxes is not None:
            for b in boxes:
                depth = np.minimum(depth, _ray_box(cam_pos, dirs_w, b[:3] * vs, b[3:] * vs))
        depth = depth + rng.normal(0.0, 0.004, depth.shape)
        poses.append(pose.astype(np.float32))
        depths.append(depth.astype(np.float32))
    feats = rng.standard_normal((n_img, feat_channels, DEPTH_H, DEPTH_W)).astype(np.float32)
    return {"feats": feats, "depths": np.stack(depths), "poses": np.stack(poses), "world2grid": world2grid}


# ----------------------------------------------------------------------------------------------
# weights
# ----------------------------------------------------------------------------------------------
def _bottleneck(prefix, inpl, planes):
    return [(f"{prefix}.conv1.weight", (planes, inpl, 1, 1, 1)), (f"{prefix}.conv1.bias", (planes,)),
            (f"{prefix}.conv2.weight", (planes, planes, 3, 3, 3)), (f"{prefix}.conv2.bias", (planes,)),
            (f"{prefix}.conv3.weight", (inpl, planes, 1, 1, 1)), (f"{prefix}.conv3.bias", (inpl,))]


def param_shapes(net="ScanNet_Backbone", use_images=True, num_classes=19, a1=3, a2=11,
                 pool=4, rpn_channels=256, use_mask=True, only_images=False, mask_images=None):
    """state_dict names -> shapes of the 3D part of the model (ENet excluded).

    ScanNet: lib/nets/backbones.py:171-231 (only_images: ONLY_IMAGES = USE_IMAGES = True, no geometry1 and a 128-channel
    colour stack); SUNCG: 118-169; heads lib/nets/network.py:35-57; mask head lib/nets/backbones.py:236-272 (mask_images:
    None, 'use' = MASK_USE_IMAGES: geometry ends 64 -> 64, a colour stack and combine; 'only' = MASK_ONLY_IMAGES too: the
    colour stack's 1x1 makes the classes).
    """
    s = []
    if only_images:
        if net != "ScanNet_Backbone" or not use_images:
            raise ValueError("only_images: ScanNet_Backbone with use_images")
        s += [("color.0.weight", (64, 128, 2, 2, 2))] + _bottleneck("color.2", 64, 32)
        s += [("color.4.weight", (128, 64, 2, 2, 2))] + _bottleneck("color.6", 128, 32)
        s += [("geometry2.0.weight", (128, 128, 3, 3, 3))]
        s += _bottleneck("geometry2.2", 128, 64) + _bottleneck("geometry2.3", 128, 64)
    elif net == "ScanNet_Backbone":
        gch, cch = (64, 64) if use_images else (128, 0)
        s += [("geometry1.0.weight", (32, 2, 2, 2, 2))]
        s += _bottleneck("geometry1.2", 32, 32) + _bottleneck("geometry1.3", 32, 32)
        s += [("geometry1.4.weight", (gch, 32, 2, 2, 2))]
        s += _bottleneck("geometry1.6", gch, 32) + _bottleneck("geometry1.7", gch, 32)
        if use_images:
            s += [("color.0.weight", (64, 128, 2, 2, 2))] + _bottleneck("color.2", 64, 32)
            s += [("color.4.weight", (cch, 64, 2, 2, 2))] + _bottleneck("color.6", cch, 32)
        s += [("geometry2.0.weight", (128, gch + cch, 3, 3, 3))]
        s += _bottleneck("geometry2.2", 128, 64) + _bottleneck("geometry2.3", 128, 64)
    elif net == "SUNCG_Backbone":
        s += [("geometry1.0.weight", (64, 2, 2, 2, 2))] + _bottleneck("geometry1.2", 64, 32)
        s += [("geometry1.3.weight", (64, 64, 2, 2, 2))] + _bottleneck("geometry1.5", 64, 32)
        if use_images:
            s += [("color.0.weight", (64, 128, 2, 2, 2))] + _bottleneck("color.2", 64, 32)
            s += [("color.3.weight", (64, 64, 2, 2, 2))] + _bottleneck("color.5", 64, 32)
        s += [("geometry2.0.weight", (128, 128 if use_images else 64, 3, 3, 3))]
        s += _bottleneck("geometry2.2", 128, 64)
    else:
        raise ValueError(net)
    s += [("classifier.0.weight", (256, 128 * pool ** 3)), ("classifier.0.bias", (256,)),
          ("classifier.2.weight", (256, 256)), ("classifier.2.bias", (256,)),
          ("classifier.4.weight", (128, 256)), ("classifier.4.bias", (128,))]
    for lvl, a in ((1, a1), (2, a2)):
        if a:
            s += [(f"rpn_net_level{lvl}.weight", (rpn_channels, 128, 3, 3, 3)),
                  (f"rpn_net_level{lvl}.bias", (rpn_channels,)),
                  (f"rpn_cls_score_net_level{lvl}.0.weight", (2 * a, rpn_channels, 1, 1, 1)),
                  (f"rpn_cls_score_net_level{lvl}.0.bias", (2 * a,)),
                  (f"rpn_bbox_pred_net_level{lvl}.weight", (6 * a, rpn_channels, 1, 1, 1)),
                  (f"rpn_bbox_pred_net_level{lvl}.bias", (6 * a,))]
    s += [("classifier_cls_score_net.weight", (num_classes, 128)), ("classifier_cls_score_net.bias", (num_classes,)),
          ("classifier_bbox_pred_net.weight", (num_classes * 6, 128)),
          ("classifier_bbox_pred_net.bias", (num_classes * 6,))]
    if use_mask:
        cin = 2
        for i in (0, 2, 4, 6, 8):
            s += [(f"mask_backbone.geometry.{i}.weight", (64, cin, 3, 3, 3))]
            cin = 64
        s += [("mask_backbone.geometry.10.weight", (64 if mask_images else num_classes, 64, 1, 1, 1))]
        if mask_images:
            cin = 128
            for i in (0, 2, 4, 6, 8):
                s += [(f"mask_backbone.color.{i}.weight", (64, cin, 3, 3, 3))]
                cin = 64
            s += [("mask_backbone.color.10.weight", (num_classes if mask_images == "only" else 64, 64, 1, 1, 1)),
                  ("mask_backbone.combine.0.weight", (128, 128, 3, 3, 3)),
                  ("mask_backbone.combine.2.weight", (num_classes, 128, 1, 1, 1))]
    return OrderedDict(s)


# gains applied on top of the U(-1/sqrt(fan_in), 1/sqrt(fan_in)) default-init bound so that a
# random network yields a non-degenerate workload (varied RPN scores, confident classes -> masks).
_GAINS = {"rpn_cls_score_net": 40.0, "rpn_bbox_pred_net": 4.0, "classifier_cls_score_net": 60.0,
          "classifier_bbox_pred_net": 3.0, "mask_backbone.geometry.10": 8.0, "mask_backbone.color.10": 8.0,
          "mask_backbone.combine.2": 8.0}


def make_weights(seed=0, **kw):
    """Deterministic numpy weights keyed like the reference state_dict (float32)."""
    rng = np.random.default_rng(seed + 77)
    out = OrderedDict()
    shapes = param_shapes(**kw)
    fan = {}
    for name, shp in shapes.items():
        if name.endswith("weight"):
            fan[name.rsplit(".", 1)[0]] = int(np.prod(shp[1:]))
    for name, shp in shapes.items():
        base = name.rsplit(".", 1)[0]
        bound = 1.0 / math.sqrt(fan[base])
        gain = 1.0
        for k, g in _GAINS.items():
            if base.startswith(k):
                gain = g
        out[name] = (rng.uniform(-bound, bound, shp) * gain).astype(np.float32)
    return out


def make_nms_boxes(seed, n=400, dims=(96, 48, 96), dup_frac=0.05):
    """Score-sorted-looking proposal boxes for operator-level NMS / RoI tests (SURVEY 8d)."""
    rng = np.random.default_rng(seed + 5)
    dims = np.asarray(dims, dtype=np.float64)
    size = _ANCHOR_SIZES[rng.integers(0, len(_ANCHOR_SIZES), n)] * np.exp(rng.normal(0, 0.2, (n, 3)))
    size = np.minimum(size, dims)
    ctr = rng.uniform(0, 1, (n, 3)) * dims
    lo = np.clip(ctr - size / 2, 0, dims)
    hi = np.clip(ctr + size / 2, 0, dims)
    boxes = np.concatenate([lo, hi], 1)
    integer = rng.uniform(size=n) < 0.3
    boxes[integer] = np.round(boxes[integer])
    ndup = int(n * dup_frac)
    if ndup:
        src = rng.integers(0, n, ndup)
        dst = rng.integers(0, n, ndup)
        boxes[dst] = boxes[src]
    return boxes.astype(np.float32)


# ---------------------------------------------------------------- named cases shared by the parity tests, smoke() and bench.py
CASES = {
    "cfg1_32": dict(cfgname="scannet", dims=(32, 32, 32), n_img=0, seed=101, use_images=False, use_mask=False),
    "odd_45x27x41": dict(cfgname="scannet", dims=(45, 27, 41), n_img=3, seed=202, use_images=True, use_mask=True),
    "cfg2_96x48x96": dict(cfgname="scannet", dims=(96, 48, 96), n_img=5, seed=303, use_images=True, use_mask=True),
    "suncg_40x24x40": dict(cfgname="suncg", dims=(40, 24, 40), n_img=3, seed=404, use_images=True, use_mask=True),
}


def build_case(port, c):
    """(oracle cfg, weights, data, views) of a named case; `port` is the CPU checker module (oracle/port.py), passed in by
    the test / bench leg that is allowed to use it."""
    cfg = port.make_cfg(c["cfgname"], USE_IMAGES=c["use_images"], USE_MASK=c["use_mask"])
    w = make_weights(seed=0, net=cfg.NET, use_images=c["use_images"], num_classes=cfg.NUM_CLASSES,
                     a1=cfg.NUM_ANCHORS_LEVEL1, a2=cfg.NUM_ANCHORS_LEVEL2, use_mask=c["use_mask"])
    data, boxes = make_scene(c["seed"], c["dims"])
    views = None
    if c["use_images"]:
        views = make_views(c["seed"], c["dims"], c["n_img"], boxes, intrinsic=np.array(cfg.INTRINSIC, dtype=np.float32))
    return cfg, w, data, views


def make_net(c, keep_debug=True, math="fp32", weights=None, enet=False, gt_rois=None, only_images=False, mask_images=None):
    """The product Network for a case: released yml config, seeded synthetic weights loaded through load_state_dict.
    enet=True: cfg.USE_IMAGES_GT=False -- the blobs carry RGB frames and the 2-D ENet encoder (seeded default init) is part
    of the forward.  gt_rois=True / False: test mode on ground-truth boxes and classes (USE_RPN = USE_CLASS = False) with
    USE_BACKBONE on / off; the weights are those of the same model without RPN and classifier heads (the ones
    oracle/make_golden_gt_rois.py loads into the reference).  only_images=True: the image-only ScanNet backbone (ONLY_IMAGES)
    with the weights of param_shapes(only_images=True).  mask_images='use' / 'only': the colour-aware mask head
    (MASK_USE_IMAGES, with MASK_ONLY_IMAGES for 'only') and the weights of param_shapes(mask_images=...)."""
    import os
    import torch
    from lib.utils.config import cfg, cfg_from_file, cfg_reset
    cfg_reset()
    yml = "SUNCG" if c["cfgname"] == "suncg" else "ScanNet"
    cfg_from_file(os.path.join(os.path.dirname(os.path.abspath(__file__)), "experiments", "cfgs", yml, "rpn_class_mask_5.yml"))
    cfg.NUM_CLASSES = 26 if c["cfgname"] == "suncg" else 19
    cfg.USE_IMAGES, cfg.USE_MASK, cfg.USE_IMAGES_GT = c["use_images"], c["use_mask"], not enet
    cfg.ONLY_IMAGES = bool(only_images)
    cfg.MASK_USE_IMAGES, cfg.MASK_ONLY_IMAGES = bool(mask_images), mask_images == "only"
    if gt_rois is not None:
        cfg.USE_RPN, cfg.USE_CLASS, cfg.USE_BACKBONE = False, False, bool(gt_rois)
    from lib.nets import backbones
    import torch as _t
    _t.manual_seed(1234)  # default-initialised tensors (the ENet encoder when enet=True) are the same in every process
    net = getattr(backbones, cfg.NET)()
    net.init_modules()
    if weights is None and gt_rois is not None:
        weights = {k: v for k, v in make_weights(seed=0, net=cfg.NET, use_images=c["use_images"], num_classes=cfg.NUM_CLASSES,
                                                 a1=0, a2=0, use_mask=c["use_mask"], mask_images=mask_images).items()
                   if not k.startswith("classifier_")}
    w = weights if weights is not None else make_weights(
        seed=0, net=cfg.NET, use_images=c["use_images"], num_classes=cfg.NUM_CLASSES, a1=cfg.NUM_ANCHORS_LEVEL1,
        a2=cfg.NUM_ANCHORS_LEVEL2, use_mask=c["use_mask"], only_images=only_images, mask_images=mask_images)
    net.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()}, strict=not enet)
    net._keep_debug = keep_debug
    net.set_conv_math(math)
    return net, cfg


def write_chunks(out_dir, c, seeds, label_seed=5):
    """Synthetic .chunk files of a case with GT for test mode's mAP: boxes from make_scene with random labels 1..18, each GT mask
    the voxels of negative SDF inside the box's floor / ceil bounds (as the dataset rounds it).  -> (paths, view_provider)."""
    import os
    from lib.datasets.scene_io import write_scene
    paths, provs = [], {}
    rng = np.random.default_rng(label_seed)
    for k, seed in enumerate(seeds):
        data, boxes = make_scene(seed, c["dims"])
        views = make_views(seed, c["dims"], c["n_img"], boxes)
        sdf = np.where(data[0, 1] > 0.5, data[0, 0], -data[0, 0]).astype(np.float32)
        sdf[(data[0, 1] < 0.5) & (data[0, 0] < 1.0)] = -1.0
        gt, masks = [], []
        for b in boxes:
            lo, hi = np.floor(b[:3]).astype(int), np.ceil(b[3:]).astype(int)
            label = int(rng.integers(1, 19))
            gt.append(list(b) + [label])
            masks.append((label, (sdf[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] < 0).astype(np.uint16)))
        p = os.path.join(out_dir, f"scene{k:04d}_00__0.chunk")
        write_scene(p, sdf, np.array(gt, np.float32), masks, world2grid=views["world2grid"], frame_ids=[0, 20, 40])
        paths.append(p)
        provs[p] = views
    provider = lambda p, ids, w2g, dims: {"images": provs[p]["feats"], "depths": provs[p]["depths"], "poses": provs[p]["poses"],
                                          "world2grid": provs[p]["world2grid"]}
    return paths, provider


def make_blobs(c, data, views, pin=False):
    """The reference's blob dict (lib/datasets/dataloader.py collate_fn) for one synthetic scene."""
    import torch
    t = (lambda a: torch.from_numpy(a).pin_memory()) if pin else torch.from_numpy
    blobs = {"data": t(data), "id": ["synthetic"], "gt_box": [torch.zeros(0, 7)], "gt_mask": [[]]}
    if views is not None:
        blobs["nearest_images"] = {"images": [t(views["feats"])], "depths": [t(views["depths"])],
                                   "poses": [t(views["poses"])], "world2grid": [t(views["world2grid"])]}
    return blobs
