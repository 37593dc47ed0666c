"""oracle/make_golden_only_images.py -- TEST INFRASTRUCTURE ONLY; runs ONLY in the build container (needs the reference tree).

Runs the UNMODIFIED reference through oracle/ref_harness.py with the image-only ScanNet backbone (ONLY_IMAGES = USE_IMAGES =
True, lib/nets/backbones.py:98-113, 171-231) and stores tests/golden/only_images_reference.npz, which pins the oracle's
image-only forward (oracle/port_only_images.py) and the GPU forward (tests/test_only_images.py, tests/test_gpu_only_images.py).

    python oracle/make_golden_only_images.py

Forward cases (Network.forward, the reference's own test-mode forward, weights sis3d_synth.make_weights(only_images=True)):
96x48x96 with 5 views, 45x27x41 with 3 views of which view 1 sees nothing within PROJ_DEPTH_MAX (killed), 88x44x88 with 8
views, all on ENet-shaped features (USE_IMAGES_GT); and 45x27x41 with 3 raw 256x328 images through the reference's ENet
(USE_IMAGES_GT = False, encoder parameters of tests/golden/enet_encoder.npz, loaded from PRETRAINED_ENET_PATH as the
reference does).

Refusals: the two neighbouring combinations the reference cannot run, SUNCG_Backbone with ONLY_IMAGES (and USE_IMAGES) and
ScanNet_Backbone with ONLY_IMAGES and USE_IMAGES = False, each built and run on a small scene; the exception is stored.

Loop set: the reference's SolverWrapper.test and SolverWrapper.benchmark (lib/model/trainval.py:634-941) on two seeded
45x27x41 scenes with 3 views, writing the result files.

Layout: step_{imageft, level, rpn_prob, mask_cls, mask_allcls} (the sample strides); sd_keys / sd_shapes (the reference
model's state_dict without the 2-D encoder); per forward case t: t_dims, t_seed, t_n_img, t_killed (views whose depth was
set beyond PROJ_DEPTH_MAX), t_images_seed (-1: features), t_killing_inds; t_imageft_sub, t_level1_sub, t_level2_sub
(strided samples, NCDHW C order, and [sum, sum |.|, max, min] as *_stats); t_rpn_prob_sub_l{1,2} (strided), t_rois,
t_roi_scores, t_level_inds, t_cls_prob, t_cls_pred, t_bbox_pred, t_pred_box (the driver's decode), t_keep, t_crops, t_mask_{j}_cls_sub (kept crop j's predicted-class mask, strided), t_mask_{j}_allcls_sub
(all classes, strided), t_mask_{j}_cls_on (voxels > 0.5), t_n_masks.  refused_{suncg, no_images}: the exception text.
Loop set: loop_n_scenes, loop_dims, loop_n_img, loop_{s}_seed, loop_{s}_id, loop_{s}_gt_box, loop_{s}_gt_bits; per mode m in
(test, benchmark): loop_{m}_{s}_{written, pred_class, pred_conf, pred_box, pred_mask_index, pred_mask_bits, pred_mask_shapes},
loop_{m}_printed.
"""
from __future__ import annotations

import contextlib
import io
import os
import pickle
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-sis_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, ROOT)
import sis3d_synth as synth  # noqa: E402
import ref_harness as rh  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "only_images_reference.npz")
YML = "ScanNet/rpn_class_mask_5.yml"
CASES = [  # tag, dims, n_img, seed, killed views, seed of the raw images (None: ENet-shaped features)
    ("cfg2_96x48x96", (96, 48, 96), 5, 303, (), None),
    ("killed_45x27x41", (45, 27, 41), 3, 202, (1,), None),
    ("scene_88x44x88", (88, 44, 88), 8, 505, (), None),
    ("enet_45x27x41", (45, 27, 41), 3, 202, (), 77),
]
LOOP_DIMS, LOOP_N_IMG, LOOP_SEEDS = (45, 27, 41), 3, (231, 232)
# strides of the stored samples (kept in the fixture as step_*): coarse enough to keep the fixture small
STEPS = dict(imageft=997, level=97, rpn_prob=53, mask_cls=29, mask_allcls=389)


def weights(cfg):
    return synth.make_weights(seed=0, net=cfg.NET, use_images=True, num_classes=cfg.NUM_CLASSES, a1=cfg.NUM_ANCHORS_LEVEL1,
                              a2=cfg.NUM_ANCHORS_LEVEL2, use_mask=True, only_images=True)


def raw_images(seed, n):
    return np.random.default_rng(seed).standard_normal((n, 3, 256, 328)).astype(np.float32)


def enet_checkpoint(path, num_2d_classes):
    """A create_enet state_dict whose encoder carries the parameters of tests/golden/enet_encoder.npz (the file
    create_enet_for_3d loads, enet.py:697-699); the 2-D classifier keeps its seeded default init (unused by the forward)."""
    from lib.nets import enet  # the reference's module
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "enet_encoder.npz")))
    params = [g[k] for k in sorted(k for k in g if k.startswith("p"))]
    torch.manual_seed(7)
    model = enet.create_enet(num_2d_classes)
    sd = model.state_dict()
    names = [k for k in sd if not k.startswith(f"{len(model) - 1}.") and not k.endswith("num_batches_tracked")]
    assert len(names) == len(params), (len(names), len(params))
    for k, p in zip(names, params):
        sd[k] = torch.from_numpy(p)
    torch.save(sd, path)


def sub(t, step):
    a = np.asarray(t, dtype=np.float32).reshape(-1)
    return a[::step].copy(), np.array([a.astype(np.float64).sum(), np.abs(a).astype(np.float64).sum(), float(a.max()),
                                       float(a.min())])


def build(cfg, w):
    from lib.nets import backbones
    net = getattr(backbones, cfg.NET)()
    net.init_modules()
    res = net.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in w.items()}, strict=False)
    assert not res.unexpected_keys and all(k.startswith("image_enet_") for k in res.missing_keys), res
    return net.eval()


def run_case(g, tag, dims, n_img, seed, killed, images_seed):
    rh.install()  # the reference's `lib` package, not this repository's
    from lib.layer_utils.projection import ProjectionHelper
    from lib.utils.bbox_transform import bbox_transform_inv, clip_boxes
    with tempfile.TemporaryDirectory() as tmp:
        over = dict(USE_IMAGES=True, ONLY_IMAGES=True, USE_IMAGES_GT=images_seed is None, USE_MASK=True)
        if images_seed is not None:
            over["PRETRAINED_ENET_PATH"] = os.path.join(tmp, "enet.pth")
            cfg = rh.load_cfg(YML, **over)
            enet_checkpoint(over["PRETRAINED_ENET_PATH"], cfg.NUM_2D_CLASSES)
        cfg = rh.load_cfg(YML, **over)
        w = weights(cfg)
        torch.manual_seed(0)
        net = build(cfg, w)
    if images_seed is None:
        assert not any(k.startswith("image_enet_") for k in net.state_dict())
        g["sd_keys"] = np.array(list(net.state_dict()))
        g["sd_shapes"] = np.array([list(v.shape) + [0] * (5 - v.dim()) for v in net.state_dict().values()], np.int64)
    levels = {}
    orig = net._backbone

    def backbone():
        out = orig()
        levels["l1"], levels["l2"] = out[0], out[1]
        return out

    net._backbone = backbone
    data, boxes = synth.make_scene(seed, dims)
    v = synth.make_views(seed, dims, n_img, boxes, intrinsic=np.array(cfg.INTRINSIC, dtype=np.float32))
    for k in killed:
        v["depths"][k][:] = 9.0  # beyond PROJ_DEPTH_MAX: no valid projection
    feats = v["feats"] if images_seed is None else raw_images(images_seed, n_img)
    blobs = {"data": torch.from_numpy(data), "id": [f"synthetic_{tag}"], "gt_box": [torch.zeros(0, 7)], "gt_mask": [[]]}
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
    g.update({k + "dims": np.array(dims), k + "seed": np.array(seed), k + "n_img": np.array(n_img),
              k + "killed": np.array(killed, np.int64), k + "images_seed": np.array(-1 if images_seed is None else images_seed),
              k + "killing_inds": np.array(killing, np.int64)})
    g[k + "imageft_sub"], g[k + "imageft_stats"] = sub(net._imageft, STEPS["imageft"])
    assert levels["l1"].shape[1] == 128 and levels["l2"].shape[1] == 128
    g[k + "level1_sub"], g[k + "level1_stats"] = sub(levels["l1"], STEPS["level"])
    g[k + "level2_sub"], g[k + "level2_stats"] = sub(levels["l2"], STEPS["level"])
    for lvl in (1, 2):
        g[k + f"rpn_prob_sub_l{lvl}"], _ = sub(P[f"rpn_cls_prob_level{lvl}"][0, 1], STEPS["rpn_prob"])
    g[k + "rois"], g[k + "roi_scores"] = P["rois"][0].numpy(), P["roi_scores"][0].numpy()
    g[k + "level_inds"] = P["level_inds"][0].numpy()
    g[k + "cls_prob"], g[k + "cls_pred"], g[k + "bbox_pred"] = P["cls_prob"].numpy(), P["cls_pred"].numpy(), P["bbox_pred"].numpy()
    pc = g[k + "cls_pred"]
    reg = np.stack([g[k + "bbox_pred"][i, pc[i] * 6:(pc[i] + 1) * 6] for i in range(len(pc))]) if len(pc) else np.zeros((0, 6))
    pb = clip_boxes(bbox_transform_inv(P["rois"][0], torch.from_numpy(reg).float()), list(dims)).numpy()
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
    print(f"[golden] {tag}: rois={len(pc)} masks={len(masks)} killed={killing}")


def refused(g, key, yml, dims, n_img, **over):
    """Build the reference model of a switch combination and run one scene through it; store what it raised."""
    cfg = rh.load_cfg(yml, USE_IMAGES_GT=True, USE_MASK=True, **over)
    from lib.nets import backbones
    torch.manual_seed(0)
    try:
        net = getattr(backbones, cfg.NET)()
        net.init_modules()
        net.eval()
        data, boxes = synth.make_scene(404, dims)
        views = synth.make_views(404, dims, n_img, boxes, intrinsic=np.array(cfg.INTRINSIC, dtype=np.float32)) if n_img else None
        rh.reference_forward(net, cfg, data, views)
    except Exception as e:  # noqa: BLE001 -- the failure is the record
        g[key] = np.array(f"{type(e).__name__}: {e}".splitlines()[0])
        print(f"[golden] {key}: {g[key]}")
        return
    raise SystemExit(f"{key}: the reference ran this combination; support it and pin its outputs instead")


def run_loops(g):
    import make_golden_gt_rois as gtr
    import types
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
    cfg = rh.load_cfg(YML, USE_IMAGES=True, ONLY_IMAGES=True, USE_IMAGES_GT=True, USE_MASK=True)
    torch.manual_seed(0)
    net = build(cfg, weights(cfg))
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
    refused(g, "refused_suncg", "SUNCG/rpn_class_mask_5.yml", (40, 24, 40), 3, USE_IMAGES=True, ONLY_IMAGES=True)
    refused(g, "refused_no_images", YML, (32, 32, 32), 0, USE_IMAGES=False, ONLY_IMAGES=True)
    run_loops(g)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {len(g)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
