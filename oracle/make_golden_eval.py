"""oracle/make_golden_eval.py -- TEST INFRASTRUCTURE ONLY; runs ONLY in the build container (needs the reference tree).

Runs the reference's UNMODIFIED lib/utils/evaluation.py (DetectionMAP.evaluate / evaluate_mask / finalize / mAP / AP, under
oracle/ref_harness.install() plus one shim of its own: np.int -> int, removed in numpy 2) on seeded synthetic evaluation sets
and stores inputs and outputs in
tests/golden/eval_reference.npz, which pins lib/utils/evaluation.py and the sis3d_mask_overlap kernel
(tests/test_eval_map.py, tests/test_gpu_eval.py).

    python oracle/make_golden_eval.py

Sets: 0 is hand-made (IoU exactly at MAP_THRESH = 0.25 for boxes and masks, boxes sharing only a face, an empty predicted and
an empty GT mask on the same box (nan IoU), masks touching the far scene border, .5 box coordinates (round half to even),
a class predicted but absent from the GT, a scene without predictions, one prediction over several GT, confidence ties).
1 and 2 are random (several predictions per GT, wrong classes, false positives, confidence ties from a short list of
values; set 2 at MAP_THRESH = 0.5 with one 208x48x160 scene).

Layout (keys; k = set, s = scene): n_sets; k_n_class, k_thresh, k_n_scenes; inputs k_s_dims, k_s_pred_box (f32), k_s_pred_class,
k_s_pred_conf (f64), k_s_gt_box (f32), k_s_gt_class (f32), k_s_pred_bits / k_s_gt_bits (np.packbits of the masks, each C order
with the shape of its rounded box, back to back; predicted masks are float32 0/1 in the reference's driver, GT masks uint8);
outputs per scene and {box, mask}: k_s_{m}_iou (after `IoU[IoU < thresh] = 0`), k_s_{m}_tp / _fp (confidences of all classes
back to back), k_s_{m}_tp_n / _fp_n / _fn (per class); per set and {box, mask}: k_{m}_ap (nan for ignored classes),
k_{m}_map, k_{m}_ignore, k_{m}_summary (the printed lines).
"""
from __future__ import annotations

import os
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(_HERE), "tests", "golden", "eval_reference.npz")
CONFS = np.array([0.55, 0.6, 0.7, 0.8, 0.9, 0.95, 0.99])


def rbox(b):
    return np.rint(np.asarray(b, np.float64)).astype(np.int64)


def blob(rng, shape, p):
    return (rng.random(shape) < p).astype(np.uint8)


def handmade(rng):
    D = (16, 12, 16)
    scenes = []
    # A: exact-threshold overlaps, face-only contact, nan masks, border masks, half-integer coordinates
    gt_box = np.array([[0, 0, 0, 4, 4, 4, 1], [4, 0, 0, 8, 4, 4, 1], [10, 0, 10, 14, 4, 14, 2], [12, 8, 12, 16, 12, 16, 2]],
                      np.float32)
    gt_mask = [np.ones((4, 4, 4), np.uint8), blob(rng, (4, 4, 4), 0.7), np.zeros((4, 4, 4), np.uint8),
               blob(rng, (4, 4, 4), 0.8)]
    gt_mask[3][-1, -1, -1] = 1
    pred_box = np.array([[0, 0, 0, 4, 4, 1], [0, 0, 0, 4, 4, 2], [4, 0, 0, 8, 4, 4], [1, 1, 1, 5, 5, 5],
                         [10, 0, 10, 14, 4, 14], [11.5, 8, 12.5, 16, 12, 16], [12.5, 7.5, 11.5, 16, 12, 16]], np.float32)
    pred_class = np.array([1, 1, 1, 3, 2, 2, 2], np.int64)
    pred_conf = np.array([0.9, 0.9, 0.8, 0.7, 0.6, 0.6, 0.9], np.float64)
    full1 = np.zeros(D, np.uint8)
    full1[4:8, 0:4, 0:4] = gt_mask[1]
    pred_mask = [np.ones((4, 4, 1), np.float32), np.ones((4, 4, 2), np.float32), full1[4:8, 0:4, 0:4].astype(np.float32),
                 blob(rng, (4, 4, 4), 0.5).astype(np.float32), np.zeros((4, 4, 4), np.float32)]
    for b in pred_box[5:]:
        lo, hi = rbox(b[:3]), rbox(b[3:])
        pred_mask.append(blob(rng, tuple(hi - lo), 0.8).astype(np.float32))
    scenes.append((D, pred_box, pred_class, pred_conf, pred_mask, gt_box, gt_mask))
    # B: no predictions
    gt_box = np.array([[2, 2, 2, 6, 5, 7, 1], [8, 0, 8, 12, 3, 13, 4]], np.float32)
    scenes.append((D, np.zeros((0, 6), np.float32), np.zeros(0, np.int64), np.zeros(0, np.float64), [], gt_box,
                   [blob(rng, (4, 3, 5), 0.6), blob(rng, (4, 3, 5), 0.6)]))
    # C: one large prediction over three GT of its class, plus tied confidences (one TP, one FP)
    gt_box = np.array([[0, 0, 0, 3, 3, 3, 1], [3, 0, 0, 6, 3, 3, 1], [0, 3, 0, 3, 6, 3, 1]], np.float32)
    gt_mask = [np.ones((3, 3, 3), np.uint8) for _ in range(3)]
    pred_box = np.array([[0, 0, 0, 6, 6, 3], [0, 0, 0, 3, 3, 3], [0, 0, 0, 3, 3, 3]], np.float32)
    pred_mask = [np.ones((6, 6, 3), np.float32), np.ones((3, 3, 3), np.float32), np.ones((3, 3, 3), np.float32)]
    scenes.append((D, pred_box, np.array([1, 1, 1], np.int64), np.array([0.8, 0.8, 0.8]), pred_mask, gt_box, gt_mask))
    return 5, 0.25, scenes


def random_scene(rng, D, n_gt, n_class, present):
    D = np.asarray(D)
    gt_box, gt_mask = [], []
    for _ in range(n_gt):
        ext = rng.integers(2, np.minimum(13, D // 2) + 1)
        lo = rng.integers(0, D - ext + 1)
        if rng.random() < 0.15:  # on the far border
            lo[rng.integers(0, 3)] = 0
            lo = np.where(rng.random(3) < 0.3, D - ext, lo)
        gt_box.append(np.concatenate([lo, lo + ext, [rng.choice(present)]]).astype(np.float32))
        gt_mask.append(blob(rng, tuple(ext), rng.choice([0.5, 0.8, 0.95])))
    gt_box = np.array(gt_box, np.float32)
    full = np.zeros((n_gt,) + tuple(D), np.uint8)
    for j in range(n_gt):
        lo, hi = gt_box[j, :3].astype(int), gt_box[j, 3:6].astype(int)
        full[j, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = gt_mask[j]
    pb, pc, pm = [], [], []
    for j in range(n_gt):
        for _ in range(rng.integers(0, 4)):  # several predictions per GT
            b = gt_box[j, :6] + rng.integers(-4, 5, 6) * 0.5
            b[:3], b[3:] = np.clip(b[:3], 0, D), np.clip(b[3:], 0, D)
            lo, hi = rbox(b[:3]), rbox(b[3:])
            if (hi <= lo).any():
                continue
            m = full[j, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] ^ blob(rng, tuple(hi - lo), 0.1)
            pb.append(b)
            pc.append(int(gt_box[j, 6]) if rng.random() < 0.8 else int(rng.integers(1, n_class)))
            pm.append(m.astype(np.float32))
    for _ in range(rng.integers(1, 4)):  # false positives, some of a class without GT
        ext = rng.integers(2, 8, 3)
        lo = rng.integers(0, D - ext + 1)
        pb.append(np.concatenate([lo, lo + ext]).astype(np.float32))
        pc.append(int(rng.integers(1, n_class)))
        pm.append(blob(rng, tuple(ext), 0.5).astype(np.float32))
    pred_box = np.array(pb, np.float32).reshape(-1, 6)
    pred_conf = rng.choice(CONFS, len(pb)).astype(np.float64)
    return tuple(int(v) for v in D), pred_box, np.array(pc, np.int64), pred_conf, pm, gt_box, gt_mask


def random_set(rng, n_class, thresh, dims, n_gts):
    present = rng.choice(np.arange(1, n_class), size=max(1, (n_class - 1) * 2 // 3), replace=False)
    return n_class, thresh, [random_scene(rng, D, g, n_class, present) for D, g in zip(dims, n_gts)]


def pack(masks):
    flat = [np.ascontiguousarray(m).reshape(-1) != 0 for m in masks]
    return np.packbits(np.concatenate(flat) if flat else np.zeros(0, bool))


def run_reference(n_class, thresh, scenes, k, out):
    from lib.utils.evaluation import DetectionMAP as RefMAP  # the reference's module (ref_harness puts its root first)
    rec = {}
    orig_iou, orig_iou_mask, orig_tp = RefMAP.compute_IoU, RefMAP.compute_IoU_mask, RefMAP.compute_TP_FP_FN

    def grab(name, f):
        def g(*a):
            r = f(*a)
            rec[name] = r  # thresholded in place by the caller
            return r
        return staticmethod(g)

    def grab_tp(pred_cls, gt_cls, pred_conf, IoU, c):
        r = orig_tp(pred_cls, gt_cls, pred_conf, IoU, c)
        rec.setdefault("tp", []).append(r)
        return r

    RefMAP.compute_IoU, RefMAP.compute_IoU_mask = grab("iou", orig_iou), grab("iou", orig_iou_mask)
    RefMAP.compute_TP_FP_FN = staticmethod(grab_tp)
    box = RefMAP(n_class, ignore_class=[0], overlap_threshold=thresh)
    mask = RefMAP(n_class, ignore_class=[0], overlap_threshold=thresh)
    try:
        for s, (D, pb, pc, pconf, pm, gb, gm) in enumerate(scenes):
            key = f"{k}_{s}_"
            out.update({key + "dims": np.array(D, np.int64), key + "pred_box": pb, key + "pred_class": pc,
                        key + "pred_conf": pconf, key + "gt_box": gb[:, :6].copy(), key + "gt_class": gb[:, 6].copy(),
                        key + "pred_bits": pack(pm), key + "gt_bits": pack(gm)})
            for name, run in (("box", lambda: box.evaluate(pb, pc, pconf, gb[:, :6], gb[:, 6])),
                              ("mask", lambda: mask.evaluate_mask(pb, pc, pconf, pm, gb[:, :6], gb[:, 6], gm, list(D)))):
                rec.clear()
                run()
                out[key + name + "_iou"] = np.asarray(rec["iou"]).reshape(len(pb), len(gb))  # [0, 6] without predictions
                tps = rec["tp"]
                out[key + name + "_tp"] = np.array([float(v) for t in tps for v in t[0]], np.float64)
                out[key + name + "_fp"] = np.array([float(v) for t in tps for v in t[1]], np.float64)
                out[key + name + "_tp_n"] = np.array([len(t[0]) for t in tps], np.int64)
                out[key + name + "_fp_n"] = np.array([len(t[1]) for t in tps], np.int64)
                out[key + name + "_fn"] = np.array([int(t[2]) for t in tps], np.int64)
    finally:
        RefMAP.compute_IoU, RefMAP.compute_IoU_mask, RefMAP.compute_TP_FP_FN = \
            staticmethod(orig_iou), staticmethod(orig_iou_mask), staticmethod(orig_tp)
    for name, title, m in (("box", "CLASSIFICATION", box), ("mask", "mask", mask)):
        m.finalize()  # printed as SolverWrapper.test does (lib/model/trainval.py:929-941)
        lines = ["mAP of {}: {}".format(title, m.mAP())]
        lines += ["class {}: {}".format(c, m.AP(c)) for c in range(n_class) if c not in m.ignore_class]
        out[f"{k}_{name}_ap"] = np.array([np.nan if c in m.ignore_class else m.AP(c) for c in range(n_class)], np.float64)
        out[f"{k}_{name}_map"] = np.float64(m.mAP())
        out[f"{k}_{name}_ignore"] = np.array(m.ignore_class, np.int64)
        out[f"{k}_{name}_summary"] = np.array("\n".join(lines))
    out[f"{k}_n_class"], out[f"{k}_thresh"], out[f"{k}_n_scenes"] = np.int64(n_class), np.float64(thresh), np.int64(len(scenes))


def main():
    sys.path.insert(0, os.path.dirname(_HERE))
    from oracle import ref_harness
    ref_harness.install()
    # numpy 2 removed the `np.int` alias the reference's evaluator casts class ids with (evaluation.py:41-42, 74-75); it
    # meant the builtin int, so it is restored for this process only, next to the harness's other shims
    if "int" not in np.__dict__:
        np.int = int
    rng = np.random.default_rng(20261015)
    sets = [handmade(rng),
            random_set(rng, 8, 0.25, [(32, 16, 32), (40, 24, 32), (48, 24, 40), (32, 16, 32), (36, 20, 28), (44, 24, 44)],
                       [4, 6, 8, 3, 5, 7]),
            random_set(rng, 19, 0.5, [(96, 48, 96), (96, 48, 96), (208, 48, 160)], [10, 12, 14])]
    out = {"n_sets": np.int64(len(sets))}
    for k, (n_class, thresh, scenes) in enumerate(sets):
        run_reference(n_class, thresh, scenes, k, out)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
