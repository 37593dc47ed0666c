"""Box and mask mAP of test mode under the reference's names: `DetectionMAP` and `APAccumulator` of
lib/utils/evaluation.py (reference lines cited per method; paths relative to the reference root).

Results equal the reference's for the same inputs, bit for bit: the same float32 box arithmetic, the same greedy matching in
the same `np.argsort` order, the same accumulator arithmetic.  What differs is how mask overlaps are counted.  The reference
expands every mask into a full-scene uint8 volume and runs two full-volume passes per (prediction, GT) pair
(evaluation.py:144-179, 293-307).  Here the masks stay packed at their boxes, and one launch of sis3d_mask_overlap
(csrc/eval.cu) counts the voxels of each mask and of each intersecting pair; the IoU follows on the host from those exact
integer counts.  Masks are binary (0/1, as the dataset and the mask stage produce them).

One departure: the reference raises (np.max of an empty array, evaluation.py:114) when a scene has predictions but no GT box;
here every such prediction counts as a false positive.
"""
from __future__ import annotations

import contextlib
import ctypes as C

import numpy as np
import torch

from lib import _sis3d as S


class DetectionMAP:
    def __init__(self, n_class, pr_samples=11, overlap_threshold=0.5, ignore_class=None, output_dir=None):
        """evaluation.py:14-27.  `ignore_class` is extended in place by finalize() with the classes that have no GT."""
        self.n_class = n_class
        self.overlap_threshold = overlap_threshold
        self.pr_scale = np.linspace(0, 1, pr_samples)
        self.ignore_class = [] if ignore_class is None else ignore_class
        self.output_dir = output_dir
        self.reset_accumulators()

    def reset_accumulators(self):
        self.total_accumulators = [APAccumulator() for _ in range(self.n_class)]

    # ---------------------------------------------------------------------------------------- per scene
    def evaluate(self, pred_bb, pred_classes, pred_conf, gt_bb, gt_classes):
        """Box mAP of one scene (evaluation.py:62-85): boxes [n, 6] = min xyz, max xyz."""
        if np.ndim(pred_bb) != 2:
            raise ValueError("pred_bb must be [n_pred, 6]")
        self._accumulate(pred_classes, pred_conf, box_iou(pred_bb, gt_bb), gt_classes)

    def evaluate_mask(self, pred_box, pred_class, pred_conf, pred_mask, gt_box, gt_class, gt_mask, scene_info=(64, 64, 32)):
        """Mask mAP of one scene from host mask lists (evaluation.py:40-60): mask i has the shape of box i rounded to voxels
        and is placed at its rounded lo corner of the [scene_info[:3]] scene.  Packs both sides and makes one H2D copy."""
        dims = tuple(int(v) for v in scene_info[:3])
        pb, po, pbox = pack_masks(pred_mask, pred_box, dims, "predicted")
        gb, go, gbox = pack_masks(gt_mask, gt_box, dims, "GT")
        self.evaluate_overlaps(pred_class, pred_conf, launch_mask_overlap(pb, po, pbox, gb, go, gbox).result(), gt_class)

    def evaluate_overlaps(self, pred_class, pred_conf, overlaps, gt_class):
        """Mask mAP of one scene from the counts of launch_mask_overlap (the form the test driver uses: its predicted masks
        are already on the device)."""
        self._accumulate(pred_class, pred_conf, mask_iou(*overlaps), gt_class)

    def _accumulate(self, pred_class, pred_conf, iou, gt_class):
        """evaluation.py:49-60 / 79-85: threshold the IoU, then greedy matching class by class."""
        pred_class = np.asarray(pred_class).astype(np.int64)
        gt_class = np.asarray(gt_class).astype(np.int64)
        iou[iou < self.overlap_threshold] = 0
        if pred_class.shape[0] and pred_class[0] == -1:  # class-agnostic predictions are matched in every class
            classes = range(self.n_class)
        else:  # a class with neither predictions nor GT adds nothing
            classes = np.union1d(pred_class, gt_class)
        for i in classes:
            if 0 <= i < self.n_class:
                TP, FP, FN = DetectionMAP.compute_TP_FP_FN(pred_class, gt_class, pred_conf, iou, int(i))
                acc = self.total_accumulators[i]
                acc.inc_predictions(TP, FP)
                acc.inc_not_predicted(FN)

    @staticmethod
    def compute_TP_FP_FN(pred_cls, gt_cls, pred_conf, IoU, class_index):
        """evaluation.py:182-226.  Predictions of the class are visited in `np.argsort(conf)[::-1]` order (numpy's default
        sort kind: tie order changes AP); each takes the unmatched GT of the class with the largest nonzero IoU, the first
        one on ties (the reference's strict `>`); a nan IoU (two empty masks) never matches."""
        gt_sel = gt_cls == class_index
        FN = int(np.count_nonzero(gt_sel))
        if pred_cls.shape[0] == 0:
            return [], [], FN
        if pred_cls[0] == -1:
            iou = IoU[:, gt_sel]
            order = np.argsort(pred_conf[:])[::-1]
        else:
            sel = pred_cls == class_index
            iou = IoU[sel][:, gt_sel]
            order = np.argsort(pred_conf[sel])[::-1]
        # matchable entries are the nonzero, non-nan ones: after thresholding with a positive MAP_THRESH they are > 0
        cand = np.where((iou != 0) & ~np.isnan(iou), iou, -1)
        free = np.ones(iou.shape[1], dtype=bool)
        TP, FP = [], []
        for i in order:
            row = np.where(free, cand[i], -1)
            j = int(np.argmax(row)) if row.size else 0
            # The reference appends pred_conf[i] with i indexing the class-filtered subset but reads the UNFILTERED array
            # (evaluation.py:221/225).  That is a bug, but it decides the published numbers, so it is reproduced here.
            if row.size and row[j] > -1:
                TP.append(pred_conf[i])
                free[j] = False
                FN -= 1
            else:
                FP.append(pred_conf[i])
        return TP, FP, FN

    # ---------------------------------------------------------------------------------------- summary
    def compute_ap(self, precisions, recalls):
        """evaluation.py:229-240."""
        previous_recall = 0
        average_precision = 0
        for precision, recall in zip(precisions[::-1], recalls[::-1]):
            average_precision += precision * (recall - previous_recall)
            previous_recall = recall
        return average_precision

    def compute_precision_recall_(self, class_index, interpolated=True):
        """evaluation.py:242-261: precision/recall at the pr_scale recall levels, highest level first; interpolated =
        running maximum of the precision from the highest level down."""
        acc = self.total_accumulators[class_index]
        pr = [acc.precision_recall(t) for t in self.pr_scale][::-1]
        precisions, recalls = [p for p, _ in pr], [r for _, r in pr]
        if interpolated:
            running = []
            for p in precisions:
                running.append(max(p, max(running)) if running else max(p, 0))
            precisions = running
        return precisions, recalls

    def mAP(self):
        """evaluation.py:263-275: mean AP over the classes not ignored (0 when every class is)."""
        aps = [self.AP(i) for i in range(self.n_class) if i not in self.ignore_class]
        return sum(aps) / len(aps) if aps else 0

    def AP(self, idx):
        precisions, recalls = self.compute_precision_recall_(idx, True)
        return self.compute_ap(precisions, recalls)

    def finalize(self):
        """evaluation.py:287-291: rank each class's predictions; classes without GT join ignore_class."""
        for i, acc in enumerate(self.total_accumulators):
            acc.ranking()
            if acc.if_ignore() and i not in self.ignore_class:
                self.ignore_class.append(i)


class APAccumulator:
    """True/false positives (with their confidences) and missed GT of one class (evaluation.py:309-370)."""

    def __init__(self):
        self.predictions = []  # [conf, 1.0 (TP) | 0.0 (FP)]; an ndarray after ranking()
        self.FN = 0
        self.TP = 0

    def inc_predictions(self, TP, FP):
        self.predictions.extend([tp, 1.0] for tp in TP)
        self.TP += len(TP)
        self.predictions.extend([fp, 0.0] for fp in FP)

    def inc_not_predicted(self, value=1):
        self.FN += value

    def ranking(self):
        """Descending confidence: np.argsort (default kind) of the stacked rows, reversed, as evaluation.py:334-340."""
        if len(self.predictions) != 0:
            self.predictions = np.stack(self.predictions, 0)
            self.predictions = self.predictions[np.argsort(self.predictions[:, 0])[::-1]]
        else:
            self.predictions = np.empty(shape=(0, 0))

    def if_ignore(self):
        return self.TP + self.FN == 0

    def precision_recall(self, thresh):
        """evaluation.py:349-370: (precision, recall) at the first ranked prediction whose recall reaches `thresh`;
        (0, 0) at thresh 0 and (0, 1) when the recall never reaches it.  Cumulative counts are exact small integers, so
        the float64 divisions below equal the reference's running Python-float divisions."""
        if thresh == 0.0:
            return (0.0, 0.0)
        n = self.predictions.shape[0]
        if n == 0:
            return (0.0, 1.0)
        total_gt = self.TP + self.FN
        if total_gt == 0:
            raise ZeroDivisionError("precision_recall of a class without GT (finalize() ignores such classes)")
        tp = np.cumsum(self.predictions[:, 1] == 1.0).astype(np.float64)
        recall = tp / float(total_gt)
        hit = np.flatnonzero(recall >= thresh)
        if hit.size == 0:
            return (0.0, 1.0)
        k = int(hit[0])
        return float(tp[k] / float(k + 1)), float(recall[k])


def summary_lines(name, dmap, num_classes):
    """The summary test mode prints for one DetectionMAP (reference trainval.py:929-941); call after finalize()."""
    lines = ["mAP of {}: {}".format(name, dmap.mAP())]
    lines += ["class {}: {}".format(c, dmap.AP(c)) for c in range(num_classes) if c not in dmap.ignore_class]
    return lines


# -------------------------------------------------------------------------------------------- IoU
def box_iou(pred, gt):
    """[n_pred, n_gt] IoU of corner boxes in the reference's operation order and dtype (evaluation.py:98-141).
    The reference clips the per-axis overlap to [0, max(overlap)].  When that max is >= 0 this is a clip at 0; when it is
    negative (no pair overlaps at all) every IoU it produces is negative for boxes of positive volume, and only values
    >= MAP_THRESH > 0 are ever used.  So a clip at 0 gives the same thresholded matrix."""
    pred, gt = np.asarray(pred), np.asarray(gt)
    if pred.shape[0] == 0:  # the reference returns an unused [0, 6] array here
        return np.zeros((0, gt.shape[0]))
    a, b = pred[:, np.newaxis, :], gt[np.newaxis, :, :]
    d = np.minimum(a[:, :, 3:], b[:, :, 3:]) - np.maximum(a[:, :, :3], b[:, :, :3])
    d = np.maximum(d, 0)
    inter = d[:, :, 0] * d[:, :, 1] * d[:, :, 2]
    area_a = (pred[:, 3] - pred[:, 0]) * (pred[:, 4] - pred[:, 1]) * (pred[:, 5] - pred[:, 2])
    area_b = (gt[:, 3] - gt[:, 0]) * (gt[:, 4] - gt[:, 1]) * (gt[:, 5] - gt[:, 2])
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / (area_a[:, np.newaxis] + area_b[np.newaxis, :] - inter)


def mask_iou(pred_count, gt_count, inter):
    """float64 IoU from exact voxel counts: inter / (|a| + |b| - inter), which equals the reference's
    inter[i, j] / sum(mask_a[i] + mask_b[j] > 0) (evaluation.py:157-163) bit for bit, nan when both masks are empty."""
    union = pred_count[:, np.newaxis] + gt_count[np.newaxis, :] - inter
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter.astype(np.float64) / union


# -------------------------------------------------------------------------------------------- overlap counts
def pack_masks(masks, boxes, dims, what="GT"):
    """Host masks -> (bits uint8 [sum of sizes], offsets int64 [n], boxes int32 [n, 6] lo | hi) in the layout
    sis3d_mask_overlap reads: each mask C order at int(round(box)) (evaluation.py:293-307).  Raises ValueError for a mask
    whose shape is not its box's extent or whose box is not inside [0, dims]."""
    boxes = np.asarray(boxes, dtype=np.float64).reshape(-1, 6)
    if len(masks) != boxes.shape[0]:
        raise ValueError(f"{len(masks)} {what} masks for {boxes.shape[0]} boxes")
    ib = np.rint(boxes).astype(np.int64)  # Python's round(): half to even
    parts, offs, o = [], np.zeros(len(masks), np.int64), 0
    for i, m in enumerate(masks):
        m = np.asarray(m)
        lo, hi = ib[i, :3], ib[i, 3:]
        if m.shape != tuple(int(v) for v in hi - lo):
            raise ValueError(f"{what} mask {i}: shape {m.shape} is not the extent {tuple(int(v) for v in hi - lo)} of its box")
        if (lo < 0).any() or (hi > np.asarray(dims)).any():
            raise ValueError(f"{what} mask {i}: box {ib[i].tolist()} is not inside the scene [0, {list(dims)}]")
        parts.append(np.ascontiguousarray(m).astype(np.uint8, copy=False).reshape(-1))
        offs[i] = o
        o += m.size
    bits = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    return bits, offs, ib.astype(np.int32)


def box_pairs(pred_box, gt_box):
    """int32 [n_pairs, 2] (prediction, GT) index pairs whose integer boxes share at least one voxel."""
    lo = np.maximum(pred_box[:, np.newaxis, :3], gt_box[np.newaxis, :, :3])
    hi = np.minimum(pred_box[:, np.newaxis, 3:], gt_box[np.newaxis, :, 3:])
    return np.argwhere((hi > lo).all(axis=2)).astype(np.int32).reshape(-1, 2)


class MaskOverlap:
    """Counts of one sis3d_mask_overlap launch; result() waits for them."""

    def __init__(self, n_pred, n_gt, pairs, counts, event, keep):
        self.n_pred, self.n_gt, self.pairs, self.counts, self.event, self._keep = n_pred, n_gt, pairs, counts, event, keep

    def result(self):
        """-> pred_count int64[n_pred], gt_count int64[n_gt], inter int64[n_pred, n_gt]."""
        if self.event is not None:
            self.event.synchronize()
        c = self.counts.numpy()
        if (c < 0).any():
            raise S.Sis3dError("sis3d_mask_overlap: pair index out of range")
        inter = np.zeros((self.n_pred, self.n_gt), np.int64)
        inter[self.pairs[:, 0], self.pairs[:, 1]] = c[self.n_pred + self.n_gt:]
        self._keep = None
        return c[:self.n_pred].copy(), c[self.n_pred:self.n_pred + self.n_gt].copy(), inter


_streams = {}


def launch_mask_overlap(pred_bits, pred_offs, pred_box, gt_bits, gt_offs, gt_box, device=None):
    """Queue the voxel counts of one scene's masks (layout of pack_masks; boxes int [n, 6] lo | hi).
    pred_bits: a uint8 tensor already on the device (the mask stage's bits; it must be complete, as it is for a scene the
    scene loop has yielded), or a host array that travels in the same H2D copy as the GT side.  Everything else is host data:
    one pinned H2D copy, one kernel and one D2H copy on a side stream, so a caller can collect the counts of one scene while
    the next one is being computed."""
    pred_box = np.ascontiguousarray(pred_box, dtype=np.int32).reshape(-1, 6)
    gt_box = np.ascontiguousarray(gt_box, dtype=np.int32).reshape(-1, 6)
    n_pred, n_gt = pred_box.shape[0], gt_box.shape[0]
    pairs = box_pairs(pred_box, gt_box)
    host_pred = not torch.is_tensor(pred_bits)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if host_pred and torch.cuda.is_available() else \
            (torch.device("cpu") if host_pred else pred_bits.device)
    sections = [np.asarray(pred_offs, np.int64)[:n_pred], np.asarray(gt_offs, np.int64)[:n_gt], pred_box, gt_box, pairs,
                np.asarray(gt_bits, np.uint8)] + ([np.asarray(pred_bits, np.uint8)] if host_pred else [])
    starts, o = [], 0
    for a in sections:
        o = (o + 7) // 8 * 8
        starts.append(o)
        o += a.nbytes
    cuda = device.type == "cuda"
    blob = torch.empty(max(o, 8), dtype=torch.uint8, pin_memory=cuda)
    bn = blob.numpy()
    for a, s in zip(sections, starts):
        bn[s:s + a.nbytes] = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    n_out = n_pred + n_gt + pairs.shape[0]
    stream = _streams.get(device) if cuda else None
    if cuda and stream is None:
        stream = _streams[device] = torch.cuda.Stream(device)
    with torch.cuda.stream(stream) if cuda else contextlib.nullcontext():
        dblob = blob.to(device, non_blocking=True)
        counts = torch.empty(max(n_out, 1), dtype=torch.int64, device=device)
        view = lambda k: dblob[starts[k]:]
        pb = view(6) if host_pred else pred_bits
        if cuda and not host_pred:
            pred_bits.record_stream(stream)
        h = C.c_void_p(stream.cuda_stream) if cuda else S.stream()
        S.check(S.lib.sis3d_mask_overlap(S.ptr(pb), S.ptr(view(0)), S.ptr(view(2)), n_pred, S.ptr(view(5)), S.ptr(view(1)),
                                         S.ptr(view(3)), n_gt, S.ptr(view(4)), int(pairs.shape[0]), S.ptr(counts),
                                         S.ptr(counts[n_pred:]), S.ptr(counts[n_pred + n_gt:]), h), "mask_overlap")
        event = None
        if cuda:
            out = torch.empty(counts.shape, dtype=torch.int64, pin_memory=True)
            out.copy_(counts, non_blocking=True)
            event = torch.cuda.Event()
            event.record(stream)
        else:
            out = counts
    return MaskOverlap(n_pred, n_gt, pairs, out[:n_out], event, (blob, dblob, counts, pred_bits))

