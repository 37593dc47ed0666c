"""ScanNet's instance annotations -> GT ids per mesh vertex, resolved once per segment (reference:
tools/scannet_benchmark/export_train_mesh_for_evaluation.py:39-98; lines cited per function).

ScanNet labels segments of the mesh, not vertices: `<scene>.aggregation.json` lists objects (`segGroups`: `objectId`, the
raw category `label`, `segments`) and `<scene>_vh_clean_2.0.010000.segs.json` gives each vertex's segment (`segIndices`).
The reference fills per-vertex arrays in Python loops.  Every vertex of a segment receives the same value, so here its rules
run once per segment into a table sorted by segment id, and sis3d_segment_gt_slots (csrc/eval.cu) spreads the table over
the vertices on the device (evaluate_predictions.segment_gt_slots).

The table reproduces the reference's last-writer-wins order:
- labels are written label by label in first-appearance order, instances object id by object id, in two separate passes,
  so a segment's label and its instance can come from different objects;
- `label_to_segs[label] = segs` keeps the first object's own list and later objects of that label extend it, so that
  object (while its id is not overwritten in object_id_to_segs) also owns, in the instance pass, the segments of every
  later object of its label.  This shows only when objects share segments or object ids repeat;
- an id is `label * 1000 + instance` in uint32 arithmetic, as the reference's uint32 arrays compute it; a label can map to
  0, which gives ids below 1000; a segment no object lists is 0.

Departures (the reference dies with KeyError in the first two cases): a segment the aggregation lists that is not in the
segs file, a raw category missing from the TSV map, an nyu40 id missing from the CSV map, a segment id beyond int32 in the
segs file and a negative segment id listed by the aggregation exit through utils.print_error, naming the scene and the key.
"""
from __future__ import annotations

import json
from typing import NamedTuple

import numpy as np

from . import utils

INT32 = np.iinfo(np.int32)


class SegmentGT(NamedTuple):
    """One scene's GT as sis3d_segment_gt_slots consumes it."""
    seg_index: np.ndarray  # int32 [n_vert]: each vertex's segment id (segIndices)
    seg_ids: np.ndarray    # int32 [n_seg]: the segments the aggregation lists, sorted ascending, unique
    seg_slot: np.ndarray   # int32 [n_seg]: each segment's slot, an index into slot_ids
    slot_ids: np.ndarray   # int64 [n_slot]: the distinct GT ids of the table and 0, sorted ascending
    seg_file: str


def read_aggregation(filename):
    """export_train_mesh_for_evaluation.py:39-55, list aliasing included: -> (object_id_to_segs, label_to_segs), object ids
    1-based."""
    object_id_to_segs, label_to_segs = {}, {}
    with open(filename) as f:
        data = json.load(f)
    for group in data["segGroups"]:
        object_id = group["objectId"] + 1
        label, segs = group["label"], group["segments"]
        object_id_to_segs[object_id] = segs
        if label in label_to_segs:
            label_to_segs[label].extend(segs)  # grows the first object's own list
        else:
            label_to_segs[label] = segs
    return object_id_to_segs, label_to_segs


def read_segmentation(filename, scene):
    """export_train_mesh_for_evaluation.py:58-70, inverted: the segment id of every vertex, int32 [n_vert]."""
    with open(filename) as f:
        seg = np.asarray(json.load(f)["segIndices"], np.int64).reshape(-1)
    if seg.size and (seg.min() < INT32.min or seg.max() > INT32.max):
        bad = seg[(seg < INT32.min) | (seg > INT32.max)][0]
        utils.print_error("%s: segment id %d in %s does not fit in int32" % (scene, bad, filename))
    return seg.astype(np.int32)


def segment_table(object_id_to_segs, label_to_segs, seg_index, label_map, label_map2, task, scene):
    """export_train_mesh_for_evaluation.py:79-94 per segment: -> (seg_ids int32 [n_seg] sorted, ids int64 [n_seg]), the GT
    id a `task` ('label' or 'instance') export writes for every vertex of each segment the aggregation lists."""
    present = set(np.unique(seg_index).tolist())
    seg_label = {}
    for label, segs in label_to_segs.items():
        if label not in label_map:
            utils.print_error("%s: raw category %r is not in the raw_category -> nyu40id label map" % (scene, label))
        if label_map[label] not in label_map2:
            utils.print_error("%s: nyu40id %r (raw category %r) is not in the nyu40id -> mappedIdConsecutive label map"
                              % (scene, label_map[label], label))
        label_id = label_map2[label_map[label]]
        for seg in segs:
            if seg not in present:
                utils.print_error("%s: segment %r of the aggregation has no vertex in the segmentation file" % (scene, seg))
            seg_label[seg] = label_id
    rows = sorted(seg_label)
    if rows and rows[0] < 0:
        utils.print_error("%s: negative segment id %d in the aggregation" % (scene, rows[0]))
    ids = np.array([seg_label[s] for s in rows], np.uint32)
    if task == "instance":
        seg_inst = {}
        for object_id, segs in object_id_to_segs.items():
            for seg in segs:  # every one of them is also in a label's list
                seg_inst[seg] = object_id
        ids = ids * 1000 + np.array([seg_inst.get(s, 0) for s in rows], np.uint32)
    elif task != "label":
        raise ValueError("task type must be 'label' or 'instance', not %r" % (task,))
    return np.array(rows, np.int32), ids.astype(np.int64)


def read_scene_gt(agg_file, seg_file, label_map, label_map2, task, scene):
    """One scene's annotations -> SegmentGT.  Slot s stands for slot_ids[s]; slot 0 is id 0."""
    object_id_to_segs, label_to_segs = read_aggregation(agg_file)
    seg_index = read_segmentation(seg_file, scene)
    seg_ids, ids = segment_table(object_id_to_segs, label_to_segs, seg_index, label_map, label_map2, task, scene)
    slot_ids = np.unique(np.concatenate([np.zeros(1, np.int64), ids]))
    return SegmentGT(seg_index, seg_ids, np.searchsorted(slot_ids, ids).astype(np.int32), slot_ids, seg_file)


def gt_ids_host(gt):
    """The per-vertex GT ids on the host (a numpy restatement of sis3d_segment_gt_slots, for tests and benchmarks)."""
    row = np.searchsorted(gt.seg_ids, gt.seg_index)
    row = np.minimum(row, max(len(gt.seg_ids) - 1, 0))
    hit = (len(gt.seg_ids) > 0) & (gt.seg_index >= 0)
    if len(gt.seg_ids):
        hit &= gt.seg_ids[row] == gt.seg_index
    slot = np.where(hit, gt.seg_slot[row] if len(gt.seg_ids) else 0, 0).astype(np.int32)
    return gt.slot_ids[slot], slot
