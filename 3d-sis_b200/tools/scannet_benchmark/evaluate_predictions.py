"""ScanNet instance AP straight from benchmark-mode result folders: vox2mesh.py followed by evaluate_semantic_instance.py,
without the per-vertex text files.

    python evaluate_predictions.py --pred_dir RESULTS --scan_path SCANS --frames FRAMES --gt_path GT [--output_file FILE]
    python evaluate_predictions.py --pred_dir RESULTS --scan_path SCANS --frames FRAMES --label_map_file TSV
        --label_map_file2 CSV [--output_file FILE]

For every result folder `<scene>` of `pred_dir` that has a mesh `<scan_path>/<scene>/<scene>_vh_clean_2.ply` (the folders
vox2mesh.py exports), with `<frames>/<scene>/world2grid.txt` and the GT ids `<gt_path>/<scene>.txt`, the scene's inputs are
uploaded in one copy and two kernels of libsis3d (csrc/eval.cu) run:
- sis3d_instance_paint: the owner of each voxel of the kept boxes' extent, i.e. the first box whose mask covers it, as
  vox2mesh.paint_instances paints its canvas;
- sis3d_vertex_instance_overlap: each vertex's voxel (or first owned neighbour, as vox2mesh.vertex_labels) and, per box,
  the number of its vertices carrying each GT id, plus the box's first vertex.
One histogram comes back.  Each box's instance id, class and confidence are then decoded from its painted float64 value by
export's expressions; boxes whose instance ids collide merge as export's dict merges them, and instances are ordered by first
vertex as export writes them.  The counts go into evaluate_semantic_instance.assign_instances and the rest of that module,
so the table printed on stdout and the CSV are byte for byte what the two-step file route produces.

Without --gt_path (then --label_map_file and --label_map_file2 are required), each scene's GT comes from ScanNet's
annotations, `<scan_path>/<scene>/<scene>.aggregation.json` and `<scene>_vh_clean_2.0.010000.segs.json`, as
export_train_mesh_for_evaluation.py --type instance would write it: annotations.py builds the per-segment table on the
host, the segment index and table travel in the same upload, and sis3d_segment_gt_slots gives every vertex its GT slot on
the device for the overlap kernel; the per-slot vertex counts come back with the histogram.

A scene with no instances is still evaluated (its GT count as false negatives).  A result folder without a GT file (or
without its annotation files) is the evaluator's exit-2 error.  There is no CPU path: without a CUDA device the launch
raises.
"""
from __future__ import annotations

import argparse
import os
import pickle
import sys

import numpy as np
import torch

if __package__:
    from . import evaluate_semantic_instance as E
    from . import annotations, utils, vox2mesh
else:  # run as a script
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
    from tools.scannet_benchmark import evaluate_semantic_instance as E
    from tools.scannet_benchmark import annotations, utils, vox2mesh

from lib import _sis3d as S

NO_VERTEX = np.iinfo(np.int32).max  # first_vertex of a box no vertex takes


# ------------------------------------------------------------------------------------------------------------ host side
def read_result_folder(pred_folder):
    """Kept boxes, classes, confidences and masks of one result folder, in vox2mesh.load_pred's order (mask b belongs to
    kept box b)."""
    pred_box = np.load(os.path.join(pred_folder, "pred_box.npy"))[:, :6]
    pred_class = np.load(os.path.join(pred_folder, "pred_class.npy"))
    pred_conf = np.load(os.path.join(pred_folder, "pred_conf.npy"))
    with open(os.path.join(pred_folder, "pred_mask"), "rb") as f:
        pred_mask = pickle.load(f)
    with open(os.path.join(pred_folder, "pred_mask_index"), "rb") as f:
        index = np.asarray(pickle.load(f))
    if index.size == 0:
        index = index.astype(np.int64)
    return pred_box[index], pred_class[index], pred_conf[index], pred_mask


def box_values(pred_class, pred_conf):
    """float64 value each box paints (vox2mesh.paint_instances: box_index*100 + class + conf - 0.01, the same expression)."""
    return np.array([b * 100 + pred_class[b] + pred_conf[b] - 0.01 for b in range(len(pred_class))], np.float64)


def pack_boxes(pred_box, values, pred_mask, dims=vox2mesh.SCENE_DIMS):
    """Masks -> (bits uint8, offs int64 [n], box int32 [n, 6] lo | hi, owner-volume lo int [3], extent int [3]) with
    vox2mesh.paint_instances' rules: corners rounded half to even; an empty box is skipped; a box leaving the canvas or a mask
    smaller than its box raises IndexError; a larger mask is cropped to the box; a voxel is set where the mask is != 0.  A
    box whose value is 0.0 paints nothing (its row is left empty).  The owner volume spans the painting boxes."""
    n = len(pred_box)
    boxes = np.asarray(pred_box, np.float64).reshape(-1, 6)
    lo_all, hi_all = np.rint(boxes[:, :3]).astype(np.int64), np.rint(boxes[:, 3:6]).astype(np.int64)
    ibox, offs, parts, o = np.zeros((n, 6), np.int32), np.zeros(n, np.int64), [], 0
    for b in range(n):
        (x0, y0, z0), (x1, y1, z1) = lo_all[b], hi_all[b]
        if x1 <= x0 or y1 <= y0 or z1 <= z0:
            continue
        if min(x0, y0, z0) < 0 or x1 > dims[0] or y1 > dims[1] or z1 > dims[2]:
            raise IndexError(f"box {b} leaves the {dims} volume")
        m = np.asarray(pred_mask[b])[:x1 - x0, :y1 - y0, :z1 - z0]
        if m.shape != (x1 - x0, y1 - y0, z1 - z0):
            raise IndexError(f"mask {b} is smaller than its box")
        if values[b] == 0:
            continue
        parts.append(np.ascontiguousarray(m != 0).view(np.uint8).reshape(-1))
        ibox[b] = (x0, y0, z0, x1, y1, z1)
        offs[b] = o
        o += parts[-1].size
    bits = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    painted = (ibox[:, 3:] > ibox[:, :3]).all(axis=1)
    if painted.any():
        lo, hi = ibox[painted, :3].min(axis=0), ibox[painted, 3:].max(axis=0)
    else:
        lo, hi = np.zeros(3, np.int64), np.zeros(3, np.int64)
    return bits, offs, ibox, lo.astype(np.int64), (hi - lo).astype(np.int64)


# ------------------------------------------------------------------------------------------------------------ device side
def _upload(sections, device):
    """One H2D copy of numpy arrays packed at 16-byte aligned offsets -> (device, views of each section's start)."""
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    starts, o = [], 0
    for a in sections:
        o = (o + 15) // 16 * 16
        starts.append(o)
        o += a.nbytes
    blob = torch.empty(max(o, 16), dtype=torch.uint8, pin_memory=device.type == "cuda")
    bn = blob.numpy()
    for a, s in zip(sections, starts):
        bn[s:s + a.nbytes] = a.reshape(-1).view(np.uint8)
    dblob = blob.to(device, non_blocking=True)
    return device, [dblob[s:] for s in starts]


def _segment_gt_slots(views, n_vert, gt, gt_slot, slot_count, h):
    S.check(S.lib.sis3d_segment_gt_slots(S.ptr(views[0]), n_vert, S.ptr(views[1]), S.ptr(views[2]), len(gt.seg_ids),
                                         len(gt.slot_ids), S.ptr(gt_slot), S.ptr(slot_count), h), "segment_gt_slots")


def _segment_sections(gt):
    return [np.ascontiguousarray(gt.seg_index, np.int32), np.ascontiguousarray(gt.seg_ids, np.int32),
            np.ascontiguousarray(gt.seg_slot, np.int32)]


def segment_gt_slots(gt, device=None):
    """sis3d_segment_gt_slots on one scene's annotations.SegmentGT: one H2D copy, one D2H copy.
    -> (gt_slot int32 [n_vert], slot_count int64 [n_slot]); the GT id of vertex v is gt.slot_ids[gt_slot[v]]."""
    n_vert, n_slot = len(gt.seg_index), len(gt.slot_ids)
    device, views = _upload(_segment_sections(gt), device)
    cuda = device.type == "cuda"
    res = torch.empty(max(n_slot + (n_vert + 1) // 2, 1), dtype=torch.int64, device=device)
    slot_count, gt_slot = res[:n_slot], res[n_slot:].view(torch.int32)
    _segment_gt_slots(views, n_vert, gt, gt_slot, slot_count, S.stream() if cuda else None)
    out = res.cpu().numpy() if cuda else res.numpy()
    return out[n_slot:].view(np.int32)[:n_vert].copy(), out[:n_slot].copy()


def vertex_instance_overlap(verts, world2grid, gt_slot, n_slot, bits, offs, ibox, lo, ext, dims=vox2mesh.SCENE_DIMS,
                            want_vertex_box=False, device=None, segment_gt=None):
    """Both kernels on one scene: one H2D copy of every input, one D2H copy of the results.
    -> (hist int64 [n_box, n_slot], first_vertex int32 [n_box], vertex_box int32 [n_vert] or None).

    With `segment_gt` (an annotations.SegmentGT), `gt_slot` and `n_slot` are ignored: the segment index and table travel
    in the same copy, sis3d_segment_gt_slots computes the slots on the device for the overlap kernel, and the result gains
    a fourth member, slot_count int64 [len(segment_gt.slot_ids)], which comes back in the same D2H copy."""
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    n_vert, n_box = verts.shape[0], ibox.shape[0]
    seg = segment_gt is not None
    if seg:
        n_slot = len(segment_gt.slot_ids)
        gt_slot = np.zeros(0, np.int32)
    sections = [np.ascontiguousarray(world2grid, np.float64).reshape(16), verts, np.ascontiguousarray(gt_slot, np.int32),
                np.ascontiguousarray(offs, np.int64), np.ascontiguousarray(ibox, np.int32), np.ascontiguousarray(bits, np.uint8)]
    device, view = _upload(sections + (_segment_sections(segment_gt) if seg else []), device)
    cuda = device.type == "cuda"
    n_hist = n_box * n_slot
    n_owner = int(np.prod(ext))
    n_res = n_hist + n_box + (n_vert if want_vertex_box else 0) + (n_slot if seg else 0)
    owner = torch.empty(max(n_owner, 1), dtype=torch.int32, device=device)
    res = torch.empty(max(n_res, 1), dtype=torch.int64, device=device)
    first = res[n_hist:n_hist + n_box].view(torch.int32)  # int32 slots inside the int64 result: one D2H copy for all
    vbox = res[n_hist + n_box:n_hist + n_box + n_vert].view(torch.int32) if want_vertex_box else None
    h = S.stream() if cuda else None  # host tensors: S.ptr raises (no CPU path)
    slots = view[2]
    if seg:
        slots = torch.empty(max(n_vert, 1), dtype=torch.int32, device=device)
        _segment_gt_slots(view[6:9], n_vert, segment_gt, slots, res[n_res - n_slot:n_res], h)
    S.check(S.lib.sis3d_instance_paint(S.ptr(view[5]), S.ptr(view[3]), S.ptr(view[4]), n_box, int(lo[0]), int(lo[1]),
                                       int(lo[2]), int(ext[0]), int(ext[1]), int(ext[2]), S.ptr(owner), h), "instance_paint")
    S.check(S.lib.sis3d_vertex_instance_overlap(
        S.ptr(view[1]), n_vert, S.ptr(view[0]), S.ptr(owner), int(lo[0]), int(lo[1]), int(lo[2]), int(ext[0]), int(ext[1]),
        int(ext[2]), int(dims[0]), int(dims[1]), int(dims[2]), S.ptr(slots), n_slot, n_box, S.ptr(res), S.ptr(first),
        S.ptr(vbox), h), "vertex_instance_overlap")
    out = res.cpu().numpy() if cuda else res.numpy()
    hist = out[:n_hist].reshape(n_box, n_slot)
    first_vertex = out[n_hist:n_hist + n_box].view(np.int32)[:n_box]
    vertex_box = out[n_hist + n_box:n_hist + n_box + n_vert].view(np.int32)[:n_vert] if want_vertex_box else None
    if seg:
        return hist, first_vertex, vertex_box, out[n_res - n_slot:n_res]
    return hist, first_vertex, vertex_box


# ------------------------------------------------------------------------------------------------------------ per scene
def decode_instances(values, hist, first_vertex):
    """Box counts -> export's instances, in export's order: [(instance id, class, confidence, hist)].  Boxes are visited by
    first vertex; the first box of an instance id owns the instance's first vertex and gives its class and confidence,
    later boxes with the same id add their counts (export's dict merge)."""
    taken = np.nonzero(first_vertex != NO_VERTEX)[0]
    taken = taken[np.argsort(first_vertex[taken], kind="stable")]
    whole = values.astype(np.int64)  # int() truncation, as export
    instances = {}
    for b in taken:
        i = int(whole[b] // 100)
        if i in instances:
            instances[i][3] = instances[i][3] + hist[b]
        else:
            instances[i] = [i, int(whole[b] % 100), float(np.modf(values[b])[0]), hist[b].copy()]
    return list(instances.values())


def scene_predictions(pred_folder, mesh_file, world2grid_file, gt_ids, mask_dir, scene):
    """(gt_uniq, gt_counts, preds) of one scene for evaluate_semantic_instance.assign_instances; each prediction's key is
    the mask path vox2mesh would have written for it under `mask_dir`.  `gt_ids` is either a GT file's per-vertex ids or
    an annotations.SegmentGT, whose slots are resolved on the device; slots no vertex takes are then dropped, which leaves
    exactly np.unique(ids, return_counts=True) of the ids an export would write."""
    pred_box, pred_class, pred_conf, pred_mask = read_result_folder(pred_folder)
    verts = utils.read_mesh_vertices(mesh_file)
    segment_gt = gt_ids if isinstance(gt_ids, annotations.SegmentGT) else None
    if segment_gt is not None and len(segment_gt.seg_index) != len(verts):
        utils.print_error("wrong number of segment indices in %s (%d) vs #mesh vertices (%d) of %s"
                          % (segment_gt.seg_file, len(segment_gt.seg_index), len(verts), mesh_file))
    if segment_gt is None and len(gt_ids) != len(verts):
        utils.print_error("wrong number of lines in GT file (%d) vs #mesh vertices (%d) of %s" % (len(gt_ids), len(verts),
                                                                                              mesh_file))
    w2g = vox2mesh.load_matrix(world2grid_file)
    values = box_values(pred_class, pred_conf)
    bits, offs, ibox, lo, ext = pack_boxes(pred_box, values, pred_mask)
    if segment_gt is not None:
        hist, first, _, slot_count = vertex_instance_overlap(verts, w2g, None, 0, bits, offs, ibox, lo, ext,
                                                             segment_gt=segment_gt)
        taken = slot_count > 0
        gt_uniq, gt_counts, hist = segment_gt.slot_ids[taken], slot_count[taken], hist[:, taken]
    else:
        gt_uniq, gt_slot, gt_counts = np.unique(gt_ids, return_inverse=True, return_counts=True)
        hist, first, _ = vertex_instance_overlap(verts, w2g, gt_slot.astype(np.int32), len(gt_uniq), bits, offs, ibox, lo,
                                                 ext)
    preds = [(os.path.abspath(os.path.join(mask_dir, "predicted_masks", scene + "_" + "{:03d}".format(i) + ".txt")), c, conf, h)
             for i, c, conf, h in decode_instances(values, hist, first)]
    return gt_uniq, gt_counts, preds


def annotation_files(scan_path, scene):
    """ScanNet's annotation files of one scan: (aggregation, segmentation)."""
    return (os.path.join(scan_path, scene, scene + ".aggregation.json"),
            os.path.join(scan_path, scene, scene + "_vh_clean_2.0.010000.segs.json"))


def evaluate_folders(pred_dir, scan_path, frames, gt_path, output_file, label_map_file=None, label_map_file2=None):
    """Scene selection of vox2mesh.main and evaluate_semantic_instance.main combined, then the evaluator's output.
    gt_path None: each scene's GT comes from its annotation files in scan_path, with the two label maps, as
    export_train_mesh_for_evaluation.py --type instance would write it.  -> (ap, avgs)."""
    scenes = [s for s in sorted(os.listdir(pred_dir)) if os.path.isdir(os.path.join(pred_dir, s))
              and os.path.exists(os.path.join(scan_path, s, s + "_vh_clean_2.ply"))]
    if not scenes:
        utils.print_error("No result files found.", user_fault=True)
    gt_files = []
    for s in scenes:
        if gt_path is None:
            for f in annotation_files(scan_path, s):
                if not os.path.isfile(f):
                    utils.print_error("Result file {} does not match any gt file: no {}".format(s + ".txt", f),
                                      user_fault=True)
            gt_files.append(annotation_files(scan_path, s)[0])
            continue
        gt_file = os.path.join(gt_path, s + ".txt")
        if not os.path.isfile(gt_file):
            utils.print_error("Result file {} does not match any gt file".format(s + ".txt"), user_fault=True)
        gt_files.append(gt_file)
    if gt_path is None:
        label_map = utils.read_label_mapping(label_map_file, label_from="raw_category", label_to="nyu40id")
        label_map2 = utils.read_label_mapping(label_map_file2, label_from="nyu40id", label_to="mappedIdConsecutive",
                                              delimiter=",")
    print("evaluating", len(scenes), "scans...")
    matches = {}
    mask_dir = os.path.dirname(os.path.abspath(output_file))
    for i, (s, gt_file) in enumerate(zip(scenes, gt_files)):
        if gt_path is None:
            gt_ids = annotations.read_scene_gt(*annotation_files(scan_path, s), label_map, label_map2, "instance", s)
        else:
            try:
                gt_ids = utils.load_ids(gt_file)
            except Exception as e:
                utils.print_error("unable to load " + gt_file + ": " + str(e))
        gt_uniq, gt_counts, preds = scene_predictions(os.path.join(pred_dir, s), os.path.join(scan_path, s, s + "_vh_clean_2.ply"),
                                                      os.path.join(frames, s, "world2grid.txt"), gt_ids, mask_dir, s)
        gt2pred, pred2gt = E.assign_instances(gt_uniq, gt_counts, preds)
        matches[os.path.abspath(gt_file)] = {"gt": gt2pred, "pred": pred2gt}
        sys.stdout.write("\rscans processed: {}".format(i + 1))
        sys.stdout.flush()
    print("")
    return E.finish(matches, output_file)


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    parser.add_argument("--pred_dir", required=True, help="benchmark-mode result folders, one per scene")
    parser.add_argument("--scan_path", required=True, help="ScanNet scans: <scene>/<scene>_vh_clean_2.ply")
    parser.add_argument("--frames", required=True, help="frames folders: <scene>/world2grid.txt")
    parser.add_argument("--gt_path", default=None,
                        help="path to directory of gt .txt files [default: the annotations in scan_path]")
    parser.add_argument("--label_map_file", default=None, help="path to scannetv2-labels.combined.tsv (without --gt_path)")
    parser.add_argument("--label_map_file2", default=None, help="path to nyu40labels_scannet.csv (without --gt_path)")
    parser.add_argument("--output_file", default="", help="output file [default: pred_dir/" + E.RESULT_FILE + "]")
    opt = parser.parse_args(argv)
    if opt.gt_path is None and (opt.label_map_file is None or opt.label_map_file2 is None):
        parser.error("without --gt_path, --label_map_file and --label_map_file2 are required")
    output_file = opt.output_file or os.path.join(opt.pred_dir, E.RESULT_FILE)
    return evaluate_folders(opt.pred_dir, opt.scan_path, opt.frames, opt.gt_path, output_file, opt.label_map_file,
                            opt.label_map_file2)


if __name__ == "__main__":
    main()
