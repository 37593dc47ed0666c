"""ScanNet instance AP straight from benchmark-mode result folders: vox2mesh.py followed by evaluate_semantic_instance.py,
without the per-vertex text files.

    python evaluate_predictions.py --pred_dir RESULTS --scan_path SCANS --frames FRAMES --gt_path GT [--output_file FILE]

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

A scene with no instances is still evaluated (its GT count as false negatives).  A result folder without a GT file is the
evaluator's exit-2 error.  There is no CPU path: without a CUDA device the launch raises.
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
    from . import utils, vox2mesh
else:  # run as a script
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
    from tools.scannet_benchmark import evaluate_semantic_instance as E
    from tools.scannet_benchmark import utils, vox2mesh

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
def vertex_instance_overlap(verts, world2grid, gt_slot, n_slot, bits, offs, ibox, lo, ext, dims=vox2mesh.SCENE_DIMS,
                            want_vertex_box=False, device=None):
    """Both kernels on one scene: one H2D copy of every input, one D2H copy of the results.
    -> (hist int64 [n_box, n_slot], first_vertex int32 [n_box], vertex_box int32 [n_vert] or None)."""
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    n_vert, n_box = verts.shape[0], ibox.shape[0]
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    cuda = device.type == "cuda"
    sections = [np.ascontiguousarray(world2grid, np.float64).reshape(16), verts, np.ascontiguousarray(gt_slot, np.int32),
                np.ascontiguousarray(offs, np.int64), np.ascontiguousarray(ibox, np.int32), np.ascontiguousarray(bits, np.uint8)]
    starts, o = [], 0
    for a in sections:
        o = (o + 15) // 16 * 16
        starts.append(o)
        o += a.nbytes
    blob = torch.empty(max(o, 16), dtype=torch.uint8, pin_memory=cuda)
    bn = blob.numpy()
    for a, s in zip(sections, starts):
        bn[s:s + a.nbytes] = a.reshape(-1).view(np.uint8)
    n_hist = n_box * n_slot
    n_owner = int(np.prod(ext))
    dblob = blob.to(device, non_blocking=True)
    owner = torch.empty(max(n_owner, 1), dtype=torch.int32, device=device)
    res = torch.empty(max(n_hist + n_box + (n_vert if want_vertex_box else 0), 1), dtype=torch.int64, device=device)
    first = res[n_hist:n_hist + n_box].view(torch.int32)  # int32 slots inside the int64 result: one D2H copy for all
    vbox = res[n_hist + n_box:].view(torch.int32) if want_vertex_box else None
    view = lambda k: dblob[starts[k]:]
    h = S.stream() if cuda else None  # host tensors: S.ptr raises (no CPU path)
    S.check(S.lib.sis3d_instance_paint(S.ptr(view(5)), S.ptr(view(3)), S.ptr(view(4)), n_box, int(lo[0]), int(lo[1]),
                                       int(lo[2]), int(ext[0]), int(ext[1]), int(ext[2]), S.ptr(owner), h), "instance_paint")
    S.check(S.lib.sis3d_vertex_instance_overlap(
        S.ptr(view(1)), n_vert, S.ptr(view(0)), S.ptr(owner), int(lo[0]), int(lo[1]), int(lo[2]), int(ext[0]), int(ext[1]),
        int(ext[2]), int(dims[0]), int(dims[1]), int(dims[2]), S.ptr(view(2)), n_slot, n_box, S.ptr(res), S.ptr(first),
        S.ptr(vbox), h), "vertex_instance_overlap")
    out = res.cpu().numpy() if cuda else res.numpy()
    hist = out[:n_hist].reshape(n_box, n_slot)
    first_vertex = out[n_hist:n_hist + n_box].view(np.int32)[:n_box]
    vertex_box = out[n_hist + n_box:].view(np.int32)[:n_vert] if want_vertex_box else None
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
    the mask path vox2mesh would have written for it under `mask_dir`."""
    pred_box, pred_class, pred_conf, pred_mask = read_result_folder(pred_folder)
    verts = utils.read_mesh_vertices(mesh_file)
    if len(gt_ids) != len(verts):
        utils.print_error("wrong number of lines in GT file (%d) vs #mesh vertices (%d) of %s" % (len(gt_ids), len(verts),
                                                                                              mesh_file))
    w2g = vox2mesh.load_matrix(world2grid_file)
    values = box_values(pred_class, pred_conf)
    bits, offs, ibox, lo, ext = pack_boxes(pred_box, values, pred_mask)
    gt_uniq, gt_slot, gt_counts = np.unique(gt_ids, return_inverse=True, return_counts=True)
    hist, first, _ = vertex_instance_overlap(verts, w2g, gt_slot.astype(np.int32), len(gt_uniq), bits, offs, ibox, lo, ext)
    preds = [(os.path.abspath(os.path.join(mask_dir, "predicted_masks", scene + "_" + "{:03d}".format(i) + ".txt")), c, conf, h)
             for i, c, conf, h in decode_instances(values, hist, first)]
    return gt_uniq, gt_counts, preds


def evaluate_folders(pred_dir, scan_path, frames, gt_path, output_file):
    """Scene selection of vox2mesh.main and evaluate_semantic_instance.main combined, then the evaluator's output.
    -> (ap, avgs)."""
    scenes = [s for s in sorted(os.listdir(pred_dir)) if os.path.isdir(os.path.join(pred_dir, s))
              and os.path.exists(os.path.join(scan_path, s, s + "_vh_clean_2.ply"))]
    if not scenes:
        utils.print_error("No result files found.", user_fault=True)
    gt_files = []
    for s in scenes:
        gt_file = os.path.join(gt_path, s + ".txt")
        if not os.path.isfile(gt_file):
            utils.print_error("Result file {} does not match any gt file".format(s + ".txt"), user_fault=True)
        gt_files.append(gt_file)
    print("evaluating", len(scenes), "scans...")
    matches = {}
    mask_dir = os.path.dirname(os.path.abspath(output_file))
    for i, (s, gt_file) in enumerate(zip(scenes, gt_files)):
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
    parser.add_argument("--gt_path", required=True, help="path to directory of gt .txt files")
    parser.add_argument("--output_file", default="", help="output file [default: pred_dir/" + E.RESULT_FILE + "]")
    opt = parser.parse_args(argv)
    output_file = opt.output_file or os.path.join(opt.pred_dir, E.RESULT_FILE)
    return evaluate_folders(opt.pred_dir, opt.scan_path, opt.frames, opt.gt_path, output_file)


if __name__ == "__main__":
    main()
