"""Voxel predictions -> ScanNet benchmark files (SURVEY row f4; reference: tools/scannet_benchmark/vox2mesh.py).

Same functions and file formats as the reference tool -- `load_pred`, `nn_search`, `export`,
`save_scannet_benchmark`, `load_matrix` -- but the two hot loops (painting the instance volume voxel by voxel,
vox2mesh.py:55-69, and the per-vertex 3x3x3 neighbour search, vox2mesh.py:71-106) are array operations, so a
scene with ~10^5 mesh vertices takes milliseconds instead of minutes.  Host-side numpy like the reference (this is
file export, not the GPU hot path).

Deviations, on purpose: vertices that land outside the volume (or whose neighbourhood would leave it) are skipped;
the reference indexes the array with them (IndexError, or a silent wrap-around for -1).

    python vox2mesh.py --pred_dir RESULTS --scan_path SCANS --frames FRAMES [--output_dir DIR]

runs the reference's command line (vox2mesh.py:123-145): for every result folder `<scene>` of `pred_dir` with a mesh
`<scan_path>/<scene>/<scene>_vh_clean_2.ply`, it reads the mesh and `<frames>/<scene>/world2grid.txt`, paints the
predictions and writes `<scene>.txt` plus `predicted_masks/` into `output_dir`, the input of evaluate_semantic_instance.py.
Folders are visited in sorted order; folders without a mesh are skipped.
"""
from __future__ import annotations

import argparse
import os
import pickle
import sys

import numpy as np

SCENE_DIMS = (400, 200, 400)  # vox2mesh.py:41


def save_scannet_benchmark(instance_class, instance_mask, instance_conf, verts_len, output_dir, scene_id):
    """<scene>.txt with one `predicted_masks/<scene>_<id:03d>.txt <class> <score>` line per instance and a 0/1 text
    mask per vertex for each instance (vox2mesh.py:23-38)."""
    os.makedirs(os.path.join(output_dir, "predicted_masks"), exist_ok=True)
    with open(os.path.join(output_dir, scene_id + ".txt"), "w") as f:
        for instance_id in instance_class:
            mask_file = "predicted_masks/" + scene_id + "_" + "{:03d}".format(instance_id) + ".txt"
            f.write(mask_file + " " + str(instance_class[instance_id]) + " " + str(float(instance_conf[instance_id])) + "\n")
            mask = np.zeros(verts_len, dtype=np.uint8)
            mask[np.asarray(instance_mask[instance_id], dtype=np.int64)] = 1
            np.savetxt(os.path.join(output_dir, mask_file), mask, fmt="%u")


def paint_instances(pred_box, pred_class, pred_conf, pred_mask, dims=SCENE_DIMS):
    """Instance volume: voxel = box_index*100 + class + conf - 0.01 for the FIRST box whose mask covers it, else 0
    (vox2mesh.py:55-69).  Box corners are rounded half to even like Python's round()."""
    scene = np.zeros(dims, dtype=np.float64)
    lo = np.rint(np.asarray(pred_box, dtype=np.float64)[:, :3]).astype(np.int64) if len(pred_box) else np.zeros((0, 3), np.int64)
    hi = np.rint(np.asarray(pred_box, dtype=np.float64)[:, 3:6]).astype(np.int64) if len(pred_box) else np.zeros((0, 3), np.int64)
    for b in range(len(lo)):
        (x0, y0, z0), (x1, y1, z1) = lo[b], hi[b]
        if x1 <= x0 or y1 <= y0 or z1 <= z0:
            continue
        if min(x0, y0, z0) < 0 or x1 > dims[0] or y1 > dims[1] or z1 > dims[2]:
            raise IndexError(f"box {b} leaves the {dims} volume")
        m = np.asarray(pred_mask[b])[:x1 - x0, :y1 - y0, :z1 - z0]
        if m.shape != (x1 - x0, y1 - y0, z1 - z0):
            raise IndexError(f"mask {b} is smaller than its box")
        region = scene[x0:x1, y0:y1, z0:z1]
        take = (m != 0) & (region == 0)
        region[take] = b * 100 + pred_class[b] + pred_conf[b] - 0.01
    return scene


def load_pred(pred_folder, dims=SCENE_DIMS):
    """Read pred_{box,class,conf}.npy and the pickled pred_mask / pred_mask_index of one scene (as written by
    lib.model.trainval.save_scene_results) and paint the instance volume (vox2mesh.py:40-69)."""
    pred_box = np.load(os.path.join(pred_folder, "pred_box.npy"))[:, :6]
    pred_class = np.load(os.path.join(pred_folder, "pred_class.npy"))
    pred_conf = np.load(os.path.join(pred_folder, "pred_conf.npy"))
    with open(os.path.join(pred_folder, "pred_mask"), "rb") as f:
        pred_mask = pickle.load(f)
    with open(os.path.join(pred_folder, "pred_mask_index"), "rb") as f:
        sort_index = pickle.load(f)
    sort_index = np.asarray(sort_index)
    return paint_instances(pred_box[sort_index], pred_class[sort_index], pred_conf[sort_index], pred_mask, dims)


_NEIGHBOURS = np.array([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)], dtype=np.int64)


def nn_search(scene, x, y, z):
    """The voxel itself if labelled, else the first labelled voxel of its 3x3x3 neighbourhood in (i, j, k) order,
    else (-1, -1, -1)  (vox2mesh.py:71-81)."""
    if scene[x, y, z] != 0:
        return x, y, z
    for i, j, k in _NEIGHBOURS:
        if scene[x + i, y + j, z + k] != 0:
            return x + i, y + j, z + k
    return -1, -1, -1


def vertex_labels(mesh_vertices, world2grid, scene):
    """Vectorised per-vertex lookup: (value, valid) with value = scene at the vertex's voxel or at the first labelled
    neighbour in the reference's scan order."""
    v = np.asarray(mesh_vertices, dtype=np.float64).reshape(-1, 3)
    homo = np.concatenate([v, np.ones((len(v), 1))], 1)
    g = np.rint(np.rint(homo @ np.asarray(world2grid, dtype=np.float64).T)[:, :3]).astype(np.int64)
    dims = np.array(scene.shape, dtype=np.int64)
    inside = np.all((g >= 1) & (g <= dims - 2), axis=1)  # the whole 3x3x3 neighbourhood exists
    gi = np.where(inside[:, None], g, 1)
    value = scene[gi[:, 0], gi[:, 1], gi[:, 2]]
    need = inside & (value == 0)
    for d in _NEIGHBOURS:  # first hit in scan order wins
        if not need.any():
            break
        idx = np.nonzero(need)[0]
        q = gi[idx] + d
        nv = scene[q[:, 0], q[:, 1], q[:, 2]]
        hit = nv != 0
        value[idx[hit]] = nv[hit]
        need[idx[hit]] = False
    return value, inside & (value != 0)


def export(mesh_vertices, world2grid, scene, output_dir, scene_id):
    """Transfer the voxel instance labels to the mesh vertices and write the benchmark files (vox2mesh.py:83-108)."""
    value, valid = vertex_labels(mesh_vertices, world2grid, scene)
    idx = np.nonzero(valid)[0]
    val = value[idx]
    whole = val.astype(np.int64)  # int() truncation; values are positive
    inst = whole // 100
    instance_mask, instance_conf, instance_class = {}, {}, {}
    uniq, first = np.unique(inst, return_index=True)
    for k in np.argsort(first, kind="stable"):  # instances in the order their first vertex appears (the reference's dict order)
        i, p = int(uniq[k]), first[k]
        instance_class[i] = int(whole[p] % 100)
        instance_conf[i] = np.modf(val[p])[0]
        instance_mask[i] = idx[inst == uniq[k]].tolist()
    save_scannet_benchmark(instance_class, instance_mask, instance_conf, len(np.asarray(mesh_vertices).reshape(-1, 3)), output_dir,
                           scene_id)
    return instance_class, instance_mask, instance_conf


def load_matrix(filename):
    """4x4 world2grid text matrix with the chunk padding removed from the translation column (vox2mesh.py:110-121)."""
    padding = [10, 16, 10, 0]
    matrix = np.zeros((4, 4))
    with open(filename) as f:
        for ind, line in enumerate(f.readlines()[:4]):
            parts = line.split()
            matrix[ind, :3] = [float(parts[0]), float(parts[1]), float(parts[2])]
            matrix[ind, 3] = float(parts[3]) - padding[ind]
    return matrix


def main(argv=None):
    """vox2mesh.py:123-145: every result folder with a mesh -> benchmark files in --output_dir."""
    if __package__:
        from . import utils
    else:  # run as a script
        import utils
    parser = argparse.ArgumentParser()
    parser.add_argument("--pred_dir", required=True, help="benchmark-mode result folders, one per scene")
    parser.add_argument("--output_dir", default="./ScanNet_Benchmark_Result", help="output directory")
    parser.add_argument("--scan_path", required=True, help="ScanNet scans: <scene>/<scene>_vh_clean_2.ply")
    parser.add_argument("--frames", required=True, help="frames folders: <scene>/world2grid.txt")
    opt = parser.parse_args(argv)
    names = sorted(os.listdir(opt.pred_dir))
    for ind, name in enumerate(names):
        print("{}/{}".format(ind, len(names)))
        mesh_file = os.path.join(opt.scan_path, name, name + "_vh_clean_2.ply")
        if not os.path.isdir(os.path.join(opt.pred_dir, name)) or not os.path.exists(mesh_file):
            continue
        os.makedirs(opt.output_dir, exist_ok=True)
        world2grid = load_matrix(os.path.join(opt.frames, name, "world2grid.txt"))
        mesh_vertices = utils.read_mesh_vertices(mesh_file)
        folder = os.path.join(opt.pred_dir, name)
        with open(os.path.join(folder, "pred_mask_index"), "rb") as f:
            kept = len(pickle.load(f))
        # a scene without detections paints nothing (load_pred cannot index with an empty list)
        scene = load_pred(folder) if kept else np.zeros(SCENE_DIMS)
        export(mesh_vertices, world2grid, scene, opt.output_dir, name)
        sys.stdout.flush()


if __name__ == "__main__":
    main()
