"""Benchmark predictions drawn on their ScanNet meshes (the reference's tools/scannet_benchmark/visualize_benchmark.py).

    python tools/scannet_benchmark/visualize_benchmark.py --result_dir RESULTS --output_dir OUT --scan_path SCANS

For every file `<scene>.txt` of RESULTS (lines `<mask file> <label> <confidence>`, mask files of one 0/1 line per mesh
vertex, paths relative to RESULTS), writes OUT/<scene>.ply: the mesh SCANS/<scene>/<scene>_vh_clean_2.ply moved by the
`axisAlignment` of SCANS/<scene>/<scene>.txt, instance i's vertices coloured palette[(i + 1) % 41] (a later instance
overwrites an earlier one's vertices), and the cylinder edges of each instance's bounding box (tools/visualization.py
write_bbox) appended to the mesh.  The file is byte for byte what the reference writes; its text is formatted on the GPU.

Every vertex no instance covers keeps the reference's colour [64, 64, 96], which is not divided by 255 as the palette
colours are, so write_ply writes it as `16320 16320 24480`.  That quirk is kept: the file is the contract.

Departures from the reference, none of which changes a file it can write: files are visited in sorted order; a scene
with no instances writes the aligned mesh alone (the reference's np.concatenate of an empty list with the mesh raises);
mask files made of exactly "0\\n" / "1\\n" lines are parsed as bytes, others with np.loadtxt as the reference does.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

if __package__:
    from .. import visualization as V
else:  # run as a script
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
    from tools import visualization as V

UNCOVERED_COLOR = np.array([64, 64, 96])  # visualize_benchmark.py:114, not scaled to [0, 1]


def coords_multiplication(A, B):
    """visualize_benchmark.py:75-87 (numpy branch): the 4x4 A applied to the rows of B [n, 3], with the same numpy calls,
    so the result has the same bits."""
    B = np.concatenate([np.transpose(B), np.ones((1, B.shape[0]))])
    return np.transpose(np.dot(A, B))[:, :3]


def load_mask(path):
    """One mask file -> float64 [n] (np.loadtxt's result for a one-column file)."""
    with open(path, "rb") as f:
        raw = f.read()
    b = np.frombuffer(raw, np.uint8)
    if b.size and b.size % 2 == 0 and (b[1::2] == 10).all() and ((b[0::2] == 48) | (b[0::2] == 49)).all():
        return (b[0::2] - 48).astype(np.float64)
    return np.loadtxt(path)


def read_instances(result_dir, txt_file):
    """Benchmark_reader.__getitem__ (visualize_benchmark.py:60-73): [(vertex mask, label)] in line order."""
    with open(os.path.join(result_dir, txt_file)) as f:
        lines = f.readlines()
    return [(load_mask(os.path.join(result_dir, line.split()[0])), int(line.split()[1])) for line in lines]


def visualize_scene(result_dir, txt_file, scan_path, output_dir, slab_lines=V.SLAB_LINES, device=None, stats=None):
    """visualize_benchmark.py:106-144 for one result file; -> the written path."""
    scene = txt_file.split(".")[0]
    ply_file = os.path.join(scan_path, scene, scene + "_vh_clean_2.ply")
    with open(os.path.join(scan_path, scene, scene + ".txt")) as f:
        alignment = f.readlines()[0]
    alignment = np.array([float(a) for a in alignment.split()[2:]]).reshape(4, 4)
    points, faces, _ = V.read_ply(ply_file)
    colors = np.zeros_like(points) + UNCOVERED_COLOR
    points = coords_multiplication(alignment, points)
    boxes = []
    palette = V.create_color_palette()
    for i, (mask, _) in enumerate(read_instances(result_dir, txt_file)):
        r, g, b = palette[(i + 1) % 41]
        idx = mask.nonzero()[0].astype(np.int32)
        pts = points[idx]
        boxes.append(np.concatenate([np.min(pts, 0), np.max(pts, 0), [i + 1]]))
        colors[idx] = [r / 255.0, g / 255.0, b / 255.0]
    output_file = os.path.join(output_dir, scene + ".ply")
    if boxes:
        bverts, bcolors, bfaces = V.write_bbox(np.array(boxes), None)
        points = np.concatenate([points, bverts])
        colors = np.concatenate([colors, bcolors])
        faces = np.concatenate([faces, bfaces + len(colors) - len(bcolors)])
    V.write_ply(points, colors, faces, output_file, slab_lines, device, stats)
    return output_file


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--result_dir", default="./ScanNet_Benchmark_Result")
    parser.add_argument("--output_dir", default="./ScanNet_Benchmark_Result_Visualization")
    parser.add_argument("--scan_path", default="/mnt/canis_datasets/ScanNet/public/v2/scans")
    opt = parser.parse_args(argv)
    os.makedirs(opt.output_dir, exist_ok=True)
    for name in sorted(os.listdir(opt.result_dir)):
        if os.path.isdir(os.path.join(opt.result_dir, name)):
            continue
        print(name)
        visualize_scene(opt.result_dir, name, opt.scan_path, opt.output_dir)


if __name__ == "__main__":
    main()
