"""oracle/make_golden_visualization.py -- TEST INFRASTRUCTURE ONLY; runs ONLY where the reference tree is present.

Runs the reference's UNMODIFIED visualisation tools in this process on seeded inputs and stores every file they write in
tests/golden/visualization_reference.npz, which pins tools/visualization.py, tools/scannet_benchmark/visualize_benchmark.py
and proj_label.py (tests/test_visualization.py, tests/test_gpu_visualization.py).

    python oracle/make_golden_visualization.py

Shims: a stub `plyfile` module whose PlyData.read parses only the ASCII fixture meshes written here (x y z red green blue
alpha vertices, list faces), `sys.argv` set for each tool's argument parsing, and runpy for each tool's __main__ block:
- tools/visualization.py --path RESULTS --mode result on result folders as test mode writes them;
- tools/scannet_benchmark/visualize_benchmark.py on benchmark result files and fixture scans;
- tools/scannet_benchmark/proj_label.py on a copy of the benchmark result files.
The inputs are regenerated from seeds by the functions below (the tests import them; nothing of the reference is involved
in making them).  They cover overlapping masks (the first box wins), a mask larger than its box, boxes on the volume
border, .5 box corners (rounded half to even), class ids >= 41 (the palette wraps) and a class 0 box (paints nothing and
leaves its voxels to later boxes), nan and 0.5 mask values, a scene without detections, test mode's GT files present and
absent, pred_roi.npy, a flat GT box (nan cylinder vertices), a box with an edge along -z, a benchmark mesh with quads,
instances that overwrite each other's vertex colours and a mask file only np.loadtxt reads.

Layout (keys): `res__<scene>__<file>` and `bench__<file>` / `proj__<file>` (uint8: the bytes of every file written),
`res_files` / `bench_files` (the written names), `bbox_<k>_verts` / `_colors` / `_faces` (write_bbox(boxes_k, None) as
float64 / float64 / int64 arrays), `palette` (int64 [41, 3]).
"""
from __future__ import annotations

import contextlib
import io
import os
import pickle
import runpy
import shutil
import sys
import tempfile
import types

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
REF = os.environ.get("SIS3D_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "visualization_reference.npz")
DIMS = (24, 16, 20)


# ------------------------------------------------------------------------------------------------------------ results
def _mask(rng, shape, p=0.6):
    m = (rng.random(shape) < p).astype(np.float32)
    if m.size:
        flat = m.reshape(-1)
        flat[rng.integers(0, m.size, 3)] = 0.5  # != 0: set
        flat[rng.integers(0, m.size, 2)] = np.nan  # != 0: set
    return m


def _ext(box):
    return tuple(int(v) for v in np.maximum(np.rint(box[3:6]) - np.rint(box[0:3]), 0))


def result_scenes(seed=5):
    """-> {scene: {file name: array or picklable}} as lib.model.trainval writes test-mode result folders."""
    rng = np.random.default_rng(seed)
    scenes = {}
    box = np.array([[2, 3, 4, 9, 10, 12], [5.5, 6, 7, 12, 14, 15], [16, 0, 10, 24, 16, 20], [1, 1, 1, 4, 4, 4],
                    [10.5, 2.5, 1.5, 14.5, 6.5, 5.5]], np.float32)
    keep = [True, True, True, False, True]
    masks = [_mask(rng, _ext(b)) for b in box]
    masks[1] = np.pad(masks[1], ((0, 1), (0, 2), (0, 0)), constant_values=1.0)  # larger than its box: cropped
    gt_box = np.array([[2, 3, 4, 8, 9, 10], [0, 0, 0, 3, 3, 0], [12, 8, 12, 20, 16, 20]], np.float32)
    scenes["scene0000_00"] = {
        "scene.npy": (rng.random(DIMS) < 0.05).astype(np.int64),
        "pred_box.npy": box, "pred_class.npy": np.array([5, 45, 12, 7, 3], np.int64),
        "pred_conf.npy": rng.random(5), "pred_mask": [m for m, k in zip(masks, keep) if k], "pred_mask_index": keep,
        "gt_box.npy": gt_box, "gt_class.npy": np.array([5, 2, 41], np.float32),
        "gt_mask": [_mask(rng, _ext(b), 0.7) for b in gt_box]}
    box = np.array([[3, 3, 3, 11, 9, 10], [6, 5, 4, 14, 12, 12]], np.float32)
    scenes["scene0001_00"] = {
        "scene.npy": (rng.random(DIMS) < 0.04).astype(np.int64),
        "pred_roi.npy": np.concatenate([rng.uniform(0, 10, (2, 3)), rng.uniform(12, 20, (2, 3))], 1).astype(np.float32),
        "pred_box.npy": box, "pred_class.npy": np.array([0, 19], np.int64), "pred_conf.npy": rng.random(2),
        "pred_mask": [_mask(rng, _ext(b)) for b in box], "pred_mask_index": [True, True]}
    scenes["scene0002_00"] = {
        "scene.npy": (rng.random(DIMS) < 0.03).astype(np.int64),
        "pred_box.npy": np.zeros((0, 6), np.float32), "pred_class.npy": np.zeros(0, np.int64),
        "pred_conf.npy": np.zeros(0), "pred_mask": [], "pred_mask_index": []}
    return scenes


def write_result_scenes(scenes, root):
    for scene, files in scenes.items():
        d = os.path.join(root, scene)
        os.makedirs(d, exist_ok=True)
        for name, v in files.items():
            if name.endswith(".npy"):
                np.save(os.path.join(d, name), v)
            else:
                with open(os.path.join(d, name), "wb") as f:
                    pickle.dump(v, f)


BBOX_SETS = {
    "f32": lambda: np.array([[0, 0, 0, 1, 2, 3, 4], [1.5, -0.25, 2, 1.5, 3, 2.75, 50], [0, 0, 5, 2, 2, 1, 1]], np.float32),
    "f64": lambda: np.array([[0.1, 0.2, 0.3, 1.7, 2.9, 0.31, 40], [-3.0, -2.0, -1.0, -1.5, -0.5, 2.0, 82]], np.float64),
}


# ---------------------------------------------------------------------------------------------------------- benchmark
def write_ascii_mesh(path, verts, faces):
    """x y z red green blue alpha vertices and list faces (any polygon size), ASCII."""
    n = len(verts)
    head = (f"ply\nformat ascii 1.0\nelement vertex {n}\nproperty float x\nproperty float y\nproperty float z\n"
            "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\n"
            f"element face {len(faces)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "w") as f:
        f.write(head)
        for i, v in enumerate(np.asarray(verts, np.float32)):
            f.write(" ".join(repr(float(x)) for x in v) + f" {i % 251} {(3 * i) % 256} {(7 * i) % 256} 255\n")
        for t in faces:
            f.write(f"{len(t)} " + " ".join(str(int(x)) for x in t) + "\n")


def benchmark_scenes(seed=9):
    """-> {scene: dict(verts float32 [n, 3], faces list, align float64 [4, 4], instances [(mask 0/1 [n], label, conf,
    loadtxt_only)])}"""
    rng = np.random.default_rng(seed)
    out = {}
    for s, (n, n_inst) in enumerate([(400, 4), (150, 1)]):
        verts = rng.uniform(0, 3, (n, 3)).astype(np.float32)
        faces = [list(rng.integers(0, n, 3 if rng.random() < 0.7 else 4)) for _ in range(n)]
        a = rng.uniform(0, 2 * np.pi)
        align = np.eye(4)
        align[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        align[:3, 3] = rng.uniform(-2, 2, 3)
        inst = []
        for i in range(n_inst):
            m = np.zeros(n, np.int64)
            lo = int(rng.integers(0, n // 2))
            m[lo:lo + int(rng.integers(n // 6, n // 2))] = 1  # overlapping spans: later instances overwrite colours
            inst.append((m, int(rng.integers(0, 19)), float(rng.choice([0.5, 0.75, 0.9])), i == 1))
        out[f"scene{100 + s:04d}_00"] = dict(verts=verts, faces=faces, align=align, instances=inst)
    return out


def write_benchmark_inputs(scenes, result_dir, scan_dir):
    os.makedirs(os.path.join(result_dir, "pred_mask"), exist_ok=True)
    for scene, c in scenes.items():
        os.makedirs(os.path.join(scan_dir, scene), exist_ok=True)
        write_ascii_mesh(os.path.join(scan_dir, scene, scene + "_vh_clean_2.ply"), c["verts"], c["faces"])
        with open(os.path.join(scan_dir, scene, scene + ".txt"), "w") as f:
            f.write("axisAlignment = " + " ".join(repr(float(v)) for v in c["align"].reshape(-1)) + "\n")
            f.write("colorHeight = 968\n")
        with open(os.path.join(result_dir, scene + ".txt"), "w") as f:
            for i, (m, label, conf, loadtxt_only) in enumerate(c["instances"]):
                rel = f"pred_mask/{scene}_{i:03d}.txt"
                if loadtxt_only:
                    np.savetxt(os.path.join(result_dir, rel), m.astype(np.float64))  # "1.000000000000000000e+00" lines
                else:
                    np.savetxt(os.path.join(result_dir, rel), m, fmt="%d")
                f.write(f"{rel}  {label}   {conf}\n" if i % 2 else f"{rel} {label} {conf}\n")


# ------------------------------------------------------------------------------------------------------------ the reference
def _plyfile_stub():
    """plyfile.PlyData.read for the ASCII fixture meshes: vertex rows as tuples of numpy scalars of the declared types,
    face rows as (int32 array,) -- what the reference's read_ply iterates."""
    types_ = {"float": np.float32, "uchar": np.uint8, "int": np.int32}

    def read(f):
        lines = f.read().decode("ascii").splitlines()
        end = lines.index("end_header")
        elements = []
        for line in lines[:end]:
            w = line.split()
            if w[0] == "element":
                elements.append((w[1], int(w[2]), []))
            elif w[0] == "property":
                elements[-1][2].append(w[1:])
        data, row = {}, end + 1
        for name, count, props in elements:
            rows = []
            for line in lines[row:row + count]:
                w = line.split()
                if props[0][0] == "list":
                    rows.append((np.array([int(x) for x in w[1:1 + int(w[0])]], np.int32),))
                else:
                    rows.append(tuple(types_[p[0]](float(x) if p[0] == "float" else int(x)) for p, x in zip(props, w)))
            data[name] = rows
            row += count
        return data
    return types.SimpleNamespace(PlyData=types.SimpleNamespace(read=read), PlyElement=None)


def _run(script, argv):
    old = sys.argv
    sys.argv = [os.path.basename(script)] + argv
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            runpy.run_path(script, run_name="__main__")
    finally:
        sys.argv = old


def _collect(root, prefix, out, skip=()):
    names = []
    for dirpath, _, files in os.walk(root):
        for fn in files:
            rel = os.path.relpath(os.path.join(dirpath, fn), root)
            if rel in skip:
                continue
            with open(os.path.join(dirpath, fn), "rb") as f:
                out[prefix + "__" + rel.replace(os.sep, "__")] = np.frombuffer(f.read(), np.uint8)
            names.append(rel)
    return sorted(names)


def main():
    sys.modules["plyfile"] = _plyfile_stub()
    sys.path.insert(0, REF)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        res = os.path.join(d, "results")
        scenes = result_scenes()
        write_result_scenes(scenes, res)
        _run(os.path.join(REF, "tools", "visualization.py"), ["--path", res, "--mode", "result"])
        inputs = {os.path.join(s, n) for s, files in scenes.items() for n in files}
        out["res_files"] = np.array(_collect(res, "res", out, skip=inputs))

        bench_res, scans, vis = (os.path.join(d, x) for x in ("bench", "scans", "vis"))
        write_benchmark_inputs(benchmark_scenes(), bench_res, scans)
        _run(os.path.join(REF, "tools", "scannet_benchmark", "visualize_benchmark.py"),
             ["--result_dir", bench_res, "--output_dir", vis, "--scan_path", scans])
        out["bench_files"] = np.array(_collect(vis, "bench", out))

        proj = os.path.join(d, "proj")
        shutil.copytree(bench_res, proj)
        _run(os.path.join(REF, "tools", "scannet_benchmark", "proj_label.py"), ["--pred_path", proj])
        for fn in sorted(os.listdir(proj)):
            if fn.endswith(".txt"):
                with open(os.path.join(proj, fn), "rb") as f:
                    out["proj__" + fn] = np.frombuffer(f.read(), np.uint8)

    ns = runpy.run_path(os.path.join(REF, "tools", "visualization.py"), run_name="ref_visualization")
    for k, make in BBOX_SETS.items():
        v, c, t = ns["write_bbox"](make(), None)
        out[f"bbox_{k}_verts"] = np.array(v, np.float64)
        out[f"bbox_{k}_colors"] = np.array(c, np.float64)
        out[f"bbox_{k}_faces"] = np.array(t, np.int64)
    out["palette"] = np.array(ns["create_color_palette"](), np.int64)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
