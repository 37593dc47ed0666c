"""Cost of writing the result visualisation's PLY files, two ways (not bench.py):

  (a) host: oracle/ply_writer.py, the reference's writers restated (numpy for the cubes, one str.format per text line,
      as the reference formats them);
  (b) GPU route: tools/visualization.py / visualize_benchmark.py, split into the mesh and formatter kernels (CUDA event
      pairs), the device-to-host copies of the text (CUDA event pairs) and the file writes (host clock); "total" is the
      wall time of the whole call, file writes included.

Workloads: one test-mode result folder of 208x48x160 (scene.npy at the given occupancy, 100 kept masks of density 0.6,
40 GT boxes with masks; scene.ply, pred_bbox.ply, pred_mask.ply, gt_bbox.ply, gt_mask.ply) and one benchmark scene of
300k mesh vertices with 60 instances.  Both routes write to a temporary directory; their files are compared by sha1 in
the same run.  Prints the card name and power limit, then one JSON line per workload.

    python tools/bench_visualization.py [--occupancy 0.12] [--verts 300000]
"""
import argparse
import hashlib
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "3d-sis_b200"), ROOT, os.path.join(ROOT, "oracle")]

import ply_writer as W  # noqa: E402
from tools import visualization as V  # noqa: E402
from tools.scannet_benchmark import visualize_benchmark as VB  # noqa: E402

DIMS = (208, 48, 160)


def result_folder(d, occupancy, seed=0, n_box=120, n_keep=100, n_gt=40):
    rng = np.random.default_rng(seed)
    os.makedirs(d, exist_ok=True)
    scene = (rng.random(DIMS) < occupancy).astype(np.int64)
    lo = rng.integers(0, np.array(DIMS) - 24, (n_box, 3)) + rng.choice([0.0, 0.5, 0.3], (n_box, 3))
    hi = np.minimum(lo + rng.integers(4, 24, (n_box, 3)) + rng.choice([0.0, 0.5], (n_box, 3)), DIMS)
    box = np.concatenate([lo, hi], 1).astype(np.float32)
    keep = np.zeros(n_box, bool)
    keep[rng.permutation(n_box)[:n_keep]] = True
    ext = lambda b: tuple(int(v) for v in np.maximum(np.rint(b[3:6]) - np.rint(b[:3]), 0))
    masks = [(rng.random(ext(b)) < 0.6).astype(np.float32) for b, k in zip(box, keep) if k]
    cls = rng.integers(1, 19, n_box).astype(np.int64)
    gbox = np.floor(box[:n_gt]).astype(np.float32)
    gcls = rng.integers(1, 19, n_gt).astype(np.float32)
    gmask = [(rng.random(ext(b)) < 0.7).astype(np.float32) for b in gbox]
    np.save(os.path.join(d, "scene.npy"), scene)
    np.save(os.path.join(d, "pred_box.npy"), box)
    np.save(os.path.join(d, "pred_class.npy"), cls)
    np.save(os.path.join(d, "gt_box.npy"), gbox)
    np.save(os.path.join(d, "gt_class.npy"), gcls)
    pickle.dump(masks, open(os.path.join(d, "pred_mask"), "wb"))
    pickle.dump([bool(k) for k in keep], open(os.path.join(d, "pred_mask_index"), "wb"))
    pickle.dump(gmask, open(os.path.join(d, "gt_mask"), "wb"))
    kb = box[keep]
    return {"scene.ply": lambda: W.mask_mesh(scene),
            "pred_bbox.ply": lambda: V.bbox_cylinders(np.concatenate([kb, cls[keep][:, None]], 1)),
            "pred_mask.ply": lambda: W.mask_mesh(W.paint_masks(DIMS, kb, masks, cls[keep])),
            "gt_bbox.ply": lambda: V.bbox_cylinders(np.concatenate([gbox, gcls[:, None]], 1)),
            "gt_mask.ply": lambda: W.mask_mesh(W.paint_masks(DIMS, gbox, gmask, gcls))}


def benchmark_scene(root, n, seed=1, n_inst=60):
    import make_golden_scannet_eval as SE
    rng = np.random.default_rng(seed)
    scene = "scene0500_00"
    verts = rng.uniform(0, 8, (n, 3)).astype(np.float32)
    faces = rng.integers(0, n, (2 * n, 3))
    os.makedirs(os.path.join(root, "scans", scene))
    SE.write_ply(os.path.join(root, "scans", scene, scene + "_vh_clean_2.ply"), verts, "binary_little_endian", faces)
    align = np.eye(4)
    align[:3, 3] = [-4.0, -4.0, 0.25]
    with open(os.path.join(root, "scans", scene, scene + ".txt"), "w") as f:
        f.write("axisAlignment = " + " ".join(repr(float(v)) for v in align.reshape(-1)) + "\n")
    res = os.path.join(root, "res")
    os.makedirs(os.path.join(res, "pred_mask"))
    with open(os.path.join(res, scene + ".txt"), "w") as f:
        for i in range(n_inst):
            m = np.zeros(n, np.int64)
            a = int(rng.integers(0, n - n // 25))
            m[a:a + int(rng.integers(n // 300, n // 25))] = 1
            np.savetxt(os.path.join(res, "pred_mask", f"{i:03d}.txt"), m, fmt="%d")
            f.write(f"pred_mask/{i:03d}.txt {int(rng.integers(0, 19))} 0.9\n")

    def host_arrays():
        pts = VB.coords_multiplication(align, verts)
        colors = np.zeros_like(verts) + VB.UNCOVERED_COLOR
        boxes = []
        for i, (m, _) in enumerate(VB.read_instances(res, scene + ".txt")):
            idx = m.nonzero()[0].astype(np.int32)
            r, g, b = V.create_color_palette()[(i + 1) % 41]
            boxes.append(np.concatenate([pts[idx].min(0), pts[idx].max(0), [i + 1]]))
            colors[idx] = [r / 255.0, g / 255.0, b / 255.0]
        bv, bc, bf = V.bbox_cylinders(np.array(boxes))
        return np.concatenate([pts, bv]), np.concatenate([colors, bc]), np.concatenate([faces, bf + n])
    return res, os.path.join(root, "scans"), scene, host_arrays


def sha1_file(path):
    with open(path, "rb") as f:
        return hashlib.sha1(f.read()).hexdigest()


def split(stats, total_s):
    return {"total_s": round(total_s, 4), "mesh_kernels_ms": round(V.event_ms(stats.get("mesh", [])), 3),
            "format_kernels_ms": round(V.event_ms(stats.get("format", [])), 3),
            "d2h_ms": round(V.event_ms(stats.get("d2h", [])), 3), "file_write_s": round(stats.get("file_write_s", 0.0), 4)}


def run(occupancy, n_verts):
    with tempfile.TemporaryDirectory() as tmp:
        # warm-up: module load, first launches, pinned allocations
        V.write_mask(np.ones((8, 8, 8), np.int64), os.path.join(tmp, "warm.ply"))
        d = os.path.join(tmp, "scene0000_00")
        makers = result_folder(d, occupancy)
        host_dir = os.path.join(tmp, "host")
        os.makedirs(host_dir)
        t = time.perf_counter()
        for name, make in makers.items():
            W.write_ply(*make(), os.path.join(host_dir, name))
        host_s = time.perf_counter() - t
        stats = {}
        torch.cuda.synchronize()
        t = time.perf_counter()
        V.visualize_result_folder(d, stats=stats)
        torch.cuda.synchronize()
        gpu_s = time.perf_counter() - t
        lines = nbytes = 0
        for name in makers:
            assert sha1_file(os.path.join(d, name)) == sha1_file(os.path.join(host_dir, name)), name
            nbytes += os.path.getsize(os.path.join(d, name))
            with open(os.path.join(d, name), "rb") as f:
                lines += f.read().count(b"\n") - 10  # minus the header's lines
        occupied = int(np.load(os.path.join(d, "scene.npy")).sum())
        yield {"workload": f"results_{DIMS[0]}x{DIMS[1]}x{DIMS[2]}", "scene_occupied_voxels": occupied, "files": len(makers),
               "lines": lines, "bytes": nbytes, "host_s": round(host_s, 3), "gpu": split(stats, gpu_s)}

        bt = os.path.join(tmp, "bench")
        res, scans, scene, host_arrays = benchmark_scene(bt, n_verts)
        out = os.path.join(bt, "out")
        os.makedirs(out)
        t = time.perf_counter()
        W.write_ply(*host_arrays(), os.path.join(bt, "host.ply"))
        host_s = time.perf_counter() - t
        stats = {}
        torch.cuda.synchronize()
        t = time.perf_counter()
        path = VB.visualize_scene(res, scene + ".txt", scans, out, stats=stats)
        torch.cuda.synchronize()
        gpu_s = time.perf_counter() - t
        assert sha1_file(path) == sha1_file(os.path.join(bt, "host.ply"))
        with open(path, "rb") as f:
            lines = f.read().count(b"\n") - 10
        yield {"workload": f"benchmark_{n_verts}_verts_60_instances", "lines": lines, "bytes": os.path.getsize(path),
               "host_s": round(host_s, 3), "gpu": split(stats, gpu_s)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--occupancy", type=float, default=0.12)
    ap.add_argument("--verts", type=int, default=300000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_visualization.py measures the GPU route: it needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("device:", torch.cuda.get_device_name(0), "|", q.stdout.strip(), flush=True)
    for rec in run(a.occupancy, a.verts):
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
