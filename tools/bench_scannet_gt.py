"""Per-scene cost of ScanNet GT from the annotation files (not bench.py):

  (a) export: tools/scannet_benchmark/export_train_mesh_for_evaluation.export (label maps, mesh, annotations, segment
      table, sis3d_segment_gt_slots, text) against the reference's per-vertex loop restated in
      oracle/make_golden_scannet_gt.loop_export_ids followed by the same text writer; the files are compared;
  (b) the fused evaluation of one scene (evaluate_predictions.scene_predictions) with the GT read from the annotations
      against the same with the GT read from the exported file (load_ids + np.unique);
  (c) sis3d_segment_gt_slots alone, CUDA events over many launches on resident inputs.

Synthetic scans: tools/bench_scannet_eval.make_scene's boxes and vertices, segments over 3-voxel cells, one object per box.
Prints the card name and power limit, then one JSON line per vertex count.

    python tools/bench_scannet_gt.py [--verts 150000 300000] [--boxes 100] [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "3d-sis_b200"), ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")]

import bench_scannet_eval as B  # noqa: E402
import make_golden_scannet_gt as GG  # noqa: E402
from lib import _sis3d as S  # noqa: E402
from tools.scannet_benchmark import annotations as A  # noqa: E402
from tools.scannet_benchmark import evaluate_predictions as F  # noqa: E402
from tools.scannet_benchmark import export_train_mesh_for_evaluation as X  # noqa: E402
from tools.scannet_benchmark import utils  # noqa: E402


def timed(f, reps=1):
    t0 = time.perf_counter()
    for _ in range(reps):
        r = f()
    return r, (time.perf_counter() - t0) / reps


def write_scene(tmp, c, seed):
    scene = "scene0000_00"
    seg, groups = GG.annotate_chain_scene(np.random.default_rng(seed), c, id_step=997)  # tens of thousands of cells
    GG.write_scan(os.path.join(tmp, "scans"), scene, c["verts"], seg, groups)
    GG.G.write_pred_folder(os.path.join(tmp, "results", scene), dict(c, keep=np.ones(len(c["box"]), bool)))
    os.makedirs(os.path.join(tmp, "frames", scene), exist_ok=True)
    GG.G.write_world2grid(os.path.join(tmp, "frames", scene, "world2grid.txt"), c["w2g"])
    for name, text in (("labels.tsv", GG.label_tsv()), ("nyu40.csv", GG.label_csv(False))):
        with open(os.path.join(tmp, name), "w") as f:
            f.write(text)
    d = os.path.join(tmp, "scans", scene)
    return scene, dict(mesh=os.path.join(d, scene + "_vh_clean_2.ply"), agg=os.path.join(d, scene + ".aggregation.json"),
                       seg=os.path.join(d, scene + "_vh_clean_2.0.010000.segs.json"), tsv=os.path.join(tmp, "labels.tsv"),
                       csv=os.path.join(tmp, "nyu40.csv"), n_groups=len(groups))


def export_times(tmp, scene, p):
    out_dev, out_loop = os.path.join(tmp, "gt_device.txt"), os.path.join(tmp, "gt_loop.txt")
    _, t_dev = timed(lambda: X.export(p["mesh"], p["agg"], p["seg"], p["tsv"], p["csv"], "instance", out_dev), 3)

    def loop():
        lm = utils.read_label_mapping(p["tsv"])
        lm2 = utils.read_label_mapping(p["csv"], label_from="nyu40id", label_to="mappedIdConsecutive", delimiter=",")
        utils.read_mesh_vertices(p["mesh"])
        ids = GG.loop_export_ids(*A.read_aggregation(p["agg"]), A.read_segmentation(p["seg"], scene), lm, lm2, "instance")
        utils.export_ids(out_loop, ids)
    _, t_loop = timed(loop)
    same = open(out_dev, "rb").read() == open(out_loop, "rb").read()
    return dict(export_device_s=t_dev, export_loop_s=t_loop, files_equal=same), out_dev


def fused_times(tmp, scene, p, gt_file):
    lm = utils.read_label_mapping(p["tsv"])
    lm2 = utils.read_label_mapping(p["csv"], label_from="nyu40id", label_to="mappedIdConsecutive", delimiter=",")
    args = (os.path.join(tmp, "results", scene), p["mesh"], os.path.join(tmp, "frames", scene, "world2grid.txt"))
    (u1, c1, p1), t_ann = timed(lambda: F.scene_predictions(*args, A.read_scene_gt(p["agg"], p["seg"], lm, lm2, "instance",
                                                                                    scene), tmp, scene), 3)
    (u2, c2, p2), t_file = timed(lambda: F.scene_predictions(*args, utils.load_ids(gt_file), tmp, scene), 3)
    same = np.array_equal(u1, u2) and np.array_equal(c1, c2) and all(
        a[1:3] == b[1:3] and np.array_equal(a[3], b[3]) for a, b in zip(p1, p2)) and len(p1) == len(p2)
    return dict(fused_annotations_s=t_ann, fused_gt_file_s=t_file, same_counts=bool(same))


def kernel_time(p, scene, iters):
    lm = utils.read_label_mapping(p["tsv"])
    lm2 = utils.read_label_mapping(p["csv"], label_from="nyu40id", label_to="mappedIdConsecutive", delimiter=",")
    gt = A.read_scene_gt(p["agg"], p["seg"], lm, lm2, "instance", scene)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = [dev(gt.seg_index), dev(gt.seg_ids), dev(gt.seg_slot)]
    slot = torch.empty(len(gt.seg_index), dtype=torch.int32, device="cuda")
    count = torch.empty(len(gt.slot_ids), dtype=torch.int64, device="cuda")
    h = S.stream()

    def run():
        S.check(S.lib.sis3d_segment_gt_slots(S.ptr(t[0]), len(gt.seg_index), S.ptr(t[1]), S.ptr(t[2]), len(gt.seg_ids),
                                             len(gt.slot_ids), S.ptr(slot), S.ptr(count), h), "segment_gt_slots")
    for _ in range(10):
        run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    ok = np.array_equal(slot.cpu().numpy(), A.gt_ids_host(gt)[1])
    return dict(kernel_us=a.elapsed_time(b) * 1000 / iters, segments=len(gt.seg_ids), slots=len(gt.slot_ids),
                slots_equal_host=bool(ok))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--verts", type=int, nargs="+", default=[150000, 300000])
    ap.add_argument("--boxes", type=int, default=100)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the kernel timings need a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("device:", torch.cuda.get_device_name(0), "|", q.stdout.strip())
    for nv in a.verts:
        with tempfile.TemporaryDirectory() as tmp:
            c = B.make_scene(nv * 3 + a.boxes, nv, a.boxes)
            scene, p = write_scene(tmp, c, nv)
            ex, gt_file = export_times(tmp, scene, p)
            rec = dict(vertices=nv, boxes=a.boxes, objects=p["n_groups"], **ex, **fused_times(tmp, scene, p, gt_file),
                       **kernel_time(p, scene, a.iters))
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
