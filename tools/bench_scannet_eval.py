"""Per-scene cost of turning voxel predictions into the ScanNet instance-AP counts, two ways (not bench.py):

  (a) file route: vox2mesh.paint_instances + export (per-vertex 0/1 text files), then the evaluator's
      assign_instances_for_scan reading them back;
  (b) fused route, host part: packing the masks, np.unique of the GT ids, decoding the boxes and assign_instances;
      and the whole fused call (one H2D copy, both kernels, one D2H copy, synchronised);
  (c) the two kernels alone (sis3d_instance_paint + sis3d_vertex_instance_overlap), CUDA events over many launches on
      resident inputs, their counts checked against the host's vertex_labels + bincount in the same run.

Synthetic scenes on the 400x200x400 canvas: boxes inside a 208x48x160 region, masks of density 0.6, vertices around the
boxes and scattered over the region, GT ids from shifted boxes.  Prints the card name and power limit, then one JSON line
per configuration.

    python tools/bench_scannet_eval.py [--verts 50000 150000 300000] [--boxes 30 100] [--iters 200]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "3d-sis_b200"), ROOT]

from lib import _sis3d as S  # noqa: E402
from tools.scannet_benchmark import evaluate_predictions as F  # noqa: E402
from tools.scannet_benchmark import evaluate_semantic_instance as E  # noqa: E402
from tools.scannet_benchmark import vox2mesh as V  # noqa: E402

REGION = np.array([208, 48, 160])


def make_scene(seed, n_vert, n_box):
    rng = np.random.default_rng(seed)
    base = np.array([96, 40, 120])
    box, masks = [], []
    for _ in range(n_box):
        lo = base + rng.integers(0, REGION - 24) + rng.choice([0.0, 0.5, -0.3], 3)
        hi = lo + rng.integers(6, 24, 3)
        box.append(np.concatenate([lo, hi]))
        shape = tuple(np.rint(hi).astype(int) - np.rint(lo).astype(int))
        masks.append((rng.random(shape) < 0.6).astype(np.float32))
    box = np.array(box, np.float32)
    cls = rng.integers(1, 19, n_box)
    conf = rng.uniform(0.05, 0.99, n_box)
    w2g = np.eye(4)
    w2g[:3, :3] *= 1 / 0.046875
    w2g[:3, 3] = rng.uniform(-2, 2, 3)
    near = rng.integers(0, n_box, n_vert // 2)
    g = np.concatenate([rng.integers(np.rint(box[near, :3]).astype(int) - 1, np.rint(box[near, 3:]).astype(int) + 1),
                        base + rng.integers(0, REGION, (n_vert - len(near), 3))]).astype(np.float64)
    grid = g + rng.uniform(-0.4, 0.4, g.shape)
    verts = ((grid - w2g[:3, 3]) * 0.046875).astype(np.float32)
    gi = g.astype(np.int64)
    gt = np.zeros(n_vert, np.int64)
    for b in range(n_box):
        lo, hi = np.rint(box[b, :3]).astype(int) + rng.integers(-1, 2, 3), np.rint(box[b, 3:]).astype(int) + rng.integers(-1, 2, 3)
        gt[np.all((gi >= lo) & (gi < hi), axis=1) & (gt == 0)] = int(rng.integers(1, 19)) * 1000 + b + 1
    return dict(box=box, cls=cls, conf=conf, masks=masks, w2g=w2g, verts=verts, gt=gt)


def timed(f, reps=1):
    t0 = time.perf_counter()
    for _ in range(reps):
        r = f()
    return r, (time.perf_counter() - t0) / reps


def file_route(c, tmp):
    scene, t_paint = timed(lambda: V.paint_instances(c["box"], c["cls"], c["conf"], c["masks"]))
    gt_file = os.path.join(tmp, "gt", "scene0000_00.txt")
    os.makedirs(os.path.dirname(gt_file), exist_ok=True)
    np.savetxt(gt_file, c["gt"], fmt="%d")
    out = os.path.join(tmp, "bench")
    _, t_export = timed(lambda: V.export(c["verts"], c["w2g"], scene, out, "scene0000_00"))
    (_, pred2gt), t_eval = timed(lambda: E.assign_instances_for_scan(os.path.join(out, "scene0000_00.txt"), gt_file, out))
    lines = sum(1 for _ in open(os.path.join(out, "scene0000_00.txt")))
    shutil.rmtree(out)
    return dict(paint_s=t_paint, export_s=t_export, evaluator_read_s=t_eval, instances=lines,
                text_lines=lines * len(c["verts"])), pred2gt


def fused_host(c):
    values = F.box_values(c["cls"], c["conf"])
    bits, offs, ibox, lo, ext = F.pack_boxes(c["box"], values, c["masks"])
    uniq, slot, counts = np.unique(c["gt"], return_inverse=True, return_counts=True)
    return values, bits, offs, ibox, lo, ext, uniq, slot.astype(np.int32), counts


def fused_route(c):
    (values, bits, offs, ibox, lo, ext, uniq, slot, counts), t_pack = timed(lambda: fused_host(c), 3)
    (hist, first, _), t_call = timed(lambda: F.vertex_instance_overlap(c["verts"], c["w2g"], slot, len(uniq), bits, offs, ibox,
                                                                       lo, ext), 5)

    def assign():
        preds = [(f"m{i}", cl, conf, h) for i, cl, conf, h in F.decode_instances(values, hist, first)]
        return E.assign_instances(uniq, counts, preds)
    (_, pred2gt), t_assign = timed(assign, 3)
    return dict(pack_unique_s=t_pack, device_call_s=t_call, decode_assign_s=t_assign,
                host_part_s=t_pack + t_assign), pred2gt


def kernels(c, iters):
    values, bits, offs, ibox, lo, ext, uniq, slot, counts = fused_host(c)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = [dev(c["verts"]), dev(c["w2g"].astype(np.float64)), dev(slot), dev(offs), dev(ibox), dev(bits)]
    n_vert, n_box, n_slot = len(c["verts"]), len(offs), len(uniq)
    owner = torch.empty(int(np.prod(ext)), dtype=torch.int32, device="cuda")
    res = torch.empty(n_box * n_slot + n_box + n_vert, dtype=torch.int64, device="cuda")
    first = res[n_box * n_slot:n_box * n_slot + n_box].view(torch.int32)
    vbox = res[n_box * n_slot + n_box:].view(torch.int32)
    h = S.stream()
    li, ex = [int(v) for v in lo], [int(v) for v in ext]

    def paint():
        S.check(S.lib.sis3d_instance_paint(S.ptr(t[5]), S.ptr(t[3]), S.ptr(t[4]), n_box, *li, *ex, S.ptr(owner), h), "paint")

    def overlap(with_box):
        S.check(S.lib.sis3d_vertex_instance_overlap(S.ptr(t[0]), n_vert, S.ptr(t[1]), S.ptr(owner), *li, *ex, *V.SCENE_DIMS,
                                                    S.ptr(t[2]), n_slot, n_box, S.ptr(res), S.ptr(first),
                                                    S.ptr(vbox) if with_box else None, h), "overlap")
    times = {}
    for name, f in (("paint_us", paint), ("overlap_us", lambda: overlap(False))):
        for _ in range(10):
            f()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            f()
        b.record()
        torch.cuda.synchronize()
        times[name] = a.elapsed_time(b) * 1000 / iters
    paint()
    overlap(True)
    torch.cuda.synchronize()
    r = res.cpu().numpy()
    hist = r[:n_box * n_slot].reshape(n_box, n_slot)
    got_box = r[n_box * n_slot + n_box:].view(np.int32)[:n_vert]
    scene = V.paint_instances(c["box"], c["cls"], c["conf"], c["masks"])
    value, valid = V.vertex_labels(c["verts"], c["w2g"], scene)
    want_box = np.full(n_vert, -1)
    for b, v in enumerate(values):
        want_box[valid & (value == v)] = b
    want_hist = np.zeros_like(hist)
    np.add.at(want_hist, (want_box[valid], slot[valid]), 1)
    times.update(owner_voxels=int(np.prod(ext)), labelled_vertices=int(valid.sum()),
                 label_disagreements=int((got_box != want_box).sum()), counts_equal=bool(np.array_equal(hist, want_hist)))
    return times


def same_pred2gt(a, b):
    strip = lambda p2g: [[(p["label_id"], p["vert_count"], p["confidence"], p["void_intersection"],
                           [(g["instance_id"], g["intersection"]) for g in p["matched_gt"]]) for p in p2g[k]] for k in sorted(p2g)]
    return strip(a) == strip(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--verts", type=int, nargs="+", default=[50000, 150000, 300000])
    ap.add_argument("--boxes", type=int, nargs="+", default=[30, 100])
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the kernel timings need a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("device:", torch.cuda.get_device_name(0), "|", q.stdout.strip())
    with tempfile.TemporaryDirectory() as tmp:
        for nv in a.verts:
            for nb in a.boxes:
                c = make_scene(nv * 7 + nb, nv, nb)
                fused, p_fused = fused_route(c)
                k = kernels(c, a.iters)
                files, p_file = file_route(c, tmp)
                rec = dict(vertices=nv, boxes=nb, file_route=files, fused=fused, kernels=k,
                           same_counts_both_routes=same_pred2gt(p_file, p_fused))
                print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
