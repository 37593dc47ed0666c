"""Scenes/s of the test loop on ground-truth boxes and classes (USE_RPN = USE_CLASS = False, USE_BACKBONE off) next to the
normal detection forward, on the same scenes: 96x48x96 ScanNet-shape chunks with 5 views and their own boxes (the cfg2
workload of bench.py), and the 208x48x160 whole scene with 40 views and 40 or 100 ground-truth boxes.  Both run through
Network.forward_pipelined in the default math mode; the timed window ends in a device synchronise.

    python tools/bench_gt_rois.py [--scenes 96] [--warmup 24]

Prints one JSON line per workload and mode, with the GPU's name, power limit and SM clock limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-sis_b200"))
import sis3d_synth as synth  # noqa: E402


def gt_boxes(n, dims, seed, own=None):
    rng = np.random.default_rng(seed + 11)
    if own is not None:
        b = np.asarray(own, np.float32)
    else:
        size = rng.uniform(4, 40, (n, 3))
        lo = rng.uniform(0, 1, (n, 3)) * (np.array(dims) - 4)
        b = np.concatenate([lo, np.minimum(lo + size, dims)], 1)
    return np.concatenate([b, rng.integers(1, 19, (len(b), 1))], 1).astype(np.float32)


def workloads():
    yield "cfg2_96x48x96_5img_own_boxes", [((96, 48, 96), 5, 1000 + j, None) for j in range(24)]
    for n in (40, 100):
        yield f"scene_208x48x160_40img_{n}_boxes", [((208, 48, 160), 40, 3000 + j, n) for j in range(4)]


def scenes(spec):
    out = []
    for dims, n_img, seed, n in spec:
        data, boxes = synth.make_scene(seed, dims)
        views = synth.make_views(seed, dims, n_img, boxes)
        b = synth.make_blobs(dict(use_images=True), data, views, pin=True)
        b["gt_box"] = [torch.from_numpy(gt_boxes(n, dims, seed, boxes if n is None else None))]
        out.append(b)
    return out


def rate(net, blobs, n, warmup):
    seq = lambda k: (blobs[i % len(blobs)] for i in range(k))
    kept = 0
    for _, P in net.forward_pipelined(seq(warmup)):
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _, P in net.forward_pipelined(seq(n)):
        kept += int((P["detections_host"][:, 8] > 0.5).sum())
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0), kept / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=96)
    ap.add_argument("--warmup", type=int, default=24)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gt_rois.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    c = dict(cfgname="scannet", use_images=True, use_mask=True)
    for name, spec in workloads():
        blobs = scenes(spec)
        for mode in ("detections", "gt_rois"):
            net, _ = synth.make_net(c, keep_debug=False, math="exact", gt_rois=False if mode == "gt_rois" else None)
            sps, kept = rate(net, blobs, a.scenes if "cfg2" in name else a.scenes // 4, a.warmup)
            print(json.dumps(dict(workload=name, mode=mode, scenes_per_sec=round(sps, 2), kept_per_scene=round(kept, 1),
                                  math="exact", gpu=gpu)), flush=True)
            del net
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
