"""Scenes/s of the colour-aware mask head next to the default ScanNet net, on the same seeded scenes: the default net, the
MASK_USE_IMAGES net and the MASK_ONLY_IMAGES net, on the cfg2 workload of bench.py (96x48x96, 5 views) and the 208x48x160
whole scene with 40 views.  All nets run Network.forward_pipelined in `exact` math on pinned inputs, in one process, the
arms alternating window by window; each timed window ends in a device synchronise.  Before timing, each arm's pipelined
outputs are checked bit for bit against its synchronous forward on the same scenes.

    python tools/bench_mask_images.py [--scenes 96] [--warmup 24] [--rounds 3]

Prints one JSON line per workload and arm (median and spread over the rounds, kept crops per scene), with the GPU's name,
power limit and SM clock limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-sis_b200"))
import sis3d_synth as synth  # noqa: E402

C = dict(cfgname="scannet", use_images=True, use_mask=True)


def workloads():
    yield "cfg2_96x48x96_5img", [((96, 48, 96), 5, 1000 + j) for j in range(24)]
    yield "scene_208x48x160_40img", [((208, 48, 160), 40, 3000 + j) for j in range(4)]


def scenes(spec):
    out = []
    for dims, n_img, seed in spec:
        data, boxes = synth.make_scene(seed, dims)
        out.append(synth.make_blobs(C, data, synth.make_views(seed, dims, n_img, boxes), pin=True))
    return out


def snap(P):
    return (P["detections_host"].copy(), P["rois"][0].cpu().clone(), [m.cpu().clone() for m in P["mask_pred"][0]])


def same(a, b):
    return (np.array_equal(a[0].view(np.int32), b[0].view(np.int32)) and torch.equal(a[1], b[1]) and len(a[2]) == len(b[2])
            and all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a[2], b[2])))


def check(net, blobs):
    want = [snap(net.forward(b, "TEST", None)) for b in blobs]
    got = [snap(P) for _, P in net.forward_pipelined(iter(blobs))]
    if len(got) != len(want) or not all(same(a, b) for a, b in zip(got, want)):
        raise SystemExit("forward_pipelined differs from forward")


def window(net, blobs, n):
    seq = (blobs[i % len(blobs)] for i in range(n))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    kept = 0
    for _, P in net.forward_pipelined(seq):
        kept += int((P["detections_host"][:, 8] > 0.5).sum())
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0), kept / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=96)
    ap.add_argument("--warmup", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mask_images.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    # the nets live in one process: a colour-aware net stays so whatever the global cfg says later
    nets = {arm: synth.make_net(C, keep_debug=False, math="exact", mask_images=mi)[0]
            for arm, mi in (("default", None), ("mask_use_images", "use"), ("mask_only_images", "only"))}
    for name, spec in workloads():
        blobs = scenes(spec)
        n = a.scenes if "cfg2" in name else max(a.scenes // 4, 8)
        for net in nets.values():
            check(net, blobs)
            window(net, blobs, a.warmup)
        rates = {arm: [] for arm in nets}
        for _ in range(a.rounds):
            for arm, net in nets.items():
                rates[arm].append(window(net, blobs, n))
        for arm, r in rates.items():
            v = [x[0] for x in r]
            print(json.dumps(dict(workload=name, arm=arm, scenes_per_sec=round(statistics.median(v), 2),
                                  spread=round((max(v) - min(v)) / statistics.median(v), 3), all_rounds=[round(x, 2) for x in v],
                                  kept_per_scene=round(r[0][1], 1), math="exact", gpu=gpu)), flush=True)
        del blobs


if __name__ == "__main__":
    main()
