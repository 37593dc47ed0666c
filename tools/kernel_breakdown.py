#!/usr/bin/env python
"""Per-kernel device-time breakdown of the cfg2 scene loop (torch.profiler, CUDA activities).
  python tools/kernel_breakdown.py --out DIR [--scenes 48] [--math exact]   (GPU box)
Runs Network.forward_pipelined (7 scenes in flight, device-resident inputs, as bench.py's `value`) over the 24 cfg2 scenes
(96x48x96, 5 views), warms it up unprofiled, then profiles `--scenes` scenes in a run of its own.  Kernel events are
grouped by their full (templated) name.  Writes DIR/kernel_breakdown.txt (one row per kernel instantiation: us per scene,
launches per scene, share of the summed kernel time) and DIR/kernel_breakdown.json; prints the table.  Tracing slows the
host, so the times are device times of each kernel, not an end-to-end rate: take that from bench.py."""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "3d-sis_b200"), ROOT):
    sys.path.insert(0, p)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import sis3d_synth as synth  # noqa: E402

DIMS, N_IMG = (96, 48, 96), 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--scenes", type=int, default=48)
    ap.add_argument("--math", default="exact")
    ap.add_argument("--top", type=int, default=40, help="rows printed (the files list every kernel)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kernel_breakdown needs a GPU")
    dev = torch.device("cuda", 0)
    case = dict(cfgname="scannet", dims=DIMS, n_img=N_IMG, seed=0, use_images=True, use_mask=True)
    net = synth.make_net(case, keep_debug=False, math=a.math)[0]
    inputs = []
    for j in range(24):  # the scenes of bench.py's cfg2 workload (rank 0)
        data, boxes = synth.make_scene(1000 + j, DIMS)
        hb = synth.make_blobs(None, data, synth.make_views(1000 + j, DIMS, N_IMG, boxes), pin=True)
        ni = hb["nearest_images"]
        inputs.append({"data": hb["data"].to(dev), "id": hb["id"],
                       "nearest_images": {"images": [ni["images"][0].to(dev)], "depths": [ni["depths"][0].to(dev)],
                                          "poses": ni["poses"], "world2grid": ni["world2grid"]}})

    def run(n):
        for _ in net.forward_pipelined(inputs[k % len(inputs)] for k in range(n)):
            pass
        for sl in net._slots:
            if sl["stream"] is not None:
                torch.cuda.current_stream().wait_stream(sl["stream"])
        torch.cuda.synchronize()

    run(48)  # warm-up: module loads, graph captures of the pipeline slots
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(a.scenes)
    tot = collections.defaultdict(float)
    cnt = collections.Counter()
    iv = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")):
            tot[e.name] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            cnt[e.name] += 1
            iv.append((e.time_range.start, e.time_range.end))
    summed = sum(tot.values())
    # span of the profiled kernels and the part of it in which at least one kernel ran (the rest: the device waited on the
    # host or on copies; tracing slows the host, so this is a lower bound on how busy the untraced loop keeps the device)
    iv.sort()
    busy, (s0, e0) = 0.0, iv[0]
    for s, e in iv[1:]:
        if s > e0:
            busy, s0, e0 = busy + e0 - s0, s, e
        else:
            e0 = max(e0, e)
    busy += e0 - s0
    span = iv[-1][1] - iv[0][0]
    rows = sorted(tot, key=lambda k: -tot[k])
    table = [dict(kernel=k, us_per_scene=tot[k] / a.scenes, launches_per_scene=cnt[k] / a.scenes, share=tot[k] / summed)
             for k in rows]
    props = torch.cuda.get_device_properties(0)
    head = (f"{props.name}, math={a.math}, {a.scenes} cfg2 scenes profiled; summed kernel time "
            f"{summed / a.scenes:.1f} us per scene over {sum(cnt.values()) / a.scenes:.1f} launches; kernel span "
            f"{span / a.scenes:.1f} us per scene, some kernel running in {100 * busy / span:.1f} % of it")
    lines = [head, f"{'us/scene':>9} {'launch/sc':>9} {'share':>6}  kernel"]
    lines += [f"{r['us_per_scene']:9.2f} {r['launches_per_scene']:9.2f} {100 * r['share']:5.1f}%  {r['kernel']}" for r in table]
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "kernel_breakdown.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    with open(os.path.join(a.out, "kernel_breakdown.json"), "w") as f:
        json.dump(dict(device=props.name, math=a.math, scenes=a.scenes, summed_us_per_scene=summed / a.scenes,
                       span_us_per_scene=span / a.scenes, busy_fraction=busy / span, kernels=table), f, indent=1)
    print("\n".join(lines[:a.top + 2]))


if __name__ == "__main__":
    main()
