"""Which kernel every layer runs on, in every conv math mode: one eager forward per (config, mode) with per-kernel timing
on (`net._prof = {}`: no CUDA graph, no parallel branches), recording

  - the ordered `_rec` timing names (`conv_tc_h3[geometry1.2.conv1]`, `conv[color.4]`, `mask_stage`, ...),
  - the libsis3d kernel launches of the forward (`kernel_launches()` delta),
  - the conv3d_k3_tc_kernel instances the mask stage launches, read through torch.profiler.

tests/golden/conv_routes.json holds this output; tests/test_gpu_conv_routes.py reruns it and requires the same, and
tests/test_pack_plan.py checks on the CPU that every pack these routes read is planned.

  python tools/capture_routes.py OUT.json
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "3d-sis_b200"), ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import sis3d_synth as synth  # noqa: E402
from lib.nets.network import Network  # noqa: E402

# the cfg2 and cfg5 bench scenes, and the cfg2 scene on its ground-truth boxes (USE_RPN = USE_CLASS = False)
CONFIGS = {
    "cfg2": dict(cfgname="scannet", dims=(96, 48, 96), n_img=5, seed=1000, gt_rois=None),
    "cfg5": dict(cfgname="suncg", dims=(96, 48, 96), n_img=3, seed=5000, gt_rois=None),
    "gt_rois": dict(cfgname="scannet", dims=(96, 48, 96), n_img=5, seed=1000, gt_rois=True),
}


def blobs_of(c):
    data, boxes = synth.make_scene(c["seed"], c["dims"])
    views = synth.make_views(c["seed"], c["dims"], c["n_img"], boxes)
    blobs = synth.make_blobs(dict(cfgname=c["cfgname"], use_images=True), data, views)
    if c["gt_rois"]:
        cls = (np.arange(len(boxes)) % 18 + 1).astype(np.float32)[:, None]
        blobs["gt_box"] = [torch.from_numpy(np.concatenate([boxes, cls], 1).astype(np.float32))]
    return blobs


def capture_case(c, mode):
    import test_gpu_mask_stage as T
    net, _ = synth.make_net(dict(cfgname=c["cfgname"], use_images=True, use_mask=True), keep_debug=False, math=mode,
                            gt_rois=c["gt_rois"])
    blobs = blobs_of(c)
    net._ensure_packed()
    net._prof = {}
    names, rec = [], net._rec
    net._rec = lambda name: (names.append(name), rec(name))[1]
    n0 = net.kernel_launches()
    P = net.forward(blobs, "TEST", None)
    torch.cuda.synchronize()
    launches = net.kernel_launches() - n0
    routes = list(names)
    det = P["detections_host"]
    n_masks = len(P["mask_pred"][0])
    want = T.expected_kernels(T.MASK_MATH_ROUTE[net._mask_math])
    found = T._launched(lambda: net._mask_branch(net._scene, det, det.shape[0]), want)
    return dict(routes=routes, kernel_launches=int(launches), n_masks=n_masks,
                mask_tc_instances=None if found is None else [list(i) for i in found[1]])


def capture():
    return {f"{name}/{mode}": capture_case(c, mode) for name, c in CONFIGS.items() for mode in Network.MATH_MODES}


if __name__ == "__main__":
    out = capture()
    with open(sys.argv[1], "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    for k, v in out.items():
        print(k, len(v["routes"]), "rec names,", v["kernel_launches"], "launches,", v["n_masks"], "masks,",
              v["mask_tc_instances"])
