"""Cost of test mode's mask mAP on the GPU (one JSON line on stdout; --out FILE also writes it there).

  1. sis3d_mask_overlap kernel time (CUDA events over back-to-back launches) at the cfg2 scene size (96x48x96, ~30 kept
     masks x ~12 GT) and at the whole-scene size 208x48x160 (~100 x ~40); masks are random crops at random places;
  2. the same counts from a vectorised numpy host version (count_nonzero per mask and over each intersecting pair's common
     box), on the same masks;
  3. scenes/s of run_scenes with and without the evaluator (test vs benchmark mode) on the same synthetic cfg2 chunks,
     alternated in one process.

    python tools/bench_eval.py [--reps 3] [--scenes 48] [--out FILE]

Writes nothing into the tree (result files go to a temporary directory)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-sis_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (v.strip() for v in q.split(","))
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def random_masks(rng, dims, n, max_ext, p):
    boxes, masks = [], []
    for _ in range(n):
        ext = rng.integers(4, np.minimum(max_ext, dims) + 1)
        lo = rng.integers(0, np.asarray(dims) - ext + 1)
        boxes.append(np.concatenate([lo, lo + ext]))
        masks.append((rng.random(tuple(ext)) < p).astype(np.uint8))
    return np.array(boxes, np.int32), masks


def host_counts(pm, pbox, gm, gbox, pairs):
    """Vectorised numpy: the masks stay at their boxes, each pair counts over the common box only."""
    pc = np.array([np.count_nonzero(m) for m in pm], np.int64)
    gc = np.array([np.count_nonzero(m) for m in gm], np.int64)
    inter = np.zeros((len(pm), len(gm)), np.int64)
    for i, j in pairs:
        lo, hi = np.maximum(pbox[i, :3], gbox[j, :3]), np.minimum(pbox[i, 3:], gbox[j, 3:])
        a = pm[i][lo[0] - pbox[i, 0]:hi[0] - pbox[i, 0], lo[1] - pbox[i, 1]:hi[1] - pbox[i, 1], lo[2] - pbox[i, 2]:hi[2] - pbox[i, 2]]
        b = gm[j][lo[0] - gbox[j, 0]:hi[0] - gbox[j, 0], lo[1] - gbox[j, 1]:hi[1] - gbox[j, 1], lo[2] - gbox[j, 2]:hi[2] - gbox[j, 2]]
        inter[i, j] = np.count_nonzero(a & b)
    return pc, gc, inter


def kernel_case(dims, n_pred, n_gt, max_ext, iters=2000):
    from lib import _sis3d as S
    from lib.utils import evaluation as E
    rng = np.random.default_rng(11)
    pbox, pm = random_masks(rng, dims, n_pred, max_ext, 0.6)
    gbox, gm = random_masks(rng, dims, n_gt, max_ext, 0.7)
    pb, po, _ = E.pack_masks(pm, pbox, dims, "predicted")
    gb, go, _ = E.pack_masks(gm, gbox, dims)
    pairs = E.box_pairs(pbox, gbox)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = [dev(pb), dev(po), dev(pbox), dev(gb), dev(go), dev(gbox), dev(pairs)]
    out = torch.empty(n_pred + n_gt + len(pairs), dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream()
    import ctypes as C
    h = C.c_void_p(st.cuda_stream)

    def launch():
        S.check(S.lib.sis3d_mask_overlap(S.ptr(t[0]), S.ptr(t[1]), S.ptr(t[2]), n_pred, S.ptr(t[3]), S.ptr(t[4]), S.ptr(t[5]),
                                         n_gt, S.ptr(t[6]), len(pairs), S.ptr(out), S.ptr(out[n_pred:]),
                                         S.ptr(out[n_pred + n_gt:]), h))
    for _ in range(50):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        launch()
    b.record()
    torch.cuda.synchronize()
    kernel_us = a.elapsed_time(b) * 1e3 / iters
    res = E.launch_mask_overlap(t[0], po, pbox, gb, go, gbox).result()  # the production path, checked against the host
    t0 = time.perf_counter()
    reps = 20
    for _ in range(reps):
        want = host_counts(pm, pbox, gm, gbox, pairs)
    host_us = (time.perf_counter() - t0) * 1e6 / reps
    assert all(np.array_equal(x, y) for x, y in zip(res, want)), "kernel counts differ from the host counts"
    return dict(dims=list(dims), n_pred=n_pred, n_gt=n_gt, n_pairs=int(len(pairs)), kernel_us=round(kernel_us, 2),
                host_numpy_us=round(host_us, 1))


def loop_rates(n_scenes, reps):
    import sis3d_synth as synth
    from lib.datasets.dataset import Dataset, collate_fn
    from lib.datasets.prefetch import Prefetcher
    from lib.model.trainval import SceneEvaluator, run_scenes
    c = synth.CASES["cfg2_96x48x96"]
    net, cfg = synth.make_net(c, keep_debug=False, math="exact")
    with tempfile.TemporaryDirectory() as tmp:
        paths, provider = synth.write_chunks(tmp, c, range(1000, 1000 + n_scenes))
        ds = Dataset(paths, "test", view_provider=provider, device_decode=True)

        def run(evaluate, k):
            out = os.path.join(tmp, f"out_{k}")
            loader = (collate_fn([it]) for it in Prefetcher((ds[i] for i in range(len(ds))), depth=6))
            ev = SceneEvaluator() if evaluate else None
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = run_scenes(net, loader, out, evaluator=ev)
            lines = ev.summary() if ev else []
            torch.cuda.synchronize()
            return n / (time.perf_counter() - t0), lines
        run(True, "warm_t")
        run(False, "warm_b")
        rates = {"test": [], "benchmark": []}
        lines = None
        for r in range(reps):
            for mode in (("test", "benchmark") if r % 2 == 0 else ("benchmark", "test")):
                rate, ln = run(mode == "test", f"{mode}_{r}")
                rates[mode].append(round(rate, 1))
                lines = ln or lines
    return dict(scenes=n_scenes, scenes_per_s=rates, summary=lines[:2] if lines else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scenes", type=int, default=48)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_eval measures the GPU: no device found"
    name, power = card()
    res = dict(gpu=name, power_limit=power,
               kernel=[kernel_case((96, 48, 96), 30, 12, (24, 20, 24)), kernel_case((208, 48, 160), 100, 40, (32, 24, 32))])
    res["loop"] = loop_rates(a.scenes, a.reps)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
