"""oracle/make_golden_scannet_eval.py -- TEST INFRASTRUCTURE ONLY; runs ONLY in the build container (needs the reference tree).

Runs the reference's UNMODIFIED tools/scannet_benchmark/evaluate_semantic_instance.py (with its utils.py) in this process
under three shims -- a stub `plyfile` module (its utils.py imports it; only read_mesh_vertices uses it), the `np.float` /
`np.bool` aliases numpy 2 removed (they meant the builtins), and `sys.argv` set for its import-time parse_args -- and stores
what it computes in tests/golden/scannet_instance_eval_reference.npz, which pins tools/scannet_benchmark/
evaluate_semantic_instance.py, vox2mesh.py's command line and evaluate_predictions.py (tests/test_scannet_eval*.py).

    python oracle/make_golden_scannet_eval.py

Two kinds of input, both regenerated from seeds by the functions below (the tests import them; nothing of the reference is
involved in making them):
- text sets (make_text_set): per-vertex GT id files and prediction files with 0/1 mask files, fed to the evaluator directly;
- chain sets (make_chain_set): prediction folders as the benchmark mode writes them, mesh vertices, world2grid.txt and GT id
  files, fed through the reference vox2mesh functions (make_golden_vox2mesh.reference_functions: load_matrix, load_pred,
  export) and then the evaluator.

The sets cover overlapping predictions, a GT matched twice (the lower score becomes a false positive), groups (ids < 1000),
small GT, void labels including id 0, predictions under 100 vertices, invalid label ids, tied confidences across scenes, a
class with GT only and classes with neither, the empty-curve branch (a class with GT and predictions where nothing
survives), a scene with an empty prediction file, a box with confidence below 0.01 (its class decodes as class - 1 and its
instance id can collide with the previous box's), and vertices outside the 400x200x400 canvas.  Chain vertices outside the
canvas sit at negative grid coordinates far from every box: the reference indexes the volume with them (numpy wraps a
negative index round to the far end, which is empty), this repo skips them, and both leave them unlabelled.  Every vertex
is at least 0.1 voxel away from a half-integer grid coordinate, so fp64 rounding cannot flip its voxel.

Layout (keys; k = set name): k_ap (float64 [1, 18, 10]), k_all_ap / k_all_ap_50 / k_all_ap_25, k_class_ap (float64 [18, 3]:
ap, ap50, ap25 per class), k_stdout (everything the evaluator printed), k_csv (the result file's text).
"""
from __future__ import annotations

import contextlib
import importlib.util
import io
import os
import pickle
import sys
import tempfile
import types

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
REF = os.environ.get("SIS3D_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "scannet_instance_eval_reference.npz")

CONFS = [0.55, 0.6, 0.7, 0.8, 0.9, 0.95]  # a short list: confidences tie within and across scenes
VOXEL = 0.046875
PADDING = np.array([10, 16, 10, 0])  # what vox2mesh.load_matrix subtracts from the translation column


# ------------------------------------------------------------------------------------------------------------ text sets
def _span(n, a, b):
    m = np.zeros(n, bool)
    m[a:b] = True
    return m


def handmade_text_set():
    """-> {scene: (gt_ids int64 [n], [(mask bool [n], label text, confidence text), ...])}"""
    sets = {}
    n = 1500
    gt = np.zeros(n, np.int64)
    gt[0:300], gt[300:500], gt[500:560], gt[560:860] = 3001, 3002, 5001, 5002  # chair, chair, small table, table
    gt[860:960], gt[960:1100], gt[1100:1250], gt[1250:1500] = 7, 0, 25001, 1001  # group, void, invalid class, cabinet
    preds = [
        (_span(n, 0, 300), "3", "0.9"),                                      # exactly GT 3001
        (_span(n, 0, 300) | _span(n, 960, 1010), "3", "0.8"),                # 3001 again: IoU 0.857 -> lower score is an FP
        (_span(n, 300, 420) | _span(n, 860, 960) | _span(n, 1100, 1150), "3.0", "0.7"),  # 3002 weakly, group + void
        (_span(n, 500, 700), "5", "0.6"),                                    # small table GT + table: IoU 0.389
        (_span(n, 560, 640), "5", "0.95"),                                   # 80 vertices: dropped before its pred_id
        (_span(n, 0, 500), "0", "0.9"),                                      # invalid labels
        (_span(n, 0, 500), "19", "0.9"),
        (_span(n, 1240, 1500), "1", "0.95"),                                 # cabinet
        (_span(n, 960, 1250), "4", "0.8"),                                   # sofa on void only: always ignored
    ]
    sets["scene0000_00"] = (gt, preds)
    n = 1200
    gt = np.zeros(n, np.int64)
    gt[0:150], gt[150:400], gt[400:700] = 4001, 11001, 3001  # sofa (never matched), desk (no prediction), chair
    sets["scene0001_00"] = (gt, [(_span(n, 400, 690), "3", "0.9"),           # ties with scene0000_00's 0.9
                                 (_span(n, 150, 300), "3", "0.7")])          # chair on a desk: a false positive
    n = 600
    gt = np.zeros(n, np.int64)
    gt[0:200], gt[200:450] = 3003, 1002
    sets["scene0002_00"] = (gt, [])                                          # empty prediction file
    return sets


def random_text_set(seed, n_scenes=5):
    rng = np.random.default_rng(seed)
    sets = {}
    for s in range(n_scenes):
        n = int(rng.integers(2000, 4000))
        gt = np.zeros(n, np.int64)
        o, objs = 0, []
        while o < n:
            size = int(rng.integers(40, 500))
            kind = rng.random()
            if kind < 0.12:
                gid = 0
            elif kind < 0.2:
                gid = int(rng.integers(1, 999))  # group
            elif kind < 0.26:
                gid = int(rng.integers(19, 40)) * 1000 + len(objs) + 1  # invalid class
            else:
                gid = int(rng.integers(1, 19)) * 1000 + len(objs) + 1
            gt[o:o + size] = gid
            objs.append((o, min(o + size, n), gid))
            o += size
        perm = rng.permutation(n)  # instances scattered over the vertex order
        gt = gt[perm]
        preds = []
        for a, b, gid in objs:
            for _ in range(int(rng.integers(0, 3))):
                m = np.zeros(n, bool)
                lo = a + int(rng.integers(-60, 60))
                hi = b + int(rng.integers(-60, 60))
                m[max(lo, 0):max(min(hi, n), 0)] = True
                m ^= rng.random(n) < 0.01
                label = gid // 1000 if gid >= 1000 and rng.random() < 0.8 else int(rng.integers(0, 21))
                text = str(label) if rng.random() < 0.8 else f"{label}.0"
                preds.append((m[perm], text, repr(float(rng.choice(CONFS)))))
        order = rng.permutation(len(preds))
        sets[f"scene{s:04d}_00"] = (gt, [preds[i] for i in order])
    return sets


def write_text_set(sets, pred_dir, gt_dir):
    os.makedirs(os.path.join(pred_dir, "predicted_masks"), exist_ok=True)
    os.makedirs(gt_dir, exist_ok=True)
    for scene, (gt, preds) in sets.items():
        np.savetxt(os.path.join(gt_dir, scene + ".txt"), gt, fmt="%d")
        with open(os.path.join(pred_dir, scene + ".txt"), "w") as f:
            for i, (m, label, conf) in enumerate(preds):
                rel = f"predicted_masks/{scene}_{i:03d}.txt"
                np.savetxt(os.path.join(pred_dir, rel), m.astype(np.uint8), fmt="%u")
                f.write(f"{rel} {label} {conf}\n")


# ------------------------------------------------------------------------------------------------------------ chain sets
def make_chain_scene(rng, n_box, conf_low=None):
    """Prediction-folder arrays, mesh vertices (float32) and the unpadded world2grid of one scene on the reference's
    400x200x400 canvas, with per-vertex GT ids from boxes near the predicted ones."""
    base = np.array([rng.integers(20, 300), rng.integers(20, 120), rng.integers(20, 300)])
    box, masks, cls = [], [], []
    for b in range(n_box):
        lo = base + rng.integers(0, [40, 20, 40]) + rng.choice([0.0, 0.3, -0.3, 0.5], 3)
        size = rng.integers(4, 11, 3)
        hi = lo + size + rng.choice([0.0, 0.4, 0.5], 3)
        box.append(np.concatenate([lo, hi]))
        shape = tuple(np.rint(hi).astype(int) - np.rint(lo).astype(int))
        m = (rng.random(shape) < 0.75).astype(np.float32)
        if rng.random() < 0.3:  # larger than its box: vox2mesh crops it
            m = np.pad(m, ((0, 1), (0, 2), (0, 0)), constant_values=1.0)
        masks.append(m)
        cls.append(int(rng.integers(1, 19)))
    box = np.array(box, np.float32)
    conf = rng.choice(CONFS, n_box).astype(np.float32)
    if conf_low is not None:  # below 0.01: box b decodes as class - 1 and confidence ~0.995; with class 0 as box b - 1's
        conf[conf_low:conf_low + 2] = 0.005  # instance id (class 99), so box conf_low + 1 merges into box conf_low
        cls[conf_low + 1] = 0
    keep = rng.random(n_box) < 0.85
    keep[0] = True
    if conf_low is not None:
        keep[conf_low:conf_low + 2] = True
    w2g = np.eye(4)
    w2g[:3, :3] *= 1 / VOXEL
    w2g[:3, 3] = rng.uniform(-2, 2, 3)
    # vertices: around each box (inside, on its shell, just outside: the 3x3x3 neighbour search), scattered, and outside
    g = []
    for b in range(n_box):
        lo, hi = np.rint(box[b, :3]), np.rint(box[b, 3:])
        k = int(rng.integers(150, 400))
        g.append(rng.integers(lo - 1, hi + 1, (k, 3)))
    g.append(rng.integers(base - 5, base + 55, (400, 3)))
    far = rng.integers([-30, 5, 5], [-4, 150, 350], (30, 3))  # outside the canvas (negative x)
    g.append(far)
    g = np.concatenate(g).astype(np.float64)
    g = g[rng.permutation(len(g))]
    grid = g + rng.uniform(-0.4, 0.4, g.shape)
    verts = ((grid - w2g[:3, 3]) @ np.linalg.inv(w2g[:3, :3]).T).astype(np.float32)
    # GT ids: the "true" objects are the predicted boxes shifted by up to one voxel; a few are small, groups or void
    gi = np.rint(g).astype(np.int64)
    gt = np.zeros(len(g), np.int64)
    for b in range(n_box):
        lo = np.rint(box[b, :3]).astype(int) + rng.integers(-1, 2, 3)
        hi = np.rint(box[b, 3:]).astype(int) + rng.integers(-1, 2, 3)
        inside = np.all((gi >= lo) & (gi < hi), axis=1) & (gt == 0)
        r = rng.random()
        if r < 0.1:
            gid = 30 + b  # group
        elif r < 0.18:
            gid = 27000 + b + 1  # invalid class
        else:
            gid = (cls[b] if rng.random() < 0.8 else int(rng.integers(1, 19))) * 1000 + b + 1
        idx = np.nonzero(inside)[0]
        if rng.random() < 0.15:
            idx = idx[:60]  # a small GT instance
        gt[idx] = gid
    return dict(box=box, cls=np.array(cls, np.int64), conf=conf, masks=masks, keep=keep, w2g=w2g, verts=verts, gt=gt)


def make_chain_set(seed, n_scenes=3):
    rng = np.random.default_rng(seed)
    return {f"scene{s:04d}_00": make_chain_scene(rng, int(rng.integers(6, 12)), conf_low=3 if s == 1 else None)
            for s in range(n_scenes)}


def write_pred_folder(d, c):
    """The result folder of one scene as lib.model.trainval.save_scene_results writes it."""
    os.makedirs(d, exist_ok=True)
    np.save(os.path.join(d, "pred_box.npy"), np.concatenate([c["box"], np.zeros((len(c["box"]), 1), np.float32)], 1))
    np.save(os.path.join(d, "pred_class.npy"), c["cls"])
    np.save(os.path.join(d, "pred_conf.npy"), c["conf"])
    with open(os.path.join(d, "pred_mask"), "wb") as f:
        pickle.dump([m for m, k in zip(c["masks"], c["keep"]) if k], f)
    with open(os.path.join(d, "pred_mask_index"), "wb") as f:
        pickle.dump([bool(k) for k in c["keep"]], f)


def write_world2grid(path, w2g):
    """world2grid.txt with the chunk padding added back, as the frames folders store it (repr: exact round trip)."""
    m = np.array(w2g, np.float64)
    m[:, 3] += PADDING
    with open(path, "w") as f:
        for row in m:
            f.write(" ".join(repr(float(v)) for v in row) + "\n")


def write_ply(path, verts, fmt="binary_little_endian", faces=None):
    """A mesh as ScanNet ships it: float x y z, uchar red green blue alpha, then a face element of int lists."""
    verts = np.asarray(verts, np.float32)
    n = len(verts)
    faces = np.zeros((0, 3), np.int32) if faces is None else np.asarray(faces, np.int32)
    head = (f"ply\nformat {fmt} 1.0\ncomment synthetic\nelement vertex {n}\nproperty float x\nproperty float y\n"
            f"property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\n"
            f"element face {len(faces)}\nproperty list uchar int vertex_indices\nend_header\n")
    rgba = (np.arange(n * 4) % 251).astype(np.uint8).reshape(n, 4)
    with open(path, "wb") as f:
        f.write(head.encode("ascii"))
        if fmt == "ascii":
            for v, c in zip(verts, rgba):
                f.write((" ".join(repr(float(x)) for x in v) + " " + " ".join(str(int(x)) for x in c) + "\n").encode())
            for t in faces:
                f.write(("3 " + " ".join(str(int(x)) for x in t) + "\n").encode())
            return
        e = "<" if fmt == "binary_little_endian" else ">"
        vdt = np.dtype([("x", e + "f4"), ("y", e + "f4"), ("z", e + "f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1"),
                        ("alpha", "u1")])
        v = np.zeros(n, vdt)
        v["x"], v["y"], v["z"] = verts[:, 0], verts[:, 1], verts[:, 2]
        v["red"], v["green"], v["blue"], v["alpha"] = rgba.T
        f.write(v.tobytes())
        fdt = np.dtype([("n", "u1"), ("i", e + "i4", (3,))])
        fa = np.zeros(len(faces), fdt)
        fa["n"], fa["i"] = 3, faces
        f.write(fa.tobytes())


def write_chain_inputs(chain, pred_dir, scan_dir, frames_dir, gt_dir, ply_fmt="binary_little_endian"):
    """Result folders, <scan>/<scene>/<scene>_vh_clean_2.ply, <frames>/<scene>/world2grid.txt and <gt>/<scene>.txt."""
    os.makedirs(gt_dir, exist_ok=True)
    for scene, c in chain.items():
        write_pred_folder(os.path.join(pred_dir, scene), c)
        os.makedirs(os.path.join(scan_dir, scene), exist_ok=True)
        n = len(c["verts"])
        faces = np.stack([np.arange(n - 2), np.arange(1, n - 1), np.arange(2, n)], 1)[:50]
        write_ply(os.path.join(scan_dir, scene, scene + "_vh_clean_2.ply"), c["verts"], ply_fmt, faces)
        os.makedirs(os.path.join(frames_dir, scene), exist_ok=True)
        write_world2grid(os.path.join(frames_dir, scene, "world2grid.txt"), c["w2g"])
        np.savetxt(os.path.join(gt_dir, scene + ".txt"), c["gt"], fmt="%d")


# ------------------------------------------------------------------------------------------------------------ the reference
def reference_evaluator():
    """The reference's evaluator module, imported unmodified under the shims of the module docstring."""
    sys.modules.setdefault("plyfile", types.SimpleNamespace(PlyData=None, PlyElement=None))
    for name, alias in (("float", float), ("bool", bool)):
        if name not in np.__dict__:
            setattr(np, name, alias)
    tools = os.path.join(REF, "tools", "scannet_benchmark")
    sys.path.insert(0, tools)
    spec = importlib.util.spec_from_file_location("utils", os.path.join(tools, "utils.py"))
    utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(utils)
    sys.modules["utils"] = utils  # the evaluator's `import utils`; reference_functions() leaves it in place
    argv = sys.argv
    sys.argv = ["evaluate_semantic_instance.py", "--pred_path", "-", "--gt_path", "-"]
    try:
        spec = importlib.util.spec_from_file_location("ref_evaluate_semantic_instance",
                                                      os.path.join(tools, "evaluate_semantic_instance.py"))
        ev = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ev)
    finally:
        sys.argv = argv
    return ev


def run_evaluator(ev, pred_dir, gt_dir, out, key):
    """The reference's main() on one prediction / GT folder pair; records AP, averages, stdout and CSV under `key`."""
    ev.opt.pred_path, ev.opt.gt_path = pred_dir, gt_dir
    ev.opt.output_file = os.path.join(pred_dir, "semantic_instance_evaluation.txt")
    rec = {}
    orig = ev.evaluate_matches

    def grab(matches):
        rec["ap"] = orig(matches)
        return rec["ap"]
    ev.evaluate_matches = grab
    buf = io.StringIO()
    try:
        with contextlib.redirect_stdout(buf):
            ev.main()
    finally:
        ev.evaluate_matches = orig
    avgs = ev.compute_averages(rec["ap"])
    out[key + "_ap"] = rec["ap"]
    out[key + "_all_ap"] = np.float64(avgs["all_ap"])
    out[key + "_all_ap_50"] = np.float64(avgs["all_ap_50%"])
    out[key + "_all_ap_25"] = np.float64(avgs["all_ap_25%"])
    out[key + "_class_ap"] = np.array([[avgs["classes"][c][k] for k in ("ap", "ap50%", "ap25%")] for c in ev.CLASS_LABELS])
    out[key + "_stdout"] = np.array(buf.getvalue())
    with open(ev.opt.output_file) as f:
        out[key + "_csv"] = np.array(f.read())
    print(f"{key}: all_ap {avgs['all_ap']:.4f} ap50 {avgs['all_ap_50%']:.4f} ap25 {avgs['all_ap_25%']:.4f}")


TEXT_SETS = {"text_hand": handmade_text_set, "text_rand0": lambda: random_text_set(11), "text_rand1": lambda: random_text_set(12)}
CHAIN_SETS = {"chain0": lambda: make_chain_set(21), "chain1": lambda: make_chain_set(22)}


def main():
    sys.path.insert(0, _HERE)
    ev = reference_evaluator()
    from make_golden_vox2mesh import reference_functions
    ns = reference_functions()
    out = {}
    for key, make in TEXT_SETS.items():
        with tempfile.TemporaryDirectory() as d:
            pred, gt = os.path.join(d, "pred"), os.path.join(d, "gt")
            write_text_set(make(), pred, gt)
            run_evaluator(ev, pred, gt, out, key)
    for key, make in CHAIN_SETS.items():
        chain = make()
        with tempfile.TemporaryDirectory() as d:
            pred, scans, frames, gt = (os.path.join(d, x) for x in ("results", "scans", "frames", "gt"))
            write_chain_inputs(chain, pred, scans, frames, gt)
            bench = os.path.join(d, "benchmark")
            for scene, c in chain.items():  # the reference main's per-folder steps (vox2mesh.py:131-145)
                w2g = ns["load_matrix"](os.path.join(frames, scene, "world2grid.txt"))
                with contextlib.redirect_stdout(io.StringIO()):
                    ns["export"](c["verts"], w2g, ns["load_pred"](os.path.join(pred, scene)), bench, scene)
            run_evaluator(ev, bench, gt, out, key)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
