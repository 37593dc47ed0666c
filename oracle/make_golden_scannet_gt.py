"""oracle/make_golden_scannet_gt.py -- TEST INFRASTRUCTURE ONLY; runs ONLY in the build container (needs the reference tree).

Runs the reference's UNMODIFIED tools/scannet_benchmark/export_train_mesh_for_evaluation.py as a script (runpy, with its
argv) on seeded synthetic ScanNet scans, and the reference chain export -> vox2mesh functions -> evaluator on seeded
benchmark result folders, and stores what they write in tests/golden/scannet_gt_export_reference.npz.  That file pins
tools/scannet_benchmark/export_train_mesh_for_evaluation.py, annotations.py and evaluate_predictions.py without --gt_path
(tests/test_scannet_gt*.py).  Run it in a process of its own:

    python oracle/make_golden_scannet_gt.py

Shims: a stub `plyfile` whose PlyData.read parses the fixture meshes written here (make_golden_scannet_eval.write_ply's
layout; the reference reads the vertex count and x, y, z), installed before the reference's utils.py is imported; the
reference evaluator and vox2mesh functions as make_golden_scannet_eval.py loads them.

Inputs (regenerated from seeds by the functions below; the tests import them):
- a synthetic scannetv2-labels.combined.tsv (label_tsv: duplicate rows, the later one wins) and the committed copy of
  datagen/fileLists/nyu40labels_scannet.csv (tests/golden/scannet_gt/), optionally with one extra row whose consecutive
  id is 0;
- export sets (EXPORT_SETS): scans with a mesh, a segs file and an aggregation; several objects of one label, segments
  shared across objects, a repeated object id, unannotated vertices, a label whose consecutive id is 0, non-contiguous and
  large segment ids, and a filelist whose last line has no newline and one of whose lines ends in CRLF; both --type values;
- chain sets (CHAIN_SETS): make_golden_scannet_eval's result folders, meshes and world2grid.txt, with annotations made
  from the predicted boxes.

Layout (keys; k = set name): export sets: k_<type>_files (str [n]: the file names written), k_<type>_<scene> (str: the
file's text), k_<type>_stdout; chain sets: k_ap, k_stdout, k_csv (as make_golden_scannet_eval).
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import runpy
import sys
import tempfile
import types

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
REF = os.environ.get("SIS3D_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "scannet_gt_export_reference.npz")
CSV = os.path.join(ROOT, "tests", "golden", "scannet_gt", "nyu40labels_scannet.csv")
sys.path.insert(0, _HERE)
import make_golden_scannet_eval as G  # noqa: E402

# consecutive class (1..18) -> a raw category mapping to it; 'wall' and 'floor' map to consecutive id 19 (ignored)
CLASS_CATEGORY = {1: "cabinet", 2: "bed", 3: "chair", 4: "sofa", 5: "table", 6: "door", 7: "window", 8: "bookshelf",
                  9: "picture", 10: "counter", 11: "desk", 12: "curtain", 13: "refridgerator", 14: "shower curtain",
                  15: "toilet", 16: "sink", 17: "bathtub", 18: "otherfurniture"}
ZERO_CATEGORY = "zero thing"  # nyu40id 41, consecutive id 0 in the extended CSV only


def label_tsv():
    """A scannetv2-labels.combined.tsv in ScanNet's column layout: raw category -> nyu40id, with duplicates."""
    nyu = {3: "cabinet", 4: "bed", 5: "chair", 6: "sofa", 7: "table", 8: "door", 9: "window", 10: "bookshelf",
           11: "picture", 12: "counter", 14: "desk", 16: "curtain", 24: "refridgerator", 28: "shower curtain", 33: "toilet",
           34: "sink", 36: "bathtub", 39: "otherfurniture", 1: "wall", 2: "floor", 40: "otherprop"}
    rows = [(name, i) for i, name in nyu.items()]
    rows += [("office chair", 5), ("kitchen cabinet", 3), ("couch", 39), ("trash can", 40), ("couch", 6),  # couch: last wins
             ("chair", 5), (ZERO_CATEGORY, 41)]
    lines = ["id\traw_category\tcategory\tcount\tnyu40id\teigen13id\tnyuClass\tnyu40class"]
    for k, (name, i) in enumerate(rows):
        lines.append(f"{k + 1}\t{name}\t{name}\t{100 - k}\t{i}\t0\t{name}\t{name}")
    return "\n".join(lines) + "\n"


def label_csv(with_zero):
    text = open(CSV).read()
    return text + ("41,zero thing,(ignore),0,0.0\n" if with_zero else "")


# ------------------------------------------------------------------------------------------------------------ scans
def write_scan(scan_dir, scene, verts, seg_indices, groups):
    """<scene>_vh_clean_2.ply, <scene>_vh_clean_2.0.010000.segs.json, <scene>.aggregation.json as ScanNet ships them.
    groups: [(objectId, raw category, [segment ids])]."""
    d = os.path.join(scan_dir, scene)
    os.makedirs(d, exist_ok=True)
    G.write_ply(os.path.join(d, scene + "_vh_clean_2.ply"), verts)
    with open(os.path.join(d, scene + "_vh_clean_2.0.010000.segs.json"), "w") as f:
        json.dump({"params": {"kThresh": "0.0001"}, "sceneId": scene, "segIndices": [int(s) for s in seg_indices]}, f)
    with open(os.path.join(d, scene + ".aggregation.json"), "w") as f:
        json.dump({"sceneId": "scannet." + scene, "appId": "synthetic", "segGroups": [
            {"id": k, "objectId": int(o), "segments": [int(s) for s in segs], "label": lab}
            for k, (o, lab, segs) in enumerate(groups)], "segmentsFile": "scannet." + scene + "_vh_clean_2.0.010000.segs.json"}, f)


def handmade_scan():
    """-> (verts, seg_indices, groups) covering each quirk on a few segments."""
    seg_ids = np.array([5, 17, 900, 901, 40000, 2 ** 31 - 2, 123456789, 77, 8, 3000, 3001, 3002])
    counts = [30, 20, 25, 10, 15, 12, 40, 18, 22, 9, 14, 11]
    seg = np.repeat(seg_ids, counts)
    seg = seg[np.random.default_rng(1).permutation(len(seg))]
    groups = [
        (0, "chair", [5, 17]),            # first chair: its list also receives every later chair's segments
        (1, "table", [900]),
        (2, "chair", [901, 900]),         # shares 900 with the table; chair wins the label, object 3 the instance
        (4, "office chair", [40000]),     # same nyu40 id as chair but another label key
        (2, "sofa", [2 ** 31 - 2]),       # repeats objectId 2: object 3 now owns only this segment
        (7, ZERO_CATEGORY, [123456789]),  # consecutive id 0: ids below 1000
        (8, "couch", [77, 5]),            # duplicate TSV rows: the later one (sofa) wins; shares segment 5 with chair
        (9, "wall", [8]),                 # consecutive id 19
        (20, "desk", [3001]),             # 3001: label from this object (desk's list comes after chair's) ...
        (21, "chair", [3001, 3002]),      # ... instance from this one (chair's list, object 1's, is extended)
    ]                                     # segment 3000 is unannotated
    verts = np.random.default_rng(2).normal(size=(len(seg), 3)).astype(np.float32)
    return verts, seg, groups


def random_scan(rng, n_vert, n_seg, n_obj, categories):
    """Random segments with large non-contiguous ids, objects of a few categories, shared segments, repeated object ids,
    and unannotated segments."""
    seg_ids = rng.choice(np.arange(1, 2 ** 31 - 1, 7919, dtype=np.int64), n_seg, replace=False)
    seg = seg_ids[rng.integers(0, n_seg, n_vert)]
    used = np.unique(seg)
    order = rng.permutation(len(used))
    groups, at = [], 0
    for o in range(n_obj):
        k = int(rng.integers(1, 6))
        segs = [int(s) for s in used[order[at:at + k]]]
        at += k
        if groups and rng.random() < 0.2:  # a segment shared with an earlier object
            segs.append(int(rng.choice(groups[int(rng.integers(0, len(groups)))][2])))
        oid = o if rng.random() > 0.1 or not groups else groups[int(rng.integers(0, len(groups)))][0]  # repeated id
        groups.append((oid, categories[int(rng.integers(0, len(categories)))], segs))
    verts = rng.normal(size=(n_vert, 3)).astype(np.float32)
    return verts, seg, groups


def export_set(key):
    """-> (scans {scene: (verts, seg, groups)}, filelist bytes, with_zero)."""
    cats = ["chair", "chair", "table", "office chair", "couch", "desk", "wall", "bed", "kitchen cabinet", "trash can"]
    if key == "exp_hand":
        scans = {"scene0000_00": handmade_scan()}
        rng = np.random.default_rng(5)
        scans["scene0001_00"] = random_scan(rng, 500, 40, 12, cats + [ZERO_CATEGORY])
        scans["scene0002_00"] = random_scan(rng, 300, 20, 6, cats)  # last filelist line, no newline: not exported
        scans["scene0003_00"] = random_scan(rng, 200, 10, 3, cats)  # not listed
        return scans, b"scene0000_00\nscene0001_00\r\nscene0002_00", True
    seed = {"exp_rand0": 7, "exp_rand1": 8}[key]
    rng = np.random.default_rng(seed)
    scans = {f"scene{s:04d}_0{seed % 2}": random_scan(rng, int(rng.integers(1000, 4000)), int(rng.integers(50, 300)),
                                                      int(rng.integers(10, 40)), cats) for s in range(3)}
    return scans, "".join(s + "\n" for s in scans).encode(), False


def write_export_inputs(key, d):
    """Scans, filelist and label maps of an export set under d -> dict of paths."""
    scans, filelist, with_zero = export_set(key)
    p = {"scans": os.path.join(d, "scans"), "filelist": os.path.join(d, "filelist.txt"), "tsv": os.path.join(d, "labels.tsv"),
         "csv": os.path.join(d, "nyu40labels_scannet.csv")}
    for scene, (verts, seg, groups) in scans.items():
        write_scan(p["scans"], scene, verts, seg, groups)
    with open(p["filelist"], "wb") as f:
        f.write(filelist)
    with open(p["tsv"], "w") as f:
        f.write(label_tsv())
    with open(p["csv"], "w") as f:
        f.write(label_csv(with_zero))
    return p


def export_argv(p, out_dir, task):
    return ["--scan_path", p["scans"], "--filelist", p["filelist"], "--output_dir", out_dir, "--label_map_file", p["tsv"],
            "--label_map_file2", p["csv"], "--type", task]


# ------------------------------------------------------------------------------------------------------------ chain sets
def annotate_chain_scene(rng, c, id_step=104729):
    """Segments over 3-voxel cells of each vertex's grid position (ids large and non-contiguous, multiples of id_step plus
    3) and one object per predicted box: the segments whose cells lie in the box shifted by up to one voxel, mostly of the
    box's class.  The default id_step leaves room for about 10k segments."""
    grid = c["verts"].astype(np.float64) @ c["w2g"][:3, :3].T + c["w2g"][:3, 3]
    cell = np.floor(grid / 3).astype(np.int64)
    cells, seg_of = np.unique(cell, axis=0, return_inverse=True)
    seg_ids = rng.choice(np.arange(3, 2 ** 30, id_step, dtype=np.int64), len(cells), replace=False)
    seg = seg_ids[seg_of.reshape(-1)]
    centre = cells * 3 + 1.5
    taken = np.zeros(len(cells), bool)
    groups = []
    for b in range(len(c["box"])):
        lo = np.rint(c["box"][b, :3]) + rng.integers(-1, 2, 3)
        hi = np.rint(c["box"][b, 3:]) + rng.integers(-1, 2, 3)
        inside = np.all((centre >= lo) & (centre < hi), axis=1)
        segs = seg_ids[inside & ~taken].tolist()
        if not segs:
            continue
        if rng.random() < 0.15 and (inside & taken).any():  # one segment shared with an earlier object
            segs.append(int(seg_ids[np.nonzero(inside & taken)[0][0]]))
        taken |= inside
        r = rng.random()
        cls = int(c["cls"][b]) if r < 0.75 and 1 <= c["cls"][b] <= 18 else int(rng.integers(1, 19))
        cat = "wall" if r > 0.92 else CLASS_CATEGORY[cls]
        groups.append((b, cat, segs))
    if len(groups) > 2:
        groups[-1] = (groups[0][0], groups[-1][1], groups[-1][2])  # a repeated object id
    return seg, groups


def chain_set(key):
    """-> (make_golden_scannet_eval chain scenes, {scene: (seg, groups)})."""
    seed = {"gtchain0": 41, "gtchain1": 42}[key]
    chain = G.make_chain_set(seed)
    rng = np.random.default_rng(seed + 100)
    return chain, {s: annotate_chain_scene(rng, c) for s, c in chain.items()}


def write_chain_scans(key, d):
    """Result folders, scans (mesh + annotations), frames, a filelist of every scene and the label maps under d."""
    chain, ann = chain_set(key)
    p = {k: os.path.join(d, k) for k in ("results", "scans", "frames", "gt_unused")}
    G.write_chain_inputs(chain, p["results"], p["scans"], p["frames"], p["gt_unused"])
    for s, (seg, groups) in ann.items():
        write_scan(p["scans"], s, chain[s]["verts"], seg, groups)
    p["filelist"], p["tsv"], p["csv"] = (os.path.join(d, f) for f in ("filelist.txt", "labels.tsv", "nyu40.csv"))
    with open(p["filelist"], "w") as f:
        f.write("".join(s + "\n" for s in chain))
    with open(p["tsv"], "w") as f:
        f.write(label_tsv())
    with open(p["csv"], "w") as f:
        f.write(label_csv(False))
    return chain, p


def loop_export_ids(object_id_to_segs, label_to_segs, seg_index, label_map, label_map2, task):
    """The reference's per-vertex export written the same way (segment -> vertex lists, then Python loops writing uint32
    arrays per segment), for timing and for checking large scans: -> uint32 [n_vert]."""
    seg_to_verts = {}
    for i, s in enumerate(seg_index.tolist()):
        seg_to_verts.setdefault(s, []).append(i)
    label_ids = np.zeros(len(seg_index), np.uint32)
    for label, segs in label_to_segs.items():
        label_id = label_map2[label_map[label]]
        for seg in segs:
            label_ids[seg_to_verts[seg]] = label_id
    if task == "label":
        return label_ids
    instance_ids = np.zeros(len(seg_index), np.uint32)
    for object_id, segs in object_id_to_segs.items():
        for seg in segs:
            instance_ids[seg_to_verts[seg]] = object_id
    return label_ids * 1000 + instance_ids


# ------------------------------------------------------------------------------------------------------------ the reference
def plyfile_stub():
    """plyfile.PlyData.read for write_ply's binary little-endian meshes: ['vertex'].count and .data[name]."""
    class PlyData:
        @staticmethod
        def read(f):
            assert f.readline().strip() == b"ply"
            props, count, in_vertex = [], 0, False
            types_ = {"float": "<f4", "uchar": "u1", "int": "<i4"}
            while True:
                w = f.readline().split()
                if w[0] == b"end_header":
                    break
                if w[0] == b"format":
                    assert w[1] == b"binary_little_endian"
                elif w[0] == b"element":
                    in_vertex = w[1] == b"vertex"
                    assert props or in_vertex  # vertex first
                    if in_vertex:
                        count = int(w[2])
                elif w[0] == b"property" and in_vertex:
                    props.append((w[2].decode(), types_[w[1].decode()]))
            dt = np.dtype(props)
            data = np.frombuffer(f.read(count * dt.itemsize), dt, count)
            return {"vertex": types.SimpleNamespace(count=count, data=data)}
    return types.SimpleNamespace(PlyData=PlyData, PlyElement=None)


def run_reference_export(argv):
    """The reference script as `python export_train_mesh_for_evaluation.py argv...` -> its stdout."""
    script = os.path.join(REF, "tools", "scannet_benchmark", "export_train_mesh_for_evaluation.py")
    old = sys.argv
    sys.argv = [script] + argv
    buf = io.StringIO()
    try:
        with contextlib.redirect_stdout(buf):
            runpy.run_path(script, run_name="__main__")
    finally:
        sys.argv = old
    return buf.getvalue()


EXPORT_SETS = ("exp_hand", "exp_rand0", "exp_rand1")
CHAIN_SETS = ("gtchain0", "gtchain1")


def main():
    sys.modules["plyfile"] = plyfile_stub()  # before the reference's utils.py binds PlyData
    sys.path.insert(0, os.path.join(REF, "tools", "scannet_benchmark"))
    ev = G.reference_evaluator()
    from make_golden_vox2mesh import reference_functions
    ns = reference_functions()
    out = {}
    for key in EXPORT_SETS:
        with tempfile.TemporaryDirectory() as d:
            p = write_export_inputs(key, d)
            for task in ("instance", "label"):
                o = os.path.join(d, "out_" + task)
                os.makedirs(o)
                out[f"{key}_{task}_stdout"] = np.array(run_reference_export(export_argv(p, o, task)))
                names = sorted(os.listdir(o))
                out[f"{key}_{task}_files"] = np.array(names)
                for n in names:
                    out[f"{key}_{task}_{n[:-4]}"] = np.array(open(os.path.join(o, n)).read())
                print(key, task, names)
    for key in CHAIN_SETS:
        with tempfile.TemporaryDirectory() as d:
            chain, p = write_chain_scans(key, d)
            gt = os.path.join(d, "gt")
            os.makedirs(gt)
            run_reference_export(export_argv(p, gt, "instance"))
            bench = os.path.join(d, "benchmark")
            for scene, c in chain.items():  # the reference vox2mesh main's per-folder steps
                w2g = ns["load_matrix"](os.path.join(p["frames"], scene, "world2grid.txt"))
                with contextlib.redirect_stdout(io.StringIO()):
                    ns["export"](c["verts"], w2g, ns["load_pred"](os.path.join(p["results"], scene)), bench, scene)
            G.run_evaluator(ev, bench, gt, out, key)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
