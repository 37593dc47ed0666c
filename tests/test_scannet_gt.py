"""CPU: ScanNet GT from the annotation files, under host emulation of sis3d_segment_gt_slots (csrc/eval.cu).

- export_train_mesh_for_evaluation.py's files against the unmodified reference's, byte for byte
  (tests/golden/scannet_gt_export_reference.npz, recorded by oracle/make_golden_scannet_gt.py from seeded inputs that are
  regenerated here), for both --type values;
- the kernel's slots and counts against a numpy restatement (random tables, ids absent from the table, negative ids,
  empty tables and meshes, more slots than the shared histogram holds);
- evaluate_predictions.py without --gt_path against the file route on the exported GT and the reference chain;
- the departures: print_error exits where the reference dies with KeyError, and the vertex-count check."""
import contextlib
import ctypes as C
import io
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden
from test_scannet_eval import eval_emu_lib, host_eval  # noqa: F401  (fixtures)

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_golden_scannet_gt as GG  # noqa: E402  (the seeded inputs; no reference code involved)

GOLDEN = "scannet_gt_export_reference.npz"


def run_quiet(f, *a):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        r = f(*a)
    return r, buf.getvalue()


def check_export_against_golden(tmp_path, key, task):
    from tools.scannet_benchmark import export_train_mesh_for_evaluation as X
    g = load_golden(GOLDEN)
    p = GG.write_export_inputs(key, str(tmp_path / "in"))
    out = tmp_path / ("out_" + task)
    out.mkdir()
    _, stdout = run_quiet(X.main, GG.export_argv(p, str(out), task))
    names = sorted(os.listdir(out))
    assert names == g[f"{key}_{task}_files"].tolist()
    for n in names:
        assert (out / n).read_bytes() == str(g[f"{key}_{task}_{n[:-4]}"]).encode(), n
    # one line per exported scene, in os.listdir order
    assert sorted(stdout.splitlines()) == sorted(str(g[f"{key}_{task}_stdout"]).splitlines())
    return p, out


@pytest.mark.parametrize("task", ["instance", "label"])
@pytest.mark.parametrize("key", GG.EXPORT_SETS)
def test_export_equals_reference_emulated(host_eval, tmp_path, key, task):
    check_export_against_golden(tmp_path, key, task)


def test_golden_sets_reach_the_quirks():
    """The hand-made scan shows each rule: list aliasing, label and instance from different objects, a repeated object id,
    consecutive id 0, duplicate TSV rows, unannotated vertices; the filelist's CRLF line is exported (readlines() in text
    mode turns it into '\\n'), its newline-less last line is not."""
    g = load_golden(GOLDEN)
    assert g["exp_hand_instance_files"].tolist() == ["scene0000_00.txt", "scene0001_00.txt"]
    verts, seg, groups = GG.handmade_scan()
    ids = np.array(str(g["exp_hand_instance_scene0000_00"]).split(), np.int64)
    at = {s: int(ids[np.nonzero(seg == s)[0][0]]) for s in np.unique(seg).tolist()}
    chair, table, sofa, desk, zero, wall = 3, 5, 4, 11, 0, 19
    assert at[5] == sofa * 1000 + 9      # couch (sofa: the later TSV row wins) is the last writer of segment 5
    assert at[17] == chair * 1000 + 1
    assert at[900] == table * 1000 + 2   # the table's label pass and its object come after the chair's
    assert at[901] == chair * 1000 + 1   # object 3's id went to the sofa: its chair segment stays with object 1's list
    assert at[40000] == chair * 1000 + 5
    assert at[2 ** 31 - 2] == sofa * 1000 + 3
    assert at[123456789] == zero * 1000 + 8
    assert at[77] == sofa * 1000 + 9 and at[8] == wall * 1000 + 10 and at[3000] == 0
    assert at[3001] == desk * 1000 + 22  # label from object 21, instance from object 22
    assert at[3002] == chair * 1000 + 22


# ------------------------------------------------------------------------------------------------------------ kernel
def slot_case(seed, n_vert, n_seg, n_slot, negative=False):
    from tools.scannet_benchmark import annotations as A
    rng = np.random.default_rng(seed)
    seg_ids = np.sort(rng.choice(np.arange(0, 2 ** 31 - 1, 9973, dtype=np.int64), n_seg, replace=False)).astype(np.int32)
    seg_slot = rng.integers(0, max(n_slot, 1), n_seg).astype(np.int32)
    pool = np.concatenate([seg_ids, rng.integers(0, 2 ** 31 - 1, 64).astype(np.int32)])  # ids absent from the table
    if negative:
        pool = np.concatenate([pool, np.array([-1, -5, -(2 ** 31)], np.int32)])
    seg_index = pool[rng.integers(0, len(pool), n_vert)] if len(pool) else np.zeros(n_vert, np.int32)
    slot_ids = np.arange(n_slot, dtype=np.int64) * 7
    return A.SegmentGT(seg_index.astype(np.int32), seg_ids, seg_slot, slot_ids, "")


SLOT_CASES = {"random": (0, 20000, 300, 40, False), "negative_ids": (1, 5000, 50, 9, True), "no_segments": (2, 3000, 0, 1, True),
              "no_vertices": (3, 0, 30, 5, False), "many_slots": (4, 30000, 3000, 2500, True)}


def check_slots(case, device=None):
    from tools.scannet_benchmark import annotations as A
    from tools.scannet_benchmark import evaluate_predictions as F
    gt = slot_case(*SLOT_CASES[case])
    slot, count = F.segment_gt_slots(gt, device=device)
    want_ids, want_slot = A.gt_ids_host(gt)
    assert slot.dtype == np.int32 and np.array_equal(slot, want_slot)
    assert np.array_equal(count, np.bincount(want_slot, minlength=len(gt.slot_ids)))
    return gt, slot, count


@pytest.mark.parametrize("case", list(SLOT_CASES))
def test_kernel_slots_equal_numpy_emulated(host_eval, case):
    import torch
    check_slots(case, torch.device("cpu"))


def test_numpy_restatement_by_hand():
    from tools.scannet_benchmark import annotations as A
    gt = A.SegmentGT(np.array([4, 9, -3, 10, 4, 7], np.int32), np.array([4, 7, 10], np.int32), np.array([2, 1, 0], np.int32),
                     np.array([0, 3001, 5002]), "")
    ids, slot = A.gt_ids_host(gt)
    assert slot.tolist() == [2, 0, 0, 0, 2, 1] and ids.tolist() == [5002, 0, 0, 0, 5002, 3001]


def test_kernel_argument_checks(host_eval):
    L = host_eval.lib
    i32, i64 = (C.c_int32 * 8)(), (C.c_int64 * 8)(*([-7] * 8))
    assert L.sis3d_segment_gt_slots(None, -1, None, None, 0, 0, None, None, None) == -1
    assert L.sis3d_segment_gt_slots(None, 0, None, None, -1, 0, None, None, None) == -1
    assert L.sis3d_segment_gt_slots(None, 0, None, None, 0, -1, None, None, None) == -1
    assert L.sis3d_segment_gt_slots(None, 1, None, None, 0, 1, i32, i64, None) == -1    # no segment index
    assert L.sis3d_segment_gt_slots(i32, 1, None, None, 0, 1, None, i64, None) == -1    # no gt_slot
    assert L.sis3d_segment_gt_slots(i32, 1, None, None, 1, 1, i32, i64, None) == -1     # table without ids
    assert L.sis3d_segment_gt_slots(i32, 1, None, None, 0, 1, i32, None, None) == -1    # no slot_count
    assert L.sis3d_segment_gt_slots(None, 0, None, None, 0, 0, None, None, None) == 0
    assert L.sis3d_segment_gt_slots(None, 0, None, None, 0, 3, None, i64, None) == 0    # no vertex: counts initialised
    assert list(i64)[:4] == [0, 0, 0, -7]


def test_real_library_exports_the_entry_point():
    from lib import _sis3d as S
    assert S.lib.sis3d_segment_gt_slots(None, -1, None, None, 0, 0, None, None, None) == -1


def test_export_without_device_raises(tmp_path):
    import torch
    from lib import _sis3d as S
    from tools.scannet_benchmark import export_train_mesh_for_evaluation as X
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    p = GG.write_export_inputs("exp_rand0", str(tmp_path / "in"))
    (tmp_path / "out").mkdir()
    with pytest.raises(S.Sis3dError):
        run_quiet(X.main, GG.export_argv(p, str(tmp_path / "out"), "instance"))


# ------------------------------------------------------------------------------------------------------------ fused route
def fused_from_annotations(p, tmp, name="fused"):
    from tools.scannet_benchmark import evaluate_predictions as F
    out_file = str(tmp / name / "result.csv")
    os.makedirs(os.path.dirname(out_file), exist_ok=True)
    (ap, _), out = run_quiet(F.main, ["--pred_dir", p["results"], "--scan_path", p["scans"], "--frames", p["frames"],
                                      "--label_map_file", p["tsv"], "--label_map_file2", p["csv"], "--output_file", out_file])
    with open(out_file) as f:
        return ap, out, f.read()


def file_route_exported(p, tmp):
    """export_train_mesh_for_evaluation.py, vox2mesh.py and evaluate_semantic_instance.py, each through its CLI."""
    from tools.scannet_benchmark import evaluate_semantic_instance as E
    from tools.scannet_benchmark import export_train_mesh_for_evaluation as X
    from tools.scannet_benchmark import vox2mesh as V
    gt, bench = str(tmp / "gt"), str(tmp / "bench")
    os.makedirs(gt)
    run_quiet(X.main, GG.export_argv(p, gt, "instance"))
    run_quiet(V.main, ["--pred_dir", p["results"], "--output_dir", bench, "--scan_path", p["scans"], "--frames", p["frames"]])
    (ap, _), out = run_quiet(E.main, ["--pred_path", bench, "--gt_path", gt])
    with open(os.path.join(bench, E.RESULT_FILE)) as f:
        return ap, out, f.read()


def check_chain(tmp_path, key):
    g = load_golden(GOLDEN)
    _, p = GG.write_chain_scans(key, str(tmp_path / "in"))
    fused = fused_from_annotations(p, tmp_path)
    assert np.array_equal(fused[0], g[key + "_ap"], equal_nan=True)
    assert fused[1] == str(g[key + "_stdout"]) and fused[2] == str(g[key + "_csv"])
    ap, out, csv = file_route_exported(p, tmp_path)
    assert np.array_equal(ap, fused[0], equal_nan=True) and out == fused[1] and csv == fused[2]


@pytest.mark.parametrize("key", GG.CHAIN_SETS)
def test_fused_from_annotations_equals_file_route_and_reference_emulated(host_eval, tmp_path, key):
    check_chain(tmp_path, key)


# ------------------------------------------------------------------------------------------------------------ departures
def edit_json(path, f):
    import json
    with open(path) as fh:
        d = json.load(fh)
    f(d)
    with open(path, "w") as fh:
        json.dump(d, fh)


@pytest.mark.parametrize("fault, match", [
    ("segment", "scene0000_00: segment 999 of the aggregation has no vertex in the segmentation file"),
    ("category", "scene0000_00: raw category 'no such thing' is not in the raw_category -> nyu40id label map"),
    ("nyu40", "scene0000_00: nyu40id 41 (raw category 'zero thing') is not in the nyu40id -> mappedIdConsecutive label map"),
])
def test_export_exits_where_the_reference_raises_keyerror(host_eval, tmp_path, capsys, fault, match):
    from tools.scannet_benchmark import export_train_mesh_for_evaluation as X
    p = GG.write_export_inputs("exp_hand", str(tmp_path / "in"))
    agg = os.path.join(p["scans"], "scene0000_00", "scene0000_00.aggregation.json")
    if fault == "segment":
        edit_json(agg, lambda d: d["segGroups"][1]["segments"].append(999))
    elif fault == "category":
        edit_json(agg, lambda d: d["segGroups"][2].update(label="no such thing"))
    else:
        with open(p["csv"], "w") as f:
            f.write(GG.label_csv(False))
    (tmp_path / "out").mkdir()
    with pytest.raises(SystemExit) as e:
        run_quiet(X.main, GG.export_argv(p, str(tmp_path / "out"), "instance"))
    assert e.value.code == -1 and match in capsys.readouterr().err


def test_export_needs_the_mesh(host_eval, tmp_path):
    from tools.scannet_benchmark import export_train_mesh_for_evaluation as X
    p = GG.write_export_inputs("exp_rand1", str(tmp_path / "in"))
    os.remove(os.path.join(p["scans"], "scene0001_00", "scene0001_00_vh_clean_2.ply"))
    (tmp_path / "out").mkdir()
    with pytest.raises(FileNotFoundError):
        run_quiet(X.main, GG.export_argv(p, str(tmp_path / "out"), "label"))


def test_fused_from_annotations_errors(host_eval, tmp_path, capsys):
    from tools.scannet_benchmark import evaluate_predictions as F
    _, p = GG.write_chain_scans("gtchain0", str(tmp_path / "in"))
    with pytest.raises(SystemExit) as e:  # label maps are required without --gt_path
        F.main(["--pred_dir", p["results"], "--scan_path", p["scans"], "--frames", p["frames"]])
    assert e.value.code == 2 and "--label_map_file" in capsys.readouterr().err
    seg_file = os.path.join(p["scans"], "scene0001_00", "scene0001_00_vh_clean_2.0.010000.segs.json")
    edit_json(seg_file, lambda d: d["segIndices"].append(d["segIndices"][0]))
    with pytest.raises(SystemExit) as e:
        fused_from_annotations(p, tmp_path)
    err = capsys.readouterr().err
    assert e.value.code == -1 and "wrong number of segment indices in " + seg_file in err and "vs #mesh vertices" in err
    os.remove(seg_file)
    with pytest.raises(SystemExit) as e:
        fused_from_annotations(p, tmp_path)
    err = capsys.readouterr().err
    assert e.value.code == 2 and "Result file scene0001_00.txt does not match any gt file: no " + seg_file in err
