"""CPU: box and mask mAP of test mode (lib/utils/evaluation.py) against the reference's own evaluation.py
(tests/golden/eval_reference.npz, recorded by oracle/make_golden_eval.py), with the mask-overlap kernel (csrc/eval.cu) compiled
for the host by tools/cuda_host_emu.py."""
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden

GOLDEN = "eval_reference.npz"


@pytest.fixture(scope="module")
def eval_emu_lib(tmp_path_factory):
    import ctypes as C
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import cuda_host_emu
    out = str(tmp_path_factory.mktemp("emu_eval") / "libsis3d_eval_emu.so")
    cuda_host_emu.build(out, [os.path.join(ROOT, "3d-sis_b200", "csrc", "eval.cu")])
    lib = C.CDLL(out)
    lib.sis3d_strerror.restype = C.c_char_p
    return lib


@pytest.fixture
def host_eval(monkeypatch, eval_emu_lib):
    """lib._sis3d pointed at the emulated library, accepting host tensors (as conftest's host_S)."""
    import ctypes as C
    from lib import _sis3d as S
    monkeypatch.setattr(S, "lib", eval_emu_lib)
    monkeypatch.setattr(S, "ptr", lambda t: None if t is None else C.c_void_p(t.data_ptr()))
    monkeypatch.setattr(S, "stream", lambda: None)
    return S


def unpack_masks(bits, boxes, dtype):
    """Inverse of the fixture's packing: masks with the shapes of the rounded boxes, back to back."""
    flat = np.unpackbits(bits).astype(dtype)
    out, o = [], 0
    for b in np.rint(np.asarray(boxes, np.float64)).astype(np.int64):
        shape = tuple(int(v) for v in b[3:6] - b[0:3])
        n = int(np.prod(shape))
        out.append(flat[o:o + n].reshape(shape))
        o += n
    return out


def golden_scenes(g, k):
    for s in range(int(g[f"{k}_n_scenes"])):
        p = f"{k}_{s}_"
        pred_box, gt_box = g[p + "pred_box"], g[p + "gt_box"]
        yield p, dict(dims=tuple(int(v) for v in g[p + "dims"]), pred_box=pred_box, pred_class=g[p + "pred_class"],
                      pred_conf=g[p + "pred_conf"], pred_mask=unpack_masks(g[p + "pred_bits"], pred_box, np.float32),
                      gt_box=gt_box, gt_class=g[p + "gt_class"], gt_mask=unpack_masks(g[p + "gt_bits"], gt_box, np.uint8))


def check_golden_set(g, k):
    """One golden set through DetectionMAP: IoU matrices array_equal (nan positions included), per-class TP/FP/FN, every AP,
    the mAP, the final ignore_class and the printed lines equal."""
    from lib.utils import evaluation as E
    n_class, thresh = int(g[f"{k}_n_class"]), float(g[f"{k}_thresh"])
    dm = {"box": E.DetectionMAP(n_class, ignore_class=[0], overlap_threshold=thresh),
          "mask": E.DetectionMAP(n_class, ignore_class=[0], overlap_threshold=thresh)}
    for p, sc in golden_scenes(g, k):
        iou = {"box": E.box_iou(sc["pred_box"], sc["gt_box"])}
        pb, po, pbox = E.pack_masks(sc["pred_mask"], sc["pred_box"], sc["dims"], "predicted")
        gb, go, gbox = E.pack_masks(sc["gt_mask"], sc["gt_box"], sc["dims"])
        iou["mask"] = E.mask_iou(*E.launch_mask_overlap(pb, po, pbox, gb, go, gbox).result())
        for name in ("box", "mask"):
            got = iou[name]
            got[got < thresh] = 0
            want = g[p + name + "_iou"]
            assert got.dtype == want.dtype and np.array_equal(got, want, equal_nan=True), (p, name)
            tp, fp, fn = [], [], []
            pc, gc = sc["pred_class"].astype(np.int64), sc["gt_class"].astype(np.int64)
            for c in range(n_class):
                t, f, n = E.DetectionMAP.compute_TP_FP_FN(pc, gc, sc["pred_conf"], got, c)
                tp.append(t), fp.append(f), fn.append(n)
            assert [len(t) for t in tp] == g[p + name + "_tp_n"].tolist(), (p, name)
            assert [len(f) for f in fp] == g[p + name + "_fp_n"].tolist(), (p, name)
            assert fn == g[p + name + "_fn"].tolist(), (p, name)
            assert [float(v) for t in tp for v in t] == g[p + name + "_tp"].tolist(), (p, name)
            assert [float(v) for f in fp for v in f] == g[p + name + "_fp"].tolist(), (p, name)
        dm["box"].evaluate(sc["pred_box"], sc["pred_class"], sc["pred_conf"], sc["gt_box"], sc["gt_class"])
        dm["mask"].evaluate_mask(sc["pred_box"], sc["pred_class"], sc["pred_conf"], sc["pred_mask"], sc["gt_box"],
                                 sc["gt_class"], sc["gt_mask"], list(sc["dims"]))
    for name, title in (("box", "CLASSIFICATION"), ("mask", "mask")):
        m = dm[name]
        m.finalize()
        assert m.ignore_class == g[f"{k}_{name}_ignore"].tolist()
        aps = [np.nan if c in m.ignore_class else m.AP(c) for c in range(n_class)]
        assert np.array_equal(np.array(aps, np.float64), g[f"{k}_{name}_ap"], equal_nan=True)
        assert m.mAP() == float(g[f"{k}_{name}_map"])
        assert E.summary_lines(title, m, n_class) == str(g[f"{k}_{name}_summary"]).split("\n")


@pytest.mark.parametrize("k", [0, 1, 2])
def test_golden_sets_emulated(host_eval, k):
    check_golden_set(load_golden(GOLDEN), k)


def brute_counts(pred_masks, pred_box, gt_masks, gt_box, dims):
    """Full-scene expansion, as the reference's unmold_mask."""
    def full(masks, boxes):
        f = np.zeros((len(masks),) + tuple(dims), bool)
        for i, (m, b) in enumerate(zip(masks, boxes)):
            f[i, b[0]:b[3], b[1]:b[4], b[2]:b[5]] = m != 0
        return f.reshape(len(masks), -1)
    a, b = full(pred_masks, pred_box), full(gt_masks, gt_box)
    return a.sum(1), b.sum(1), a.astype(np.int64) @ b.T.astype(np.int64)


def random_masks(rng, dims, n, max_ext, p):
    boxes, masks = [], []
    for _ in range(n):
        ext = rng.integers(1, np.minimum(max_ext, dims) + 1)
        lo = rng.integers(0, np.asarray(dims) - ext + 1)
        boxes.append(np.concatenate([lo, lo + ext]))
        masks.append((rng.random(tuple(ext)) < p).astype(np.uint8))
    return np.array(boxes, np.int64).reshape(-1, 6), masks


def check_counts(pred_box, pred_masks, gt_box, gt_masks, dims):
    from lib.utils import evaluation as E
    pb, po, pbox = E.pack_masks(pred_masks, pred_box, dims, "predicted")
    gb, go, gbox = E.pack_masks(gt_masks, gt_box, dims)
    got = E.launch_mask_overlap(pb, po, pbox, gb, go, gbox).result()
    want = brute_counts(pred_masks, pred_box, gt_masks, gt_box, dims)
    for x, y in zip(got, want):
        assert np.array_equal(x, y)
    return got


def test_counts_brute_force_emulated(host_eval):
    rng = np.random.default_rng(7)
    # the 208x48x160 whole scene at the size test mode sees (~100 kept masks x ~40 GT)
    pb, pm = random_masks(rng, (208, 48, 160), 100, (24, 16, 24), 0.6)
    gb, gm = random_masks(rng, (208, 48, 160), 40, (24, 16, 24), 0.7)
    check_counts(pb, pm, gb, gm, (208, 48, 160))
    # crops of size 1 (single voxels and 1-wide slabs), densely overlapping
    pb, pm = random_masks(rng, (6, 5, 7), 30, (1, 5, 1), 0.8)
    gb, gm = random_masks(rng, (6, 5, 7), 20, (1, 1, 7), 0.8)
    check_counts(pb, pm, gb, gm, (6, 5, 7))


def test_face_touching_boxes_have_no_pairs(host_eval):
    from lib.utils import evaluation as E
    pred_box = np.array([[0, 0, 0, 4, 4, 4], [0, 0, 0, 4, 4, 4], [2, 2, 2, 6, 6, 6]])
    gt_box = np.array([[4, 0, 0, 8, 4, 4], [0, 4, 0, 4, 8, 4], [0, 0, 4, 4, 4, 8]])
    ones = [np.ones((4, 4, 4), np.uint8)] * 3
    assert E.box_pairs(pred_box[:2], gt_box).shape == (0, 2)  # sharing a face is no common voxel
    pc, gc, inter = check_counts(pred_box, ones, gt_box, ones, (8, 8, 8))
    assert inter[:2].sum() == 0 and inter[2].tolist() == [8, 8, 8]


def test_mask_shape_and_bounds_checks(host_eval):
    from lib.utils import evaluation as E
    dm = E.DetectionMAP(3, ignore_class=[0], overlap_threshold=0.25)
    pred = dict(pred_box=np.array([[0, 0, 0, 2, 2, 2]], np.float32), pred_class=np.array([1]), pred_conf=np.array([0.9]),
                pred_mask=[np.ones((2, 2, 2), np.float32)])
    with pytest.raises(ValueError, match="GT mask 1: shape"):
        dm.evaluate_mask(**pred, gt_box=np.array([[0, 0, 0, 2, 2, 2], [1, 1, 1, 3, 3, 4]], np.float32),
                         gt_class=np.array([1, 1]), gt_mask=[np.ones((2, 2, 2)), np.ones((2, 2, 2))], scene_info=[4, 4, 4])
    with pytest.raises(ValueError, match="GT mask 0: box"):  # numpy slicing would wrap the negative bound silently
        dm.evaluate_mask(**pred, gt_box=np.array([[-1, 0, 0, 1, 2, 2]], np.float32), gt_class=np.array([1]),
                         gt_mask=[np.ones((2, 2, 2))], scene_info=[4, 4, 4])
    with pytest.raises(ValueError, match="GT mask 0: box"):
        dm.evaluate_mask(**pred, gt_box=np.array([[3, 0, 0, 5, 2, 2]], np.float32), gt_class=np.array([1]),
                         gt_mask=[np.ones((2, 2, 2))], scene_info=[4, 4, 4])
    with pytest.raises(ValueError, match="predicted mask 0: shape"):
        dm.evaluate_mask(pred["pred_box"], pred["pred_class"], pred["pred_conf"], [np.ones((2, 2, 3))],
                         np.array([[0, 0, 0, 2, 2, 2]], np.float32), np.array([1]), [np.ones((2, 2, 2))], [4, 4, 4])
    with pytest.raises(ValueError, match="2 GT masks for 1 boxes"):
        dm.evaluate_mask(**pred, gt_box=np.array([[0, 0, 0, 2, 2, 2]], np.float32), gt_class=np.array([1]),
                         gt_mask=[np.ones((2, 2, 2))] * 2, scene_info=[4, 4, 4])


def test_predictions_without_gt_are_false_positives():
    """The reference raises here (np.max of an empty array); every prediction counts as a false positive instead."""
    from lib.utils import evaluation as E
    dm = E.DetectionMAP(3, ignore_class=[0], overlap_threshold=0.25)
    dm.evaluate(np.array([[0, 0, 0, 2, 2, 2], [1, 1, 1, 3, 3, 3]], np.float32), np.array([1, 2]), np.array([0.9, 0.8]),
                np.zeros((0, 6), np.float32), np.zeros(0, np.float32))
    dm.evaluate(np.array([[0, 0, 0, 2, 2, 2]], np.float32), np.array([1]), np.array([0.7]),
                np.array([[0, 0, 0, 2, 2, 2]], np.float32), np.array([1], np.float32))
    acc = dm.total_accumulators
    assert (acc[1].TP, acc[1].FN, len(acc[1].predictions), acc[2].TP, acc[2].FN, len(acc[2].predictions)) == (1, 0, 2, 0, 0, 1)
    dm.finalize()
    assert dm.ignore_class == [0, 2]
    assert acc[1].predictions.tolist() == [[0.9, 0.0], [0.7, 1.0]]


def test_mask_overlap_rejects_bad_arguments(host_eval):
    import ctypes as C
    L = host_eval.lib
    buf = (C.c_int64 * 8)()
    assert L.sis3d_mask_overlap(None, None, None, -1, None, None, None, 0, None, 0, None, None, None, None) == -1
    assert L.sis3d_mask_overlap(None, None, None, 1, None, None, None, 0, None, 0, buf, None, None, None) == -1
    assert L.sis3d_mask_overlap(None, None, None, 0, None, None, None, 2, None, 0, None, buf, None, None) == -1
    assert L.sis3d_mask_overlap(None, None, None, 0, None, None, None, 0, buf, 1, None, None, buf, None) == -1  # pairs, no masks
    assert L.sis3d_mask_overlap(None, None, None, 0, None, None, None, 0, None, 0, None, None, None, None) == 0  # nothing to do


def test_mask_overlap_flags_out_of_range_pairs(host_eval):
    import ctypes as C
    bits = (C.c_uint8 * 8)(*([1] * 8))
    offs = (C.c_int64 * 1)(0)
    box = (C.c_int32 * 6)(0, 0, 0, 2, 2, 2)
    pairs = (C.c_int32 * 4)(0, 0, 0, 3)
    pc, gc, out = (C.c_int64 * 1)(), (C.c_int64 * 1)(), (C.c_int64 * 2)()
    assert host_eval.lib.sis3d_mask_overlap(bits, offs, box, 1, bits, offs, box, 1, pairs, 2, pc, gc, out, None) == 0
    assert (pc[0], gc[0], out[0], out[1]) == (8, 8, 8, -1)


def test_real_library_exports_the_entry_point():
    from lib import _sis3d as S
    assert hasattr(S.lib, "sis3d_mask_overlap")
    assert S.lib.sis3d_mask_overlap(None, None, None, -1, None, None, None, 0, None, 0, None, None, None, None) == -1
