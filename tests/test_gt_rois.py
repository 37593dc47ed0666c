"""CPU: test mode on ground-truth boxes and classes (USE_RPN = USE_CLASS = False).

- oracle/port_gt_rois.py's forward_gt_rois equals the unmodified reference (tests/golden/gt_rois_reference.npz, written by
  oracle/make_golden_gt_rois.py) on every forward case, with USE_BACKBONE on and off;
- the host detection-table builder (lib.nets.network.gt_detection_table) equals the reference's bbox_transform_inv +
  clip_boxes + round filter bit for bit, on the golden boxes and on a grid of fractional and half-integer corners around
  every scene face;
- the combinations the reference cannot run are refused, naming the combination."""
import numpy as np
import pytest
import torch

import sis3d_synth as synth
from conftest import load_golden
from lib import _sis3d as S
from lib.nets.network import Network, gt_detection_table
from lib.utils.config import cfg
from oracle.port_gt_rois import forward_gt_rois

GOLDEN = "gt_rois_reference.npz"
FORWARD = ("cfg1_32", "odd_45x27x41", "cfg2_96x48x96", "suncg_40x24x40", "thresh1_45x27x41")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def case_inputs(port, g, tag):
    name = str(g[f"{tag}_cfgname"])
    ocfg = port.make_cfg(name, CLASS_THRESH=float(g[f"{tag}_class_thresh"]))
    w = synth.make_weights(seed=0, net=ocfg.NET, use_images=bool(g[f"{tag}_n_img"] > 0), num_classes=ocfg.NUM_CLASSES,
                           a1=0, a2=0, use_mask=True)
    data, _ = synth.make_scene(int(g[f"{tag}_seed"]), tuple(int(v) for v in g[f"{tag}_dims"]))
    return ocfg, w, data


def reference_decode(port, gt, dims, thresh):
    """The reference's decode of ground-truth RoIs, op for op (network.py:276-301 / trainval.py:825-858): zero deltas through
    bbox_transform_inv, clip_boxes, conf = 1.0 > CLASS_THRESH, Python round() on each corner."""
    rois = torch.from_numpy(np.ascontiguousarray(gt[:, :6], np.float32))
    pb = port.clip_boxes(port.bbox_transform_inv(rois, torch.zeros(len(gt), 6)), dims).numpy() if len(gt) else np.zeros((0, 6),
                                                                                                                      np.float32)
    keep = np.array([1.0 > thresh] * len(gt), bool)
    crops = np.array([[round(float(v)) for v in b] for b in pb], np.int64).reshape(-1, 6)
    keep &= (crops[:, :3] < crops[:, 3:]).all(1)
    return pb, keep, crops


@pytest.mark.parametrize("tag", FORWARD)
def test_oracle_equals_reference(oracle, golden, tag):
    g = golden
    ocfg, w, data = case_inputs(oracle, g, tag)
    gt = g[f"{tag}_gt_box"]
    out = forward_gt_rois(ocfg, w, data, gt)
    for b in (1, 0):  # USE_BACKBONE on and off: the reference gives the same predictions
        k = f"{tag}_b{b}_"
        assert np.array_equal(out["rois"].numpy(), g[k + "rois"])
        assert np.array_equal(out["roi_scores"].numpy(), g[k + "roi_scores"])
        assert np.array_equal(out["cls_pred"].numpy(), g[k + "cls_pred"])
        assert np.array_equal(out["cls_prob"].numpy(), g[k + "cls_prob"])
        assert np.array_equal(out["bbox_pred"].numpy(), g[k + "bbox_pred"])
        assert np.array_equal(out["pred_box"].view(np.int32), g[k + "pred_box"].view(np.int32))
        assert np.array_equal(out["mask_keep"], g[k + "keep"])
        assert np.array_equal(out["mask_crops"], g[k + "crops"])
        assert len(out["mask_pred"]) == int(g[k + "n_masks"]) == int(g[k + "keep"].sum())
    pc = out["cls_pred"].numpy()[out["mask_keep"]]
    for j, m in enumerate(out["mask_pred"]):
        m = m[0].numpy()
        np.testing.assert_allclose(m[pc[j]].reshape(-1)[::7], g[f"{tag}_b1_mask_{j}_cls_sub"], atol=1e-5)
        np.testing.assert_allclose(m.reshape(-1)[::97], g[f"{tag}_b1_mask_{j}_allcls_sub"], atol=1e-5)
        assert int((m[pc[j]] >= 0.5).sum()) == int(g[f"{tag}_b1_mask_{j}_cls_on"])


def test_golden_cases_cover_the_edges(golden):
    g = golden
    keeps = {t: g[f"{t}_b1_keep"] for t in FORWARD}
    assert not keeps["thresh1_45x27x41"].any() and float(g["thresh1_45x27x41_class_thresh"]) >= 1.0
    for t in FORWARD[:4]:
        gt, dims = g[f"{t}_gt_box"], g[f"{t}_dims"]
        assert (gt[:, :3] < 0).any() and (gt[:, 3:6] > dims).any(axis=0).all() and (gt[:, :3] < 0).any(axis=0).all()
        assert (gt[:, 6] == 0).any() and keeps[t][gt[:, 6] == 0].all()
        assert keeps[t].any() and not keeps[t].all()
        assert (np.modf(gt[:, :6])[0] == 0.5).any() and (np.modf(np.abs(gt[:, :6]))[0] % 0.5 != 0).any()
        crops = g[f"{t}_b1_crops"]
        assert ((crops[:, :3] == 0).all(1) & (crops[:, 3:] == dims).all(1)).any(), "no crop spans the whole scene"


@pytest.mark.parametrize("tag", FORWARD)
def test_host_table_equals_reference_on_golden(golden, tag):
    g = golden
    gt, dims = g[f"{tag}_gt_box"], tuple(int(v) for v in g[f"{tag}_dims"])
    nc = 26 if str(g[f"{tag}_cfgname"]) == "suncg" else 19
    det = gt_detection_table(gt, dims, float(g[f"{tag}_class_thresh"]), nc)
    k = f"{tag}_b0_"
    assert det.shape == (len(gt), 16) and det.dtype == np.float32
    assert np.array_equal(det[:, 0:6].view(np.int32), g[k + "pred_box"].view(np.int32))
    assert np.array_equal(det[:, 6], g[k + "cls_prob"][np.arange(len(gt)), g[k + "cls_pred"]])
    assert np.array_equal(det[:, 7].astype(np.int64), g[k + "cls_pred"])
    assert np.array_equal(det[:, 8] > 0.5, g[k + "keep"])
    assert np.array_equal(det[:, 9:15].astype(np.int64), g[k + "crops"])
    assert det[0, 15] == len(gt) and not det[1:, 15].any()


def test_host_table_equals_reference_on_a_corner_grid(oracle):
    """Every corner on a 1/8-voxel grid from 2 voxels outside to 2 voxels past each face, plus float32 neighbours of the
    half-integers, against the reference's decode."""
    dims = (13, 7, 11)
    rng = np.random.default_rng(5)
    base = np.arange(-16, 8 * 13 + 17) / 8.0
    half = np.arange(-2, 16) + 0.5
    near = np.concatenate([np.nextafter(half.astype(np.float32), np.float32(-np.inf)),
                           np.nextafter(half.astype(np.float32), np.float32(np.inf))])
    vals = np.concatenate([base, half, near]).astype(np.float32)
    n = 20000
    gt = np.zeros((n, 7), np.float32)
    for a, d in enumerate(dims):
        v = vals[(vals >= -2) & (vals <= d + 2)]
        gt[:, a], gt[:, a + 3] = rng.choice(v, n), rng.choice(v, n)
    gt[:, 6] = rng.integers(0, 19, n)
    for thresh in (0.5, 0.999999999, 1.0):
        det = gt_detection_table(gt, dims, thresh, 19)
        pb, keep, crops = reference_decode(oracle, gt, dims, thresh)
        assert np.array_equal(det[:, 0:6].view(np.int32), pb.view(np.int32))
        assert np.array_equal(det[:, 8] > 0.5, keep)
        assert np.array_equal(det[:, 9:15].astype(np.int64), crops)
        assert np.array_equal(det[:, 7], gt[:, 6])
        if thresh < 1.0:
            assert keep.any() and not keep.all()
        else:
            assert not keep.any()


def test_host_table_without_boxes():
    det = gt_detection_table(np.zeros((0, 7), np.float32), (8, 8, 8), 0.5, 19)
    assert det.shape == (0, 16) and det.dtype == np.float32


@pytest.mark.parametrize("gt,what", [(np.zeros((3, 6), np.float32), "shape"),
                                     (np.array([[0, 0, 0, 2, 2, 2, 19]], np.float32), "class"),
                                     (np.array([[0, 0, 0, 2, 2, 2, -1]], np.float32), "class"),
                                     (np.array([[0, 0, np.nan, 2, 2, 2, 1]], np.float32), "non-finite")])
def test_host_table_rejects_malformed_boxes(gt, what):
    with pytest.raises(S.Sis3dError, match=what):
        gt_detection_table(gt, (8, 8, 8), 0.5, 19)


@pytest.fixture
def switches():
    saved = {k: cfg[k] for k in ("USE_BACKBONE", "USE_RPN", "USE_CLASS")}
    yield cfg
    for k, v in saved.items():
        cfg[k] = v


@pytest.mark.parametrize("backbone,rpn,cls,refused", [
    (True, True, True, None), (True, True, False, None),                  # detections; RPN-only predictions
    (True, False, False, None), (False, False, False, None),              # ground-truth RoIs, with or without the backbone
    (True, False, True, "USE_RPN=False with USE_CLASS=True"), (False, False, True, "USE_RPN=False with USE_CLASS=True"),
    (False, True, True, "USE_BACKBONE=False with USE_RPN=True"), (False, True, False, "USE_BACKBONE=False with USE_RPN=True")])
def test_mode_switches(switches, backbone, rpn, cls, refused):
    switches.USE_BACKBONE, switches.USE_RPN, switches.USE_CLASS = backbone, rpn, cls
    if refused is None:
        Network._check_mode(None, "TEST")
    else:
        with pytest.raises(NotImplementedError, match=refused):
            Network._check_mode(None, "TEST")
    with pytest.raises(NotImplementedError, match="TEST"):
        Network._check_mode(None, "TRAIN")
