"""GPU: the mask-overlap kernel (csrc/eval.cu) on the golden evaluation sets, inside a CUDA graph, and test mode's box / mask
mAP end to end (lib.model.trainval.test on synthetic .chunk files)."""
import ctypes as C
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import load_golden
from test_eval_map import GOLDEN, check_golden_set, golden_scenes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", [0, 1, 2])
def test_golden_sets_on_device(k):
    check_golden_set(load_golden(GOLDEN), k)


def test_graph_capture_equals_eager():
    from lib import _sis3d as S
    from lib.utils import evaluation as E
    g = load_golden(GOLDEN)
    _, sc = list(golden_scenes(g, 2))[2]  # the 208x48x160 scene
    pb, po, pbox = E.pack_masks(sc["pred_mask"], sc["pred_box"], sc["dims"], "predicted")
    gb, go, gbox = E.pack_masks(sc["gt_mask"], sc["gt_box"], sc["dims"])
    pairs = E.box_pairs(pbox, gbox)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = [dev(pb), dev(po), dev(pbox), dev(gb), dev(go), dev(gbox), dev(pairs)]
    n_pred, n_gt, n_pairs = len(po), len(go), len(pairs)
    assert n_pairs > 0

    def launch(out, stream):
        S.check(S.lib.sis3d_mask_overlap(S.ptr(t[0]), S.ptr(t[1]), S.ptr(t[2]), n_pred, S.ptr(t[3]), S.ptr(t[4]), S.ptr(t[5]),
                                         n_gt, S.ptr(t[6]), n_pairs, S.ptr(out), S.ptr(out[n_pred:]),
                                         S.ptr(out[n_pred + n_gt:]), C.c_void_p(stream.cuda_stream)), "mask_overlap")

    eager = torch.full((n_pred + n_gt + n_pairs,), -7, dtype=torch.int64, device="cuda")
    launch(eager, torch.cuda.current_stream())
    replayed = torch.full_like(eager, -7)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch(replayed, torch.cuda.current_stream())
    torch.cuda.synchronize()
    assert (replayed == -7).all()  # captured, not run
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager, replayed)
    e = eager.cpu().numpy()
    inter = np.zeros((n_pred, n_gt), np.int64)
    inter[pairs[:, 0], pairs[:, 1]] = e[n_pred + n_gt:]
    want = E.mask_iou(e[:n_pred], e[n_pred:n_pred + n_gt], inter)
    want[want < float(g["2_thresh"])] = 0
    assert np.array_equal(want, g["2_2_mask_iou"], equal_nan=True)


def _summary(out):
    return [ln for ln in out.splitlines() if ln.startswith(("mAP of ", "class "))]


def test_test_mode_reports_map_end_to_end(tmp_path, capsys):
    import sis3d_synth as synth
    from lib.model import trainval
    from lib.model.trainval import scene_key
    from lib.utils.evaluation import DetectionMAP, summary_lines
    c = synth.CASES["odd_45x27x41"]
    net, cfg = synth.make_net(c, keep_debug=False, math="exact")
    torch.save({k: v.detach().cpu().clone() for k, v in net.state_dict().items()}, str(tmp_path / "step_1.pth"))
    paths, provider = synth.write_chunks(str(tmp_path), c, (202, 7, 8, 9, 10, 11, 12))
    cfg.TEST_FILELIST = paths
    args = SimpleNamespace(output_dir=str(tmp_path), step=1, num_workers=0)
    printed = {}
    for mode in ("pipelined", "sync"):
        cfg.TEST_SAVE_DIR = str(tmp_path / mode)
        capsys.readouterr()
        assert trainval.test(args, view_provider=provider, pipelined=(mode == "pipelined")) == len(paths)
        printed[mode] = _summary(capsys.readouterr().out)
    assert printed["pipelined"] == printed["sync"]
    lines = printed["pipelined"]
    assert lines[0].startswith("mAP of CLASSIFICATION: ") and sum(ln.startswith("mAP of mask: ") for ln in lines) == 1

    # the same numbers from the written result files, through the host-list path of DetectionMAP
    box = DetectionMAP(cfg.NUM_CLASSES, ignore_class=[0], overlap_threshold=cfg.MAP_THRESH)
    mask = DetectionMAP(cfg.NUM_CLASSES, ignore_class=[0], overlap_threshold=cfg.MAP_THRESH)
    n_kept = 0
    for p in paths:
        d = os.path.join(str(tmp_path / "pipelined"), scene_key(p))
        ld = lambda f: np.load(os.path.join(d, f + ".npy"))
        pk = lambda f: pickle.load(open(os.path.join(d, f), "rb"))
        keep = np.array(pk("pred_mask_index"), bool)
        pc, pconf, pbox, gb, gc = ld("pred_class"), ld("pred_conf"), ld("pred_box"), ld("gt_box"), ld("gt_class")
        assert gb.shape[0] > 0 and len(pk("gt_mask")) == gb.shape[0]
        box.evaluate(pbox[keep], pc[keep], pconf[keep], gb, gc)
        mask.evaluate_mask(pbox[keep], pc[keep], pconf[keep], pk("pred_mask"), gb, gc, pk("gt_mask"), ld("scene").shape)
        n_kept += int(keep.sum())
    assert n_kept > 0
    box.finalize()
    mask.finalize()
    assert lines == summary_lines("CLASSIFICATION", box, cfg.NUM_CLASSES) + summary_lines("mask", mask, cfg.NUM_CLASSES)
