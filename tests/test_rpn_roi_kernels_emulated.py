"""CPU: the SHIPPED proposal-stage and RoI kernels (csrc/rpn.cu, csrc/roi.cu: anchor scoring, histogram/radix top-N, bitonic
sort, decode, NMS bitmask + greedy reduce, RoI pooling) compiled for the host by tools/cuda_host_emu.py and driven through the
same Python wrappers / C entry points, against the oracle -- the bit-exact integer outputs (keep lists, top-N order, RoI bins)
without a GPU.  The GPU parity tests proper are tests/test_gpu_ops.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sis3d_synth as synth
from conftest import ROOT
from lib import _sis3d as S

sys.path.insert(0, os.path.join(ROOT, "tools"))


@pytest.fixture(scope="module")
def emu(emu_lib):
    return emu_lib


def _p(t):
    return C.c_void_p(t.data_ptr())


@pytest.mark.parametrize("seed,n,thr", [(0, 400, 0.1), (1, 400, 0.35), (3, 64, 0.1), (4, 65, 0.7), (5, 1, 0.1), (2, 700, 0.5)])
def test_nms_emulated_bit_exact(oracle, emu, seed, n, thr):
    b = torch.from_numpy(synth.make_nms_boxes(seed, n))
    keep = torch.empty(max(n, 1), dtype=torch.int64)
    num = torch.zeros(1, dtype=torch.int32)
    ws = torch.empty(max(int(emu.sis3d_nms_workspace_bytes(n)), 8), dtype=torch.uint8)
    assert emu.sis3d_nms(_p(b), n, C.c_float(thr), _p(keep), _p(num), _p(ws), None) == 0
    assert np.array_equal(keep[:int(num)].numpy(), oracle.nms3d(b.numpy(), thr, fma_mode=1))


@pytest.mark.parametrize("dims,seed", [((11, 7, 10), 2), ((8, 8, 8), 3)])
def test_rpn_proposals_emulated_vs_oracle(oracle, host_S, dims, seed):
    from lib.layer_utils.proposal_layer import rpn_proposals
    from lib.utils.config import cfg_from_file, cfg_reset
    cfg_reset()
    cfg_from_file(os.path.join(ROOT, "3d-sis_b200", "experiments", "cfgs", "ScanNet", "rpn_class_mask_5.yml"))
    ocfg = oracle.make_cfg("scannet")
    rng = np.random.default_rng(seed)
    scene = tuple(4 * d for d in dims)
    levels, olevels, logit_pairs = [], [], []
    for A, tab in ((3, "scannet14_3.txt"), (11, "scannet14_11.txt")):
        n = dims[0] * dims[1] * dims[2]
        cls = (rng.standard_normal((n, 2 * A)) * 2).astype(np.float32)
        logit_pairs.append((cls, A))
        dl = (rng.standard_normal((n, 6 * A)) * 0.2).astype(np.float32)
        sizes = oracle.read_anchor_table(tab)
        levels.append(dict(cls=torch.from_numpy(cls), deltas=torch.from_numpy(dl), sizes=torch.tensor(sizes, dtype=torch.float32),
                           grid=dims, A=A, cls_mode=0))
        prob = F.softmax(torch.from_numpy(cls).view(n, 2, A), dim=1)[:, 1, :].reshape(-1)
        olevels.append((prob, torch.from_numpy(dl).view(-1, 6), oracle.generate_anchors(dims, sizes, 4)))
    want = oracle.proposal_layer(ocfg, olevels, scene, fma_mode=1)
    rois, scores, lvl, num, order = rpn_proposals(levels, scene, "TEST", want_order=True)
    n = int(num.item())
    inside = np.concatenate([oracle.inside_mask(l[2], scene) for l in olevels])
    want_flat = np.nonzero(inside)[0][want["order"]]
    got_flat = order.numpy()[:len(want_flat)]
    if not np.array_equal(got_flat, want_flat):  # expf of two math libraries: only near-tied neighbours may permute
        from test_gpu_decision_kernels import check_order_margin
        p64 = np.concatenate([1.0 / (1.0 + np.exp(c[:, :A].astype(np.float64) - c[:, A:].astype(np.float64))).reshape(-1)
                              for c, A in logit_pairs])
        check_order_margin(got_flat, np.nonzero(inside)[0], p64, len(want_flat))
    assert n == len(want["rois"])
    np.testing.assert_allclose(rois[:n].numpy(), want["rois"].numpy(), atol=1e-4, rtol=1e-5)
    assert np.array_equal(lvl[:n].numpy(), want["level_inds"].numpy().astype(np.int32))
    assert not rois[n:].any()


def test_rpn_fused_tail_huge_tie_and_unfused_chain_agree(oracle, host_S, monkeypatch):
    """The single-CTA fused tail (sort in shared memory, NMS bitmask in shared memory) against the four-kernel chain, and its
    exact fallback when more candidates share the histogram bin of the K-th best than fit in shared memory: with every
    foreground probability EQUAL all ~7.5k inside anchors are candidates, and the stable order (lower flat index first) decides."""
    from lib.layer_utils.proposal_layer import rpn_proposals
    from lib.utils.config import cfg_from_file, cfg_reset
    cfg_reset()
    cfg_from_file(os.path.join(ROOT, "3d-sis_b200", "experiments", "cfgs", "ScanNet", "rpn_class_mask_5.yml"))
    ocfg = oracle.make_cfg("scannet")
    rng = np.random.default_rng(9)
    dims = (20, 10, 18)
    scene = tuple(4 * d for d in dims)
    for tie in (True, False):
        levels, olevels = [], []
        for A, tab in ((3, "scannet14_3.txt"), (11, "scannet14_11.txt")):
            n = dims[0] * dims[1] * dims[2]
            prob = np.full((n, A), 0.625, np.float32) if tie else rng.uniform(0, 1, (n, A)).astype(np.float32)
            dl = (rng.standard_normal((n, 6 * A)) * 0.2).astype(np.float32)
            sizes = oracle.read_anchor_table(tab)
            levels.append(dict(cls=torch.from_numpy(prob), deltas=torch.from_numpy(dl), sizes=torch.tensor(sizes, dtype=torch.float32),
                               grid=dims, A=A, cls_mode=1))
            olevels.append((torch.from_numpy(prob).reshape(-1), torch.from_numpy(dl).view(-1, 6), oracle.generate_anchors(dims, sizes, 4)))
        want = oracle.proposal_layer(ocfg, olevels, scene, fma_mode=1)
        inside = np.concatenate([oracle.inside_mask(l[2], scene) for l in olevels])
        if tie:
            assert inside.sum() > 4096  # more candidates than the fused kernel sorts in shared memory
        outs = {}
        for unfused in (False, True):
            if unfused:
                monkeypatch.setenv("SIS3D_RPN_UNFUSED", "1")
            else:
                monkeypatch.delenv("SIS3D_RPN_UNFUSED", raising=False)
            rois, scores, lvl, num, order = rpn_proposals(levels, scene, "TEST", want_order=True)
            n = int(num.item())
            outs[unfused] = (rois.clone(), scores.clone(), lvl.clone(), n, order.clone())
            assert np.array_equal(order.numpy()[:len(want["order"])], np.nonzero(inside)[0][want["order"]])
            assert n == len(want["rois"])
            np.testing.assert_allclose(rois[:n].numpy(), want["rois"].numpy(), atol=1e-4, rtol=1e-5)
            assert np.array_equal(lvl[:n].numpy(), want["level_inds"].numpy().astype(np.int32))
            assert not rois[n:].any()
        a, b = outs[False], outs[True]
        assert a[3] == b[3] and all(torch.equal(x, y) for x, y in zip(a[:3], b[:3])) and torch.equal(a[4], b[4])
    monkeypatch.delenv("SIS3D_RPN_UNFUSED", raising=False)


def test_roi_pool_emulated_vs_oracle(oracle, emu):
    rng = np.random.default_rng(1)
    Cn, dims = 8, (12, 6, 11)
    feat = rng.standard_normal((Cn,) + dims).astype(np.float32)
    rois = np.array([[0, 0, 0, 47, 23, 43], [3.2, 1.7, 5.5, 20.1, 9.9, 30.3], [10, 4, 8, 10.5, 4.2, 8.1], [40, 20, 40, 48, 24, 44]],
                    dtype=np.float32)
    want_out, want_arg = oracle.roi_pool3d(feat[None], rois, (4, 4, 4), 0.25)
    f = torch.from_numpy(feat).contiguous()
    r = torch.from_numpy(rois)
    out = torch.empty(len(rois), Cn, 4, 4, 4)
    arg = torch.empty(len(rois), Cn, 4, 4, 4, dtype=torch.int32)
    rc = emu.sis3d_roi_pool_fwd(_p(f), 0, C.c_float(0.25), len(rois), *dims, Cn, 4, 4, 4, _p(r), _p(out), _p(arg), None)
    assert rc == 0
    assert np.array_equal(out.numpy(), np.asarray(want_out)) and np.array_equal(arg.numpy(), np.asarray(want_arg))


def test_mlp_tail_emulated_vs_torch(emu):
    """Classifier tail (FC2, FC3, both heads in one kernel with shared-memory weight slabs) under emulation."""
    torch.manual_seed(0)
    R, d1, d2, d3, nc, nb = 23, 256, 256, 128, 19, 114
    x1 = torch.randn(R, d1).relu()
    lin = lambda i, o: (torch.randn(o, i) / i ** 0.5, torch.randn(o) * 0.1)
    (w2, b2), (w3, b3), (wc, bc), (wb, bb) = lin(d1, d2), lin(d2, d3), lin(d3, nc), lin(d3, nb)

    def pack(w):  # [K][ldw], the layout of sis3d_pack_conv_weight(ks=1)
        o, i = w.shape
        pk = torch.zeros(i, (o + 3) // 4 * 4)
        pk[:, :o] = w.t()
        return pk.contiguous()
    pw2, pw3, pwc, pwb = pack(w2), pack(w3), pack(wc), pack(wb)
    cls, box = torch.full((R, nc), 9.0), torch.full((R, nb), 9.0)
    rc = emu.sis3d_mlp_tail(_p(x1), R, d1, _p(pw2), _p(b2), d2, _p(pw3), _p(b3), d3, _p(pwc), _p(bc), nc, _p(pwb), _p(bb), nb, _p(cls),
                            _p(box), None)
    assert rc == 0
    h = F.relu(F.linear(F.relu(F.linear(x1, w2, b2)), w3, b3))
    torch.testing.assert_close(cls, F.linear(h, wc, bc), atol=1e-4, rtol=1e-4)
    torch.testing.assert_close(box, F.linear(h, wb, bb), atol=1e-4, rtol=1e-4)


# ---------------------------------------------------------------- edge cases of the C entry points (no GPU needed)
def test_nms_emulated_empty_identical_and_many_blocks(oracle, emu):
    """n = 0 (the reference's gpu_nms is never called with it; the entry point must still report 0 survivors), every box
    identical (one survivor), disjoint boxes (all survive) and a list spanning many 64-box bitmask words."""
    num = torch.full((1,), 77, dtype=torch.int32)
    keep = torch.empty(1, dtype=torch.int64)
    ws = torch.empty(max(int(emu.sis3d_nms_workspace_bytes(0)), 8), dtype=torch.uint8)
    assert emu.sis3d_nms(None, 0, C.c_float(0.1), _p(keep), _p(num), _p(ws), None) == 0
    assert int(num) == 0
    for name, boxes, thr in (
            ("identical", np.tile(np.array([[3, 4, 5, 20, 21, 22]], np.float32), (130, 1)), 0.5),
            ("disjoint", np.array([[10 * i, 0, 0, 10 * i + 5, 5, 5] for i in range(200)], np.float32), 0.1),
            ("many words", synth.make_nms_boxes(8, 1500), 0.3)):
        b = torch.from_numpy(boxes)
        n = len(boxes)
        keep = torch.empty(n, dtype=torch.int64)
        num = torch.zeros(1, dtype=torch.int32)
        ws = torch.empty(int(emu.sis3d_nms_workspace_bytes(n)), dtype=torch.uint8)
        assert emu.sis3d_nms(_p(b), n, C.c_float(thr), _p(keep), _p(num), _p(ws), None) == 0, name
        want = oracle.nms3d(boxes, thr, fma_mode=1)
        assert np.array_equal(keep[:int(num)].numpy(), want), name
        if name == "identical":
            assert int(num) == 1
        if name == "disjoint":
            assert int(num) == n


def test_roi_pool_emulated_zero_rois_and_degenerate_boxes(oracle, emu):
    rng = np.random.default_rng(4)
    Cn, dims = 4, (9, 5, 7)
    feat = torch.from_numpy(rng.standard_normal((Cn,) + dims).astype(np.float32))
    out = torch.full((1, Cn, 4, 4, 4), 5.0)
    none = torch.zeros(1, 6)
    assert emu.sis3d_roi_pool_fwd(_p(feat), 0, C.c_float(0.25), 0, *dims, Cn, 4, 4, 4, _p(none), _p(out), None, None) == 0
    assert (out == 5.0).all()  # nothing written for zero RoIs
    assert emu.sis3d_roi_pool_fwd(_p(feat), 0, C.c_float(0.25), 0, *dims, Cn, 4, 4, 4, None, _p(out), None, None) != 0  # NULL rois: EINVAL
    # zero-extent box, a box entirely outside the map (empty bins -> 0 / argmax -1), a box hanging over the far border
    rois = np.array([[8, 8, 8, 8, 8, 8], [100, 100, 100, 120, 110, 115], [30, 15, 22, 60, 40, 50], [-5, -5, -5, 3, 3, 3]], np.float32)
    want_out, want_arg = oracle.roi_pool3d(feat.numpy()[None], rois, (4, 4, 4), 0.25)
    r = torch.from_numpy(rois)
    out = torch.empty(len(rois), Cn, 4, 4, 4)
    arg = torch.empty(len(rois), Cn, 4, 4, 4, dtype=torch.int32)
    assert emu.sis3d_roi_pool_fwd(_p(feat), 0, C.c_float(0.25), len(rois), *dims, Cn, 4, 4, 4, _p(r), _p(out), _p(arg), None) == 0
    assert np.array_equal(out.numpy(), np.asarray(want_out)) and np.array_equal(arg.numpy(), np.asarray(want_arg))


def test_rpn_proposals_emulated_scene_smaller_than_every_anchor(oracle, host_S):
    """No anchor lies inside a 1x1x1-cell level grid of a 4^3 scene with ALLOW_BORDER = 0: zero candidates, zero RoIs, padded rows
    all zero (lib/layer_utils/proposal_layer.py:36-43 keeps nothing; the reference would then fail in torch.cat -- here the
    stage reports an empty result)."""
    from lib.layer_utils.proposal_layer import rpn_proposals
    from lib.utils.config import cfg_from_file, cfg_reset
    cfg_reset()
    cfg_from_file(os.path.join(ROOT, "3d-sis_b200", "experiments", "cfgs", "ScanNet", "rpn_class_mask_5.yml"))
    dims, scene = (1, 1, 1), (4, 4, 4)
    rng = np.random.default_rng(0)
    levels = []
    for A, tab in ((3, "scannet14_3.txt"), (11, "scannet14_11.txt")):
        sizes = oracle.read_anchor_table(tab)
        assert not oracle.inside_mask(oracle.generate_anchors(dims, sizes, 4), scene).any()
        levels.append(dict(cls=torch.from_numpy(rng.standard_normal((1, 2 * A)).astype(np.float32)),
                           deltas=torch.from_numpy(rng.standard_normal((1, 6 * A)).astype(np.float32)),
                           sizes=torch.tensor(sizes, dtype=torch.float32), grid=dims, A=A, cls_mode=0))
    rois, scores, lvl, num, order = rpn_proposals(levels, scene, "TEST", want_order=True)
    assert int(num.item()) == 0 and not rois.any() and not lvl.any()
