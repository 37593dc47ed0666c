"""GPU: the detection head -- proposals, RoI pooling, the MLP tail and detection decode -- step by step on its own inputs, in
every conv math mode, on the bench scenes.

One eager forward per row runs with `net._keep_debug = True` and per-kernel timing on (`net._prof = {}`: no CUDA graph, no
parallel branches).  It keeps the level features, the merged RPN heads, the pre-NMS order and `pool5`; `_linear` is wrapped
(test_gpu_static_stage.Capture) for classifier.0's input and output, and `_static_stage` for the carved result buffer (rois,
scores, level ids, count, class scores, box deltas, class probabilities, argmax, detection table).  Every reference is fp64,
built from the live parameters (`net.state_dict()`) and the cfg's anchor tables (oracle.port), never from packed weights.
Each step reads the device's own upstream outputs (teacher forcing), so a near-tied decision may go either way and the next
step follows the device's choice:

  - proposals, from the captured heads: fp64 two-way softmax, anchors, inside filter, decode + clip.  The pre-NMS order is
    exact outside the 12u p near-tie band (check_order_margin; a top-K boundary inside the band accepts either set).  Each
    kept row is the next candidate of the device's order whose level equals it, whose fp64 score is within 12u p and whose
    fp64 box is within 12u (|half extent| + |coordinate|).  The keep list is consistent along the greedy chain: a kept
    candidate has no IoU > thresh + IOU_BAND with an earlier kept one, a dropped candidate has one > thresh - IOU_BAND.  The
    count is min(post-NMS count, survivors) and rows from it on are zero;
  - RoI pooling: oracle.port's roi_pool3d on the captured level features, the device's rois and level ids, flattened in the
    reference's [C][P][P][P] order, equals `pool5` bit for bit; classifier.0 reads `pool5`'s bits;
  - the MLP tail, from classifier.0's captured output: within the fp64 bound carried through the layers (mlp_forward);
  - detection decode, from the device's rois, count, class scores and box deltas: probabilities within (nc + 8)u p of the
    fp64 softmax, the argmax that of the fp32 scores, boxes within the 12u rule on the predicted class's slice, the keep flag
    `conf > CLASS_THRESH` on the device's own conf, crops Python's round() of the device's own box floats and degenerate crops
    dropped, the count in det[0, 15] and every row from it on zero;
  - transport: the returned predictions and the host copy of the detection table equal the carved buffer bit for bit, and a
    default forward (CUDA graph, branches; the dense colour path the eager run takes) reproduces every head output bit for
    bit.

Power: fp64 models of broken wiring (MUTANTS) must fail their step's check by POWER in every row where they apply.  In the
rows after an in-place parameter update, the static-stage checks of test_gpu_static_stage run as well, so a stale merged RPN
head fails there.  HEAD_CHECKS lists what checks each `_rec` name of the head (tests/test_head_stage_coverage.py keeps it
complete)."""
import math

import numpy as np
import pytest
import torch

import sis3d_synth as synth
from test_gpu_decision_kernels import IOU_BAND, RPN_KERNELS, check_order_margin, kernel_names
from test_gpu_simt_accuracy import mlp_forward
from test_gpu_static_stage import CYCLE, SCENES as STATIC_SCENES, Capture, Row as StaticRow, blobs_of, same_bits
from test_gpu_tc_accuracy import POWER, _check

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
TINY = 2.0 ** -122    # absolute floor of a score bound: fp32 expf / division results near the subnormal range

HEAD_CHECKS = {  # `_rec` name of the head -> the step that checks it
    "rpn_proposals": "proposals",
    "roi_pool_levels": "roi_pool",
    "mlp_tail": "mlp_tail",
    "detect_decode": "decode",
}
STEPS = ("proposals", "roi_pool", "link", "mlp_tail", "decode", "transport")
MUTANTS = {  # fp64 model of broken wiring -> the step whose check it must fail
    "fg_bg_logits_swapped": "proposals",
    "anchor_index_a_major": "proposals",
    "level2_deltas_at_level1_offset": "proposals",
    "nms_skipped": "proposals",
    "all_rois_from_level1": "roi_pool",
    "scale_one_half": "roi_pool",
    "pool5_channels_last": "roi_pool",
    "cls_box_heads_swapped": "mlp_tail",
    "weights_before_update": "mlp_tail",
    "class_slice_off_by_one": "decode",
    "ge_for_gt": "decode",
    "round_half_up": "decode",
    "conf_from_class0": "decode",
}
# parameters updated in place before the last exact pass of a cycle: the tail's last hidden layer, the box head's bias, the
# level-2 RPN box head (merged into rpn_heads_level2)
UPDATES = (("classifier.4.weight", lambda p: p.mul_(1.25)), ("classifier_bbox_pred_net.bias", lambda p: p.add_(0.25)),
           ("rpn_bbox_pred_net_level2.weight", lambda p: p.mul_(1.25)))
LIBRARY_PRE_NMS = 6000  # TEST.RPN_PRE_NMS_TOP_N of lib/utils/config.py (the released ymls use 400)
SMALL_POST_NMS = 7


def empty_volume(tables):
    """The largest cube d^3 whose level grid (d // 4 per axis) holds no anchor of any of `tables` inside the volume."""
    from oracle import port
    best = None
    for d in range(4, 65):
        g = (d // 4,) * 3
        if any(port.inside_mask(port.generate_anchors(g, port.read_anchor_table(t), 4), (d, d, d)).any() for t in tables):
            break
        best = d
    return best


EMPTY_D = empty_volume(("scannet14_3.txt", "scannet14_11.txt"))
SCENES = dict(STATIC_SCENES, suncg_40x24x40=synth.CASES["suncg_40x24x40"],
              empty=dict(cfgname="scannet", dims=(EMPTY_D,) * 3, n_img=0, seed=909, use_images=False, use_mask=True))


def _rows():
    rows = []
    for scene in ("cfg2", "cfg5", "odd_45x27x41", "suncg_40x24x40"):
        rows += [dict(scene=scene, mode=m, step=i, kind="cycle") for i, m in enumerate(CYCLE)]
        rows.append(dict(scene=scene, mode="exact", step=len(CYCLE), kind="updated"))
    n = len(CYCLE) + 1
    rows += [dict(scene="cfg2", mode="exact", step=n, kind="post_nms_7"),
             dict(scene="cfg2", mode="exact", step=n + 1, kind="thresh_exact"),
             dict(scene="cfg2", mode="exact", step=n + 2, kind="thresh_one")]
    rows += [dict(scene="cfg3", mode=m, step=i, kind="cycle") for i, m in enumerate(("exact", "fp16"))]
    rows.append(dict(scene="cfg3", mode="exact", step=2, kind="pre_nms_6000"))
    rows += [dict(scene="cfg1_32", mode=m, step=i, kind="cycle") for i, m in enumerate(("exact", "fp32"))]
    rows.append(dict(scene="empty", mode="exact", step=0, kind="empty"))
    for r in rows:
        r["id"] = f"{r['scene']}-{r['step']}-{r['mode']}" + ("" if r["kind"] == "cycle" else "-" + r["kind"].replace("_", "-"))
    return rows


ROWS = _rows()


# ------------------------------------------------------------------------------------------------ capture
PRED_KEYS = ("rois", "roi_scores", "level_inds", "cls_score", "cls_pred", "cls_prob", "bbox_pred", "detections")


def _pred(P):
    """Clones of the returned head predictions (the dict is reused by the next forward)."""
    out = {k: (P[k][0] if isinstance(P[k], list) else P[k]).clone() for k in PRED_KEYS if k in P}
    if "detections_host" in P:
        out["detections_host"] = torch.from_numpy(np.array(P["detections_host"], copy=True))
    return out


def run_eager(net, blobs, full=False):
    """One eager forward with the debug tensors kept: (capture, carved result buffer, debug tensors, predictions, prof names)."""
    cap = Capture(net) if full else Capture(net, hooked=("_linear",))
    stage = {}
    orig = net._static_stage

    def static_stage(*a, **k):
        out = orig(*a, **k)
        stage.update(out)
        return out

    net.__dict__["_static_stage"] = static_stage
    net._keep_debug, net._prof = True, {}
    try:
        P = net.forward(blobs, "TEST", None)
        torch.cuda.synchronize()
        prof = set(net._prof)
        carved = {k: v.clone() for k, v in stage.items() if k != "pack"}
        debug = {k: P[k].clone() for k in P if k.startswith(("level1_vc", "level2_vc", "rpn_heads_level", "rpn_order", "pool5"))}
        pred = _pred(P)
        pred["mask_pred"] = [len(m) for m in P.get("mask_pred", [])]
    finally:
        net.__dict__.pop("_static_stage", None)
        cap.detach()
        net._keep_debug, net._prof = False, None
    return cap, carved, debug, pred, prof


# ------------------------------------------------------------------------------------------------ fp64 pieces
def decode64(anchors, deltas, dims):
    """fp64 bbox_transform_inv + clip: ([n][6] boxes, [n][6] bound 12u (|half extent| + |coordinate|))."""
    a, d = anchors.astype(np.float64), deltas.astype(np.float64)
    w = a[:, 3:] - a[:, :3]
    pc = d[:, :3] * w + (a[:, :3] + 0.5 * w)
    hw = 0.5 * np.exp(d[:, 3:]) * w
    dm = np.asarray(dims, np.float64)
    box = np.concatenate([np.clip(pc - hw, 0, dm), np.clip(pc + hw, 0, dm)], 1)
    return box, 12 * U * (np.concatenate([hw, hw], 1) + np.abs(box)) + 1e-30


def iou64(a, b):
    """[n][m] IoU of the reference's NMS (extents + 1) in fp64."""
    lo = np.maximum(a[:, None, :3], b[None, :, :3])
    hi = np.minimum(a[:, None, 3:], b[None, :, 3:])
    inter = np.prod(np.maximum(hi - lo + 1, 0), -1)
    va, vb = np.prod(a[:, 3:] - a[:, :3] + 1, -1), np.prod(b[:, 3:] - b[:, :3] + 1, -1)
    return inter / (va[:, None] + vb[None, :] - inter)


def _ratio(got, ref, bound):
    """max |got - ref| / bound (0 where equal, inf where the bound is 0 and they differ); 0 when empty."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if got.size == 0:
        return 0.0
    e = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(e == 0, 0.0, e / bound)
    return float(np.nan_to_num(r, nan=math.inf).max())


def _exact(a, b):
    """Ratio of a bit-exact check: 0 when equal, inf otherwise."""
    a, b = np.asarray(a), np.asarray(b)
    return 0.0 if a.shape == b.shape and np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                                        b.view(np.int32) if b.dtype == np.float32 else b) else math.inf


class Head:
    """The checks of one captured forward (module docstring)."""

    def __init__(self, row, net, cfg, cap, carved, debug, pred, prof, old=None):
        from oracle import port
        self.port, self.row, self.net, self.cfg = port, row, net, cfg
        self.cap, self.c, self.debug, self.pred, self.prof, self.old = cap, carved, debug, pred, prof, old
        self.rid = row["id"]
        self.sd = {k: v.detach().to(DEV, torch.float64) for k, v in net.state_dict().items()}
        self.dims = tuple(SCENES[row["scene"]]["dims"])
        self.num = int(carved["num"][0])
        self.R, self.nc = int(cfg.TEST.RPN_POST_NMS_TOP_N), int(cfg.NUM_CLASSES)
        self.err, self.mut, self.band = {}, {}, {}

    def mutant(self, name, ratio):
        assert MUTANTS[name]
        self.mut[name] = ratio

    # -------------------------------------------------------------- proposals
    def levels(self):
        cfg = self.cfg
        out = []
        for lvl in (1, 2, 3):
            A = int(cfg.get("NUM_ANCHORS_LEVEL%d" % lvl, 0) or 0)
            if not A:
                continue
            grid = tuple((d // 2) // 2 for d in self.dims)   # two stride-2 convolutions
            feat = self.debug[f"level{lvl}_vc"].reshape(*grid, -1)
            N, ld = int(np.prod(grid)), self.net._layers[f"rpn_heads_level{lvl}"][1]
            heads = self.debug[f"rpn_heads_level{lvl}"].reshape(-1)[:N * ld].view(N, ld).double().cpu().numpy()
            out.append(dict(lvl=lvl, A=A, grid=grid, N=N, ld=ld, heads=heads, feat=feat,
                            anchors=self.port.generate_anchors(grid, self.port.read_anchor_table(cfg["ANCHORS_TYPE_LEVEL%d" % lvl]), 4)))
        return out

    @staticmethod
    def score64(s0, s1):
        return 1.0 / (1.0 + np.exp(s0 - s1))

    def flat(self, lvls, a_major=False, deltas_col=None):
        """Concatenated per-flat-anchor fp64 scores, deltas, anchors and level ids (flat = vox * A + a per level).
        a_major: scores and deltas read as if flat were a * N + vox; deltas_col: level -> first delta column."""
        p, d, an, lv = [], [], [], []
        for L in lvls:
            A, N, h = L["A"], L["N"], L["heads"]
            f = np.arange(N * A)
            vox, a = (f % N, f // N) if a_major else (f // A, f % A)
            c0 = (deltas_col or {}).get(L["lvl"], 2 * A)
            p.append(self.score64(h[vox, a], h[vox, A + a]))
            d.append(np.stack([h[vox, c0 + 6 * a + k] for k in range(6)], 1))
            an.append(L["anchors"])
            lv.append(np.full(N * A, L["lvl"], np.int32))
        return np.concatenate(p), np.concatenate(d), np.concatenate(an), np.concatenate(lv)

    def proposals(self):
        cfg, rid, num = self.cfg, self.rid, self.num
        pre, post, thr = int(cfg.TEST.RPN_PRE_NMS_TOP_N), int(cfg.TEST.RPN_POST_NMS_TOP_N), float(cfg.TEST.RPN_NMS_THRESH)
        lvls = self.levels()
        self.lvls = lvls
        p64, d64, anchors, lv = self.flat(lvls)
        inside = self.port.inside_mask(anchors, self.dims, int(cfg.ALLOW_BORDER))
        flat_inside = np.nonzero(inside)[0]
        keff = min(pre, len(flat_inside))
        order = self.debug["rpn_order"].cpu().numpy()
        assert order.shape[0] == pre and bool((order[keff:] == -1).all()), f"{rid}: order rows past {keff} are not -1"
        got = order[:keff].astype(np.int64)
        st = {}
        check_order_margin(got, flat_inside, p64, keff, either_set=True, stats=st)
        self.band.update(order=st["order_in_band"], topk_boundary=int(st["boundary_in_band"]))
        # the kept rows: each the next candidate of the device's order it matches
        box64, bnd64 = decode64(anchors[got], d64[got], self.dims)
        ps, lvp = p64[got], lv[got]
        rois = self.c["rois"].double().cpu().numpy()
        scores = self.c["scores"].double().cpu().numpy()
        lids = self.c["level_ids"].cpu().numpy()
        assert 0 <= num <= min(post, keff), f"{rid}: {num} proposals of {keff} candidates, post-NMS {post}"
        kept, prev, s_err, b_err = [], -1, 0.0, 0.0
        for j in range(num):
            ok = (lvp == lids[j]) & (np.abs(scores[j] - ps) <= 12 * U * ps + TINY) & (np.abs(rois[j] - box64) <= bnd64).all(1)
            ok[:prev + 1] = False
            hit = np.nonzero(ok)[0]
            assert len(hit), f"{rid}: proposal {j} (level {lids[j]}) matches no candidate of the order after position {prev}"
            prev = int(hit[0])
            kept.append(prev)
            s_err = max(s_err, _ratio(scores[j], ps[prev], 12 * U * ps[prev] + TINY))
            b_err = max(b_err, _ratio(rois[j], box64[prev], bnd64[prev]))
        kept = np.asarray(kept, np.int64)
        self.err["proposals"] = max(s_err, b_err)
        # NMS along the greedy chain; the count: every candidate after the last kept one is dropped unless the count is full
        last = keff if num < post else (kept[-1] + 1 if num else 0)
        n_band = 0
        if num:
            iou = iou64(box64[:last], box64[kept])
            before = kept[None, :] < np.arange(last)[:, None]
            m = np.where(before, iou, -1.0).max(1)
            is_kept = np.zeros(last, bool)
            is_kept[kept] = True
            bad_keep = is_kept & (m > thr + IOU_BAND)
            bad_drop = ~is_kept & (m <= thr - IOU_BAND)
            assert not bad_keep.any(), f"{rid}: kept candidate {int(np.nonzero(bad_keep)[0][0])} overlaps an earlier kept one"
            assert not bad_drop.any(), f"{rid}: candidate {int(np.nonzero(bad_drop)[0][0])} was dropped with no kept overlap"
            n_band = int((np.abs(m - thr) <= IOU_BAND).sum())
        else:
            assert keff == 0 or post == 0, f"{rid}: no proposal from {keff} candidates"
        self.band["nms"] = n_band
        for k, t in (("rois", self.c["rois"]), ("scores", self.c["scores"]), ("level_ids", self.c["level_ids"])):
            assert not t[num:].any(), f"{rid}: {k} rows from {num} on are not zero"
        self.kept, self.got_order = kept, got
        # wiring models: the rows the device emitted, as a kernel wired that way would have decoded them
        if num:
            fk = got[kept]

            def rows_ratio(p, d, order_flat=None):
                fl = fk if order_flat is None else order_flat
                b, bb = decode64(anchors[fl], d[fl], self.dims)
                return max(_ratio(scores[:num], p[fl], 12 * U * p[fl] + TINY), _ratio(rois[:num], b, bb),
                           0.0 if np.array_equal(lids[:num], lv[fl]) else math.inf)

            self.mutant("fg_bg_logits_swapped", rows_ratio(1.0 - p64, d64))
            pa, da, _, _ = self.flat(lvls, a_major=True)
            self.mutant("anchor_index_a_major", rows_ratio(pa, da))
            if len(lvls) > 1 and lvls[0]["A"] != lvls[1]["A"] and (lids[:num] == 2).any():
                _, dw, _, _ = self.flat(lvls, deltas_col={2: 2 * lvls[0]["A"]})
                self.mutant("level2_deltas_at_level1_offset", rows_ratio(p64, dw))
            if not np.array_equal(kept, np.arange(num)):
                self.mutant("nms_skipped", rows_ratio(p64, d64, got[:num]))

    # -------------------------------------------------------------- RoI pooling and the link to classifier.0
    def pool(self, feats, rois, lids, scale, channels_last=False):
        P = int(self.cfg.CLASS_POOLING_SIZE)
        out = np.zeros((len(rois), feats[0].shape[0], P, P, P), np.float32)
        for i, f in enumerate(feats, 1):
            sel = np.nonzero(lids == i)[0]
            if len(sel):
                out[sel] = self.port.roi_pool3d(f, rois[sel], (P, P, P), scale)[0]
        if channels_last:
            out = out.transpose(0, 2, 3, 4, 1)
        return out.reshape(len(rois), feats[0].shape[0] * P ** 3)

    def roi_pool(self):
        rid, num = self.rid, self.num
        pool5 = self.debug["pool5"].cpu().numpy()
        assert pool5.shape[0] == self.R and not pool5[num:].any(), f"{rid}: pool5 rows from {num} on are not zero"
        feats = [np.ascontiguousarray(L["feat"].permute(3, 0, 1, 2).cpu().numpy()) for L in self.lvls]
        rois, lids = self.c["rois"][:num].cpu().numpy(), self.c["level_ids"][:num].cpu().numpy()
        scale = 1.0 / self.net._feat_stride[0]
        got = pool5[:num]
        self.err["roi_pool"] = _exact(got, self.pool(feats, rois, lids, scale))
        assert self.err["roi_pool"] == 0, f"{rid}: pool5 differs from the reference's RoI pooling of the device's rois"
        if num:
            if (lids == 2).any():
                self.mutant("all_rois_from_level1", _exact(got, self.pool(feats, rois, np.ones_like(lids), scale)))
            self.mutant("scale_one_half", _exact(got, self.pool(feats, rois, lids, 0.5)))
            self.mutant("pool5_channels_last", _exact(got, self.pool(feats, rois, lids, scale, channels_last=True)))
        lin = [o for o in self.cap.ops if o["kind"] == "linear" and o["name"] == "classifier.0"]
        assert len(lin) == 1, f"{rid}: classifier.0 ran {len(lin)} times"
        self.x1 = lin[0]["y"]
        self.err["link"] = _exact(lin[0]["x"].cpu().numpy(), pool5)
        assert self.err["link"] == 0, f"{rid}: classifier.0 does not read pool5's bits"

    # -------------------------------------------------------------- MLP tail
    def layers(self, sd):
        return [(sd[f"{k}.weight"], sd[f"{k}.bias"]) for k in ("classifier.2", "classifier.4", "classifier_cls_score_net",
                                                             "classifier_bbox_pred_net")]

    def mlp_tail(self):
        L = self.layers(self.sd)
        ref, bound = mlp_forward(self.x1, L)
        got = torch.cat([self.c["cls_score"].reshape(-1), self.c["bbox_pred"].reshape(-1)])
        nc = self.nc
        (wc, bc), (wb, bb) = L[2], L[3]
        pad = lambda t: torch.cat([t, t.new_zeros(5 * nc, *t.shape[1:])])
        mut = {"cls_box_heads_swapped": mlp_forward(self.x1, L[:2] + [(wb[:nc], bb[:nc]), (pad(wc), pad(bc))])[0]}
        if self.old is not None:
            sd = dict(self.sd, **{k: v.to(DEV, torch.float64) for k, v in self.old.items()})
            mut["weights_before_update"] = mlp_forward(self.x1, self.layers(sd))[0]
        k, _ = _check(got, ref, bound, {}, 0, f"{self.rid} mlp_tail")
        self.err["mlp_tail"] = k
        for name, v in mut.items():
            e = (v - got.double()).abs()
            self.mutant(name, torch.where(e == 0, torch.zeros_like(e), e / bound).max().item())

    # -------------------------------------------------------------- detection decode
    def decode(self):
        rid, num, nc, R = self.rid, self.num, self.nc, self.R
        cs = self.c["cls_score"].cpu().numpy()
        bp = self.c["bbox_pred"].cpu().numpy()
        prob = self.c["cls_prob"].cpu().numpy()
        pred = self.c["cls_pred"].cpu().numpy()
        det = self.c["det"].cpu().numpy()
        rois = self.c["rois"].cpu().numpy()
        thresh = np.float32(self.cfg.CLASS_THRESH)
        assert det[0, 15] == num and not det[1:, 15].any(), f"{rid}: det[0, 15] is {det[0, 15]}, the count {num}"
        assert not det[num:, :15].any() and not pred[num:].any() and not prob[num:].any(), f"{rid}: rows from {num} on are not zero"
        if num == 0:
            self.err["decode"] = 0.0
            return
        s, pr, pd, dt = cs[:num].astype(np.float64), prob[:num], pred[:num], det[:num]
        e = np.exp(s - s.max(1, keepdims=True))
        p64 = e / e.sum(1, keepdims=True)
        e_prob = _ratio(pr, p64, (nc + 8) * U * p64)
        assert e_prob <= 1, f"{rid}: class probabilities err/bound {e_prob:.3g}"
        assert np.array_equal(pd, cs[:num].argmax(1)), f"{rid}: cls_pred is not the first maximum of the class scores"
        assert np.array_equal(dt[:, 7], pd.astype(np.float32)), f"{rid}: det[:, 7] is not cls_pred"
        rows = np.arange(num)

        def boxes(c):
            d = np.stack([bp[rows, 6 * c + k] for k in range(6)], 1)
            return decode64(rois[:num], d, self.dims)

        b64, bb = boxes(pd)
        e_box = _ratio(dt[:, :6], b64, bb)
        assert e_box <= 1, f"{rid}: detection boxes err/bound {e_box:.3g}"
        conf = dt[:, 6]
        assert _exact(conf, pr[rows, pd]) == 0, f"{rid}: conf is not the predicted class's probability"
        crops = np.rint(dt[:, :6].astype(np.float64)).astype(np.float32)   # round half to even, as Python's round()
        assert _exact(dt[:, 9:15], crops) == 0, f"{rid}: crops are not round() of the device's boxes"
        solid = (crops[:, 0] < crops[:, 3]) & (crops[:, 1] < crops[:, 4]) & (crops[:, 2] < crops[:, 5])
        keep = (conf > thresh) & solid
        assert np.array_equal(dt[:, 8], keep.astype(np.float32)), f"{rid}: keep flags are not conf > CLASS_THRESH on solid crops"
        self.err["decode"] = max(e_prob, e_box)
        self.kept_det = keep
        # wiring models
        self.mutant("class_slice_off_by_one", _ratio(dt[:, :6], *boxes(np.where(pd + 1 < nc, pd + 1, pd - 1))))
        if ((conf == thresh) & solid).any():
            self.mutant("ge_for_gt", _exact(dt[:, 8], ((conf >= thresh) & solid).astype(np.float32)))
        if (np.abs(dt[:, :6] - np.floor(dt[:, :6])) == 0.5).any():
            self.mutant("round_half_up", _exact(dt[:, 9:15], np.floor(dt[:, :6].astype(np.float64) + 0.5).astype(np.float32)))
        if (pr[:, 0] != conf).any():
            self.mutant("conf_from_class0", _exact(conf, pr[:, 0]))

    # -------------------------------------------------------------- transport
    def transport(self):
        rid, num, p, c = self.rid, self.num, self.pred, self.c
        want = dict(rois=c["rois"][:num], roi_scores=c["scores"][:num].view(-1, 1), level_inds=c["level_ids"][:num].float(),
                    cls_score=c["cls_score"][:num], cls_pred=c["cls_pred"][:num], cls_prob=c["cls_prob"][:num],
                    bbox_pred=c["bbox_pred"][:num], detections=c["det"][:num])
        for k, v in want.items():
            assert same_bits(p[k], v), f"{rid}: the returned {k} is not the carved buffer's"
        if self.cfg.USE_MASK:
            assert same_bits(p["detections_host"], c["det"][:num].cpu()), f"{rid}: the host detection table is not the device's"
        self.err["transport"] = 0.0

    def run(self):
        names = [n for n in self.cap.loose if n in HEAD_CHECKS or n == "mask_stage"]
        want = list(HEAD_CHECKS) + (["mask_stage"] if self.cfg.USE_MASK and sum(self.pred["mask_pred"]) else [])
        assert names == want, f"{self.rid}: the head ran {names}"
        for step in (self.proposals, self.roi_pool, self.mlp_tail, self.decode, self.transport):
            step()
        weak = {k: v for k, v in self.mut.items() if v < POWER}
        assert not weak, f"{self.rid}: wiring models pass their step's check: {weak}"
        return dict(err=self.err, min_model=min(self.mut.items(), key=lambda kv: kv[1], default=(None, math.inf)),
                    models=self.mut, in_band=self.band, num=self.num)


# ------------------------------------------------------------------------------------------------ the test
def _default_forward_same(net, blobs, got, rid):
    """Two default forwards (the second replays a captured CUDA graph) give the eager run's head outputs bit for bit.  They
    take the dense colour path, as the eager run does (`_keep_debug` keeps the dense back-projected volume): the sparse
    path sums colour.0 in another order, so its detections may differ in near-tied decisions."""
    sparse = net._sparse_color
    net._sparse_color = False
    try:
        for attempt in range(2):
            d = _pred(net.forward(blobs, "TEST", None))
            torch.cuda.synchronize()
            assert set(d) == set(got) - {"mask_pred"}, f"{rid}: default forward returned {sorted(d)}"
            for k, v in d.items():
                assert same_bits(v.cpu(), got[k].cpu()), f"{rid}: {k} of the default forward (pass {attempt}) differs from the eager run"
    finally:
        net._sparse_color = sparse


@pytest.mark.parametrize("scene", list(dict.fromkeys(r["scene"] for r in ROWS)))
def test_head_stage_against_fp64(scene, record_property):
    c = SCENES[scene]
    rows = [r for r in ROWS if r["scene"] == scene]
    net, cfg = synth.make_net(c, keep_debug=False, math="exact")
    blobs = blobs_of(c)
    base = {k: (cfg.TEST[k] if k.startswith("RPN") else cfg[k]) for k in ("RPN_PRE_NMS_TOP_N", "RPN_POST_NMS_TOP_N",
                                                                            "CLASS_THRESH")}
    old, last_exact = None, None
    for row in rows:
        kind, rid = row["kind"], row["id"]
        if kind == "updated":
            with torch.no_grad():
                ps = dict(net.named_parameters())
                old = {k: ps[k].detach().clone() for k, _ in UPDATES}
                for k, fn in UPDATES:
                    fn(ps[k])
        if kind == "pre_nms_6000":
            cfg.TEST.RPN_PRE_NMS_TOP_N = LIBRARY_PRE_NMS
        elif kind == "post_nms_7":
            cfg.TEST.RPN_POST_NMS_TOP_N = SMALL_POST_NMS
        elif kind == "thresh_exact":
            # a detection with a solid crop: kept at a threshold just below its conf, dropped at exactly its conf
            det = last_exact["det"].cpu().numpy()
            solid = np.nonzero((det[:, 9:12] < det[:, 12:15]).all(1))[0]
            assert len(solid), f"{rid}: the previous exact pass has no detection with a solid crop"
            cfg.CLASS_THRESH = float(det[solid[0], 6])
        elif kind == "thresh_one":
            cfg.CLASS_THRESH = 1.0
        net.set_conv_math(row["mode"])
        try:
            cap, carved, debug, pred, prof = run_eager(net, blobs, full=kind == "updated")
            chk = Head(row, net, cfg, cap, carved, debug, pred, prof, old if kind == "updated" else None)
            res = chk.run()
            if kind == "updated":  # every static-stage layer against the live parameters: a stale merged RPN head fails here
                srow = dict(id=rid, mode=row["mode"], sparse=False)
                vol = blobs["data"][0].permute(1, 2, 3, 0).contiguous().to(DEV)
                StaticRow(srow, net, cap, None, c["use_images"], vol).run()
            num = res["num"]
            if kind == "pre_nms_6000":
                def eager():
                    net._prof = {}
                    try:
                        net.forward(blobs, "TEST", None)
                    finally:
                        net._prof = None
                names = kernel_names(eager)
                assert names is not None and set(RPN_KERNELS["unfused"]) <= set(names) and \
                    not {"rpn_sort_decode_kernel", "nms_reduce_smem_kernel"} & set(names), f"{rid}: proposal kernels {names}"
                assert debug["rpn_order"].shape[0] == LIBRARY_PRE_NMS
            if kind == "post_nms_7":
                assert num == SMALL_POST_NMS and carved["rois"].shape[0] == SMALL_POST_NMS, f"{rid}: {num} proposals"
            if kind == "thresh_exact":
                d = carved["det"].cpu().numpy()
                hit = np.nonzero(d[:, 6] == np.float32(cfg.CLASS_THRESH))[0]
                assert len(hit) and not d[hit, 8].any(), f"{rid}: a detection with conf == CLASS_THRESH is kept"
                assert "ge_for_gt" in res["models"]
            if kind == "thresh_one":
                assert not carved["det"][:, 8].any() and "mask_stage" not in prof, f"{rid}: CLASS_THRESH = 1 kept a detection"
            if kind == "empty":
                assert num == 0 and not carved["det"].any(), f"{rid}: {num} proposals in a volume no anchor fits"
                assert "mask_stage" not in prof and pred["rois"].shape[0] == 0 and pred["detections"].shape[0] == 0
                assert pred["mask_pred"] in ([], [0]), pred["mask_pred"]
            _default_forward_same(net, blobs, pred, rid)
        finally:
            cfg.TEST.RPN_PRE_NMS_TOP_N, cfg.TEST.RPN_POST_NMS_TOP_N = base["RPN_PRE_NMS_TOP_N"], base["RPN_POST_NMS_TOP_N"]
            cfg.CLASS_THRESH = base["CLASS_THRESH"]
        if row["mode"] == "exact" and kind in ("cycle", "updated"):  # the released counts: classifier.0's split-K depends on them
            last_exact = carved
        summary = dict(err=res["err"], min_model=res["min_model"], models=res["models"], in_band=res["in_band"], num=num)
        print(f"{rid}: num {num}, err/bound {res['err']}, models {res['models']}, in band {res['in_band']}")
        record_property(rid, summary)
        del chk, cap
    record_property("rows", len(rows))
