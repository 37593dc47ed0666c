"""oracle/port_gt_rois.py -- TEST INFRASTRUCTURE ONLY.

CPU restatement of the TEST forward on ground-truth boxes and classes (USE_RPN = USE_CLASS = False), the checker for that
mode of the sm_90a path.  It composes oracle/port.py's decode and mask head, which are pinned to the reference on their own;
this forward is pinned to the reference by tests/golden/gt_rois_reference.npz (oracle/make_golden_gt_rois.py,
tests/test_gt_rois.py).  The product path never imports it.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import port


def forward_gt_rois(cfg, w, data, gt_box):
    """network.py:262-265, 276-317 with USE_RPN = USE_CLASS = False: rois = gt_box[:, :6], roi_scores = 1,
    cls_pred = gt_box[:, 6].long(), a one-hot cls_prob, zero bbox_pred, then the usual decode and one mask crop per kept box.
    USE_BACKBONE and USE_IMAGES cannot change any of it, so neither runs."""
    with torch.no_grad():
        scene = torch.as_tensor(data, dtype=torch.float32)
        dims = tuple(int(v) for v in scene.shape[2:])
        gt = torch.as_tensor(np.asarray(gt_box, dtype=np.float32).reshape(-1, 7))
        n = gt.shape[0]
        cls_pred = gt[:, 6].long()
        cls_prob = torch.zeros(n, cfg.NUM_CLASSES)
        cls_prob[torch.arange(n), cls_pred] = 1.0
        bbox_pred = torch.zeros(n, cfg.NUM_CLASSES * 6)
        out = dict(rois=gt[:, :6].clone(), roi_scores=torch.ones(n, 1), cls_pred=cls_pred, cls_prob=cls_prob,
                   bbox_pred=bbox_pred)
        if cfg.USE_MASK:
            pred_box, conf, keep, crops = port.detection_boxes(cfg, out["rois"].numpy(), cls_pred.numpy(), cls_prob.numpy(),
                                                               bbox_pred.numpy(), dims)
            masks = [port.mask_head(w, scene[:, :, c[0]:c[3], c[1]:c[4], c[2]:c[5]]) for c in crops[keep]]
            out.update(pred_box=pred_box, pred_conf=conf, mask_keep=keep, mask_crops=crops, mask_pred=masks)
    return out
