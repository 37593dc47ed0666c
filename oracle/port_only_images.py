"""oracle/port_only_images.py -- TEST INFRASTRUCTURE ONLY.

CPU restatement of the TEST forward with the image-only ScanNet backbone (ONLY_IMAGES = USE_IMAGES = True), the checker for
that mode of the sm_90a path.  It composes oracle/port.py's back-projection, layer sequences, RPN, proposal layer, RoI
pooling, classifier, decode and mask head, which are pinned to the reference on their own; this forward is pinned to the
reference by tests/golden/only_images_reference.npz (oracle/make_golden_only_images.py, tests/test_only_images.py).  The
product path never imports it.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import port

# ScanNet_Backbone with ONLY_IMAGES (backbones.py:174-176, 186, 201-220): no geometry1; the colour stack (128 channels
# after color.4) and geometry2 keep the layer positions of the image + geometry net
SPEC = dict(color=[("k2s2", 0), ("bneck", 2), ("pool", 3), ("k2s2", 4), ("bneck", 6), ("pool", 7)],
            geometry2=[("k3", 0), ("bneck", 2), ("bneck", 3), ("pool", 4)])


def backbone(w, imageft):
    """Base_Backbone._backbone, image-only branch (backbones.py:99-101): level 1 = color(imageft), level 2 = geometry2(level 1)."""
    level1 = port._seq(imageft, w, "color", SPEC["color"])
    return level1, port._seq(level1, w, "geometry2", SPEC["geometry2"])


def forward(cfg, w, data, views, fma_mode=0):
    """network.py:187-317 with the image-only backbone; the mask head still reads the scene (MaskBackbone.forward,
    backbones.py:274-287, MASK_ONLY_IMAGES off).  views = dict(feats, depths, poses, world2grid).  Returns the keys of
    port.forward."""
    if cfg.NET != "ScanNet_Backbone":
        raise ValueError("ONLY_IMAGES: the reference runs it with ScanNet_Backbone only")
    out = {}
    with torch.no_grad():
        scene = torch.as_tensor(data, dtype=torch.float32)
        dims = tuple(int(v) for v in scene.shape[2:])
        imageft, killing = port.backproject_views(cfg, views["feats"], views["depths"], views["poses"], views["world2grid"],
                                                  dims)
        out["imageft"], out["killing_inds"] = imageft, killing
        level1, level2 = backbone(w, imageft)
        out["level1"], out["level2"] = level1, level2
        levels = []
        for lvl, (feat, A, tab) in enumerate(((level1, cfg.NUM_ANCHORS_LEVEL1, cfg.ANCHORS_TYPE_LEVEL1),
                                              (level2, cfg.NUM_ANCHORS_LEVEL2, cfg.ANCHORS_TYPE_LEVEL2)), 1):
            prob, deltas, _ = port.rpn_heads(w, feat, lvl, A)
            levels.append((prob, deltas, port.generate_anchors(feat.shape[2:], port.read_anchor_table(tab), 4)))
            out[f"rpn_prob_level{lvl}"], out[f"rpn_deltas_level{lvl}"] = prob, deltas
        prop = port.proposal_layer(cfg, levels, dims, fma_mode)
        out.update(rois=prop["rois"], roi_scores=prop["scores"], level_inds=prop["level_inds"], rpn_order=prop["order"],
                   nms_keep=prop["keep"])
        pool5 = port.roi_pool_levels(cfg, (level1, level2), prop["rois"].numpy(), prop["level_inds"].numpy())
        cls_score, cls_pred, cls_prob, bbox_pred = port.classifier(w, pool5)
        out.update(cls_score=cls_score, cls_pred=cls_pred, cls_prob=cls_prob, bbox_pred=bbox_pred)
        pred_box, conf, keep, crops = port.detection_boxes(cfg, prop["rois"].numpy(), cls_pred.numpy(), cls_prob.numpy(),
                                                           bbox_pred.numpy(), dims)
        masks = [port.mask_head(w, scene[:, :, c[0]:c[3], c[1]:c[4], c[2]:c[5]]) for c in crops[np.nonzero(keep)[0]]]
        out.update(pred_box=pred_box, pred_conf=conf, mask_keep=keep, mask_crops=crops, mask_pred=masks)
    return out
