"""oracle/port_mask_images.py -- TEST INFRASTRUCTURE ONLY.

CPU restatement of the TEST forward with the colour-aware mask head (MASK_USE_IMAGES, optionally MASK_ONLY_IMAGES), the
checker for that mode of the sm_90a path.  It composes oracle/port.py's back-projection, backbone, RPN, proposal layer, RoI
pooling, classifier and decode (and oracle/port_only_images.py's image-only backbone), which are pinned to the reference on
their own; the mask head is MaskBackbone.forward (reference: lib/nets/backbones.py:236-287) on the crops of network.py:302-317.
This forward is pinned to the reference by tests/golden/mask_images_reference.npz (oracle/make_golden_mask_images.py,
tests/test_mask_images.py).  The product path never imports it.
"""
from __future__ import annotations

import copy

import numpy as np
import torch
import torch.nn.functional as F

from oracle import port


def _stack(x, w, prefix):
    for i in (0, 2, 4, 6, 8):
        x = F.relu(F.conv3d(x, port._t(w, f"mask_backbone.{prefix}.{i}.weight"), None, padding=1))
    return F.conv3d(x, port._t(w, f"mask_backbone.{prefix}.10.weight"), None)


def mask_head(w, scene_crop, imageft_crop, only_images=False):
    """MaskBackbone.forward at test time: sigmoid(color(imageft)) with MASK_ONLY_IMAGES, else
    sigmoid(combine(cat[geometry(scene), color(imageft)]))."""
    if only_images:
        return torch.sigmoid(_stack(imageft_crop, w, "color"))
    x = torch.cat([_stack(scene_crop, w, "geometry"), _stack(imageft_crop, w, "color")], 1)
    x = F.relu(F.conv3d(x, port._t(w, "mask_backbone.combine.0.weight"), None, padding=1))
    return torch.sigmoid(F.conv3d(x, port._t(w, "mask_backbone.combine.2.weight"), None))


def masks(w, scene, imageft, crops, keep, only_images=False):
    """One mask per kept crop (network.py:302-317): the scene and the back-projected features cropped at the same box."""
    return [mask_head(w, scene[:, :, c[0]:c[3], c[1]:c[4], c[2]:c[5]], imageft[:, :, c[0]:c[3], c[1]:c[4], c[2]:c[5]], only_images)
            for c in crops[np.nonzero(keep)[0]]]


def forward(cfg, w, data, views, only_images=False, backbone_only_images=False, fma_mode=0):
    """network.py:187-317 with the colour-aware mask head; backbone_only_images: the image-only ScanNet backbone
    (ONLY_IMAGES).  views = dict(feats, depths, poses, world2grid).  Returns the keys of port.forward."""
    if backbone_only_images:
        from oracle import port_only_images
        out = port_only_images.forward(cfg, w, data, views, fma_mode=fma_mode)  # its scene-only masks are replaced below
    else:
        nomask = copy.copy(cfg)
        nomask.USE_MASK = False
        out = port.forward(nomask, w, data, views, fma_mode=fma_mode)
    with torch.no_grad():
        scene = torch.as_tensor(data, dtype=torch.float32)
        dims = tuple(int(v) for v in scene.shape[2:])
        pred_box, conf, keep, crops = port.detection_boxes(cfg, out["rois"].numpy(), out["cls_pred"].numpy(),
                                                           out["cls_prob"].numpy(), out["bbox_pred"].numpy(), dims)
        out.update(pred_box=pred_box, pred_conf=conf, mask_keep=keep, mask_crops=crops,
                   mask_pred=masks(w, scene, out["imageft"], crops, keep, only_images))
    return out


def forward_gt_rois(cfg, w, data, views, gt_box, only_images=False):
    """Ground-truth RoIs (USE_RPN = USE_CLASS = False; oracle/port_gt_rois.py) with the colour-aware mask head: the
    reference still back-projects the views (network.py:194-239), and only the mask head reads them."""
    from oracle import port_gt_rois
    nomask = copy.copy(cfg)
    nomask.USE_MASK = False
    out = port_gt_rois.forward_gt_rois(nomask, w, data, gt_box)
    with torch.no_grad():
        scene = torch.as_tensor(data, dtype=torch.float32)
        dims = tuple(int(v) for v in scene.shape[2:])
        imageft, killing = port.backproject_views(cfg, views["feats"], views["depths"], views["poses"], views["world2grid"], dims)
        pred_box, conf, keep, crops = port.detection_boxes(cfg, out["rois"].numpy(), out["cls_pred"].numpy(),
                                                           out["cls_prob"].numpy(), out["bbox_pred"].numpy(), dims)
        out.update(imageft=imageft, killing_inds=killing, pred_box=pred_box, pred_conf=conf, mask_keep=keep, mask_crops=crops,
                   mask_pred=masks(w, scene, imageft, crops, keep, only_images))
    return out
