"""Backbone definitions (reference: lib/nets/backbones.py).

Each backbone is a *layer program*: a list of ops per stage that `Network` executes with libsis3d
kernels.  Op tuples: ("k2s2", idx, cin, cout) 2x2x2/stride-2 conv + ReLU (no bias); ("k3", idx, cin,
cout) 3x3x3 conv + ReLU (no bias); ("bneck", idx, inplanes, planes) residual bottleneck; ("pool", idx)
MaxPool3d(3,1,1).  `idx` is the position inside the reference's nn.Sequential, which fixes the
state_dict key (e.g. geometry1.2.conv1.weight) so reference checkpoints load unchanged.
"""
import torch
from torch import nn

from lib import _sis3d as S
from lib.nets.network import Act, Network
from lib.utils.config import cfg


class Base_Backbone(Network):
    def __init__(self):
        super().__init__()
        self._fc7_channels = 128
        self._net_conv_level1_channels = self._net_conv_level2_channels = self._net_conv_level3_channels = 128

    def _program(self):
        raise NotImplementedError

    def _init_backbone_classifier(self):
        self.SPEC = self._program()
        for stage in ("geometry1", "color", "geometry2"):
            if stage in self.SPEC:
                self._declare_stack(stage, self.SPEC[stage])
        p = int(cfg.CLASS_POOLING_SIZE)
        self._declare_linear("classifier.0", 256, self._net_conv_level1_channels * p ** 3)
        self._declare_linear("classifier.2", 256, 256)
        self._declare_linear("classifier.4", 128, 256)


class ScanNet_Backbone(Base_Backbone):
    """reference: backbones.py:171-231.  With ONLY_IMAGES the program has no geometry1: the 128-channel colour stack is level
    1 by itself (backbones.py:99-101, 174-176, 186)."""

    def _program(self):
        if cfg.ONLY_IMAGES:
            if not cfg.USE_IMAGES:
                raise NotImplementedError("ScanNet_Backbone with ONLY_IMAGES and USE_IMAGES=False: the reference builds a "
                                          "0-channel geometry1 and its forward fails in geometry2.0; turn USE_IMAGES on")
            ci = int(cfg.NUM_IMAGE_CHANNELS)
            return dict(color=[("k2s2", 0, ci, 64), ("bneck", 2, 64, 32), ("pool", 3),
                               ("k2s2", 4, 64, 128), ("bneck", 6, 128, 32), ("pool", 7)],
                        geometry2=[("k3", 0, 128, 128), ("bneck", 2, 128, 64), ("bneck", 3, 128, 64), ("pool", 4)])
        g, c = (64, 64) if cfg.USE_IMAGES else (128, 0)
        prog = dict(geometry1=[("k2s2", 0, 2, 32), ("bneck", 2, 32, 32), ("bneck", 3, 32, 32),
                               ("k2s2", 4, 32, g), ("bneck", 6, g, 32), ("bneck", 7, g, 32)],
                    geometry2=[("k3", 0, g + c, 128), ("bneck", 2, 128, 64), ("bneck", 3, 128, 64), ("pool", 4)])
        if cfg.USE_IMAGES:
            ci = int(cfg.NUM_IMAGE_CHANNELS)
            prog["color"] = [("k2s2", 0, ci, 64), ("bneck", 2, 64, 32), ("pool", 3),
                             ("k2s2", 4, 64, c), ("bneck", 6, c, 32), ("pool", 7)]
        return prog


class SUNCG_Backbone(Base_Backbone):
    """reference: backbones.py:118-169."""

    def _program(self):
        if cfg.ONLY_IMAGES and cfg.USE_IMAGES:  # without USE_IMAGES the reference ignores ONLY_IMAGES here (:124, :148-153)
            raise NotImplementedError("SUNCG_Backbone with ONLY_IMAGES: its level 1 is the 64-channel colour output, but the "
                                      "reference builds rpn_net_level1 and classifier.0 for 128 channels, so its first "
                                      "level-1 RPN conv fails")
        prog = dict(geometry1=[("k2s2", 0, 2, 64), ("bneck", 2, 64, 32), ("k2s2", 3, 64, 64), ("bneck", 5, 64, 32)],
                    geometry2=[("k3", 0, 128 if cfg.USE_IMAGES else 64, 128), ("bneck", 2, 128, 64)])
        if cfg.USE_IMAGES:
            ci = int(cfg.NUM_IMAGE_CHANNELS)
            prog["color"] = [("k2s2", 0, ci, 64), ("bneck", 2, 64, 32), ("k2s2", 3, 64, 64), ("bneck", 5, 64, 32)]
        return prog


class MaskBackbone(nn.Module):
    """Per-RoI mask head: 5 x (conv3x3x3 -> ReLU) + 1x1 -> sigmoid, no biases (reference: backbones.py:236-287).  Parameters
    live here (state_dict keys mask_backbone.geometry.N.weight); the kernels are launched through the owning Network so the
    packed weights are shared.  With MASK_USE_IMAGES the geometry stack ends in a 64 -> 64 1x1, a colour stack (128 -> 64, four
    64 -> 64, 1x1) runs on the crop of the back-projected image features, and `combine` (128 -> 128 + ReLU, 1x1 -> classes)
    runs on [geometry | colour]; with MASK_ONLY_IMAGES the colour stack alone makes the masks (its 1x1 -> classes), and
    geometry and combine are declared but not run.  The switches are read once, here: a net built colour-aware stays so."""

    @staticmethod
    def refuse_unrunnable():
        """The two mask-switch combinations the reference cannot run, refused before any parameter is declared."""
        if cfg.MASK_USE_IMAGES and not cfg.USE_IMAGES:
            raise NotImplementedError("MASK_USE_IMAGES with USE_IMAGES=False: the reference has no image features to crop "
                                      "(self.color(None) fails); turn USE_IMAGES on")
        if cfg.MASK_ONLY_IMAGES and not cfg.MASK_USE_IMAGES:
            raise NotImplementedError("MASK_ONLY_IMAGES without MASK_USE_IMAGES: the reference builds no colour stack and its "
                                      "forward fails with an AttributeError; turn MASK_USE_IMAGES on too")

    def __init__(self):
        super().__init__()
        self.refuse_unrunnable()
        from lib.nets.network import _declare
        nc = int(cfg.NUM_CLASSES)
        self.colour, self.only_images = bool(cfg.MASK_USE_IMAGES), bool(cfg.MASK_ONLY_IMAGES)
        stacks = [("geometry", 2, 64 if self.colour else nc)]
        if self.colour:
            stacks.append(("color", 128, nc if self.only_images else 64))
        for stack, cin, last in stacks:
            for i in (0, 2, 4, 6, 8):
                _declare(self, f"{stack}.{i}.weight", (64, cin, 3, 3, 3), cin * 27)
                cin = 64
            _declare(self, f"{stack}.10.weight", (last, 64, 1, 1, 1), 64)
        if self.colour:
            _declare(self, "combine.0.weight", (128, 128, 3, 3, 3), 128 * 27)
            _declare(self, "combine.2.weight", (nc, 128, 1, 1, 1), 128)
        self._owner = None

    def forward(self, scene, imageft=None):
        """scene [1,2,w,h,l] crop (NCDHW), imageft its [1,128,w,h,l] crop of the back-projected image features (colour-aware
        heads) -> sigmoid mask [1,num_classes,w,h,l]."""
        net = self._owner() if self._owner is not None else None
        if net is None:
            raise S.Sis3dError("mask_backbone is launched through its owning Network (which is gone)")
        net._ensure_packed()
        if scene.shape[0] != 1:
            raise S.Sis3dError("mask_backbone: batch size 1")
        dev = next(net.parameters()).device
        scene = scene.to(dev, torch.float32).contiguous()
        w, h, l = (int(v) for v in scene.shape[2:])
        color = None
        if self.colour:
            if imageft is None or tuple(imageft.shape) != (1, 128, w, h, l):
                raise S.Sis3dError(f"mask_backbone: a colour-aware head takes the [1, 128, {w}, {h}, {l}] image-feature crop, got "
                                   f"{None if imageft is None else tuple(imageft.shape)}")
            color = dict(crop_in=imageft[0].to(dev, torch.float32).permute(1, 2, 3, 0).contiguous())
        det = torch.zeros(1, 16)
        det[0, 8] = 1.0
        det[0, 12:15] = torch.tensor([w, h, l], dtype=torch.float32)
        masks = net._mask_branch(scene, det.numpy(), 1, color=color)
        return masks[0].contiguous()
