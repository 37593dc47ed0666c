"""`Network`: the TEST-mode forward of 3D-SIS on libsis3d kernels.

Public surface kept from the reference (lib/nets/network.py): `init_modules()`, `load_state_dict()`
with the reference's parameter names/shapes, `forward(blobs, 'TEST', killing_inds)`, the
`_predictions` dict (`rois, roi_scores, level_inds, cls_score, cls_pred, cls_prob, bbox_pred,
mask_pred`), `_scene_info`, and `mask_backbone(scene_crop, imageft)`.

Everything between the input blobs and `_predictions` runs as hand-written CUDA (csrc/*.cu) on VC
(channels-last) activations; nn.Module is used only as the parameter container so checkpoints of the
reference load unchanged.  Training mode is out of scope (inference-only hot path).  With USE_RPN = USE_CLASS = False the
forward runs on the ground-truth boxes and classes of blobs['gt_box'] (`gt_detection_table`): only the mask stage runs, and
`_predictions` has no `level_inds` or `cls_score`, as in the reference.
"""
from __future__ import annotations

import ctypes as C
import gc
import math
import operator
import os
import weakref

import numpy as np
import torch
from torch import nn

from lib import _sis3d as S
from lib.layer_utils import projection as proj
from lib.layer_utils.generate_anchors import read_anchor_sizes
from lib.layer_utils.proposal_layer import rpn_proposals
from lib.utils.config import cfg


_VERSION = operator.attrgetter("_version")  # in-place update counter of a tensor


class Act:
    """A voxel activation: tensor + spatial dims + channels; layout 'vc' ([X,Y,Z,C]) or 'ncdhw'."""
    __slots__ = ("t", "dims", "C", "layout", "ld", "coff", "h")

    def __init__(self, t, dims, Cn, layout="vc", ld=None, coff=0, h=None):
        self.t, self.dims, self.C, self.layout = t, tuple(int(d) for d in dims), int(Cn), layout
        self.ld, self.coff = int(ld if ld is not None else Cn), int(coff)
        self.h = h  # optional dense fp16 twin [X,Y,Z,C] (fp16-operand tensor-core mode); `t` may be None when only `h` exists

    @property
    def nvox(self):
        return self.dims[0] * self.dims[1] * self.dims[2]


def _declare(root, dotted, shape, fan_in):
    """Register parameter `dotted` (e.g. 'geometry1.2.conv1.weight') on nested container modules,
    default-initialised like torch's Conv/Linear (U(-1/sqrt(fan_in), 1/sqrt(fan_in)))."""
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, nn.Module())
        mod = mod._modules[p]
    bound = 1.0 / math.sqrt(fan_in)
    mod.register_parameter(parts[-1], nn.Parameter(torch.empty(shape).uniform_(-bound, bound), requires_grad=False))


def _declare_tensor(root, dotted, tensor, kind):
    """Register `tensor` as parameter / buffer `dotted` on nested container modules (state_dict key == dotted)."""
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, nn.Module())
        mod = mod._modules[p]
    if kind == "param":
        mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))
    else:
        mod.register_buffer(parts[-1], tensor)


class _MaskList:
    """Sequence of per-RoI mask tensors [1, num_classes, w, h, l] (the reference's `mask_pred[i]` list,
    lib/nets/network.py:303-317) as lazily created views of the packed [total_voxels, num_classes] output."""

    def __init__(self, packed, offs, sizes, ncls):
        self.packed, self.offs, self.sizes, self.ncls = packed, offs, sizes, ncls

    def __len__(self):
        return len(self.sizes)

    def __getitem__(self, j):
        if isinstance(j, slice):
            return [self[i] for i in range(*j.indices(len(self)))]
        if j < 0:
            j += len(self)
        if not 0 <= j < len(self):
            raise IndexError(j)
        w, h, l = (int(v) for v in self.sizes[j])
        m = self.packed[int(self.offs[j]) * self.ncls:int(self.offs[j + 1]) * self.ncls].view(w, h, l, self.ncls)
        return m.permute(3, 0, 1, 2).unsqueeze(0)  # view in the reference layout

    def __iter__(self):
        return (self[i] for i in range(len(self)))

    def __eq__(self, other):
        return list(self) == other if isinstance(other, list) else NotImplemented


def gt_detection_table(gt_box, dims, class_thresh, num_classes):
    """The [n, 16] detection table of ground-truth RoIs (USE_RPN = USE_CLASS = False; reference: network.py:262-265, 276-301),
    built on the host in the layout and float32 operation order of detect_decode_kernel (csrc/roi.cu): the box decoded with
    zero deltas and clipped to the scene, conf = 1.0 (the one-hot cls_prob at the ground-truth class), the class, the keep
    flag (conf > CLASS_THRESH, compared in float64 as the reference's driver does, and a non-empty rounded extent on every
    axis), the crop bounds (round half to even) and n in row 0, column 15.  gt_box: [n, >= 7] (x0, y0, z0, x1, y1, z1,
    class)."""
    g = np.asarray(gt_box, dtype=np.float32)
    if g.ndim != 2 or g.shape[1] < 7:
        raise S.Sis3dError(f"gt_box must be [n, 7] (box, class), got shape {tuple(g.shape)}")
    if not np.isfinite(g[:, :7]).all():
        raise S.Sis3dError("gt_box holds a non-finite value")
    n = g.shape[0]
    cls = np.trunc(g[:, 6]).astype(np.int64)  # gt_box[:, 6].long()
    if n and (cls.min() < 0 or cls.max() >= num_classes):
        raise S.Sis3dError(f"gt_box class out of range [0, {num_classes}): {cls.min()} .. {cls.max()}")
    det = np.zeros((n, 16), dtype=np.float32)
    lo, hi = g[:, 0:3], g[:, 3:6]
    w = hi - lo
    ctr = lo + np.float32(0.5) * w
    pc = np.float32(0.0) * w + ctr                # dx * w + ctr with dx = 0
    hw = np.float32(0.5) * (np.float32(1.0) * w)  # 0.5 * (exp(0) * w)
    d = np.asarray(dims, dtype=np.float32)
    det[:, 0:3] = np.minimum(np.maximum(pc - hw, np.float32(0.0)), d)
    det[:, 3:6] = np.minimum(np.maximum(pc + hw, np.float32(0.0)), d)
    crop = np.rint(det[:, 0:6])
    det[:, 6] = 1.0
    det[:, 7] = cls
    det[:, 8] = (1.0 > float(class_thresh)) & (crop[:, 0:3] < crop[:, 3:6]).all(1)
    det[:, 9:15] = crop
    if n:
        det[0, 15] = n
    return det


class Network(nn.Module):
    # layer programs of the concrete backbones are provided by subclasses (lib/nets/backbones.py)
    SPEC = None

    def __init__(self):
        super().__init__()
        self._predictions = {}
        self._feat_stride = [4, 4, 4]
        self._packs = {}   # form -> layer -> packed weight (pack_plan)
        self._layers = {}  # layer -> (fp32 bias or None, cout, cin, ks)
        self._packed_version = None
        self._region_cache = {}
        self._const_cache = {}
        self._keep_debug = False
        # conv math (see set_conv_math).  Default 'exact': error-compensated split products (fp32-class accuracy, wgmma) in the
        # static stage -- everything that decides an integer output: proposal order, NMS keep list, class argmax, crop
        # bounds -- and fp16-stored operands in the ragged mask stage, whose outputs carry the 1e-3 tolerance.
        self.set_conv_math(os.environ.get("SIS3D_CONV_MATH", str(cfg.get("CONV_MATH", "exact"))).lower())
        self._graphs = {}
        self._slots = []
        self._branches = os.environ.get("SIS3D_BRANCHES", "1") != "0"
        self._replayed_kernels = 0  # libsis3d kernels executed through CUDA-graph replays
        self._sparse_color = os.environ.get("SIS3D_SPARSE_COLOR", "1") != "0"
        # host waits yield the core instead of spinning: with one process per GPU on a CPU-quota'd node, eight spinning
        # waiters plus the Python loops would eat the whole quota (cgroup throttling stalls every rank at once)
        # (spinning is ~9 % faster on an otherwise idle host, so it stays the default while cores are plentiful)
        bs = os.environ.get("SIS3D_BLOCKING_SYNC")
        if bs is None:
            try:
                cores = len(os.sched_getaffinity(0))
                with open("/sys/fs/cgroup/cpu.max") as f:
                    quota, period = f.read().split()
                if quota != "max":
                    cores = min(cores, max(1, int(quota) // int(period)))
            except (OSError, ValueError, AttributeError):
                cores = os.cpu_count() or 1
            self._blocking_sync = cores < 3 * int(os.environ.get("LOCAL_WORLD_SIZE", "1"))
        else:
            self._blocking_sync = bs != "0"
        self._pack_dirty = True
        self._arena = {}  # grow-only device/pinned workspaces for the ragged (per-scene sized) stage
        self._use_graph = os.environ.get("SIS3D_CUDA_GRAPH", "1") != "0"
        # a shape is captured the SIS3D_GRAPH_AFTER-th time it is seen (whole-scene inference meets many one-off shapes: those
        # run eagerly), and every stream slot keeps at most SIS3D_GRAPH_CACHE captured shapes (LRU; a graph owns its static
        # buffers and a private memory pool, so an unbounded cache would grow until OOM)
        self._graph_after = max(1, int(os.environ.get("SIS3D_GRAPH_AFTER", "2")))
        self._graph_cache = max(1, int(os.environ.get("SIS3D_GRAPH_CACHE", "4")))
        self._shape_seen = {}
        self._prof = None  # name -> [(start_event, end_event)] when per-kernel timing is on (bench.py)

    # ------------------------------------------------------------------ parameters
    def _declare_conv(self, name, cout, cin, ks, bias):
        _declare(self, name + ".weight", (cout, cin, ks, ks, ks), cin * ks ** 3)
        if bias:
            _declare(self, name + ".bias", (cout,), cin * ks ** 3)

    def _declare_bottleneck(self, name, inpl, planes):
        self._declare_conv(name + ".conv1", planes, inpl, 1, True)
        self._declare_conv(name + ".conv2", planes, planes, 3, True)
        self._declare_conv(name + ".conv3", inpl, planes, 1, True)

    def _declare_linear(self, name, cout, cin):
        _declare(self, name + ".weight", (cout, cin), cin)
        _declare(self, name + ".bias", (cout,), cin)

    def _declare_stack(self, prefix, spec):
        for op in spec:
            if op[0] in ("k2s2", "k3"):
                self._declare_conv(f"{prefix}.{op[1]}", op[3], op[2], 2 if op[0] == "k2s2" else 3, False)
            elif op[0] == "bneck":
                self._declare_bottleneck(f"{prefix}.{op[1]}", op[2], op[3])

    def _init_backbone_classifier(self):
        raise NotImplementedError

    def init_modules(self):
        """Declare every parameter of the 3D model (reference: network.py:35-64)."""
        if cfg.USE_MASK:
            from lib.nets.backbones import MaskBackbone
            MaskBackbone.refuse_unrunnable()
        self._init_backbone_classifier()
        if cfg.USE_RPN:
            for lvl in (1, 2, 3):
                A = cfg["NUM_ANCHORS_LEVEL%d" % lvl]
                if A:
                    self._declare_conv(f"rpn_net_level{lvl}", cfg.RPN_CHANNELS, 128, 3, True)
                    self._declare_conv(f"rpn_cls_score_net_level{lvl}.0", 2 * A, cfg.RPN_CHANNELS, 1, True)
                    self._declare_conv(f"rpn_bbox_pred_net_level{lvl}", 6 * A, cfg.RPN_CHANNELS, 1, True)
        if cfg.USE_CLASS:
            self._declare_linear("classifier_cls_score_net", cfg.NUM_CLASSES, 128)
            self._declare_linear("classifier_bbox_pred_net", cfg.NUM_CLASSES * 6, 128)
        if cfg.USE_MASK:
            from lib.nets import backbones
            self.mask_backbone = getattr(backbones, cfg.MASK_BACKBONE)()
            # weak back-reference: no parent<->child cycle, so a dropped Network (graphs, streams, arenas) is freed by
            # reference counting right away instead of by a later cyclic GC pass in the middle of someone else's capture
            self.mask_backbone._owner = weakref.ref(self)
        if cfg.USE_IMAGES and not cfg.USE_IMAGES_GT:
            self._declare_enet()

    def _declare_enet(self):
        """2-D ENet encoder (SURVEY 8f2; reference: network.py:62-63 -> enet.create_enet_for_3d, enet.py:697-715): parameters and
        BatchNorm buffers under the reference's state_dict names (lib/nets/enet_keys.py), default-initialised, then overwritten
        by cfg.PRETRAINED_ENET_PATH when that file exists (the reference loads it at this point too).  The forward runs on the
        sis3d_enet_* kernels (lib/nets/enet.py); image_enet_classification is kept only for the checkpoint contract."""
        from lib.nets.enet_keys import ENET_KEYS
        n2d = int(cfg.NUM_2D_CLASSES)
        names = {k[0] for k in ENET_KEYS}
        enc = []
        for name, shape, kind, dt in ENET_KEYS:
            if name.startswith("image_enet_classification"):
                shape = (n2d,) + tuple(shape[1:])
            if dt == "int64":
                t = torch.zeros(shape, dtype=torch.int64)
            elif name.endswith("running_var"):
                t = torch.ones(shape)
            elif name.endswith(("running_mean", ".bias")):
                t = torch.zeros(shape)
            elif len(shape) == 4:
                bound = 1.0 / math.sqrt(shape[1] * shape[2] * shape[3])
                t = torch.empty(shape).uniform_(-bound, bound)
            else:  # 1-D weight: BatchNorm scale (has running statistics beside it) or PReLU slope
                t = torch.ones(shape) if name[:-len("weight")] + "running_mean" in names else torch.full(shape, 0.25)
            _declare_tensor(self, name, t, kind)
            if not name.startswith("image_enet_classification") and not name.endswith("num_batches_tracked"):
                enc.append(name)
        self.__dict__["_enet_names"] = enc
        path = str(cfg.get("PRETRAINED_ENET_PATH", "") or "")
        if path and os.path.exists(path):
            src = torch.load(path, map_location="cpu")  # plain create_enet keys ('0.0.weight', ...), same order as ENET_KEYS
            own = dict(self.named_parameters())
            own.update(dict(self.named_buffers()))
            if len(src) != len(ENET_KEYS):
                raise S.Sis3dError(f"{path}: {len(src)} tensors, the ENet of lib/nets/enet.py has {len(ENET_KEYS)}")
            with torch.no_grad():
                for (name, _, _, _), v in zip(ENET_KEYS, src.values()):
                    own[name].copy_(v)

    # ------------------------------------------------------------------ packed weights
    def load_state_dict(self, *a, **k):
        self._pack_dirty = True
        return super().load_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):  # .cuda() / .to() / .float() move parameters -> repack
        self._pack_dirty = True
        return super()._apply(fn, *a, **k)

    def _ws(self, name, numel, dtype, dev, pinned=False):
        """Grow-only workspace: steady-state forwards never hit cudaMalloc for per-scene sized buffers."""
        t = self._arena.get(name)
        if t is None or t.numel() < numel or t.dtype != dtype:
            cap = int(numel * 1.5) + 1024
            t = torch.empty(cap, dtype=dtype, pin_memory=True) if pinned else torch.empty(cap, dtype=dtype, device=dev)
            self._arena[name] = t
        return t[:numel]

    def _versioned(self):
        """The tensors the packed weights are made from: every parameter, and the 2-D encoder's buffers."""
        ts = [p for _, p in self.named_parameters()]
        if self.__dict__.get("_enet_names"):  # BatchNorm statistics of the 2-D encoder are buffers
            ts += [b for _, b in self.named_buffers()]
        return ts

    def _version(self):
        v = tuple((n, p._version, p.data_ptr()) for n, p in self.named_parameters())
        if self.__dict__.get("_enet_names"):
            v += tuple((n, b._version, b.data_ptr()) for n, b in self.named_buffers())
        return v

    MATH_MODES = {  # mode -> (static-stage conv math, mask-stage conv math)
        "exact": ("f16x3", "fp16"),    # default: integer outputs equal the fp32 path, masks within 1e-3
        "f16x3": ("f16x3", "tf32"),    # error-compensated fp16 split (3 f16 wgmmas per product, fp32-class accuracy)
        "tf32x3": ("tf32x3", "tf32"),  # the same compensation with a TF32 split (3 TF32 wgmmas: half the f16 tensor rate)
        "mixed": ("tf32", "fp16"),     # fastest; detections equal the reference only up to near-tied scores
        "tf32": ("tf32", "tf32"),
        "fp16": ("fp16", "fp16"),
        "fp32": ("fp32", "fp32"),      # CUDA-core kernels throughout
    }
    # A conv math names the weight form its kernels read.  Mode -> forms its static-stage convs fall back to when a layer has
    # no pack of the mode's own form ('fp16': TF32 when no fp16 twin of the output is requested, else the CUDA-core kernel).
    FALLBACK_FORMS = {"fp16": ("tf32",)}
    MASK_ROUTES = ("fp32", "tf32", "fp16")  # mask-stage form -> route index of the mask stage (MaskStage.math)
    _TC32_SUFFIX = {"tf32": "", "tf32x3": "_x3", "f16x3": "_h3"}  # tensor-core forms of the fp32-output kernels -> name suffix

    @classmethod
    def mode_forms(cls, mode):
        """The weight forms conv math `mode` reads: the CUDA-core fp32 form, which every mode keeps (the first and last mask
        layers, the MLP tail and the sparse colour path read it), the static-stage form, its fallbacks and the mask-stage form."""
        static, mask = cls.MATH_MODES[mode]
        return tuple(dict.fromkeys(("fp32", static, *cls.FALLBACK_FORMS.get(mode, ()), mask)))

    @staticmethod
    def pack_layout(form, shape):
        """(shape, dtype) of the `form` pack of a layer whose weight has `shape` ([cout, cin, ks, ks, ks] conv or [cout, cin]
        nn.Linear); () when the form's kernel reads the fp32 weight as it is; None when no kernel of the form takes the layer."""
        cout, cin = shape[0], shape[1]
        ks = shape[2] if len(shape) == 5 else 1
        K = ks ** 3 * cin
        if form == "fp32":  # CUDA-core kernels: [K][cout rounded up to 4]
            return (K, (cout + 3) // 4 * 4), torch.float32
        if len(shape) == 2:  # the tensor-core GEMM; its TF32 route reads nn.Linear's [N][K] weight, already K-major
            if form == "fp16" or cin < 1024 or not S.lib.sis3d_linear_tc_supported(cin, cout):
                return None
            if form == "tf32":
                return ()
        elif ks not in (1, 2, 3) or not S.lib.sis3d_conv3d_k3_tc_supported(cin, cout):
            return None
        elif form == "fp16" and (ks == 2 or (cin % 64 and cin != 32)):  # fp16-operand kernel: no 2x2x2 taps, cin 32 or 64k
            return None
        rows = 2 if form in ("tf32x3", "f16x3") else 1  # the split forms keep a hi and a lo row per output channel
        return (rows * cout, K), (torch.float16 if form in ("f16x3", "fp16") else torch.float32)

    @classmethod
    def pack_plan(cls, shapes, mode):
        """{form: {layer: pack_layout}}: the packs `_ensure_packed` makes in conv math `mode`, from the layers' weight shapes
        (layer -> shape): every form the mode reads, each with the layers a kernel of that form takes."""
        return {form: {k: lay for k, s in shapes.items() if (lay := cls.pack_layout(form, s)) is not None}
                for form in cls.mode_forms(mode)}

    def set_conv_math(self, mode):
        """'exact' (error-compensated fp16-split static stage + fp16-operand mask stage) | 'f16x3' | 'tf32x3' | 'mixed' (TF32 +
        fp16) | 'tf32' | 'fp16' | 'fp32' (CUDA-core path)."""
        if mode not in self.MATH_MODES:
            raise S.Sis3dError(f"unknown conv math {mode!r} ({' | '.join(self.MATH_MODES)})")
        d = self.__dict__
        old = d.get("_math_mode")
        d["_math"], d["_mask_math"] = self.MATH_MODES[mode]
        d["_math_mode"] = mode
        # the static-stage forms that fp32-output tensor-core kernels read, in the order _conv tries them
        d["_tc32_forms"] = tuple(f for f in (d["_math"], *self.FALLBACK_FORMS.get(mode, ())) if f in self._TC32_SUFFIX)
        if old is not None and set(self.mode_forms(old)) != set(self.mode_forms(mode)):
            d["_pack_dirty"], d["_packed_version"] = True, None  # the next forward packs the forms of this mode

    def _layer_weights(self):
        """layer -> (fp32 weight, fp32 bias or None) of every conv and linear of the 3-D model, plus per RPN level both heads
        as ONE 1x1 conv: [2A | 6A] output channels, zero-padded to a tensor-core friendly width (32/64/128k) so the merged
        head runs on the wgmma kernel as well."""
        params = dict(self.named_parameters())
        out = {}
        for name, p in params.items():
            if name.endswith(".weight") and not name.startswith("image_enet_"):
                b = params.get(name[:-7] + ".bias")
                out[name[:-7]] = (p.detach().float().contiguous(), None if b is None else b.detach().float().contiguous())
        for lvl in (1, 2, 3):
            c, b = out.get(f"rpn_cls_score_net_level{lvl}.0"), out.get(f"rpn_bbox_pred_net_level{lvl}")
            if c is not None and b is not None:
                cout = c[0].shape[0] + b[0].shape[0]
                cpad = 32 if cout <= 32 else (64 if cout <= 64 else (cout + 127) // 128 * 128)
                wp, bp = c[0].new_zeros(cpad, *c[0].shape[1:]), c[1].new_zeros(cpad)
                wp[:cout], bp[:cout] = torch.cat([c[0], b[0]], 0), torch.cat([c[1], b[1]], 0)
                out[f"rpn_heads_level{lvl}"] = (wp, bp)
        return out

    _PACKERS = {"fp32": "sis3d_pack_conv_weight", "tf32": "sis3d_pack_conv_weight_tc", "tf32x3": "sis3d_pack_conv_weight_tc_x3",
                "f16x3": "sis3d_pack_conv_weight_tc_h3", "fp16": "sis3d_pack_conv_weight_tc_f16"}

    def _pack(self, form, layer, w, layout):
        """The `form` pack (pack_layout) of the fp32 weight `w` of `layer`."""
        if layout == ():
            return w
        out = torch.empty(layout[0], dtype=layout[1], device=w.device)
        _, cout, cin, ks = self._layers[layer]
        S.check(getattr(S.lib, self._PACKERS[form])(S.ptr(w), cout, cin, ks, S.ptr(out), S.stream()), f"{self._PACKERS[form]}[{layer}]")
        return out

    def _ensure_packed(self):
        d = self.__dict__
        if not d["_pack_dirty"] and d["_packed_version"] is not None:  # per-scene fast path: no module traversal
            # a parameter updated in place (p.mul_(), p.copy_(), an optimizer step) bumps its version counter and must be
            # repacked; inside the scene loop (scenes in flight on the slots) the check runs once, when the loop starts
            if d.get("_home_stream") is not None or list(map(_VERSION, d["_packed_from"])) == d["_packed_versions"]:
                return
        if not torch.cuda.is_available():
            raise S.Sis3dError("the sm_90a hot path needs a CUDA device (no CPU fallback)")
        if next(self.parameters()).device.type != "cuda":
            self.cuda()
        d["_dev"] = next(self.parameters()).device
        v = self._version()
        self._pack_dirty = False
        d["_packed_from"] = self._versioned()
        d["_packed_versions"] = list(map(_VERSION, d["_packed_from"]))
        if v == self._packed_version:
            return
        self.__dict__["_enet"] = None
        if self.__dict__.get("_enet_names"):
            from lib.nets.enet import EnetEncoder
            sd = dict(self.named_parameters())
            sd.update(dict(self.named_buffers()))
            self.__dict__["_enet"] = EnetEncoder([sd[n].detach() for n in self._enet_names], d["_dev"])
        weights = self._layer_weights()
        self._layers = {k: (b, w.shape[0], w.shape[1], w.shape[2] if w.dim() == 5 else 1) for k, (w, b) in weights.items()}
        plan = self.pack_plan({k: tuple(w.shape) for k, (w, _) in weights.items()}, self._math_mode)
        self._packs = {form: {k: self._pack(form, k, weights[k][0], lay) for k, lay in layers.items()} for form, layers in plan.items()}
        torch.cuda.current_stream().synchronize()
        self._packed_version = v
        # captured graphs hold the addresses of the previous packed weights: drop them (re-captured on next use)
        self.__dict__["_graphs"] = {}
        for sl in self._slots:
            sl["graphs"].clear()

    # ------------------------------------------------------------------ per-kernel timing hooks
    def _rec(self, name):
        if self._prof is None:
            return None
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return name, e

    def _rec_end(self, tok):
        if tok is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self._prof.setdefault(tok[0], []).append((tok[1], e))

    # ------------------------------------------------------------------ primitive ops
    def _regions_single(self, x: Act, out_dims, stride):
        key = ("single", x.dims, x.C, x.layout, x.ld, tuple(out_dims), stride)
        hit = self._region_cache.get(key)
        if hit is None:
            X, Y, Z = x.dims
            strides = (Y * Z * x.ld, Z * x.ld, x.ld) if x.layout == "vc" else (Y * Z, Z, 1)
            hit = S.make_regions([dict(in_off=0, out_off=0, res_off=0, in_dim=x.dims, out_dim=out_dims,
                                       in_stride=strides)], x.t.device)
            self._region_cache[key] = hit
        return hit

    def _half(self, x: Act):
        """fp16 twin of an activation (cast once, cached on the Act)."""
        if x.h is None:
            x.h = torch.empty(*x.dims, x.C, dtype=torch.float16, device=x.t.device)
            tok = self._rec("cast_f16")
            S.check(S.lib.sis3d_cast_f16(S.ptr(x.t), x.ld, x.coff, C.c_int64(x.nvox), x.C, S.ptr(x.h), S.stream()), "cast_f16")
            self._rec_end(tok)
        return x.h

    def _conv(self, x: Act, name, stride=1, pad=None, act=0, residual: Act = None, out: Act = None,
              regions=None, out_dims=None, want32=True, want16=False, out16=None):
        """One convolution.  Dispatch: wgmma fp16-operand kernel ('fp16' math), else the fp32-output wgmma kernel of the first
        of the mode's forms that has a pack of the layer, else the fp32 CUDA-core kernel.  want32/want16 choose which of the
        fp32 output / dense fp16 twin are produced (the twin feeds the next tensor-core layer in 'fp16' math); out16 =
        caller-provided fp16 destination (ragged mask stage)."""
        bias, cout, cin, ks = self._layers[name]
        W = self._packs
        if cin != x.C:
            raise S.Sis3dError(f"{name}: expected {cin} input channels, got {x.C}")
        if pad is None:
            pad = 1 if ks == 3 else 0
        if out_dims is None:
            out_dims = tuple(d // 2 for d in x.dims) if stride == 2 else x.dims
        regions_given = regions
        dev = (x.t if x.t is not None else x.h).device
        f16 = self._math == "fp16"
        if ks == 2:  # the 2x2x2 / stride-2 downsampling convs run on the tensor cores too (element-strided TMA boxes)
            geom_ok = stride == 2 and pad == 0 and min(x.dims) >= 2
        else:
            geom_ok = stride == 1 and pad == (1 if ks == 3 else 0)
        tc_ok = (regions_given is None and geom_ok and x.layout == "vc" and x.ld == x.C and x.coff == 0 and act in (0, 1))
        if not f16:
            want32, want16 = True, False
        if out is None:
            t32 = torch.empty(*out_dims, cout, dtype=torch.float32, device=dev) if want32 else None
            out = Act(t32, out_dims, cout)
        twin_ok = out.ld == cout and out.coff == 0  # the twin shares the geometry of the fp32 output
        if want16 and twin_ok and out16 is None:
            out.h = torch.empty(*out_dims, cout, dtype=torch.float16, device=dev)
        h_ptr = S.ptr(out16) if out16 is not None else (S.ptr(out.h) if (want16 and twin_ok) else None)
        res_args = (S.ptr(residual.t) if residual is not None else None, residual.ld if residual is not None else 0,
                    residual.coff if residual is not None else 0)
        if f16 and tc_ok and name in W["fp16"]:
            tok = self._rec(f"conv_tc16[{name}]")
            S.check(S.lib.sis3d_conv3d_tc_f16(S.ptr(self._half(x)), S.ptr(W["fp16"][name]), S.ptr(bias), *res_args,
                                              S.ptr(out.t) if out.t is not None else None, h_ptr, out.ld, out.coff, *x.dims,
                                              cin, cout, ks, None, 0, act, S.stream()), f"conv3d_tc_f16[{name}]")
            self._rec_end(tok)
            return out
        if x.t is None:
            raise S.Sis3dError(f"{name}: this layer needs the fp32 activation but only the fp16 twin was produced")
        if out.t is None and h_ptr is None:
            out.t = torch.empty(*out_dims, cout, dtype=torch.float32, device=dev)
        # the fp32-output tensor-core kernels (out.t is set here unless an fp16 twin was requested, which they cannot write)
        form = next((f for f in self._tc32_forms if name in W[f]), None) if tc_ok and h_ptr is None else None
        if form is not None:
            sfx = self._TC32_SUFFIX[form]
            tok = self._rec(f"conv_tc{sfx}[{name}]")
            fn = getattr(S.lib, f"sis3d_conv3d_k3_tc{sfx}")
            S.check(fn(S.ptr(x.t), S.ptr(W[form][name]), S.ptr(bias), *res_args, S.ptr(out.t), out.ld, out.coff, *x.dims,
                       cin, cout, ks, *((None, 0) if form == "tf32" else ()), act, S.stream()), f"conv3d_k3_tc{sfx}[{name}]")
            self._rec_end(tok)
            return out
        if regions is None:
            regions, n_tiles = self._regions_single(x, out_dims, stride)
        else:
            regions, n_tiles = regions
        in_sc = 1 if x.layout == "vc" else x.nvox
        xin = x.t if x.coff == 0 else x.t.reshape(-1)[x.coff:]
        tok = self._rec(f"conv[{name}]")
        S.check(S.lib.sis3d_conv3d_ex(S.ptr(xin), C.c_int64(in_sc), S.ptr(W["fp32"][name]), S.ptr(bias), *res_args,
                                      S.ptr(out.t) if out.t is not None else None, h_ptr, out.ld, out.coff, S.ptr(regions),
                                      regions.numel() // S.REGION_BYTES, n_tiles, cin, cout, ks, stride, pad, act, S.stream()),
                f"conv3d[{name}]")
        self._rec_end(tok)
        return out

    def _linear(self, x, name, act):
        """y = act(x W^T + b) through the split-K kernel (classifier MLP + heads)."""
        bias, cout, cin, _ = self._layers[name]
        M = x.shape[0]
        y = torch.empty(M, cout, dtype=torch.float32, device=x.device)
        sfx = self._TC32_SUFFIX.get(self._math)
        w = self._packs[self._math].get(name) if sfx is not None else None
        if w is not None:
            nbytes = int(S.lib.sis3d_linear_tc_workspace_bytes(M, cout, cin))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            tok = self._rec(f"linear_tc{sfx}[{name}]")
            S.check(getattr(S.lib, f"sis3d_linear_tc{sfx}")(S.ptr(x), S.ptr(w), S.ptr(bias), S.ptr(y), M, cin, cout, act,
                                                            S.ptr(ws), C.c_size_t(nbytes), S.stream()), f"linear_tc{sfx}[{name}]")
            self._rec_end(tok)
            return y
        nbytes = int(S.lib.sis3d_linear_workspace_bytes(M, cout, cin))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        tok = self._rec(f"linear[{name}]")
        S.check(S.lib.sis3d_linear(S.ptr(x), S.ptr(self._packs["fp32"][name]), S.ptr(bias), S.ptr(y), M, cin, cout, act, S.ptr(ws),
                                   C.c_size_t(nbytes), S.stream()), f"linear[{name}]")
        self._rec_end(tok)
        return y

    def _bottleneck(self, x: Act, name, out: Act = None):
        """1x1 -> relu -> 3x3x3 -> relu -> 1x1 (+x) -> relu  (reference: backbones.py:28-40).  In 'fp16' math the two inner
        activations exist only as fp16 (they feed tensor-core layers only); the block output is fp32 (+ fp16 twin when it
        is a dense tensor, for the next block's first conv)."""
        n1, n2, n3 = name + ".conv1", name + ".conv2", name + ".conv3"
        L, wt = self._layers, self._packs[self._math]
        sfx = self._TC32_SUFFIX.get(self._math)  # the fused conv2 + conv3 kernels take the fp32-output tensor-core forms
        if (self._math == "f16x3" and n1 in wt and n2 in wt and n3 in wt and x.t is not None and x.layout == "vc"
                and x.ld == x.C and x.coff == 0):
            b1, c1, cin1, ks1 = L[n1]
            _, cmid, cin, _ = L[n2]
            cout = L[n3][1]
            if ks1 == 1 and cin1 == x.C and c1 == cin and S.lib.sis3d_conv3d_k3_tc_fused_supported(cin, cmid, cout):
                # conv1 writes its activation already split into fp16 hi / lo pairs, the form the tail's MMAs read: the tail
                # needs no operand split on the SM (the result bits are those of the fp32 hand-off below)
                ys = torch.empty(*x.dims, 2 * c1, dtype=torch.float16, device=x.t.device)
                tok = self._rec(f"conv_tc_h3_split[{n1}]")
                S.check(S.lib.sis3d_conv3d_k1_tc_h3_split(S.ptr(x.t), S.ptr(wt[n1]), S.ptr(b1), S.ptr(ys), *x.dims, cin1, c1, 1,
                                                          S.stream()), f"conv3d_k1_tc_h3_split[{n1}]")
                self._rec_end(tok)
                if out is None:
                    out = Act(torch.empty(*x.dims, cout, dtype=torch.float32, device=x.t.device), x.dims, cout)
                tok = self._rec(f"conv_tc_fused_h3_split[{name}]")
                S.check(S.lib.sis3d_conv3d_k3_tc_fused_h3_split(
                    S.ptr(ys), S.ptr(wt[n2]), S.ptr(L[n2][0]), S.ptr(wt[n3]), S.ptr(L[n3][0]), S.ptr(x.t),
                    x.ld, x.coff, S.ptr(out.t), out.ld, out.coff, *x.dims, cin, cmid, cout, 1, S.stream()),
                    f"conv3d_k3_tc_fused_h3_split[{name}]")
                self._rec_end(tok)
                return out
        y = self._conv(x, n1, act=1, want32=False, want16=True)
        if sfx is not None and n2 in wt and n3 in wt and y.t is not None:
            _, cmid, cin, _ = L[n2]
            cout = L[n3][1]
            if y.ld == y.C and y.coff == 0 and S.lib.sis3d_conv3d_k3_tc_fused_supported(cin, cmid, cout):
                # conv2 + conv3 (+x, ReLU) in one wgmma kernel: the cmid-wide activation never leaves the SM
                if out is None:
                    out = Act(torch.empty(*y.dims, cout, dtype=torch.float32, device=y.t.device), y.dims, cout)
                tok = self._rec(f"conv_tc_fused{sfx}[{name}]")
                S.check(getattr(S.lib, f"sis3d_conv3d_k3_tc_fused{sfx}")(
                    S.ptr(y.t), S.ptr(wt[n2]), S.ptr(L[n2][0]), S.ptr(wt[n3]), S.ptr(L[n3][0]), S.ptr(x.t), x.ld, x.coff,
                    S.ptr(out.t), out.ld, out.coff, *y.dims, cin, cmid, cout, 1, S.stream()), f"conv3d_k3_tc_fused{sfx}[{name}]")
                self._rec_end(tok)
                return out
        y = self._conv(y, n2, act=1, want32=False, want16=True)
        return self._conv(y, n3, act=1, residual=x, out=out, want32=True, want16=True)

    def _pool(self, x: Act, out: Act = None):
        if out is None:
            out = Act(torch.empty(*x.dims, x.C, dtype=torch.float32, device=x.t.device), x.dims, x.C)
        if x.ld != x.C or x.coff:
            raise S.Sis3dError("maxpool3 expects a dense VC input")
        tok = self._rec("maxpool3")
        S.check(S.lib.sis3d_maxpool3(S.ptr(x.t), S.ptr(out.t), out.ld, out.coff, *x.dims, x.C, S.stream()), "maxpool3")
        self._rec_end(tok)
        return out

    def _run_stack(self, x: Act, prefix, spec, final_out=None):
        """Execute a backbone stage program; the last op writes into `final_out` (a slice of the
        concatenated level-1 tensor) when given."""
        for i, op in enumerate(spec):
            dst = final_out(x, op) if (final_out is not None and i == len(spec) - 1) else None
            if op[0] == "k2s2":
                x = self._conv(x, f"{prefix}.{op[1]}", stride=2, pad=0, act=1, out=dst, want16=True)
            elif op[0] == "k3":
                x = self._conv(x, f"{prefix}.{op[1]}", act=1, out=dst, want16=True)
            elif op[0] == "bneck":
                x = self._bottleneck(x, f"{prefix}.{op[1]}", out=dst)
            elif op[0] == "pool":
                x = self._pool(x, out=dst)
        return x

    # ------------------------------------------------------------------ stages of the forward
    def _const(self, key, builder):
        v = self._const_cache.get(key)
        if v is None:
            v = builder()
            self._const_cache[key] = v
        return v

    def _view_maps(self, blobs, killing_inds, dims, dev, fused=None):
        """Views -> (features [n,C,h,w], voxel->pixel maps, (feature, map) pairs, pair count): the inputs of every
        back-projection (reference: trainval.py:797-820 + network.py:194-223)."""
        w, h = int(cfg.DEPTH_SHAPE[0]), int(cfg.DEPTH_SHAPE[1])
        if fused is not None:
            feats = fused["feats"]
        else:
            feats = blobs["nearest_images"]["images"][0]
            feats = feats.to(dev, torch.float32, non_blocking=True)
        if not cfg.USE_IMAGES_GT:
            # raw images [n,3,H,W] -> ENet features [n,128,H/8,W/8] on the sis3d_enet_* kernels (reference: network.py:204-205)
            if self.__dict__.get("_enet") is None:
                raise S.Sis3dError("USE_IMAGES_GT=False but the 2-D ENet encoder was not declared (init_modules with this cfg)")
            tok = self._rec("enet_encoder")
            try:
                feats = self._enet(feats)
            except ValueError as e:  # an input shape the encoder refuses, before anything is launched
                raise S.Sis3dError(str(e)) from None
            self._rec_end(tok)
        n = feats.shape[0]
        if fused is None:
            # reference calling convention: precomputed, stacked index lists + killing_inds
            l3 = blobs["proj_ind_3d"][0].to(dev).contiguous()
            l2 = blobs["proj_ind_2d"][0].to(dev).contiguous()
            nreal = l3.shape[0]
            pix = torch.empty(nreal, dims[0] * dims[1] * dims[2], dtype=torch.int16, device=dev)
            S.check(S.lib.sis3d_project_scatter_lists(S.ptr(l3), S.ptr(l2), nreal, *dims, S.ptr(pix), S.stream()), "scatter")
            kill = set(int(k) for k in (killing_inds or []))
            pl = [(k, k) for k in range(min(n, nreal)) if k not in kill]  # zip(imageft, proj3d) + skip by position
            if not pl:
                raise S.Sis3dError("every view was skipped: nothing to back-project")
            pairs = torch.tensor([v for p in pl for v in p], dtype=torch.int32).to(dev)
            n_pairs = torch.tensor([len(pl)], dtype=torch.int32, device=dev)
            self._proj_counts = None
        else:
            # fused path: depth/pose/world2grid in, no index lists ever materialised
            vp, depths = fused["vp"], fused["depths"]
            intr = (cfg.INTRINSIC[0][0], cfg.INTRINSIC[1][1], cfg.INTRINSIC[0][2], cfg.INTRINSIC[1][2])
            tok = self._rec("project_map")
            pix, counts = proj.project_maps(vp, depths, intr, (cfg.PROJ_DEPTH_MIN, cfg.PROJ_DEPTH_MAX, cfg.VOXEL_SIZE),
                                            dims, w, h)
            self._rec_end(tok)
            pairs = torch.empty(3 * n, dtype=torch.int32, device=dev)
            n_pairs = torch.empty(1, dtype=torch.int32, device=dev)
            S.check(S.lib.sis3d_backproject_pairs(S.ptr(counts), n, S.ptr(pairs), S.ptr(n_pairs), S.stream()), "pairs")
            self._proj_counts = counts
        return feats, pix, pairs, n_pairs

    def _backproject(self, blobs, killing_inds, dims, dev, fused=None):
        """Views -> VC feature volume (reference: trainval.py:797-820 + network.py:194-239).  A colour-aware mask head gathers
        its crops from the same maps later: for it they and the channels-last features are left in self._color_src."""
        w, h = int(cfg.DEPTH_SHAPE[0]), int(cfg.DEPTH_SHAPE[1])
        feats, pix, pairs, n_pairs = self._view_maps(blobs, killing_inds, dims, dev, fused)
        feats = feats.contiguous()
        feats_t = torch.empty(feats.shape[0], w * h, feats.shape[1], dtype=torch.float32, device=dev)
        if self._mask_colour():
            self.__dict__["_color_src"] = dict(feats_t=feats_t, pix=pix, pairs=pairs, n_pairs=n_pairs, n_views=feats.shape[0],
                                               hw=w * h)
        first = self.SPEC["color"][0]
        if (self._sparse_color and not self._keep_debug and first[0] == "k2s2" and feats.shape[1] % 16 == 0
                and first[3] in (32, 64)):
            # fused + sparse: never materialise the back-projected volume (csrc/sparse.cu)
            packed, cout = self._packs["fp32"][f"color.{first[1]}"], self._layers[f"color.{first[1]}"][1]
            od = tuple(d // 2 for d in dims)
            out = Act(torch.empty(*od, cout, dtype=torch.float32, device=dev), od, cout)
            if self._math == "fp16":
                out.h = torch.empty(*od, cout, dtype=torch.float16, device=dev)
            nbytes = int(S.lib.sis3d_backproject_conv_k2s2_workspace_bytes(*dims, cout))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            tok = self._rec("backproject_conv_k2s2")
            S.check(S.lib.sis3d_backproject_conv_k2s2_ex(S.ptr(feats), S.ptr(feats_t), S.ptr(pix), S.ptr(pairs), S.ptr(n_pairs),
                                                         feats.shape[0], feats.shape[1], w, h, *dims, S.ptr(packed), cout,
                                                         S.ptr(out.t), S.ptr(out.h), out.ld, 0, S.ptr(ws), C.c_size_t(nbytes),
                                                         S.stream()),
                    "backproject_conv_k2s2")
            self._rec_end(tok)
            return ("color0", out)
        tok = self._rec("backproject_max")
        vol = proj.backproject(feats, pix, pairs, n_pairs, dims, w, h, feats_t=feats_t)
        self._rec_end(tok)
        return Act(vol, dims, feats.shape[1])

    def _parallel(self, fns):
        """Run independent launch sequences as parallel branches: forked side streams that join back, which CUDA-graph
        capture records as concurrent graph branches.  The layers at 24x12x24 launch only 54-108 CTAs on 132 SMs, so
        independent stacks (colour || geometry, RPN level 1 || level 2) overlap instead of queueing."""
        if not self._branches or self._prof is not None or len(fns) < 2:
            return [f() for f in fns]
        cur = torch.cuda.current_stream()
        key = ("branch_streams", cur.device)
        side = self._const(key, lambda: [torch.cuda.Stream() for _ in range(3)])[:len(fns) - 1]
        out = [None] * len(fns)
        for st in side:
            st.wait_stream(cur)
        pin = S.pin_stream(None)  # launches must follow torch's current stream inside the branches
        try:
            for i, st in enumerate(side, 1):
                with torch.cuda.stream(st):
                    out[i] = fns[i]()
            out[0] = fns[0]()
        finally:
            S.pin_stream(pin)
        for st in side:
            cur.wait_stream(st)
        return out

    def _backbone(self, scene: Act, imageft: Act):
        """reference: backbones.py:98-113.  Concatenation is free: both producers write their slice of
        the level-1 tensor directly (colour channels first, then geometry).  A program without geometry1 (ONLY_IMAGES) is
        image-only: the colour stack's last op writes the whole dense level 1."""
        spec = self.SPEC
        dev = scene.t.device
        if "geometry1" not in spec:
            level1 = (self._run_stack(imageft[1], "color", spec["color"][1:]) if isinstance(imageft, tuple)
                      else self._run_stack(imageft, "color", spec["color"]))
        elif cfg.USE_IMAGES:
            d4 = tuple((d // 2) // 2 for d in scene.dims)
            level1 = Act(torch.empty(*d4, 128, dtype=torch.float32, device=dev), d4, 128)
            def colour():
                if isinstance(imageft, tuple):  # ("color0", act): color.0 already produced by the fused sparse path
                    return self._run_stack(imageft[1], "color", spec["color"][1:],
                                           final_out=lambda x, op: Act(level1.t, d4, 64, ld=128, coff=0))
                return self._run_stack(imageft, "color", spec["color"],
                                       final_out=lambda x, op: Act(level1.t, d4, 64, ld=128, coff=0))

            def geometry():
                return self._run_stack(scene, "geometry1", spec["geometry1"],
                                       final_out=lambda x, op: Act(level1.t, d4, 64, ld=128, coff=64))

            self._parallel([colour, geometry])
        else:
            level1 = self._run_stack(scene, "geometry1", spec["geometry1"])
        level2 = self._run_stack(level1, "geometry2", spec["geometry2"])
        return level1, level2

    def _region_proposal(self, feats, dims, out=None):
        """reference: network.py:537-587 + 657-683 (softmax/anchors/decode/top-N/NMS fused on device)."""
        def head(lvl, f, A):
            h = self._conv(f, f"rpn_net_level{lvl}", act=1, want32=False, want16=True)  # hidden feeds only the merged head
            heads = self._conv(h, f"rpn_heads_level{lvl}")  # [N, ld]: [2A class logits | 6A box deltas | zero pad]
            heads.t.record_stream(torch.cuda.current_stream())
            return heads

        todo = [(lvl, f, cfg["NUM_ANCHORS_LEVEL%d" % lvl]) for lvl, f in enumerate(feats, 1)
                if f is not None and cfg["NUM_ANCHORS_LEVEL%d" % lvl]]
        if [t[0] for t in todo] != list(range(1, len(todo) + 1)):
            # the proposal kernel numbers the levels it is given 1..n and RoI pooling reads level k's features for id k; a gap
            # (e.g. NUM_ANCHORS_LEVEL1 = 0 with level 2 active; the reference keeps the true pyramid level,
            # proposal_layer.py:150-157) would pool from the wrong map.  No released config has one: refuse instead of guessing.
            raise S.Sis3dError("active RPN levels must be contiguous from level 1 (NUM_ANCHORS_LEVELn = 0 only for trailing levels)")
        main = torch.cuda.current_stream()
        outs = self._parallel([(lambda t=t: head(*t)) for t in todo])
        levels = []
        for (lvl, f, A), heads in zip(todo, outs):
            heads.t.record_stream(main)
            ld = heads.C  # padded head width
            cls = Act(heads.t, f.dims, 2 * A, ld=ld, coff=0)
            bbox = Act(heads.t.reshape(-1)[2 * A:], f.dims, 6 * A, ld=ld, coff=0)
            name = cfg["ANCHORS_TYPE_LEVEL%d" % lvl]
            sizes = self._const(("anchors", name, f.t.device), lambda: torch.tensor(
                read_anchor_sizes(name), dtype=torch.float32, device=f.t.device).contiguous())
            if sizes.shape[0] != A:
                raise S.Sis3dError(f"anchor table {name} has {sizes.shape[0]} rows, cfg says {A}")
            levels.append(dict(cls=cls.t, deltas=bbox.t, sizes=sizes, grid=f.dims, A=A, cls_mode=0, cls_ld=ld, deltas_ld=ld))
            if self._keep_debug:
                self._predictions[f"rpn_heads_level{lvl}"] = heads.t  # [..., :2A] class logits, [..., 2A:] box deltas
        tok = self._rec("rpn_proposals")
        res = rpn_proposals(levels, dims, "TEST", want_order=self._keep_debug, out=out)
        self._rec_end(tok)
        if self._keep_debug:
            self._predictions["rpn_order"] = res[4]
        return res[:4]

    def _classify(self, feats, rois, level_ids, out=None):
        """RoI pooling per pyramid level + MLP + heads (reference: network.py:503-534, backbones.py:92-96,
        network.py:589-604).  Always processes the padded post-NMS row count; rows >= num are zeros."""
        P = int(cfg.CLASS_POOLING_SIZE)
        R = rois.shape[0]
        f1 = feats[0]
        dev = rois.device
        pool5 = torch.empty(R, f1.C * P ** 3, dtype=torch.float32, device=dev)
        f = [x.t if x is not None else None for x in feats] + [None, None]
        tok = self._rec("roi_pool_levels")
        S.check(S.lib.sis3d_roi_pool_levels(S.ptr(f[0]), S.ptr(f[1]), S.ptr(f[2]), S.ptr(level_ids),
                                            S.f32(1.0 / self._feat_stride[0]), R, *f1.dims, f1.C, P, P, P, S.ptr(rois),
                                            S.ptr(pool5), None, S.stream()), "roi_pool_levels")
        self._rec_end(tok)
        x1 = self._linear(pool5, "classifier.0", 1)
        nc = int(cfg.NUM_CLASSES)
        if out is not None:
            cls_t, box_t = out
        else:
            cls_t = torch.empty(R, nc, dtype=torch.float32, device=dev)
            box_t = torch.empty(R, nc * 6, dtype=torch.float32, device=dev)
        W, L = self._packs["fp32"], self._layers
        tail = [a for k in ("classifier.2", "classifier.4", "classifier_cls_score_net", "classifier_bbox_pred_net")
                for a in (S.ptr(W[k]), S.ptr(L[k][0]), L[k][1])]  # CUDA-core pack, bias, cout of each layer
        tok = self._rec("mlp_tail")
        S.check(S.lib.sis3d_mlp_tail(S.ptr(x1), R, L["classifier.2"][2], *tail, S.ptr(cls_t), S.ptr(box_t), S.stream()), "mlp_tail")
        self._rec_end(tok)
        cls_score, bbox_pred = Act(cls_t, (R, 1, 1), nc), Act(box_t, (R, 1, 1), nc * 6)
        if self._keep_debug:
            self._predictions["pool5"] = pool5
        return cls_score.t.view(R, -1), bbox_pred.t.view(R, -1)

    def _mask_colour(self):
        """The mask head runs the colour stack (built with MASK_USE_IMAGES)."""
        mb = self._modules.get("mask_backbone")
        return mb is not None and mb.colour

    def _mask_plan(self, det_host, n, X, Y, Z, ncls, canvas, dev, colour):
        """The planner's tables (and the colour stage's, appended) in the pinned staging blob: (plan, color plan, blob)."""
        plan, cplan = S.MaskPlan(), S.MaskColorPlan()
        cap = self._arena["mask_tables_host"].numel() if "mask_tables_host" in self._arena else 1 << 18
        while True:
            stage = self._ws("mask_tables_host", cap, torch.uint8, dev, pinned=True)
            blob, size = C.c_void_p(stage.data_ptr()), C.c_size_t(stage.numel())
            rc = S.lib.sis3d_mask_plan_build(C.c_void_p(det_host.ctypes.data), n, X, Y, Z, ncls, 1 if canvas else 0, blob, size,
                                             C.byref(plan))
            if rc == 0 and colour:
                rc = S.lib.sis3d_mask_color_plan_build(C.c_void_p(det_host.ctypes.data), n, C.byref(plan), blob, size, C.byref(cplan))
                if rc == -3:
                    cap = int(cplan.bytes) * 2
                    continue
            if rc == -3:  # SIS3D_EWORKSPACE: grow the pinned staging buffer and retry
                cap = int(plan.bytes) * 2
                continue
            S.check(rc, "mask_plan_build")
            return plan, cplan, stage

    def _mask_branch(self, scene_ncdhw, det_host, n, extras=None, color=None):
        """Ragged per-RoI mask head (reference: network.py:283-317).  All kept crops are packed along x on
        one zeroed canvas [sum(w_j + 1), max h, max l, 64] (one zero slab between crops = the crop-border
        zero padding), so each of the six layers is ONE launch: layer 1 (C_in = 2, windowed NCDHW scene) and
        the 1x1 head on the fp32 CUDA-core kernel, the four 64->64 3x3x3 layers on the wgmma kernel driven
        by an explicit list of 4x4x8 bricks.  The tables come from the native planner (sis3d_mask_plan_build)
        and travel in ONE pinned H2D copy; all buffers come from a grow-only arena.  A colour-aware head runs
        _mask_branch_color on `color` (the static stage's colour sources, or crop_in: a dense crop of the image features)."""
        if self._mask_colour():
            return self._mask_branch_color(scene_ncdhw, det_host, n, extras, color)
        dev = scene_ncdhw.device
        X, Y, Z = (int(v) for v in scene_ncdhw.shape[2:])
        ncls = self._layers["mask_backbone.geometry.10"][1]
        math = self.MASK_ROUTES.index(self._mask_math)  # route: 0 CUDA-core, 1 TF32, 2 fp16 operands (the 64->64 layers)
        W = self._packs
        det_host = np.ascontiguousarray(det_host[:n], dtype=np.float32)
        plan, _, stage = self._mask_plan(det_host, n, X, Y, Z, ncls, math != 0, dev, False)
        nk = int(plan.n_kept)
        if nk == 0:
            return []
        nbytes, total = int(plan.bytes), int(plan.total_voxels)
        host = stage.numpy()
        offs = host[plan.off_offs:plan.off_offs + 8 * (nk + 1)].view(np.int64).copy()
        sizes = host[plan.off_sizes:plan.off_sizes + 12 * nk].view(np.int32).reshape(nk, 3).copy()
        cvox = int(plan.canvas[0]) * int(plan.canvas[1]) * int(plan.canvas[2])
        a = S.MaskStage()
        a.scene, a.X, a.Y, a.Z, a.ncls, a.math = scene_ncdhw.data_ptr(), X, Y, Z, ncls, math
        a.w_first = W["fp32"]["mask_backbone.geometry.0"].data_ptr()
        a.w_last = W["fp32"]["mask_backbone.geometry.10"].data_ptr()
        for i, idx in enumerate((2, 4, 6, 8)):
            a.w_mid[i] = W[self._mask_math][f"mask_backbone.geometry.{idx}"].data_ptr()
        a.tables = self._ws("mask_tables", nbytes, torch.uint8, dev).data_ptr()
        a.canvas_bytes = 2 * 64 * (total * 4 if math == 0 else cvox * (2 if math == 2 else 4))
        a.canvas = self._ws("mask_canvas", a.canvas_bytes, torch.uint8, dev).data_ptr()
        if math == 2:
            a.canvas32_bytes = cvox * 64 * 4
            a.canvas32 = self._ws("mask_canvas32", a.canvas32_bytes, torch.uint8, dev).data_ptr()
        # handed to the caller (mask_pred views / packed bits): fresh allocations, not arena memory
        outb = torch.empty(total * ncls, dtype=torch.float32, device=dev)
        bits = torch.empty(total, dtype=torch.uint8, device=dev)
        a.masks, a.bits, a.thresh = outb.data_ptr(), bits.data_ptr(), float(cfg.MASK_THRESH)
        if extras is not None:  # the scene loop reads the thresholded masks back: ONE small D2H, queued by the same call
            pin = self._ws("bits_host", total, torch.uint8, dev, pinned=True)
            a.bits_host = pin.data_ptr()
            extras.update(mask_bits=bits, mask_offsets=offs, mask_sizes=sizes, bits_pin=pin[:total])
        tok = self._rec("mask_stage")
        S.check(S.lib.sis3d_mask_stage_launch(C.byref(plan), C.c_void_p(stage.data_ptr()), C.byref(a), S.stream()), "mask_stage")
        self._rec_end(tok)
        return _MaskList(outb, offs, sizes, ncls)

    def _mask_branch_color(self, scene_ncdhw, det_host, n, extras, color):
        """The colour-aware ragged mask stage (MASK_USE_IMAGES / MASK_ONLY_IMAGES; reference: backbones.py:236-287): the
        layout of _mask_branch with a 128-channel colour input per crop, gathered on the device from the view maps and
        features in `color` (or copied from color['crop_in']), and ONE call of sis3d_mask_stage_color_launch."""
        if color is None:
            raise S.Sis3dError("the colour-aware mask head needs the scene's image features (USE_IMAGES inputs)")
        dev = scene_ncdhw.device
        X, Y, Z = (int(v) for v in scene_ncdhw.shape[2:])
        mb, pre = self.mask_backbone, "mask_backbone."
        only = mb.only_images
        ncls = self._layers[pre + ("color.10" if only else "combine.2")][1]
        math = self.MASK_ROUTES.index(self._mask_math)
        W, F = self._packs, self._mask_math
        det_host = np.ascontiguousarray(det_host[:n], dtype=np.float32)
        plan, cplan, stage = self._mask_plan(det_host, n, X, Y, Z, ncls, math != 0, dev, True)
        nk = int(plan.n_kept)
        if nk == 0:
            return []
        total = int(plan.total_voxels)
        host = stage.numpy()
        offs = host[plan.off_offs:plan.off_offs + 8 * (nk + 1)].view(np.int64).copy()
        sizes = host[plan.off_sizes:plan.off_sizes + 12 * nk].view(np.int32).reshape(nk, 3).copy()
        cvox = int(plan.canvas[0]) * int(plan.canvas[1]) * int(plan.canvas[2])
        a = S.MaskStageColor()
        a.scene, a.X, a.Y, a.Z, a.ncls, a.math, a.only_images = scene_ncdhw.data_ptr(), X, Y, Z, ncls, math, int(only)
        a.w_color_first = W[F][pre + "color.0"].data_ptr()
        a.w_color_last = W["fp32"][pre + "color.10"].data_ptr()
        for i, idx in enumerate((2, 4, 6, 8)):
            a.w_color_mid[i] = W[F][f"{pre}color.{idx}"].data_ptr()
        if not only:
            a.w_geom_first = W["fp32"][pre + "geometry.0"].data_ptr()
            a.w_geom_last = W["fp32"][pre + "geometry.10"].data_ptr()
            for i, idx in enumerate((2, 4, 6, 8)):
                a.w_geom_mid[i] = W[F][f"{pre}geometry.{idx}"].data_ptr()
            a.w_combine = W[F][pre + "combine.0"].data_ptr()
            a.w_combine_last = W["fp32"][pre + "combine.2"].data_ptr()
        if "crop_in" in color:
            a.crop_in = color["crop_in"].data_ptr()
        else:
            a.feats_t, a.pix = color["feats_t"].data_ptr(), color["pix"].data_ptr()
            a.pairs, a.n_pairs = color["pairs"].data_ptr(), color["n_pairs"].data_ptr()
            a.n_views, a.hw = int(color["n_views"]), int(color["hw"])
        a.tables = self._ws("mask_tables", int(cplan.bytes), torch.uint8, dev).data_ptr()
        a.canvas_bytes = 4 * 64 * (total * 4 if math == 0 else cvox * (2 if math == 2 else 4))
        a.canvas = self._ws("mask_canvas", a.canvas_bytes, torch.uint8, dev).data_ptr()
        if math == 2:
            a.canvas32_bytes = cvox * (64 if only else 128) * 4
            a.canvas32 = self._ws("mask_canvas32", a.canvas32_bytes, torch.uint8, dev).data_ptr()
        outb = torch.empty(total * ncls, dtype=torch.float32, device=dev)
        bits = torch.empty(total, dtype=torch.uint8, device=dev)
        a.masks, a.bits, a.thresh = outb.data_ptr(), bits.data_ptr(), float(cfg.MASK_THRESH)
        if extras is not None:
            pin = self._ws("bits_host", total, torch.uint8, dev, pinned=True)
            a.bits_host = pin.data_ptr()
            extras.update(mask_bits=bits, mask_offsets=offs, mask_sizes=sizes, bits_pin=pin[:total])
        tok = self._rec("mask_stage_color")
        S.check(S.lib.sis3d_mask_stage_color_launch(C.byref(plan), C.byref(cplan), C.c_void_p(stage.data_ptr()), C.byref(a),
                                                    S.stream()), "mask_stage_color")
        self._rec_end(tok)
        return _MaskList(outb, offs, sizes, ncls)

    # ------------------------------------------------------------------ forward
    _carve_layouts = {}

    @staticmethod
    def _carve(pack, R, nc):
        """Typed views of the packed result buffer of the static stage (one buffer -> one clone / one copy)."""
        lay = Network._carve_layouts.get((R, nc))
        if lay is not None and pack.device.type != "meta":
            return {name: pack[a:b].view(dt).view(shape) for name, a, b, dt, shape in lay[0]}, lay[1]
        o, out, rec = 0, {}, []
        for name, shape, dt in (("rois", (R, 6), torch.float32), ("scores", (R,), torch.float32), ("level_ids", (R,), torch.int32),
                                ("num", (4,), torch.int32), ("cls_score", (R, nc), torch.float32),
                                ("bbox_pred", (R, nc * 6), torch.float32), ("cls_prob", (R, nc), torch.float32),
                                ("det", (R, 16), torch.float32), ("cls_pred", (R,), torch.int64)):
            nb = int(np.prod(shape)) * torch.empty(0, dtype=dt).element_size()
            o = (o + 15) // 16 * 16
            out[name] = pack[o:o + nb].view(dt).view(*shape)
            rec.append((name, o, o + nb, dt, shape))
            o += nb
        Network._carve_layouts[(R, nc)] = (rec, o)
        return out, o

    def _static_stage(self, scene_t, dims, blobs=None, killing_inds=None, fused=None):
        """Every fixed-shape step: back-projection -> backbone -> RPN/NMS -> RoI pool -> classifier ->
        detection decode.  No host synchronisation inside, so the whole stage can be replayed as one CUDA
        graph per (scene shape, #views)."""
        dev = scene_t.device
        P = self._predictions
        scene = Act(scene_t, dims, 2, layout="ncdhw")
        imageft = color_src = None
        if cfg.USE_IMAGES:
            imageft = self._backproject(blobs, killing_inds, dims, dev, fused)
            color_src = self.__dict__.pop("_color_src", None)
            self._imageft_vc = imageft.t if (self._keep_debug and not isinstance(imageft, tuple)) else None
        level1, level2 = self._backbone(scene, imageft)
        if self._keep_debug:
            P["level1_vc"], P["level2_vc"] = level1.t, level2.t
        R, nc = int(cfg.TEST.RPN_POST_NMS_TOP_N), max(int(cfg.NUM_CLASSES), 1)
        probe, total = self._carve(torch.empty(1 << 22, dtype=torch.uint8, device="meta"), R, nc)
        pack = torch.empty(total + 16, dtype=torch.uint8, device=dev)
        out, _ = self._carve(pack, R, nc)
        out["pack"] = pack
        if color_src is not None:
            # the colour-aware mask stage gathers its crops from these after the stage; referenced here, they outlive a
            # captured graph's own use of them (its private pool would otherwise hand their memory to later layers)
            out["color_src"] = color_src
        rois, scores, level_ids = out["rois"], out["scores"], out["level_ids"]
        num = out["num"][:1]
        out["num"] = num
        self._region_proposal((level1, level2, None), dims, out=(rois, scores, level_ids, num))
        if cfg.USE_CLASS:
            cls_score, bbox_pred = self._classify((level1, level2, None), rois, level_ids, out=(out["cls_score"], out["bbox_pred"]))
            cls_prob, cls_pred, det = out["cls_prob"], out["cls_pred"], out["det"]
            tok = self._rec("detect_decode")
            S.check(S.lib.sis3d_detect_decode(S.ptr(rois), S.ptr(num), R, S.ptr(cls_score), S.ptr(bbox_pred), nc,
                                              *dims, S.f32(cfg.CLASS_THRESH), S.ptr(cls_prob), S.ptr(cls_pred),
                                              S.ptr(det), S.stream()), "detect_decode")
            self._rec_end(tok)
        return out

    def _graph_state(self, key, dims, n_views, feat_shape, dev):
        """Static input buffers + captured graph of `_static_stage` for one input shape (feat_shape = shape of one view's
        2-D input: [128,32,41] ENet features, or [3,256,328] images when the encoder is part of the graph)."""
        st = self._graphs.get(key)
        if st is not None:
            if next(reversed(self._graphs)) != key:
                self._graphs[key] = self._graphs.pop(key)  # most recently used last
            return st
        while len(self._graphs) >= self._graph_cache:  # LRU eviction: drops the graph, its static buffers and its pool
            self._graphs.pop(next(iter(self._graphs)))
        w, h = int(cfg.DEPTH_SHAPE[0]), int(cfg.DEPTH_SHAPE[1])
        st = dict(scene=torch.zeros(1, 2, *dims, dtype=torch.float32, device=dev))
        if cfg.USE_IMAGES:
            st.update(feats=torch.zeros(n_views, *feat_shape, dtype=torch.float32, device=dev),
                      depths=torch.zeros(n_views, h, w, dtype=torch.float32, device=dev),
                      vp=torch.zeros(n_views, 40, dtype=torch.float32, device=dev))
        st["graph"] = None
        self._graphs[key] = st
        return st

    # -- a forward is four host steps (stage inputs, static stage, ragged stage, finalize); `forward` runs them back to back,
    #    `forward_pipelined` overlaps them across consecutive scenes on stream slots (each slot owns its graphs, static
    #    buffers and arena)
    def _slot(self, i):
        while len(self._slots) <= i:
            self._slots.append(dict(stream=torch.cuda.Stream() if self._slots else None, graphs={}, arena={}))
        return self._slots[i]

    class _UseSlot:
        def __init__(self, net, slot):
            self.net, self.slot = net, slot

        def __enter__(self):
            n, sl = self.net, self.slot
            d = n.__dict__  # plain attribute writes: nn.Module.__setattr__ costs ~5 us each
            self.saved = (d["_graphs"], d["_arena"])
            d["_graphs"], d["_arena"] = sl["graphs"], sl["arena"]
            self.prev = None
            if sl["stream"] is not None:  # set_stream is several times cheaper than the torch.cuda.stream() context manager
                self.prev = d.get("_home_stream")  # the scene loop looks it up once, not three times per scene
                if self.prev is None:
                    self.prev = torch.cuda.current_stream()
                torch.cuda.set_stream(sl["stream"])
                handle = sl.get("handle")
                if handle is None:
                    handle = sl["handle"] = C.c_void_p(sl["stream"].cuda_stream)
            else:
                handle = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            self.old_pin = S.pin_stream(handle)

        def __exit__(self, *exc):
            S.pin_stream(self.old_pin)
            if self.prev is not None:
                torch.cuda.set_stream(self.prev)
            d = self.net.__dict__
            d["_graphs"], d["_arena"] = self.saved

    def _submit(self, blobs, killing_inds, slot):
        """Step 1 (async): input copies, static stage (graph replay), packed results -> pinned host (async D2H)."""
        return self._run_static(self._stage_inputs(blobs, killing_inds, slot))

    def _stage_inputs(self, blobs, killing_inds, slot):
        """Step 1a (async): per-view constants on the host + the scene's input copies into the slot's static buffers.
        The scene loop issues this one scene ahead of the graph replay so the H2D transfer hides behind compute."""
        self._ensure_packed()
        dev = self.__dict__["_dev"]
        data = blobs["data"]
        if data.shape[0] != 1:
            raise S.Sis3dError("batch size 1 only (as the reference's RoI pooling / proposal layer)")
        dims = tuple(int(v) for v in data.shape[2:])
        home = self.__dict__.get("_home_stream")  # set while the pipelined scene loop runs
        h = dict(slot=slot, dims=dims, id=blobs["id"][0] if "id" in blobs else None, scene_info=data.shape[2:], blobs=blobs,
                 killing_inds=killing_inds, dev=dev, fresh=home is None)
        if home is not None and slot["stream"] is not None:
            # tensors yielded by the scene loop live in slot-owned buffers (result ring, arena): whatever the consumer queued
            # on its own stream to read them (a clone, a D2H copy) must finish before this slot's stream overwrites them
            slot["stream"].wait_stream(home)
        if not cfg.USE_RPN:
            # ground-truth RoIs: the detection table is known on the host before any launch; nothing of the static stage
            # (ENet, back-projection, backbone, RPN, classifier) can change an output, so none of it runs
            if "gt_box" not in blobs:
                raise S.Sis3dError("USE_RPN=False takes its RoIs from blobs['gt_box'], which these blobs lack")
            gt = blobs["gt_box"][0]
            gt = gt.cpu().numpy() if isinstance(gt, torch.Tensor) else np.asarray(gt)
            h.update(use_graph=False, fused=None, gt_box=gt,
                     gt_det=gt_detection_table(gt, dims, cfg.CLASS_THRESH, int(cfg.NUM_CLASSES)))
            if self._mask_colour():  # its crops' image features come from the views (reference: network.py:194-239)
                h["fused"] = self._fused_inputs(blobs, dims)
            return h
        with torch.no_grad(), Network._UseSlot(self, slot):
            lists = cfg.USE_IMAGES and "proj_ind_3d" in blobs
            use_graph = self._use_graph and not (self._keep_debug or self._prof is not None or lists)
            fused = self._fused_inputs(blobs, dims) if cfg.USE_IMAGES else None
            h.update(use_graph=use_graph, fused=fused)
            if use_graph:
                nv = fused["feats"].shape[0] if fused else 0
                fc = tuple(fused["feats"].shape[1:]) if fused else ()
                # the head's test-time settings are kernel arguments and buffer sizes of the captured graph: a changed
                # pre / post-NMS count, NMS or class threshold must not replay a graph captured with the old ones
                t = cfg.TEST
                head = (int(t.RPN_PRE_NMS_TOP_N), int(t.RPN_POST_NMS_TOP_N), float(t.RPN_NMS_THRESH), float(cfg.CLASS_THRESH),
                        int(cfg.ALLOW_BORDER))
                key = (dims, nv, fc, self._math, head)
                seen = self._shape_seen[key] = self._shape_seen.get(key, 0) + 1
                if seen < self._graph_after and key not in self._graphs:
                    use_graph = h["use_graph"] = False  # first sight of this shape: run eagerly, capture when it comes back
            if use_graph:
                st = self._graph_state(key, dims, nv, fc, dev)
                st["scene"].copy_(data, non_blocking=True)
                if fused:
                    st["feats"].copy_(fused["feats"], non_blocking=True)
                    st["depths"].copy_(fused["depths"], non_blocking=True)
                    vph = self._ws("vp_host", fused["vp"].numel(), torch.float32, dev, pinned=True)
                    vph.copy_(fused["vp"].reshape(-1))
                    st["vp"].copy_(vph.view_as(st["vp"]), non_blocking=True)
                    h["fdev"] = dict(vp=st["vp"], feats=st["feats"], depths=st["depths"])
                else:
                    h["fdev"] = None
                h["st"] = st
        return h

    @staticmethod
    def _fused_inputs(blobs, dims):
        """Per-view constants (host) and inputs of the on-device projection; None for blobs with precomputed index lists."""
        if "proj_ind_3d" in blobs:
            return None
        imgs = blobs["nearest_images"]
        w, hh = int(cfg.DEPTH_SHAPE[0]), int(cfg.DEPTH_SHAPE[1])
        vp = proj.view_params(cfg.INTRINSIC, (w, hh), cfg.PROJ_DEPTH_MIN, cfg.PROJ_DEPTH_MAX, dims, None,
                              imgs["poses"][0], imgs["world2grid"][0])
        return dict(vp=vp, feats=imgs["images"][0], depths=torch.as_tensor(imgs["depths"][0]))

    @staticmethod
    def _fused_to(fused, dev):
        return dict(vp=fused["vp"].to(dev, non_blocking=True), feats=fused["feats"].to(dev, torch.float32, non_blocking=True),
                    depths=fused["depths"].to(dev, torch.float32, non_blocking=True).contiguous())

    def _color_sources(self, blobs, killing_inds, dims, dev, fused):
        """Ground-truth RoIs with a colour-aware mask head: the view maps and channels-last view features its gather reads,
        made without the static stage (ENet when the views are images, projection maps, pairs; no feature volume)."""
        feats, pix, pairs, n_pairs = self._view_maps(blobs, killing_inds, dims, dev, self._fused_to(fused, dev) if fused else None)
        feats = feats.contiguous()
        n, Cn, hw = feats.shape[0], feats.shape[1], feats.shape[2] * feats.shape[3]
        feats_t = torch.empty(n, hw, Cn, dtype=torch.float32, device=dev)
        S.check(S.lib.sis3d_mask_color_feats_t(S.ptr(feats), n, Cn, hw, S.ptr(feats_t), S.stream()), "mask_color_feats_t")
        return dict(feats_t=feats_t, pix=pix, pairs=pairs, n_pairs=n_pairs, n_views=n, hw=hw)

    def _run_static(self, h):
        """Step 1b (async): static stage (graph replay) on the staged inputs, packed results -> pinned host (async D2H)."""
        blobs, killing_inds, slot, dims, dev = h.pop("blobs"), h.pop("killing_inds"), h["slot"], h["dims"], h.pop("dev")
        data = blobs["data"]
        fused = h.pop("fused")
        before = set(self._predictions) if self._keep_debug else None
        with torch.no_grad(), Network._UseSlot(self, slot):
            if h.pop("use_graph"):
                st, fdev = h.pop("st"), h.pop("fdev")
                if st["graph"] is None:
                    # eager warm-up (fills the region/constant caches, sets kernel attributes), then capture
                    self._static_stage(st["scene"], dims, blobs, None, fdev)
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    n0 = S.launch_count()
                    pin = S.pin_stream(None)  # capture runs on torch's capture stream
                    gc_was_on = gc.isenabled()
                    gc.disable()  # a cyclic-GC pass in the middle of a capture may free CUDA objects (illegal while capturing)
                    try:
                        with torch.cuda.graph(g):
                            st["outs"] = self._static_stage(st["scene"], dims, blobs, None, fdev)
                    finally:
                        if gc_was_on:
                            gc.enable()
                        S.pin_stream(pin)
                    st["graph"], st["n_kernels"] = g, S.launch_count() - n0
                st["graph"].replay()
                self.__dict__["_replayed_kernels"] += st["n_kernels"]
                # results must not alias the replay buffers: ONE copy of the packed result buffer into one of two
                # slot-owned, pre-carved result buffers (valid until this slot has been reused twice)
                ring = st.get("result_ring")
                if h["fresh"]:
                    # reference-compatible forward(): the caller may keep _predictions across scenes (the reference returns
                    # fresh tensors), so hand out a private copy of the packed results and of the scene
                    pk = torch.empty_like(st["outs"]["pack"])
                    outs, _ = self._carve(pk, int(cfg.TEST.RPN_POST_NMS_TOP_N), max(int(cfg.NUM_CLASSES), 1))
                    outs["num"] = outs["num"][:1]
                    outs["pack"] = pk
                    ring = False
                elif ring is None:
                    ring = st["result_ring"] = []
                    for _ in range(2):
                        pk = torch.empty_like(st["outs"]["pack"])
                        o, _ = self._carve(pk, int(cfg.TEST.RPN_POST_NMS_TOP_N), max(int(cfg.NUM_CLASSES), 1))
                        o["num"] = o["num"][:1]
                        o["pack"] = pk
                        ring.append(o)
                    st["ring_pos"] = 0
                if ring is not False:
                    outs = ring[st["ring_pos"]]
                    st["ring_pos"] ^= 1
                outs["pack"].copy_(st["outs"]["pack"], non_blocking=True)
                if "color_src" in st["outs"]:
                    outs["color_src"] = st["outs"]["color_src"]
                scene_t = st["scene"].clone() if h["fresh"] else st["scene"]
            elif "gt_det" in h:  # ground-truth RoIs: the scene's input copy (and a colour head's view maps) before the mask stage
                scene_t = data.to(dev, torch.float32, non_blocking=True).contiguous()
                outs = None
                if self._mask_colour():
                    h["color_src"] = self._color_sources(blobs, killing_inds, dims, dev, fused)
            else:
                scene_t = data.to(dev, torch.float32, non_blocking=True).contiguous()
                if fused:
                    fused = self._fused_to(fused, dev)
                outs = self._static_stage(scene_t, dims, blobs, killing_inds, fused)
            h["outs"], h["scene_t"] = outs, scene_t
            # the one host round trip of a scene: decoded detections with the RoI count in row 0 / col 15 (12.8 KB)
            if cfg.USE_CLASS:
                det_pin = self._ws("det_host", outs["det"].numel(), torch.float32, dev, pinned=True).view_as(outs["det"])
                det_pin.copy_(outs["det"], non_blocking=True)
                h["det_pin"] = det_pin
            h["ev_static"] = torch.cuda.Event(blocking=self._blocking_sync)
            h["ev_static"].record()
        if self._keep_debug:  # intermediate tensors the static stage left in _predictions (parity tests)
            h["debug"] = {k: v for k, v in self._predictions.items()
                          if k.startswith(("level", "rpn_", "pool5")) or k not in before}
        return h

    def _launch_ragged(self, h):
        """Step 2: wait for the detections of this scene, plan + launch its ragged mask stage, queue the readback."""
        if "gt_det" in h:
            return self._launch_ragged_gt(h)
        h["ev_static"].synchronize()
        outs = h["outs"]
        P = {}
        with torch.no_grad(), Network._UseSlot(self, h["slot"]):
            if cfg.USE_CLASS:
                det_all = h["det_pin"].numpy()
                n = int(det_all[0, 15])
            else:
                n = int(outs["num"].item())
            P["rois"], P["roi_scores"] = [outs["rois"][:n]], [outs["scores"][:n].view(-1, 1)]
            P["level_inds"] = [outs["level_ids"][:n].float()]
            if cfg.USE_CLASS:
                P["cls_score"], P["cls_pred"], P["cls_prob"] = outs["cls_score"][:n], outs["cls_pred"][:n], outs["cls_prob"][:n]
                P["bbox_pred"] = outs["bbox_pred"][:n]
                P["detections"] = outs["det"][:n]
                if cfg.USE_MASK:
                    det_host = det_all[:n].copy()
                    extras = {}
                    P["mask_pred"] = [self._mask_branch(h["scene_t"], det_host, n, extras, outs.get("color_src"))]
                    P["detections_host"] = det_host
                    if "bits_pin" in extras:  # thresholded predicted-class masks -> pinned host (queued by the mask stage)
                        h["bits_pin"] = extras.pop("bits_pin")
                    P.update(extras)
            h["ev_done"] = torch.cuda.Event(blocking=self._blocking_sync)
            h["ev_done"].record()
        h["P"] = P
        return h

    def _launch_ragged_gt(self, h):
        """Step 2 with ground-truth RoIs (reference: network.py:262-265, 276-317): the table was built on the host, so there
        is nothing to wait for.  The predictions other than the masks are host tensors, as the reference's cls_pred /
        cls_prob / bbox_pred are: the scene's only GPU work is its input copy and the mask stage."""
        gt, det = h.pop("gt_box"), h.pop("gt_det")
        n, nc = det.shape[0], int(cfg.NUM_CLASSES)
        cls = torch.from_numpy(det[:, 7].astype(np.int64))
        prob = torch.zeros(n, nc, dtype=torch.float32)
        prob[torch.arange(n), cls] = 1.0
        P = dict(rois=[torch.from_numpy(np.ascontiguousarray(gt[:, :6], dtype=np.float32))],
                 roi_scores=[torch.ones(n, 1, dtype=torch.float32)], cls_pred=cls, cls_prob=prob,
                 bbox_pred=torch.zeros(n, 6 * nc, dtype=torch.float32), detections=torch.from_numpy(det), detections_host=det)
        with torch.no_grad(), Network._UseSlot(self, h["slot"]):
            if cfg.USE_MASK:
                extras = {}
                P["mask_pred"] = [self._mask_branch(h["scene_t"], det, n, extras, h.get("color_src"))]
                if "bits_pin" in extras:
                    h["bits_pin"] = extras.pop("bits_pin")
                P.update(extras)
            h["ev_done"] = torch.cuda.Event(blocking=self._blocking_sync)
            h["ev_done"].record()
        h["P"] = P
        return h

    def _finalize(self, h):
        """Step 3: wait for the scene's last kernel / copy and hand out its predictions."""
        h["ev_done"].synchronize()
        P = h["P"]
        if "bits_pin" in h:
            P["mask_bits_host"] = h["bits_pin"].numpy().copy()
        self.__dict__.update(_scene_info=h["scene_info"], _id=h["id"], _scene=h["scene_t"], batch_size=1, _mode="TEST")
        self._predictions.clear()
        self._predictions.update(h.get("debug", {}))
        self._predictions.update(P)
        return self._predictions

    def _check_mode(self, mode):
        if mode != "TEST":
            raise NotImplementedError("only the inference (TEST) forward is implemented on the GPU path")
        # ground-truth RoIs run with USE_RPN = USE_CLASS = False (USE_BACKBONE either way); the reference cannot run the
        # other combinations either
        if cfg.USE_RPN and not cfg.USE_BACKBONE:
            raise NotImplementedError("USE_BACKBONE=False with USE_RPN=True: the RPN reads the backbone's features (the "
                                      "reference fails with a NameError); turn USE_RPN and USE_CLASS off for ground-truth RoIs")
        if not cfg.USE_RPN and cfg.USE_CLASS:
            raise NotImplementedError("USE_RPN=False with USE_CLASS=True: ground-truth boxes with the classifier have no test-"
                                      "time semantics (the reference fails with KeyError 'level_inds'); turn USE_CLASS off too")

    def forward(self, blobs, mode="TEST", killing_inds=None):
        """Reference-compatible synchronous forward of one scene (lib/nets/network.py:72,187-317)."""
        self._check_mode(mode)
        return self._finalize(self._launch_ragged(self._submit(blobs, killing_inds, self._slot(0))))

    def forward_pipelined(self, blobs_iter, mode="TEST"):
        """Throughput form of the scene loop (lib/model/trainval.py:787-822): yields (blobs, predictions) in order while
        seven scenes are in flight on seven stream slots -- scene i+1: input H2D (issued one scene ahead so the transfer
        hides behind compute); scenes i .. i-3: static stage (four graph replays overlapping: one alone is a latency
        chain of small grids; measured 3 -> 4: +1 %, 5: no further gain); then the ragged mask stage and the read-back.
        The yielded dict is only valid until the next iteration."""
        self._check_mode(mode)
        self._ensure_packed()
        blobs_iter = self._reject_index_lists(blobs_iter)
        self.__dict__["_home_stream"] = torch.cuda.current_stream()  # restored after every slot switch of this loop
        finished = False
        try:
            yield from self._scene_loop(blobs_iter)
            finished = True
        finally:
            self.__dict__["_home_stream"] = None
            if not finished:
                # a consumer that stopped early (break, exception) leaves scenes in flight on their slots; the host writes
                # those slots' pinned staging buffers (vp_host, mask tables) when it next uses them, so let the queued work end
                for sl in self._slots:
                    if sl["stream"] is not None:
                        sl["stream"].synchronize()

    @staticmethod
    def _reject_index_lists(blobs_iter):
        """The scene loop computes the projection on the device from depth / pose / world2grid; blobs that carry precomputed
        proj_ind_3d/2d lists need their killing_inds (lib/model/trainval.py:805-822), which this API has no slot for: they go
        through the synchronous forward(blobs, 'TEST', killing_inds)."""
        for b in blobs_iter:
            if "proj_ind_3d" in b:
                raise S.Sis3dError("forward_pipelined takes depth/pose/world2grid blobs; use forward(blobs, 'TEST', killing_inds) "
                                   "for blobs with precomputed proj_ind_3d/2d lists")
            yield b

    def _scene_loop(self, blobs_iter):
        from collections import deque
        q = deque()      # [blobs, handle, ragged_launched] of scenes whose static stage has been launched
        staged = None    # (blobs, handle) of the scene whose inputs are uploading
        i = 0
        n_static = max(1, int(os.environ.get("SIS3D_PIPE_STATIC", "4")))  # static stages (graph replays) in flight at once
        depth = max(n_static + 2, int(os.environ.get("SIS3D_PIPE_DEPTH", str(n_static + 3))))  # scenes in flight (= stream slots)
        for blobs in blobs_iter:
            if len(q) == depth - 1:  # frees the slot the new scene is about to use
                b, h, _ = q.popleft()
                yield b, self._finalize(h)
            nxt = (blobs, self._stage_inputs(blobs, None, self._slot(1 + i % depth)))
            i += 1
            if staged is not None:
                q.append([staged[0], self._run_static(staged[1]), False])
            staged = nxt
            # the mask stage of a scene needs its detections on the host: wait for the static stage launched n_static
            # iterations ago, so that n_static graph replays overlap on the GPU (one alone is a latency chain of small grids)
            if len(q) > n_static and not q[-n_static - 1][2]:
                self._launch_ragged(q[-n_static - 1][1])
                q[-n_static - 1][2] = True
        if staged is not None:
            q.append([staged[0], self._run_static(staged[1]), False])
        while q:
            b, h, launched = q.popleft()
            if not launched:
                self._launch_ragged(h)
            yield b, self._finalize(h)

    def kernel_launches(self):
        """libsis3d kernels executed so far by this process: direct launches + kernels inside replayed graphs."""
        return S.launch_count() + self._replayed_kernels

    def delete_intermediate_states(self):
        self._predictions.clear()
