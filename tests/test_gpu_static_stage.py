"""GPU: every layer of the static stage against fp64 on its own inputs, in every conv math mode, on the bench scenes.

The static stage is back-projection -> colour / geometry stacks -> level-1 concat -> geometry2 -> RPN hidden and merged
heads -> classifier.0.  One eager forward per (scene, mode) runs with per-kernel timing on (`net._prof = {}`: no CUDA graph,
no parallel branches, the sparse colour path kept) and with `_conv`, `_bottleneck`, `_linear`, `_pool` and `_backproject`
wrapped on the instance: each call's inputs (fp32 activation and / or fp16 twin, residual), outputs and the `_rec` route
names it emitted are cloned after a device synchronisation.  The fp64 references come from the live parameters
(`net.state_dict()`), never from the packed weights, so a stale or wrongly built pack fails; the merged RPN heads are
rebuilt from the two heads' own parameters.

Every layer must meet
  - the bound of the route it took (ROUTE_CHECKS: the per-element bounds of tests/test_gpu_tc_accuracy.py and
    tests/test_gpu_simt_accuracy.py), and
  - the bound its math mode promises whatever the route (PROMISE): compensated products in exact / f16x3 / tf32x3, one TF32
    or fp16 product in mixed / tf32 / fp16, the fmaf chain in fp32.  A layer silently demoted to a cheaper route fails here.
fp16 twins equal fp16(fp32) bit for bit wherever both exist, maxpool3 is bit exact, each op reads what the op before it in
its program wrote, the level-1 halves and the merged heads' channel blocks are where the next layers read them.  Power:
the broken-kernel models of the tables and the wiring models (residual or bias omitted, input shifted by one channel,
level-1 halves swapped, input of the previous scene) must each miss the bound by POWER somewhere in every layer they apply
to.  Modes that share a static form (exact / f16x3, mixed / tf32) give identical bits, and the hooked eager forward gives
the detections of the default forward (CUDA graph, parallel branches) bit for bit.

Out of scope here, each checked by its own file (OUT_OF_SCOPE): projection, back-projection max, proposals, RoI pooling,
the MLP tail, detection decode, the mask stage and the 2-D encoder."""
import inspect
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sis3d_synth as synth
from test_gpu_simt_accuracy import fmaf_chain_accuracy, linear_splits
from test_gpu_tc_accuracy import C_T, _conv, _product, conv_accuracy, fused_accuracy, linear_accuracy

pytestmark = pytest.mark.gpu
DEV = "cuda"

# route family (a `_rec` name without its [layer]) -> (check, kernel-table mode, what the check is)
ROUTE_CHECKS = {
    "conv_tc": ("tc", "tf32", "conv_accuracy, one TF32 product"),
    "conv_tc_x3": ("tc", "x3", "conv_accuracy, TF32 split"),
    "conv_tc_h3": ("tc", "h3", "conv_accuracy, fp16 split"),
    "conv_tc16": ("tc", "f16", "conv_accuracy, fp16 operands (+ fp16 output rounding when only the twin exists)"),
    "conv_tc_fused": ("fused", "tf32", "fused_accuracy on conv1's captured output"),
    "conv_tc_fused_x3": ("fused", "x3", "fused_accuracy on conv1's captured output"),
    "conv_tc_h3_split": ("split_conv1", "h3", "conv1 of a split block: its bound feeds the block's"),
    "conv_tc_fused_h3_split": ("split_block", "h3s", "the whole block from its fp32 input, conv1's bound carried through w2"),
    "conv": ("fmaf", None, "fmaf_chain_accuracy, n = K + 2"),
    "backproject_conv_k2s2": ("sparse", None, "fmaf_chain_accuracy, n = C + 8, on the dense back-projected volume"),
    "linear_tc": ("linear", "tf32", "linear_accuracy"),
    "linear_tc_x3": ("linear", "x3", "linear_accuracy"),
    "linear_tc_h3": ("linear", "h3", "linear_accuracy"),
    "linear": ("linear_fmaf", None, "fmaf_chain_accuracy, split-K depth"),
    "maxpool3": ("pool", None, "bit exact against F.max_pool3d(3, 1, 1)"),
    "cast_f16": ("twin", None, "the twin equals fp16(fp32) bit for bit"),
}
OUT_OF_SCOPE = {
    "project_map": "tests/test_gpu_decision_kernels.py",
    "backproject_max": "tests/test_gpu_decision_kernels.py, tests/test_gpu_forward.py (bit exact to the oracle)",
    "rpn_proposals": "tests/test_gpu_head_stage.py, tests/test_gpu_decision_kernels.py",
    "roi_pool_levels": "tests/test_gpu_head_stage.py, tests/test_gpu_decision_kernels.py",
    "mlp_tail": "tests/test_gpu_head_stage.py, tests/test_gpu_simt_accuracy.py",
    "detect_decode": "tests/test_gpu_head_stage.py, tests/test_gpu_decision_kernels.py",
    "mask_stage": "tests/test_gpu_mask_stage.py",
    "enet_encoder": "tests/test_gpu_enet.py",
}
# the bound each math mode promises for every conv and linear of the stage: compensated (C_X3 s2 + C_T + C_FLOOR terms),
# one product (C_1X s2 + C_T terms), the fmaf chain
PROMISE = {"exact": "h3", "f16x3": "h3", "tf32x3": "h3", "mixed": "tf32", "tf32": "tf32", "fp16": "tf32", "fp32": "fmaf"}
SAME_STATIC = (("exact", "f16x3"), ("mixed", "tf32"))  # modes with the same static-stage form: identical bits

SCENES = {  # the cfg2 / cfg5 / cfg3 bench scenes, and two golden cases: partial bricks everywhere, geometry only
    "cfg2": dict(cfgname="scannet", dims=(96, 48, 96), n_img=5, seed=1000, use_images=True, use_mask=True),
    "cfg5": dict(cfgname="suncg", dims=(96, 48, 96), n_img=3, seed=5000, use_images=True, use_mask=True),
    "odd_45x27x41": synth.CASES["odd_45x27x41"],
    "cfg1_32": synth.CASES["cfg1_32"],
    "cfg3": dict(cfgname="scannet", dims=(208, 48, 160), n_img=40, seed=3000, use_images=True, use_mask=True),
}
CYCLE = ("exact", "f16x3", "tf32x3", "mixed", "fp16", "tf32", "fp32", "exact")  # mixed -> fp16 keeps the form set
# parameters updated in place before the last exact pass of a cycle: a conv weight and a bottleneck bias
UPDATES = (("geometry2.0.weight", lambda p: p.mul_(1.25)), ("geometry1.2.conv2.bias", lambda p: p.add_(0.25)))


def _rows():
    rows = []
    for scene in ("cfg2", "cfg5", "odd_45x27x41", "cfg1_32"):
        rows += [dict(scene=scene, mode=m, step=i, sparse=True, updated=False) for i, m in enumerate(CYCLE)]
        rows.append(dict(scene=scene, mode="exact", step=len(CYCLE), sparse=True, updated=True))
    rows.append(dict(scene="cfg2", mode="exact", step=len(CYCLE) + 1, sparse=False, updated=True))  # dense colour.0
    rows += [dict(scene="cfg3", mode=m, step=i, sparse=True, updated=False) for i, m in enumerate(("exact", "fp16"))]
    for r in rows:
        r["id"] = f"{r['scene']}-{r['step']}-{r['mode']}" + ("-updated" if r["updated"] else "") + ("" if r["sparse"] else "-dense")
    return rows


ROWS = _rows()


def active_levels():
    from lib.utils.config import cfg
    return tuple(lvl for lvl in (1, 2, 3) if cfg.get("NUM_ANCHORS_LEVEL%d" % lvl, 0))


def stage_layers(spec, images, levels):
    """Every conv / linear layer of the static stage of a backbone program (conv layers of the blocks by name)."""
    out = []
    for stage in ("color", "geometry1", "geometry2"):
        if stage == "color" and not images:
            continue
        for op in spec.get(stage, ()):
            if op[0] in ("k2s2", "k3"):
                out.append(f"{stage}.{op[1]}")
            elif op[0] == "bneck":
                out += [f"{stage}.{op[1]}.conv{i}" for i in (1, 2, 3)]
    out += [f"rpn_{k}_level{lvl}" for lvl in levels for k in ("net", "heads")]
    return out + ["classifier.0"]


# ------------------------------------------------------------------------------------------------ capture
def _dense(a):
    """The channels of activation `a` as a dense fp32 [X][Y][Z][C] clone (None when it has no fp32 tensor)."""
    if a is None or a.t is None:
        return None
    if a.layout == "ncdhw":
        return a.t.reshape(a.C, *a.dims).permute(1, 2, 3, 0).clone()
    t = a.t.reshape(-1)[:a.nvox * a.ld].view(a.nvox, a.ld)[:, a.coff:a.coff + a.C]
    return t.reshape(*a.dims, a.C).clone()


def _twin(a):
    return None if a is None or getattr(a, "h", None) is None else a.h.clone()


class Capture:
    """Wraps the static stage's op methods on one Network instance and records every call (see the module docstring)."""
    HOOKED = ("_conv", "_bottleneck", "_linear", "_pool", "_backproject")

    def __init__(self, net, hooked=HOOKED):
        self.hooked = tuple(hooked)
        self.net, self.ops, self.stack, self.loose, self.mute = net, [], [], [], False
        rec = net._rec

        def on_rec(name):
            if not self.mute:
                (self.stack[-1]["routes"] if self.stack else self.loose).append(name)
            return rec(name)

        net.__dict__["_rec"] = on_rec
        for fn in self.hooked:
            net.__dict__[fn] = self._wrap(fn[1:], getattr(net, fn))

    def detach(self):
        for fn in self.hooked + ("_rec",):
            self.net.__dict__.pop(fn, None)

    def _wrap(self, kind, orig):
        sig = inspect.signature(orig)

        def hook(*a, **k):
            bound = sig.bind(*a, **k)
            bound.apply_defaults()
            v = bound.arguments
            torch.cuda.synchronize()
            op = dict(kind=kind, routes=[], parent=self.stack[-1]["i"] if self.stack else None, i=len(self.ops))
            if kind in ("conv", "bottleneck", "pool"):
                op.update(name=v.get("name"), x=_dense(v["x"]), act=v.get("act", 1), res=_dense(v.get("residual")))
            elif kind == "linear":
                op.update(name=v["name"], x=v["x"].clone(), act=v["act"])
            self.ops.append(op)
            self.stack.append(op)
            try:
                res = orig(*a, **k)
            finally:
                self.stack.pop()
            torch.cuda.synchronize()
            if kind in ("conv", "bottleneck", "pool"):
                op.update(x16=_twin(v["x"]), y=_dense(res), y16=_twin(res))
            elif kind == "linear":
                op["y"] = res.clone()
            else:  # backproject: the dense volume, fetched once more on the dense path
                act = res[1] if isinstance(res, tuple) else res
                op.update(name="color.0" if isinstance(res, tuple) else None, y=_dense(act), y16=_twin(act))
                if isinstance(res, tuple):
                    self.mute, sparse = True, self.net._sparse_color
                    self.net._sparse_color = False
                    try:
                        op["vol"] = _dense(orig(*a, **k))
                    finally:
                        self.net._sparse_color, self.mute = sparse, False
                    torch.cuda.synchronize()
                else:
                    op["vol"] = op["y"]
            return res

        return hook


def _results(P):
    out = {"rois": P["rois"][0].clone(), "cls_prob": P["cls_prob"].clone(), "detections": P["detections"].clone()}
    if "detections_host" in P:
        out["detections_host"] = torch.from_numpy(np.array(P["detections_host"], copy=True))
    return out


def run_hooked(net, blobs):
    cap = Capture(net)
    net._prof = {}
    try:
        P = net.forward(blobs, "TEST", None)
        torch.cuda.synchronize()
        res = _results(P)
    finally:
        cap.detach()
        net._prof = None
    return cap, res


def _bits(t):
    return t.view({torch.float32: torch.int32, torch.float16: torch.int16, torch.float64: torch.int64}.get(t.dtype, t.dtype))


def same_bits(a, b):
    return a is None and b is None or (a is not None and b is not None and a.shape == b.shape and a.dtype == b.dtype
                                       and torch.equal(_bits(a), _bits(b)))


# ------------------------------------------------------------------------------------------------ references
def live_weights(net):
    """layer -> (fp32 weight, fp32 bias or None) from the live parameters; per RPN level the merged heads rebuilt from the
    class and box heads' parameters: [2A class | 6A box | zero pad up to the kernel's width]."""
    sd = {k: v.detach().to(DEV, torch.float32) for k, v in net.state_dict().items()}
    W = {k[:-7]: (v, sd.get(k[:-7] + ".bias")) for k, v in sd.items() if k.endswith(".weight")}
    for lvl in (1, 2, 3):
        c, b = W.get(f"rpn_cls_score_net_level{lvl}.0"), W.get(f"rpn_bbox_pred_net_level{lvl}")
        if c is not None and b is not None:
            W[f"rpn_heads_level{lvl}"] = ("heads", c, b)
    return W


def heads_weights(entry, width):
    _, (wc, bc), (wb, bb) = entry
    w = torch.zeros(width, *wc.shape[1:], device=DEV)
    b = torch.zeros(width, device=DEV)
    n2, n6 = wc.shape[0], wb.shape[0]
    w[:n2], b[:n2], w[n2:n2 + n6], b[n2:n2 + n6] = wc, bc, wb, bb
    return w, b, n2 + n6


def _energy_slice(x):
    """The 32-channel slice of the last axis with the most input energy (the slice a broken-kernel model drops)."""
    c = x.shape[-1]
    if c < 64 or c % 32:
        return None
    e = (x.double() ** 2).reshape(-1, c).sum(0).view(-1, 32).sum(1)
    return int(e.argmax())


def _swap_halves(x):
    return torch.cat([x[..., 64:], x[..., :64]], -1)


class Row:
    """The checks of one captured forward."""

    def __init__(self, row, net, cap, prev, images, scene):
        self.row, self.net, self.cap, self.prev, self.images, self.scene = row, net, cap, prev, images, scene
        self.mode = row["mode"]
        self.W = live_weights(net)
        self.results = []      # (layer, route, kernel err / bound, smallest model err / bound)
        self.checked = set()   # route families checked in this row

    def what(self, layer, route):
        return f"{self.row['id']} {route}[{layer}]"

    def weights(self, layer, got=None):
        e = self.W[layer]
        if e[0] == "heads":
            w, b, n = heads_weights(e, got.shape[-1])
            pad = got[..., n:]
            assert bool((pad == 0).all()), f"{self.row['id']} [{layer}]: pad channels {n}.. of the merged heads are not 0"
            return w, b
        return e

    # -------------------------------------------------------------- wiring models (pre-activation, epilogue included)
    def conv_models(self, layer, x, w, b, r, prev_x):
        d = lambda t: t.to(DEV).double()
        epi = (d(b) if b is not None else 0) + (d(r) if r is not None else 0)
        ks, m = w.shape[2], {}
        lin = lambda a: _conv(d(a), d(w), ks) + epi
        if r is not None:
            m["residual_omitted"] = lambda ref: ref - d(r)
        if b is not None and bool((b != 0).any()):
            m["bias_omitted"] = lambda ref: ref - d(b)
        if x.shape[-1] > 1:
            m["input_shifted_one_channel"] = lin(torch.roll(x, 1, -1))
        if self.images and layer in ("geometry2.0", "rpn_net_level1"):
            m["level1_halves_swapped"] = lin(_swap_halves(x))
        if prev_x is not None and prev_x.shape == x.shape:
            m["previous_scene_input"] = lin(prev_x)
        return m

    def prev_input(self, kind, layer):
        return None if self.prev is None else self.prev.get((kind, layer))

    # -------------------------------------------------------------- per-op checks
    def promise_conv(self, layer, got, x, w, b, r, act, out16, n):
        p = PROMISE[self.mode]
        what = self.what(layer, "promise of " + self.mode)
        if p == "fmaf":
            return self.fmaf_conv(layer, got, x, w, b, r, act, n, None, what)
        return conv_accuracy(p, got, x, w, b, r, act, what=what, models=False, out16=out16)

    def fmaf_conv(self, layer, got, x, w, b, r, act, n, models, what):
        d = lambda t: t.to(DEV).double()
        ks = w.shape[2]
        acc = _conv(d(x), d(w), ks)
        absum = _conv(d(x).abs(), d(w).abs(), ks)
        epi = torch.zeros_like(acc) + (d(b) if b is not None else 0) + (d(r) if r is not None else 0)
        if models is None:
            return fmaf_chain_accuracy(got, acc, absum, n, epi, act, what=what), math.inf
        full = {k: v(acc + epi) if callable(v) else v for k, v in models.items()}
        return fmaf_chain_accuracy(got, acc, absum, n, epi, act, mutants=full, what=what)

    def check_conv(self, op, fam):
        layer = op["name"]
        chk, kmode, _ = ROUTE_CHECKS[fam]
        x = op["x"] if op["x"] is not None else op["x16"].float()
        got = op["y"] if op["y"] is not None else op["y16"].float()
        out16 = op["y"] is None
        w, b = self.weights(layer, got)
        r, act = op["res"], op["act"]
        n = w.shape[2] ** 3 * w.shape[1] + 2
        models = self.conv_models(layer, x, w, b, r, self.prev_input("conv", layer))
        what = self.what(layer, fam)
        if chk == "tc":
            k, m = conv_accuracy(kmode, got, x, w, b, r, act, what=what, slice_=_energy_slice(x), extra=models, out16=out16)
        else:
            assert not out16, f"{what}: the CUDA-core kernel wrote no fp32 output"
            k, m = self.fmaf_conv(layer, got, x, w, b, r, act, n, models, what)
        kp, _ = self.promise_conv(layer, got, x, w, b, r, act, out16, n)
        return k, m, kp

    def block_ref(self, name, x, r):
        """fp64 bottleneck output (before the final ReLU) from block input x and residual r."""
        d = lambda t: t.to(DEV).double()
        y = x
        for i, ks in ((1, 1), (2, 3), (3, 1)):
            w, b = self.W[f"{name}.conv{i}"]
            y = _conv(d(y), d(w), ks) + d(b)
            if i < 3:
                y = F.relu(y)
        return y + d(r)

    def block_models(self, name, x_block, b3, tail_x=None):
        d = lambda t: t.to(DEV).double()
        m = {"residual_omitted": lambda ref: ref - d(x_block), "bias_omitted": lambda ref: ref - d(b3)}
        if tail_x is None:
            m["input_shifted_one_channel"] = self.block_ref(name, torch.roll(x_block, 1, -1), x_block)
        else:  # the tail reads conv1's output: shift that
            w2, b2 = self.W[f"{name}.conv2"]
            w3, _ = self.W[f"{name}.conv3"]
            y = F.relu(_conv(d(torch.roll(tail_x, 1, -1)), d(w2), 3) + d(b2))
            m["input_shifted_one_channel"] = _conv(y, d(w3), 1) + d(b3) + d(x_block)
        px = self.prev_input("bottleneck", name)
        if px is not None and px.shape == x_block.shape:
            m["previous_scene_input"] = self.block_ref(name, px, px)
        return m

    def check_block(self, op, fam, conv1):
        name = op["name"]
        chk, kmode, _ = ROUTE_CHECKS[fam]
        (w2, b2), (w3, b3) = self.W[f"{name}.conv2"], self.W[f"{name}.conv3"]
        x, got = op["x"], op["y"]
        what = self.what(name, fam)
        p = PROMISE[self.mode]
        assert p != "fmaf", f"{what}: {self.mode} promises the CUDA-core chain, the block ran fused on the tensor cores"
        if chk == "split_block":
            w1, b1 = self.W[f"{name}.conv1"]
            y, e_in = self.split_conv1(x, w1, b1)
            models = self.block_models(name, x, b3)
            k, m = fused_accuracy(kmode, got, y, w2, b2, w3, b3, x, 1, what, bound_in=e_in, slice_=_energy_slice(y),
                                  extra=models)
            kp, _ = fused_accuracy(p, got, y, w2, b2, w3, b3, x, 1, self.what(name, "promise of " + self.mode),
                                   bound_in=e_in, models=False)
        else:
            y = conv1["y"]
            models = self.block_models(name, x, b3, tail_x=y)
            k, m = fused_accuracy(kmode, got, y, w2, b2, w3, b3, x, 1, what, slice_=_energy_slice(y), extra=models)
            kp, _ = fused_accuracy(p, got, y, w2, b2, w3, b3, x, 1, self.what(name, "promise of " + self.mode), models=False)
        return k, m, kp

    @staticmethod
    def split_conv1(x, w1, b1):
        """fp64 conv1 output of a split block and its error bound (the compensated 1x1 conv: C_X3 s2 + floor + C_T)."""
        d = lambda t: t.to(DEV).double()
        acc, bnd, _ = _product("h3", lambda a, v: _conv(a, v, 1), d(x), d(w1), models=False)
        pre = acc + d(b1)
        return F.relu(pre), bnd + C_T * (d(b1).abs() + pre.abs())

    def check_sparse(self, op):
        vol, got = op["vol"], op["y"]
        w, _ = self.W["color.0"]
        d = lambda t: t.to(DEV).double()
        what = self.what("color.0", "backproject_conv_k2s2")
        models = {"input_shifted_one_channel": _conv(d(torch.roll(vol, 1, -1)), d(w), 2)}
        pv = self.prev_input("sparse", "color.0")
        if pv is not None and pv.shape == vol.shape:
            models["previous_scene_input"] = _conv(d(pv), d(w), 2)
        n = w.shape[1] + 8
        k, m = self.fmaf_conv("color.0", got, vol, w, None, None, 1, n, models, what)
        kp, _ = self.promise_conv("color.0", got, vol, w, None, None, 1, False, n)
        return k, m, kp

    def check_linear(self, op, fam):
        layer, x, got, act = op["name"], op["x"], op["y"], op["act"]
        chk, kmode, _ = ROUTE_CHECKS[fam]
        w, b = self.W[layer]
        d = lambda t: t.to(DEV).double()
        M, K = x.shape
        N = w.shape[0]
        s, kps = linear_splits(M, N, K)
        n = kps + s + 1 if s > 1 else K + 2
        lin = lambda a: d(a) @ d(w).T + d(b)
        models = {"bias_omitted": lambda ref: ref - d(b), "input_shifted_one_channel": lin(torch.roll(x, 1, -1))}
        px = self.prev_input("linear", layer)
        if px is not None and px.shape == x.shape:
            models["previous_scene_input"] = lin(px)
        what = self.what(layer, fam)

        def fmaf(models, what):
            acc, absum = d(x) @ d(w).T, d(x).abs() @ d(w).abs().T
            if models is None:
                return fmaf_chain_accuracy(got, acc, absum, n, d(b).expand_as(acc), act, what=what), math.inf
            full = {k: v(acc + d(b)) if callable(v) else v for k, v in models.items()}
            return fmaf_chain_accuracy(got, acc, absum, n, d(b).expand_as(acc), act, mutants=full, what=what)

        if chk == "linear":
            k, m = linear_accuracy(kmode, got, x, w, b, act, what, slice_=_energy_slice(x), extra=models)
        else:
            k, m = fmaf(models, what)
        p = PROMISE[self.mode]
        wp = self.what(layer, "promise of " + self.mode)
        kp = fmaf(None, wp)[0] if p == "fmaf" else linear_accuracy(p, got, x, w, b, act, wp, models=False)[0]
        return k, m, kp

    def check_twins(self, op):
        """Every fp16 twin next to an fp32 tensor is fp16 of it, bit for bit."""
        for a, h in (("x", "x16"), ("y", "y16")):
            if op.get(a) is not None and op.get(h) is not None:
                assert torch.equal(_bits(op[h]), _bits(op[a].half())), \
                    f"{self.row['id']} [{op.get('name')}]: the fp16 twin of the {'input' if a == 'x' else 'output'} is not fp16 of it"

    # -------------------------------------------------------------- the row
    def run(self):
        ops = self.cap.ops
        for name in self.cap.loose:
            fam = name.split("[")[0]
            assert fam in OUT_OF_SCOPE, f"{self.row['id']}: route {name} ran outside the hooked ops"
        for op in ops:
            self.check_twins(op)
            own = op["routes"]
            fams = [n.split("[")[0] for n in own]
            for n, f in zip(own, fams):
                assert f in ROUTE_CHECKS or f in OUT_OF_SCOPE, f"{self.row['id']}: route {n} has no check"
            if "cast_f16" in fams:
                assert op["kind"] == "conv" and op["x"] is not None and op["x16"] is not None
                self.checked.add("cast_f16")
            kind = op["kind"]
            res = None
            if kind == "conv":
                main = [n for n in own if n != "cast_f16"]
                assert len(main) == 1 and main[0].endswith(f"[{op['name']}]"), f"{self.row['id']}: [{op['name']}] ran {own}"
                fam = main[0].split("[")[0]
                res = (op["name"], fam, *self.check_conv(op, fam))
            elif kind == "bottleneck":
                res = self.block(op, own)
            elif kind == "linear":
                assert len(own) == 1 and own[0].endswith(f"[{op['name']}]"), f"{self.row['id']}: [{op['name']}] ran {own}"
                fam = own[0].split("[")[0]
                res = (op["name"], fam, *self.check_linear(op, fam))
            elif kind == "pool":
                assert own == ["maxpool3"], f"{self.row['id']}: pool ran {own}"
                ref = F.max_pool3d(op["x"].permute(3, 0, 1, 2)[None], 3, 1, 1)[0].permute(1, 2, 3, 0)
                assert torch.equal(_bits(op["y"]), _bits(ref.contiguous())), f"{self.row['id']}: maxpool3 is not bit exact"
                fam = "maxpool3"
            elif kind == "backproject":
                if "backproject_conv_k2s2" in own:
                    fam = "backproject_conv_k2s2"
                    res = ("color.0", fam, *self.check_sparse(op))
                else:
                    fam = None
                    assert "backproject_max" in own, f"{self.row['id']}: back-projection ran {own}"
            if kind in ("conv", "linear", "pool", "backproject") and fam:
                self.checked.add(fam)
            if res is not None:
                self.results.append(res)
        seen = {n.split("[")[0] for op in ops for n in op["routes"]} - set(OUT_OF_SCOPE)
        assert seen <= self.checked, f"{self.row['id']}: routes ran without a check: {sorted(seen - self.checked)}"
        self.wiring()
        return self.results

    def block(self, op, own):
        name = op["name"]
        kids = [o for o in self.cap.ops if o["parent"] == op["i"]]
        fams = [n.split("[")[0] for n in own]
        if fams == ["conv_tc_h3_split", "conv_tc_fused_h3_split"]:
            assert own == [f"conv_tc_h3_split[{name}.conv1]", f"conv_tc_fused_h3_split[{name}]"] and not kids, own
            self.checked.update(fams)
            return (name, fams[1], *self.check_block(op, fams[1], None))
        if len(fams) == 1 and fams[0] in ("conv_tc_fused", "conv_tc_fused_x3"):
            assert own == [f"{fams[0]}[{name}]"] and [k["name"] for k in kids] == [f"{name}.conv1"], (own, kids)
            c1 = kids[0]
            assert same_bits(c1["x"], op["x"]), f"{self.row['id']} [{name}.conv1]: input is not the block input"
            self.checked.add(fams[0])
            return (name, fams[0], *self.check_block(op, fams[0], c1))
        # three separate convs, each checked on its own: wire them
        assert not own and [k["name"] for k in kids] == [f"{name}.conv{i}" for i in (1, 2, 3)], (own, [k["name"] for k in kids])
        c1, c2, c3 = kids
        rid = self.row["id"]
        assert same_bits(c1["x"], op["x"]), f"{rid} [{name}.conv1]: input is not the block input"
        for a, b in ((c1, c2), (c2, c3)):
            assert self.follows(a, b), f"{rid} [{b['name']}]: input is not [{a['name']}]'s output"
        assert same_bits(c3["res"], op["x"]), f"{rid} [{name}.conv3]: residual is not the block input"
        assert same_bits(c3["y"], op["y"]), f"{rid} [{name}]: block output is not conv3's output"
        return None

    @staticmethod
    def follows(a, b):
        """b's captured input is a's captured output, fp32 and fp16 twin wherever both sides have one."""
        pairs = [(a["y"], b["x"]), (a["y16"], b["x16"])]
        both = [(p, q) for p, q in pairs if p is not None and q is not None]
        return bool(both) and all(same_bits(p, q) for p, q in both)

    def wiring(self):
        """Each op reads the output of the op before it in its program; the stacks start where they should."""
        rid, spec = self.row["id"], self.net.SPEC
        top = [o for o in self.cap.ops if o["parent"] is None]
        # the ops of each stack in the order they ran (branches are off); a pool carries no name and belongs to the stack
        # whose op ran before it
        seq, cur = {s: [] for s in ("color", "geometry1", "geometry2")}, None
        for o in top:
            if o["kind"] == "pool":
                seq[cur].append(o)
            elif o["kind"] in ("conv", "bottleneck") and o["name"].split(".")[0] in seq:
                cur = o["name"].split(".")[0]
                seq[cur].append(o)
        for stage, ops in seq.items():
            want = [op for op in spec.get(stage, ())]
            if stage == "color" and ops and self.row["sparse"] and self.images:
                want = want[1:]
            assert len(ops) == len(want), f"{rid}: {stage} ran {len(ops)} ops, its program has {len(want)}"
            for o, w in zip(ops, want):
                assert o["kind"] == {"k2s2": "conv", "k3": "conv", "bneck": "bottleneck", "pool": "pool"}[w[0]]
                if o["kind"] != "pool":
                    assert o["name"] == f"{stage}.{w[1]}", (o["name"], w)
            for a, b in zip(ops, ops[1:]):
                assert self.follows(a, b), f"{rid} [{b.get('name') or 'maxpool3'}]: input is not the previous op's output"
        bp = [o for o in top if o["kind"] == "backproject"]
        assert same_bits(seq["geometry1"][0]["x"], self.scene), f"{rid} [geometry1.0]: input is not the scene"
        if self.images:
            assert len(bp) == 1
            if self.row["sparse"]:
                assert self.follows(bp[0], seq["color"][0]), f"{rid} [{seq['color'][0]['name']}]: input is not colour.0's output"
            else:
                assert same_bits(seq["color"][0]["x"], bp[0]["y"]), f"{rid} [color.0]: input is not the back-projected volume"
        g2 = seq["geometry2"][0]
        level1 = g2["x"]
        if self.images:
            assert same_bits(level1[..., :64].contiguous(), seq["color"][-1]["y"]), f"{rid}: level1[..., :64] is not the colour output"
            assert same_bits(level1[..., 64:].contiguous(), seq["geometry1"][-1]["y"]), f"{rid}: level1[..., 64:] is not the geometry output"
        else:
            assert same_bits(level1, seq["geometry1"][-1]["y"]), f"{rid} [geometry2.0]: input is not level 1"
        level2 = seq["geometry2"][-1]["y"]
        rpn = {o["name"]: o for o in top if o["kind"] == "conv" and o["name"].startswith("rpn_")}
        for lvl, feat in ((1, level1), (2, level2)):
            hid, heads = rpn.get(f"rpn_net_level{lvl}"), rpn.get(f"rpn_heads_level{lvl}")
            if hid is None:
                continue
            assert same_bits(hid["x"], feat), f"{rid} [rpn_net_level{lvl}]: input is not level {lvl}"
            assert self.follows(hid, heads), f"{rid} [rpn_heads_level{lvl}]: input is not rpn_net_level{lvl}'s output"


# ------------------------------------------------------------------------------------------------ the test
def blobs_of(c, seed=None):
    seed = c["seed"] if seed is None else seed
    data, boxes = synth.make_scene(seed, c["dims"])
    views = synth.make_views(seed, c["dims"], c["n_img"], boxes) if c["use_images"] else None
    return synth.make_blobs(dict(cfgname=c["cfgname"], use_images=c["use_images"]), data, views)


def prev_inputs(cap):
    out = {}
    for o in cap.ops:
        if o["kind"] == "backproject" and "vol" in o:
            out[("sparse", "color.0")] = o["vol"]
        elif o["kind"] in ("conv", "bottleneck", "linear") and o.get("x") is not None:
            out[(o["kind"], o["name"])] = o["x"]
    return out


def static_tensors(cap):
    return [(o["kind"], o.get("name"), k, o[k]) for o in cap.ops for k in ("x", "x16", "res", "y", "y16", "vol")
            if o.get(k) is not None]


def assert_same_capture(a, b, what):
    ta, tb = static_tensors(a), static_tensors(b)
    assert [t[:3] for t in ta] == [t[:3] for t in tb], f"{what}: different op sequences"
    for p, q in zip(ta, tb):
        assert same_bits(p[3], q[3]), f"{what}: [{p[1]}] {p[2]} differs"


@pytest.mark.parametrize("scene", list(dict.fromkeys(r["scene"] for r in ROWS)))
def test_static_stage_layers_against_fp64(scene, record_property):
    c = SCENES[scene]
    rows = [r for r in ROWS if r["scene"] == scene]
    net, _ = synth.make_net(c, keep_debug=False, math="exact")
    blobs = blobs_of(c)
    scene_vc = blobs["data"][0].permute(1, 2, 3, 0).contiguous().to(DEV)
    prev_cap, _ = run_hooked(net, blobs_of(c, c["seed"] + 1))  # the previous scene: same shape, other content
    prev = prev_inputs(prev_cap)
    del prev_cap
    kept, summary = {}, {}
    for row in rows:
        if row["updated"] and not any(r["updated"] for r in rows[:rows.index(row)]):
            with torch.no_grad():
                sd = dict(net.named_parameters())
                for k, fn in UPDATES:
                    fn(sd[k])
        net.set_conv_math(row["mode"])
        net._sparse_color = row["sparse"]
        try:
            cap, got = run_hooked(net, blobs)
        finally:
            net._sparse_color = True
        chk = Row(row, net, cap, prev, c["use_images"], scene_vc)
        res = chk.run()
        worst = max(res, key=lambda t: t[2])
        weakest = min(res, key=lambda t: t[3])
        promise = max(res, key=lambda t: t[4])
        summary[row["id"]] = dict(kernel=worst[2], model=weakest[3], promise=promise[4])
        reached = set()
        for layer, fam, *_ in res:
            block = ROUTE_CHECKS[fam][0] in ("fused", "split_block")
            reached |= {f"{layer}.conv{i}" for i in (1, 2, 3)} if block else {layer}
        want = set(stage_layers(net.SPEC, c["use_images"], active_levels()))
        assert reached == want, f"{row['id']}: layers checked {sorted(reached ^ want)} differ from the program's"
        print(f"{row['id']}: worst kernel err/bound {worst[2]:.3g} ({worst[1]}[{worst[0]}]), smallest model ratio "
              f"{weakest[3]:.3g} ({weakest[1]}[{weakest[0]}]), worst promise err/bound {promise[4]:.3g} ({promise[0]})")
        # the hooked eager run gives the default forward's detections (CUDA graph on the second sight, parallel branches)
        if row["sparse"]:
            for attempt in range(2):
                P = net.forward(blobs, "TEST", None)
                torch.cuda.synchronize()
                d = _results(P)
                for k, v in got.items():
                    assert same_bits(v, d[k]), f"{row['id']}: {k} of the default forward (pass {attempt}) differs from the hooked run"
        # modes that share a static form, and the cycle back to exact, give identical bits
        for a, b in SAME_STATIC:
            if row["mode"] == b and a in kept:
                assert_same_capture(kept[a], cap, f"{row['id']} vs {a}")
        if row["mode"] == "exact" and "exact" in kept and row["sparse"] and not row["updated"]:
            assert_same_capture(kept["exact"], cap, f"{row['id']} vs the first exact pass")
        if row["mode"] in ("exact", "mixed") and row["mode"] not in kept:
            kept[row["mode"]] = cap
        record_property(row["id"], summary[row["id"]])
        del chk, cap
    record_property("rows", len(rows))
