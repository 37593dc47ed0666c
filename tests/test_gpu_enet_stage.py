"""The 2-D ENet encoder launch by launch on the GPU, against fp64 built from the reference's own (unfolded) parameters.

One encoder call is recorded through a proxy of libsis3d.so: after a sync around every sis3d_enet_* launch it keeps the
launch's arguments, its input, its residual and its output buffer before and after.  Each launch is then checked on its
own recorded input against an fp64 model of the reference's layer, built in the reference's order -- conv (+ bias) ->
eval BatchNorm (eps 1e-3) -> Dropout2d factor (1 - p) -> PReLU, and for a bottleneck's last conv CAdd with the zero-padded
(down-sampling: floor-mode 2x2/2 max-pooled) skip -> PReLU -- never from compile_enet's folded program, so a folding error
shows here.  Bounds:

  - sis3d_enet_conv2d: the fmaf chain of the kernel rows (enet_conv_accuracy), gamma_(K+2) (sum |x w'| + |epi|), plus the
    fp32 rounding of the fold: 6 u per folded weight (var + eps, sqrt, divide, times (1 - p), times w) and 9 u on the
    folded bias's two terms;
  - sis3d_enet_pool_affine: one fma (or a product and a sum) on the folded scale / shift, the same fold rounding;
  - sis3d_enet_to_nchw: bit-exact.

Every check also proves its power: the fp64 models of broken encoders in MODELS each miss the bound by POWER in every
launch they apply to.  Wiring: every launch reads the previous launch's output, writes only its channel slice (the
initial block: conv channels 0-12, pooled channels 13-15), adds the residual to channels < res_c only, and the launch
geometry and kernel instance are those encoder_launches() derives from the block structure and the launch rule of
sis3d_enet_conv2d.  Batch independence: each view of a batch equals, bit for bit, the same image encoded alone (every
kernel instance sums k = 0..K-1 in order).  fp64 is evaluated on views {0, 1, n-2, n-1} of each batch (consecutive pairs
for the off-by-one-view model); the others are tied to them by batch independence.

Rows: 256 x 328 at the view counts that straddle every half- / full-height M-tile switch of the launch rule (n = 1 .. 40),
the sizes whose pooled skip has an odd height or width at the first (250 x 328) or second (244 x 328, 256 x 324)
down-sampling bottleneck, the host-emulation shape 48 x 72, and the golden parameters; odd image sizes are refused before
any launch.  The last test runs a whole forward from raw images at IMAGE_SHAPE [328, 244] against the CPU oracle."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sis3d_synth as synth
from conftest import load_golden
from test_gpu_simt_accuracy import U, _check, enet_conv_accuracy, enet_inst
from test_gpu_tc_accuracy import POWER

pytestmark = pytest.mark.gpu
DEV = "cuda"
BN_EPS = 1e-3
FOLD_W = 6 * U      # relative rounding of a folded weight w * g / sqrt(var + eps) * (1 - p) computed in fp32
FOLD_B = 9 * U      # of each term of a folded bias (b - mean) * s + beta * (1 - p)

# The reference encoder (ENet's initial block and bottlenecks 1.0 .. 3.8 in eval mode), in its parameter order:
#   initial block: conv 3->13 k3 s2 p1 (w, b) || 2x2/2 max-pool of the image; concat -> BatchNorm(16) -> PReLU(16)
#   bottleneck (kind, mid, cout, p[, d]):
#     conv1: 1x1 (down: 2x2 stride 2), no bias -> BatchNorm -> PReLU
#     conv2: reg: 3x3 dilation d padding d (w, b) -> BatchNorm -> PReLU
#            asym: 1x5 padding (0, 2), no bias, no BatchNorm -> 5x1 padding (2, 0) (w, b) -> BatchNorm -> PReLU
#     conv3: 1x1 no bias -> BatchNorm -> Dropout2d (x (1 - p) at inference)
#     out = PReLU(conv3 + skip), skip = the block input (down: its 2x2/2 max-pool), channels zero-padded to cout
# BatchNorm parameters come as (weight, bias, running_mean, running_var).
_STAGE23 = [("reg", 1), ("reg", 2), ("asym", 5), ("reg", 4), ("reg", 1), ("reg", 8), ("asym", 5), ("reg", 16)]
BLOCKS = ([("down", 16, 64, 0.01, 1)] + [("reg", 16, 64, 0.01, 1)] * 4 + [("down", 32, 128, 0.1, 1)] +
          [(k, 32, 128, 0.1, d) for k, d in _STAGE23 * 2])

# what checks each op kind of compile_enet's program (tests/test_enet_stage_coverage.py keeps this complete)
CHECKS = {"conv": "enet_conv_accuracy on the launch's own input (fmaf chain + fold rounding)",
          "pool": "inside the initial block's pool_affine launch, and the pooled skip of the down-sampling conv3 epilogue",
          "affine_prelu": "pool_affine bound: one fma on the folded scale / shift",
          "cat": "channel-slice wiring: conv writes channels 0-12, pool_affine 13-15 of one tensor",
          "add_prelu": "the conv3 epilogue's residual (zero beyond res_c) and PReLU, in enet_conv_accuracy"}


def _odd_skip(r):
    return (r["H"] // 2) % 2 == 1 or (r["W"] // 2) % 2 == 1 or (r["H"] // 4) % 2 == 1 or (r["W"] // 4) % 2 == 1


# fp64 models of broken encoders -> the rows they apply to; each must miss the bound by POWER in every launch it applies to
MODELS = {
    "batchnorm_not_folded": lambda r: True,
    "dropout_factor_missing": lambda r: True,
    "pooled_skip_even_extent": _odd_skip,          # the skip addressed as [N][2Ho][2Wo] (the bug fixed with res_h / res_w)
    "pooled_skip_top_left": lambda r: True,
    "asym_taps_swapped": lambda r: True,           # the 1x5 and 5x1 taps exchanged
    "dilation_1": lambda r: True,
    "neighbour_slope": lambda r: True,             # the PReLU slope of the neighbouring layer
    "initial_halves_swapped": lambda r: True,      # pool channels first, conv channels after
    "previous_view": lambda r: r["n"] > 1,         # batch offset off by one image
}


def row(n, H, W, params="seeded", seed=0):
    return dict(id=f"{params}-n{n}-{H}x{W}", n=n, H=H, W=W, params=params, seed=seed)


ROWS = ([row(n, 256, 328, seed=n) for n in (1, 3, 4, 12, 13, 25, 26, 40)] +
        [row(2, 250, 328, seed=101), row(2, 244, 328, seed=102), row(2, 256, 324, seed=103), row(3, 48, 72, seed=104),
         row(2, 256, 328, params="golden", seed=105)])
REFUSED = [(255, 328), (256, 327)]


# ------------------------------------------------------------------------------------------------ structure
def _conv_out(h, w, k, stride, pad, dil):
    return (h + 2 * pad[0] - dil * (k[0] - 1) - 1) // stride + 1, (w + 2 * pad[1] - dil * (k[1] - 1) - 1) // stride + 1


def encoder_launches(n, H, W):
    """The sis3d_enet_conv2d launches of one encoder call, from the block structure: dicts of the geometry and the kernel
    instance the launch rule picks (enet_inst)."""
    out = []

    def conv(h, w, cin, cout, k, stride=1, pad=(0, 0), dil=1, nchw=False, res=None):
        ho, wo = _conv_out(h, w, k, stride, pad, dil)
        out.append(dict(N=n, H=h, W=w, cin=cin, cout=cout, kh=k[0], kw=k[1], stride=stride, pad=pad, dil=dil, Ho=ho, Wo=wo,
                        res=res, inst=enet_inst(n, ho, wo, cin, cout, nchw)))
        return ho, wo

    h, w = conv(H, W, 3, 13, (3, 3), 2, (1, 1), nchw=True)
    c = 16
    for kind, mid, cout, _, d in BLOCKS:
        down = kind == "down"
        hh, ww = conv(h, w, c, mid, (2, 2) if down else (1, 1), 2 if down else 1)
        if kind == "asym":
            conv(hh, ww, mid, mid, (1, 5), pad=(0, 2))
            conv(hh, ww, mid, mid, (5, 1), pad=(2, 0))
        else:
            conv(hh, ww, mid, mid, (3, 3), pad=(d, d), dil=d)
        conv(hh, ww, mid, cout, (1, 1), res=("pool" if down else "res", h, w, c))
        h, w, c = hh, ww, cout
    return out


def instances_reached(rows=ROWS):
    return {L["inst"] for r in rows for L in encoder_launches(r["n"], r["H"], r["W"])}


def _roles():
    """Role of every encoder parameter, in the reference's order."""
    bn = ["bn_g", "bn_b", "bn_mean", "bn_var"]
    roles = ["w", "b"] + bn + ["slope"]
    for kind, *_ in BLOCKS:
        roles += ["w"] + bn + ["slope"]
        roles += (["w", "w", "b"] if kind == "asym" else ["w", "b"]) + bn + ["slope"]
        roles += ["w"] + bn + ["slope"]
    return roles


def seeded_params(seed, like):
    """Parameters of the encoder's shapes with non-trivial BatchNorm statistics (mean != 0, var in [0.5, 2], gamma != 1)
    and PReLU slopes of both signs."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for role, t in zip(_roles(), like, strict=True):
        shp = t.shape
        u = lambda lo, hi: lo + (hi - lo) * torch.rand(shp, generator=g)
        if role == "w":
            out.append(torch.randn(shp, generator=g) * math.sqrt(2.0 / (t[0].numel())))
        elif role == "b":
            out.append(0.2 * torch.randn(shp, generator=g))
        elif role == "bn_g":
            out.append(u(0.6, 1.4) * torch.where(torch.rand(shp, generator=g) < 0.1, -1.0, 1.0))
        elif role == "bn_b":
            out.append(0.3 * torch.randn(shp, generator=g))
        elif role == "bn_mean":
            out.append(0.5 * torch.randn(shp, generator=g) + 0.1)
        elif role == "bn_var":
            out.append(u(0.5, 2.0))
        else:
            out.append(u(-0.5, 0.5))
    return out


def reference_layers(params):
    """The launches' fp64 layer models from the unfolded parameters, in launch order (the initial block is one entry)."""
    it = iter(p.to(DEV, torch.float64) for p in params)
    take = lambda k: [next(it) for _ in range(k)]
    w0, b0 = take(2)
    L = [dict(kind="init", w=w0, b=b0, bn=take(4), slope=next(it))]
    for kind, mid, cout, p, d in BLOCKS:
        down = kind == "down"
        L.append(dict(kind="conv1", w=next(it), b=None, bn=take(4), slope=next(it), stride=2 if down else 1, pad=(0, 0), dil=1))
        if kind == "asym":
            wa = next(it)
            L.append(dict(kind="asym_1x5", w=wa, b=None, bn=None, slope=None, stride=1, pad=(0, 2), dil=1))
            wb, bb = take(2)
            L.append(dict(kind="asym_5x1", w=wb, b=bb, bn=take(4), slope=next(it), stride=1, pad=(2, 0), dil=1))
        else:
            w2, b2 = take(2)
            L.append(dict(kind="conv2", w=w2, b=b2, bn=take(4), slope=next(it), stride=1, pad=(d, d), dil=d))
        L.append(dict(kind="conv3", w=next(it), b=None, bn=take(4), drop=1.0 - p, down=down, stride=1, pad=(0, 0), dil=1))
        L[-1]["slope"] = next(it)  # the CAdd's PReLU
    assert next(it, None) is None
    return L


# ------------------------------------------------------------------------------------------------ recording proxy
class _DevPtr:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<f4", "data": (int(ptr), False), "version": 3}


def _dev(ptr, n):
    """fp32 CUDA memory at a raw pointer as a (non-owning) tensor of n elements."""
    return torch.as_tensor(_DevPtr(ptr, n), device=DEV)


def _strided(ptr, shape, strides):
    span = 1 + sum((s - 1) * st for s, st in zip(shape, strides))
    return _dev(ptr, span).as_strided(shape, strides).clone()


class Recorder:
    """libsis3d.so's sis3d_enet_* entry points, forwarded after a sync that snapshots each launch."""

    def __init__(self, lib):
        self.lib, self.launches = lib, []

    def sis3d_enet_pack_weight(self, *a):
        return self.lib.sis3d_enet_pack_weight(*a)

    def sis3d_enet_conv2d(self, args, stream):
        from lib.nets.enet import _Conv
        a = C.cast(args, C.POINTER(_Conv)).contents
        f = {k: getattr(a, k) for k, _ in _Conv._fields_}
        torch.cuda.synchronize()
        rec = dict(op="conv", f=f, x=_strided(f["inp"], (a.N, a.H, a.W, a.cin), (a.in_sn, a.in_sy, a.in_sx, a.in_sc)),
                   out_ptr=f["out"], res_ptr=f["res"], in_ptr=f["inp"])
        nout = a.N * a.Ho * a.Wo * a.out_ld
        rec["before"] = _dev(a.out, nout).clone()
        if a.res:
            rec["res"] = _strided(a.res, (a.N, a.res_h, a.res_w, a.res_c), (a.res_h * a.res_w * a.res_ld, a.res_w * a.res_ld,
                                                                           a.res_ld, 1))
            rec["res_flat"] = _dev(a.res, a.N * a.res_h * a.res_w * a.res_ld).clone().view(-1, a.res_ld)[:, :a.res_c]
        rc = self.lib.sis3d_enet_conv2d(args, stream)
        torch.cuda.synchronize()
        rec["after"] = _dev(a.out, nout).clone()
        self.launches.append(rec)
        return rc

    def sis3d_enet_pool_affine(self, inp, sn, sy, sx, sc, N, H, W, Cn, scale, shift, slope, out, out_ld, out_coff, stream):
        torch.cuda.synchronize()
        nout = N * (H // 2) * (W // 2) * out_ld
        rec = dict(op="pool_affine", x=_strided(inp.value, (N, H, W, Cn), (sn, sy, sx, sc)), in_ptr=inp.value,
                   out_ptr=out.value, f=dict(N=N, H=H, W=W, C=Cn, out_ld=out_ld, out_coff=out_coff),
                   before=_dev(out.value, nout).clone())
        rc = self.lib.sis3d_enet_pool_affine(inp, sn, sy, sx, sc, N, H, W, Cn, scale, shift, slope, out, out_ld, out_coff,
                                             stream)
        torch.cuda.synchronize()
        rec["after"] = _dev(out.value, nout).clone()
        self.launches.append(rec)
        return rc

    def sis3d_enet_to_nchw(self, inp, ld, coff, N, P, Cn, out, stream):
        torch.cuda.synchronize()
        P_ = P.value
        rec = dict(op="to_nchw", x=_dev(inp.value, N * P_ * ld).clone().view(N, P_, ld)[..., coff:coff + Cn],
                   in_ptr=inp.value, f=dict(N=N, P=P_, C=Cn))
        rc = self.lib.sis3d_enet_to_nchw(inp, ld, coff, N, P, Cn, out, stream)
        torch.cuda.synchronize()
        rec["after"] = _dev(out.value, N * Cn * P_).clone()
        self.launches.append(rec)
        return rc


# ------------------------------------------------------------------------------------------------ fp64 models
def _bn(layer):
    """Per-channel scale and shift of BatchNorm (x Dropout factor) and the fold rounding of the bias, fp64."""
    cout = layer["w"].shape[0]
    zero = torch.zeros(cout, dtype=torch.float64, device=DEV)
    b = layer["b"] if layer["b"] is not None else zero
    if layer.get("bn") is None:
        return torch.ones_like(zero), b, zero
    g, beta, mean, var = layer["bn"]
    e = layer.get("drop", 1.0)
    s = g / torch.sqrt(var + BN_EPS) * e
    bias = (b - mean) * s + beta * e
    return s, bias, FOLD_B * ((b - mean).abs() * s.abs() + (beta * e).abs())


def _conv(x, w, layer, swap=False, dil=None):
    pad, d = layer["pad"], layer["dil"] if dil is None else dil
    if swap:
        w, pad = w.transpose(2, 3), pad[::-1]
    if dil is not None:
        pad = (d * (w.shape[2] // 2), d * (w.shape[3] // 2))
    return F.conv2d(x, w, stride=layer["stride"], padding=pad, dilation=d)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


class Stats:
    def __init__(self):
        self.k, self.models = 0.0, {}

    def add(self, k, m, names):
        self.k = max(self.k, k)
        for nm in names:
            self.models[nm] = min(self.models.get(nm, math.inf), m[nm] if isinstance(m, dict) else m)


def _check_named(got, ref, bound, models, what, stats):
    """_check per model, so that every model's smallest ratio is known (each must be >= POWER)."""
    k = 0.0
    mins = {}
    for nm, v in models.items():
        k, mins[nm] = _check(got, ref, bound, {nm: v}, 0, f"{what} [{nm}]")
    if not models:
        k, _ = _check(got, ref, bound, {}, 0, what)
    stats.add(k, mins, models)


def _conv_named(got, acc, absum, K, epi, slope, models, operand_err, what, stats):
    k = 0.0
    mins = {}
    for nm, v in models.items():
        k, mins[nm] = enet_conv_accuracy(got, acc, absum, K, epi, slope, {nm: v}, operand_err, f"{what} [{nm}]")
    if not models:
        k, _ = enet_conv_accuracy(got, acc, absum, K, epi, slope, None, operand_err, what)
    stats.add(k, mins, models)


def _prev(t, views):
    """Model of the off-by-one batch offset: view j takes view j - 1's values where both are checked."""
    out = t.clone()
    for i, j in enumerate(views):
        if i > 0 and views[i - 1] == j - 1:
            out[i] = t[i - 1]
    return out


def check_initial(pool_rec, layer, next_slope, views, r, stats):
    """Initial block: the 16-channel tensor after both launches, on the image."""
    img = pool_rec["x"][views].permute(0, 3, 1, 2).double()           # [v,3,H,W]
    x16 = pool_rec["after"].view(r["n"], r["H"] // 2, r["W"] // 2, 16)[views]
    g, beta, mean, var = layer["bn"]
    s = g / torch.sqrt(var + BN_EPS)
    sl = layer["slope"]
    # conv half, channels 0..12
    raw = _nhwc(F.conv2d(img, layer["w"], stride=2, padding=1))
    absum = _nhwc(F.conv2d(img.abs(), layer["w"].abs(), stride=2, padding=1)) * s[:13].abs()
    acc = raw * s[:13]
    bias = (layer["b"] - mean[:13]) * s[:13] + beta[:13]
    bias_err = FOLD_B * ((layer["b"] - mean[:13]).abs() * s[:13].abs() + beta[:13].abs())
    pooled = _nhwc(F.max_pool2d(img, 2))
    pool_pre = pooled * s[13:] + (beta[13:] - mean[13:] * s[13:])
    both = torch.cat((acc + bias, pool_pre), -1)
    swapped = torch.cat((both[..., 13:], both[..., :13]), -1)
    models = {"batchnorm_not_folded": raw + layer["b"], "neighbour_slope": (acc + bias, next_slope[:13]),
              "initial_halves_swapped": swapped[..., :13]}
    if len(views) > 1:
        models["previous_view"] = _prev(acc + bias, views)
    _conv_named(x16[..., :13], acc, absum, 27, bias, sl[:13], models, FOLD_W * absum + bias_err, f"{r['id']} initial conv",
                stats)
    # pool half, channels 13..15: fold rounding of scale / shift + one fma (or product and sum)
    ps = (pooled * s[13:]).abs()
    pre_bound = FOLD_W * (ps + (mean[13:] * s[13:]).abs()) + 2 * U * beta[13:].abs() + U * (ps + pool_pre.abs())
    pr = lambda v, q: torch.where(v >= 0, v, v * q)
    bound = pre_bound * sl[13:].abs().clamp(min=1.0) + U * pr(pool_pre, sl[13:]).abs()
    pm = {"batchnorm_not_folded": pr(pooled, sl[13:]), "neighbour_slope": pr(pool_pre, next_slope[13:16]),
          "initial_halves_swapped": pr(swapped[..., 13:], sl[13:])}
    if len(views) > 1:
        pm["previous_view"] = _prev(pr(pool_pre, sl[13:]), views)
    _check_named(x16[..., 13:], pr(pool_pre, sl[13:]), bound, pm, f"{r['id']} initial pool_affine", stats)


def check_conv(rec, layer, neighbour, views, r, stats, applied):
    f = rec["f"]
    x = rec["x"][views].permute(0, 3, 1, 2).double()
    w = layer["w"]
    cout = f["cout"]
    got = rec["after"].view(f["N"], f["Ho"], f["Wo"], f["out_ld"])[views][..., f["out_coff"]:f["out_coff"] + cout]
    s, bias, bias_err = _bn(layer)
    raw = _nhwc(_conv(x, w, layer))
    absum = _nhwc(_conv(x.abs(), w.abs(), layer)) * s.abs()
    acc = raw * s
    res = torch.zeros_like(acc)
    models = {}
    what = f"{r['id']} launch {layer['i']} ({layer['kind']}, {f['Ho']}x{f['Wo']}x{cout}, {rec['inst']})"
    if layer["kind"] == "conv3":
        rr = rec["res"][views].double()
        if layer["down"]:
            pool = lambda t: _nhwc(F.max_pool2d(t.permute(0, 3, 1, 2), 2))
            skip = pool(rr)
            Ho, Wo = f["Ho"], f["Wo"]
            models["pooled_skip_top_left"] = rr[:, :2 * Ho:2, :2 * Wo:2]
            if (f["res_h"], f["res_w"]) != (2 * Ho, 2 * Wo):  # image n at n * 4HoWo pixels, rows of 2Wo pixels
                flat = rec["res_flat"][:f["N"] * 4 * Ho * Wo].reshape(f["N"], 2 * Ho, 2 * Wo, f["res_c"])[views].double()
                models["pooled_skip_even_extent"] = pool(flat)
        else:
            skip = rr
        pad = lambda t: F.pad(t, (0, cout - t.shape[-1]))
        res = pad(skip)
        models = {k: acc + bias + pad(v) for k, v in models.items()}
        models["dropout_factor_missing"] = (acc + bias) / layer["drop"] + res
    epi = bias + res
    if layer["bn"] is not None:
        b = layer["b"] if layer["b"] is not None else 0.0
        models["batchnorm_not_folded"] = (raw + b) * layer.get("drop", 1.0) + res
    if layer["kind"].startswith("asym"):
        models["asym_taps_swapped"] = _nhwc(_conv(x, w, layer, swap=True)) * s + epi
    if layer["dil"] > 1:
        models["dilation_1"] = _nhwc(_conv(x, w, layer, dil=1)) * s + epi
    slope = layer["slope"]
    if slope is not None:
        models["neighbour_slope"] = (acc + epi, neighbour)
    if len(views) > 1:
        models["previous_view"] = _prev(acc + epi, views)
    K = f["kh"] * f["kw"] * f["cin"]
    _conv_named(got, acc, absum, K, epi, slope, models, FOLD_W * absum + bias_err, what, stats)
    applied.update(models)


# ------------------------------------------------------------------------------------------------ the rows
def _golden():
    g = load_golden("enet_encoder.npz")
    return g, [torch.from_numpy(g[k]) for k in sorted(k for k in g if k.startswith("p"))]


def _params(r):
    g, golden = _golden()
    return golden if r["params"] == "golden" else seeded_params(1000 + r["seed"], golden)


def _images(r):
    x = torch.randn(r["n"], 3, r["H"], r["W"], generator=torch.Generator().manual_seed(r["seed"]))
    if r["params"] == "golden":
        g, _ = _golden()
        x[0] = torch.from_numpy(np.random.default_rng(int(g["seed"])).standard_normal((3, 256, 328)).astype(np.float32))
    return x.to(DEV)


@pytest.fixture(scope="module")
def S():
    from lib import _sis3d
    return _sis3d


def _views(n):
    return sorted({0, 1, n - 2, n - 1} & set(range(n)))


@pytest.mark.parametrize("r", ROWS, ids=[r["id"] for r in ROWS])
def test_encoder_launch_by_launch_against_fp64(S, r, record_property):
    from lib.nets.enet import EnetEncoder
    params = _params(r)
    x = _images(r)
    rec = Recorder(S.lib)
    enc = EnetEncoder(params, DEV, lib=rec)
    rec.launches.clear()
    y = enc(x)
    torch.cuda.synchronize()
    n, views = r["n"], _views(r["n"])
    L = rec.launches
    plan = encoder_launches(n, r["H"], r["W"])
    assert [l["op"] for l in L] == ["conv", "pool_affine"] + ["conv"] * (len(plan) - 1) + ["to_nchw"]
    convs = [l for l in L if l["op"] == "conv"]
    for l, p in zip(convs, plan, strict=True):  # geometry and kernel instance of every launch
        f = l["f"]
        got = dict(N=f["N"], H=f["H"], W=f["W"], cin=f["cin"], cout=f["cout"], kh=f["kh"], kw=f["kw"], stride=f["stride"],
                   pad=(f["pad_y"], f["pad_x"]), dil=f["dil"], Ho=f["Ho"], Wo=f["Wo"])
        assert got == {k: p[k] for k in got}, (got, p)
        l["inst"] = p["inst"]
        if p["res"] is None:
            assert not f["res"]
        else:
            kind, rh, rw, rc = p["res"]
            assert (f["res_pool"], f["res_h"], f["res_w"], f["res_c"]) == (int(kind == "pool"), rh, rw, rc)

    # wiring: each launch reads the previous one's output and writes only its channel slice
    init_conv, pool = L[0], L[1]
    assert init_conv["in_ptr"] == pool["in_ptr"] == x.data_ptr() and init_conv["out_ptr"] == pool["out_ptr"]
    assert torch.equal(pool["x"], x.permute(0, 2, 3, 1))
    for l in (init_conv, pool):
        ld, coff, c = 16, l["f"]["out_coff"], l["f"]["cout"] if l["op"] == "conv" else l["f"]["C"]
        assert (coff, c) == ((0, 13) if l["op"] == "conv" else (13, 3))
        keep = torch.ones(ld, dtype=torch.bool, device=DEV)
        keep[coff:coff + c] = False
        a, b = l["before"].view(-1, ld), l["after"].view(-1, ld)
        assert torch.equal(a[:, keep].view(torch.int32), b[:, keep].view(torch.int32)), "written outside the channel slice"
    prev = pool["after"]
    block_in = prev
    for i, l in enumerate(L[2:], start=2):
        if l["op"] == "to_nchw":
            assert torch.equal(l["x"].reshape(-1), prev.view(-1, l["f"]["C"]).reshape(-1))
            nchw = prev.view(n, l["f"]["P"], l["f"]["C"]).transpose(1, 2).reshape(-1)
            assert torch.equal(l["after"].view(torch.int32), nchw.view(torch.int32))  # to_nchw: a bit-exact transpose
            break
        f = l["f"]
        assert torch.equal(l["x"].reshape(-1), prev.view(-1, f["cin"]).reshape(-1)), f"launch {i} does not read launch {i - 1}"
        if f["res"]:
            assert torch.equal(l["res_flat"].reshape(-1), block_in.view(-1, f["res_c"]).reshape(-1)), "skip is not the block input"
        prev = l["after"].view(-1, f["out_ld"])[:, f["out_coff"]:f["out_coff"] + f["cout"]]
        assert f["out_ld"] == f["cout"] and f["out_coff"] == 0
        if f["res"]:
            block_in = prev

    # fp64, launch by launch, on the launch's own recorded input
    layers = reference_layers(params)
    stats, applied = Stats(), set()
    slopes = [ly["slope"] for ly in layers if ly["slope"] is not None]

    def neighbour(ly):
        i = next(k for k, s in enumerate(slopes) if s is ly["slope"])
        o = slopes[i + 1] if i + 1 < len(slopes) else slopes[i - 1]
        c = ly["slope"].numel()
        return o[:c] if o.numel() >= c else o.repeat(-(-c // o.numel()))[:c]

    check_initial(pool, layers[0], slopes[1].repeat(2)[:16], views, r, stats)
    applied |= {"batchnorm_not_folded", "neighbour_slope", "initial_halves_swapped"} | ({"previous_view"} if n > 1 else set())
    for i, (l, ly) in enumerate(zip(convs[1:], layers[1:], strict=True), start=1):
        ly["i"] = i
        nb = neighbour(ly) if ly["slope"] is not None else None
        check_conv(l, ly, nb, views, r, stats, applied)
    want = {m for m, applies in MODELS.items() if applies(r)}
    assert applied == want, f"models applied {sorted(applied)} != expected {sorted(want)}"
    record_property("max_err_over_bound", stats.k)
    record_property("min_model_ratio", stats.models)
    print(f"\n{r['id']}: max err/bound {stats.k:.3g}; smallest model ratio " +
          ", ".join(f"{k} {v:.3g}" for k, v in sorted(stats.models.items())))
    assert min(stats.models.values()) >= POWER

    # batch independence: every view equals the same image encoded alone, bit for bit
    plain = EnetEncoder(params, DEV)
    y_batch = plain(x)
    assert torch.equal(y_batch.view(torch.int32), y.view(torch.int32))
    for j in range(n):
        assert torch.equal(plain(x[j:j + 1])[0].view(torch.int32), y_batch[j].view(torch.int32)), f"view {j} of {n}"


@pytest.mark.parametrize("hw", REFUSED, ids=[f"{h}x{w}" for h, w in REFUSED])
def test_encoder_refuses_odd_image_sizes_before_launching(S, hw):
    from lib.nets.enet import EnetEncoder
    enc = EnetEncoder(_golden()[1], DEV)
    x = torch.zeros((2, 3) + hw, device=DEV)
    torch.cuda.synchronize()
    n0 = S.launch_count()
    with pytest.raises(ValueError, match="even H and W"):
        enc(x)
    torch.cuda.synchronize()
    assert S.launch_count() == n0


# ------------------------------------------------------------------------------------------------ whole forward
class _Tap:
    """The network's encoder, keeping every output tensor it returns (the features the back-projection receives)."""

    def __init__(self, enc):
        self.enc, self.outs = enc, []

    def __call__(self, images):
        y = self.enc(images)
        self.outs.append(y)
        return y


def test_forward_from_raw_images_at_an_odd_quarter_size(oracle):
    """IMAGE_SHAPE [328, 244] (61 rows at the second down-sampling bottleneck), DEPTH_SHAPE [41, 30]: the whole TEST
    forward from raw images against the CPU oracle (integer outputs exact, masks within 1e-3), eager then CUDA-graph
    replay, with the features the back-projection receives equal bit for bit to the encoder's own output."""
    from lib.nets.enet import EnetEncoder
    from test_gpu_enet import _net_from_images
    c = synth.CASES["odd_45x27x41"]
    _, params = _golden()
    ocfg, w, data, views = synth.build_case(oracle, c)
    ocfg.DEPTH_SHAPE = [41, 30]
    views = dict(views, depths=np.ascontiguousarray(views["depths"][:, :30]))  # the same cameras, 30 rows
    images = np.random.default_rng(78).standard_normal((c["n_img"], 3, 244, 328)).astype(np.float32)
    with torch.no_grad():
        feats = oracle.enet_encoder(params, torch.from_numpy(images)).numpy()
    assert feats.shape == (c["n_img"], 128, 30, 41)
    want = oracle.forward(ocfg, w, data, dict(views, feats=feats), fma_mode=1)
    net, cfg = _net_from_images(c, params)
    saved = list(cfg.IMAGE_SHAPE), list(cfg.DEPTH_SHAPE)
    cfg.IMAGE_SHAPE, cfg.DEPTH_SHAPE = [328, 244], [41, 30]
    try:
        net._ensure_packed()  # builds the network's encoder
        tap = _Tap(net.__dict__["_enet"])
        net.__dict__["_enet"] = tap
        blobs = synth.make_blobs(c, data, dict(views, feats=images))
        own = EnetEncoder(params, DEV)(torch.from_numpy(images).to(DEV))
        torch.cuda.synchronize()

        def check(P):
            got, ref = P["rois"][0].cpu().numpy(), want["rois"].numpy()
            assert got.shape == ref.shape
            np.testing.assert_allclose(got, ref, atol=2e-3)
            assert np.array_equal(P["level_inds"][0].cpu().numpy(), want["level_inds"].numpy())
            assert np.array_equal(P["cls_pred"].cpu().numpy(), want["cls_pred"].numpy())
            det = P["detections_host"]
            assert np.array_equal(det[:, 8] > 0.5, want["mask_keep"])
            assert np.array_equal(det[:, 9:15].astype(np.int64), want["mask_crops"])
            assert len(P["mask_pred"][0]) == len(want["mask_pred"])
            for m, r in zip(P["mask_pred"][0], want["mask_pred"]):
                assert float((m.cpu() - r).abs().max()) < 1e-3
            torch.cuda.synchronize()
            assert torch.equal(tap.outs[-1].view(torch.int32), own.view(torch.int32))

        check(net.forward(blobs, "TEST", None))   # eager
        check(net.forward(blobs, "TEST", None))   # captured with the encoder inside the graph
        seen = len(tap.outs)
        tap.outs[-1].fill_(float("nan"))           # the graph's own feature buffer: only a replay refills it
        check(net.forward(blobs, "TEST", None))
        assert len(tap.outs) == seen, "the third forward did not replay the graph"
        with pytest.raises(synth_error()):
            bad = synth.make_blobs(c, data, dict(views, feats=np.zeros((c["n_img"], 3, 243, 328), np.float32)))
            net.forward(bad, "TEST", None)
    finally:
        cfg.IMAGE_SHAPE, cfg.DEPTH_SHAPE = saved


def synth_error():
    from lib import _sis3d
    return _sis3d.Sis3dError
