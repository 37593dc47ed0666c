"""Per-element accuracy of every tensor-core convolution and GEMM instance against fp64.

Every layer of the detection path runs on conv3d_k3_tc_kernel (3d-sis_b200/csrc/conv_tc.cu), one template instantiated
through launch_tc<BN, KS, EB, ROWB, BY, N2, X3, CL, PS> per math mode, kernel size, N tile, fused tail and cluster size.
Each row of the case table below names the instance it reaches (checked against the name of the kernel it launches;
tests/test_tc_instance_coverage.py keeps the table complete) and asserts, element by element,

    |got - ref| <= c * s2 + 2^-22 * (|bias| + |residual| + |ref|),        s2 = sqrt(sum_k (x_k w_k)^2)

with ref and s2 in fp64, c = 2^-15 for the error-compensated products (x3: TF32 split, h3: fp16 split) and 2^-7 for a single
TF32 / fp16 product.  A bound relative to s2 separates a correct compensated kernel from one that lost part of the
compensation (tests/test_split_product_model.py models both); a norm over the volume would hide a wrong edge brick.
Each case also proves the test's power: fp64 models of broken kernels on the same inputs must exceed the bound by 4x
somewhere -- the uncompensated product and the cross terms of one x-tap (of one 32-channel K slice for 1x1 convs and
GEMMs) dropped for the compensated modes, one 32-channel K slice of one tap dropped for the 1x modes.

Layout: outputs go to a NaN-filled tensor wider than cout (channel offset 4, guard voxels after the last row), residuals
come from a wider tensor (channel offset 8, NaN elsewhere); nothing outside the written slice may change.  Every launch
runs twice with identical bits, and one case per family is replayed from a CUDA graph."""
import ctypes as C
import math
import os
import re
import subprocess
import sys
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"

C_X3 = 2.0 ** -15     # compensated products: 22-bit operands, short fresh accumulation chains per pipeline stage
C_1X = 2.0 ** -7      # one TF32 (operands truncated to 11 bits by the tensor core) or fp16 (rounded) product
C_T = 2.0 ** -22      # fp32 roundings of the epilogue (bias, residual, output) relative to |bias| + |residual| + |ref|
C_FLOOR = 2.0 ** -34  # fp16 split of an operand below 2^-14 (subnormal hi): 2^-35 absolute (tests/test_split_product_model.py)
C_H = 2.0 ** -11      # rounding of an output stored as fp16 only, relative to |ref|
POWER = 4.0           # every broken-kernel model exceeds the bound by this factor somewhere in the case
COMPENSATED = ("x3", "h3", "h3s")
X3_OF = {"tf32": 0, "f16": 0, "x3": 1, "h3": 2, "h3s": 2}
EWORKSPACE = -3
GUARD = 3             # guard voxels (rows) after the last output row


@pytest.fixture(scope="module")
def S():
    from lib import _sis3d
    return _sis3d


# ------------------------------------------------------------------------------------------------ instances and case table
INST_DEFAULTS = (None, None, 4, 128, 2, 0, 0, 1, False)  # launch_tc<BN, KS, EB = 4, ROWB = 128, BY = 2, N2 = 0, X3 = 0, CL = 1, PS>


def inst(*args):
    """launch_tc<args...> with the template's defaults filled in: (BN, KS, EB, ROWB, BY, N2, X3, CL, PS)."""
    return tuple(args) + INST_DEFAULTS[len(args):]


def parse_inst(text):
    """'32, 3, 4, 128, 2, 0, 2, 1, false' (template arguments as written or demangled) -> instance tuple."""
    vals = [a.strip() for a in text.split(",") if a.strip()]
    return inst(*[a == "true" if a in ("true", "false") else int(a) for a in vals])


def reached(r):
    """The launch_tc<...> instance the C entry point dispatches row r to (conv_tc.cu)."""
    k, m, cl = r["kind"], r["mode"], r["cl"]
    if k == "linear":
        return inst(min(r["N"], 128), 0, *{"tf32": (), "x3": (4, 64, 2, 0, 1), "h3": (4, 128, 2, 0, 2)}[m])
    if k == "fused":
        cl = cl if m == "h3" and r["cmid"] == 64 else 1
        return inst(r["cmid"], 3, 4, 64 if m == "x3" else 128, 2, r["cout"], X3_OF[m], cl, m == "h3s")
    ks, cin, cout = r["ks"], r["cin"], r["cout"]
    by = 4 if r["tiles"] and ks == 3 and cout == 64 and cin % 64 == 0 else 2
    if m == "f16":
        wide = cin % 64 == 0
        return inst(min(cout, 128 if wide else 64), ks, 2, 128 if wide else 64, by, 0, 0, cl if by == 4 else 1)
    cl = cl if by == 4 or (m == "h3" and ks == 3 and cout >= 128) else 1
    return inst(min(cout, 128), ks, 4, 64 if m == "x3" else 128, by, 0, X3_OF[m], cl)


def _row(r):
    if r["mode"] not in COMPENSATED:
        r["w"] = "normal"  # weights below fp16's normal range are a property of the split; 1x fp16 operands would flush them
    r["inst"] = reached(r)
    r["id"] = "-".join(str(v) for v in (r["kind"], r["mode"], r["shape"], r["x"], "res" if r.get("res") else "",
                                        "tiny" if r["w"] == "tiny" else "", "act0" if r["act"] == 0 else "",
                                        "cl2" if r["cl"] == 2 else "") if v != "")
    return r


def conv(mode, ks, cin, cout, dims, *, res=False, act=1, bias=True, x="relu", w="normal", tiles=None, graph=False, cl=1):
    if tiles:  # crops packed along x on a zero canvas, one zero plane apart
        dims = (sum(s[0] + 1 for s in tiles), max(s[1] for s in tiles), max(s[2] for s in tiles))
    shape = f"k{ks}_{cin}to{cout}_{'x'.join(map(str, dims))}" + ("_tiles" if tiles else "")
    return _row(dict(kind="conv", mode=mode, ks=ks, cin=cin, cout=cout, dims=dims, res=res, act=act, bias=bias, x=x, w=w,
                     tiles=tiles, graph=graph, cl=cl, shape=shape))


def fused(mode, cin, cmid, cout, dims, *, res=True, act=1, x="relu", w="normal", graph=False, cl=1):
    shape = f"{cin}to{cmid}to{cout}_{'x'.join(map(str, dims))}"
    return _row(dict(kind="fused", mode=mode, cin=cin, cmid=cmid, cout=cout, dims=dims, res=res, act=act, x=x, w=w, graph=graph,
                     cl=cl, shape=shape))


def linear(mode, M, K, N, *, act=1, x="relu", w="normal", graph=False):
    return _row(dict(kind="linear", mode=mode, M=M, K=K, N=N, act=act, x=x, w=w, graph=graph, cl=1, shape=f"{M}x{K}to{N}"))


# ks, cin, cout, dims, options: every ks x cout in {32, 64, 128, 256} (256 = two N blocks); partial bricks on every axis
# (17x9x11, 45x27x41), one-voxel volumes, 2x2x2 / 3x5x7 (ks = 2, floor), a thin 70x3x3 volume, many bricks per SM (96x48x96),
# cin = 96 (an odd number of 32-channel slices)
CONV_SHAPES = [
    (3, 32, 32, (96, 48, 96), dict(graph=True)), (3, 64, 64, (17, 9, 11), dict(res=True, x="wide")),
    (3, 32, 128, (9, 5, 7), dict(x="signed", act=0)), (3, 128, 256, (6, 5, 7), dict(res=True, w="tiny")),
    (3, 96, 32, (45, 27, 41), dict(x="wide")), (3, 32, 64, (1, 1, 1), dict(res=True)),
    (3, 64, 32, (70, 3, 3), dict(w="tiny", bias=False)),
    (2, 64, 32, (45, 27, 41), dict(x="wide")), (2, 96, 64, (17, 9, 11), dict(res=True)),
    (2, 32, 128, (3, 5, 7), dict(x="signed", act=0)), (2, 64, 256, (2, 2, 2), dict(w="tiny")),
    (1, 32, 32, (70, 3, 3), {}), (1, 64, 64, (96, 48, 96), dict(x="wide")), (1, 96, 128, (1, 1, 1), dict(res=True)),
    (1, 256, 256, (8, 6, 5), dict(x="signed", res=True, w="tiny")), (1, 32, 64, (17, 9, 11), dict(x="wide", w="tiny")),
]
# fp16-operand kernel: cin = 32 (64-byte rows, N tiles of at most 64: 32 -> 128 at ks = 3 runs two 64-wide N blocks) and
# cin % 64 == 0 (128-byte rows)
F16_SHAPES = [
    (3, 32, 32, (17, 9, 11), dict(graph=True)), (3, 32, 64, (45, 27, 41), dict(x="wide", res=True)), (3, 32, 128, (9, 5, 7), {}),
    (1, 32, 32, (70, 3, 3), {}), (1, 32, 256, (8, 6, 5), dict(res=True, x="signed", act=0)),
    (3, 64, 32, (17, 9, 11), dict(x="signed")), (3, 64, 64, (45, 27, 41), dict(res=True)), (3, 128, 256, (6, 5, 7), dict(x="wide")),
    (3, 64, 128, (1, 1, 1), {}), (1, 64, 32, (96, 48, 96), {}), (1, 128, 64, (1, 1, 1), dict(res=True)),
    (1, 256, 128, (9, 4, 7), dict(res=True, act=0)),
]
CROPS = ((10, 7, 5), (6, 9, 12), (3, 3, 3))  # 4x4x8 bricks: 6 + 12 + 1 = 19, an odd count (the cluster's padding CTA)
FUSED_SHAPES = [  # cin, cmid, cout, dims: the three (cmid, cout) tails
    (32, 32, 32, (17, 9, 11), dict(res=False, graph=True)), (64, 32, 64, (45, 27, 41), dict(x="wide")),
    (64, 64, 128, (9, 5, 7), dict(w="tiny")), (96, 32, 32, (8, 2, 8), {}), (32, 64, 128, (70, 3, 3), dict(x="signed")),
]
LINEAR_SHAPES = [  # M, K, N: K = 1056 leaves an uneven last split-K chunk.  A fault in one of K / 32 slices is visible at
    # K = 8192 only where heavy-tailed ("wide") activations put much of a row's weight into the slice
    (1, 256, 32, dict(graph=True)), (7, 1056, 64, dict(x="signed")), (65, 1056, 128, dict(x="signed", act=0)),
    (200, 8192, 256, dict(x="wide", w="tiny")), (64, 2048, 128, {}), (200, 1056, 32, dict(x="wide")), (65, 8192, 64, dict(x="wide")),
]

ROWS = (
    [conv(m, ks, ci, co, d, **o) for m in ("h3", "x3", "tf32") for ks, ci, co, d, o in CONV_SHAPES]
    + [conv("f16", ks, ci, co, d, **o) for ks, ci, co, d, o in F16_SHAPES]
    + [conv("tf32", 3, 64, 64, None, tiles=CROPS, res=True, graph=True), conv("f16", 3, 64, 64, None, tiles=CROPS, x="wide"),
       conv("tf32", 3, 32, 32, None, tiles=CROPS), conv("f16", 3, 32, 64, None, tiles=CROPS, res=True)]
    + [fused(m, ci, cm, co, d, **o) for m in ("h3", "h3s", "x3", "tf32") for ci, cm, co, d, o in FUSED_SHAPES]
    + [fused("h3", 32, 32, 64, (96, 48, 96)), fused("h3s", 32, 32, 64, (96, 48, 96), x="wide")]
    + [linear(m, M, K, N, **o) for m in ("h3", "x3", "tf32") for M, K, N, o in LINEAR_SHAPES]
)
# 2-CTA clusters (SIS3D_CLUSTER=1), odd brick counts: 17x5x8 = 9 bricks of 8x2x8, CROPS = 19 bricks of 4x4x8
CLUSTER_ROWS = [conv("h3", 3, 128, 128, (17, 5, 8), x="wide", res=True, cl=2), conv("tf32", 3, 64, 64, None, tiles=CROPS, cl=2),
                fused("h3", 64, 64, 128, (17, 5, 8), cl=2), conv("f16", 3, 64, 64, None, tiles=CROPS, res=True, cl=2)]


# ------------------------------------------------------------------------------------------------ fp64 reference and bound
def tf32_rna(v):
    """fp32 -> nearest TF32 value, ties away from zero (cvt.rna.tf32.f32)."""
    return ((v.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def hi_part(v, mode):
    """fp64 value of the hi part of the operand split of `mode` (x3: tf32(v); h3: fp16(v))."""
    v = v.float()
    return (tf32_rna(v) if mode == "x3" else v.clamp(-65504, 65504).half().float()).double()


def _conv(x, w, ks):
    """VC [X][Y][Z][cin] x [cout][cin][k][k][k] -> VC, as the kernel: pad 1 (ks 3), stride 2 (ks 2)."""
    y = F.conv3d(x.permute(3, 0, 1, 2)[None], w, stride=2 if ks == 2 else 1, padding=1 if ks == 3 else 0)
    return y[0].permute(1, 2, 3, 0)


def _gemm(x, w):
    return x @ w.T


def _drop_mask(mode, w, slice_=None):
    """Weights whose products a broken-kernel model loses: the centre x-tap (compensated, ks 3 / 2; every output voxel has
    it), else one 32-channel K slice (of the centre tap for the 1x modes): slice `slice_` when given, else the last.  Real
    activations can leave a slice all zero (dead ReLU channels); their callers pick the slice with the most input energy."""
    m = torch.zeros_like(w)
    ks = slice(-32, None) if slice_ is None else slice(32 * slice_, 32 * slice_ + 32)
    if w.dim() == 2 or w.shape[2] == 1:
        m[:, ks] = 1
    elif mode in COMPENSATED:
        m[:, :, w.shape[2] // 2] = 1
    else:
        c = w.shape[2] // 2
        m[:, ks, c, c, c] = 1
    return m


def _product(mode, lin, x, w, slice_=None, models=True):
    """fp64 accumulator of the linear operator lin(x, w), its error bound c * s2 (+ the subnormal floor of the fp16 split),
    and the accumulators of the broken-kernel models (none when models is False; slice_: see _drop_mask)."""
    acc = lin(x, w)
    bound = (C_X3 if mode in COMPENSATED else C_1X) * lin(x * x, w * w).sqrt()
    if mode in ("h3", "h3s"):
        small = lambda v: (v.abs() < 2.0 ** -14).double()
        bound = bound + C_FLOOR * (lin(x.abs(), small(w)) + lin(small(x), w.abs()))
    if not models:
        return acc, bound, {}
    m = _drop_mask(mode, w, slice_)
    if mode in COMPENSATED:
        xh, wh = hi_part(x, mode), hi_part(w, mode)
        mutants = {"uncompensated": lin(xh, wh), "one_tap_no_cross": acc - lin(x, w * m) + lin(xh, wh * m)}
    else:
        mutants = {"one_slice_dropped": acc - lin(x, w * m)}
    return acc, bound, mutants


def _check(got, ref, bound, mutants, act, what):
    """Assert |got - ref| <= bound everywhere and that every broken-kernel model exceeds it by POWER somewhere.
    Returns (kernel's max err / bound, smallest model max err / bound; inf without models)."""
    f = F.relu if act == 1 else (lambda v: v)
    ref = f(ref)

    def ratio(v):
        e = (v - ref).abs()
        return torch.where(e == 0, torch.zeros_like(e), e / bound).max().item()  # e > 0 where bound = 0: inf

    k = ratio(got.double())
    m = {name: ratio(f(v)) for name, v in mutants.items()}
    msg = f"{what}: kernel max err/bound {k:.3g}; broken-kernel models " + ", ".join(f"{n} {v:.3g}" for n, v in m.items())
    assert k <= 1.0, msg
    assert not m or min(m.values()) >= POWER, "bound too loose to reject a broken kernel: " + msg
    return k, min(m.values(), default=math.inf)


def _models(extra, ref):
    """Extra fp64 models of a caller (name -> pre-activation output, or a function of the pre-activation reference)."""
    return {k: v(ref) if callable(v) else v for k, v in (extra or {}).items()}


def _d(t):
    return None if t is None else t.to(DEV).double()


def conv_accuracy(mode, got, x, w, b=None, r=None, act=1, where=None, what="conv", slice_=None, models=True, extra=None,
                  out16=False):
    """got: VC output [Xo][Yo][Zo][cout] of the conv of VC x [X][Y][Z][cin] with w [cout][cin][k][k][k] (+ b, + r, ReLU if
    act == 1) in math mode `mode`; where: optional bool [Xo][Yo][Zo] of the voxels to compare.  models: whether the
    broken-kernel models must miss the bound; extra: further models (_models); out16: got was stored as fp16 (adds its
    rounding, 2^-11 |ref|, and 2^-25 below fp16's normal range)."""
    ks = w.shape[2]
    acc, bound, mut = _product(mode, lambda a, v: _conv(a, v, ks), _d(x), _d(w), slice_, models)
    epi = torch.zeros_like(acc)
    if b is not None:
        epi = epi + _d(b)
    if r is not None:
        epi = epi + _d(r)
    ref = acc + epi
    bound = bound + C_T * ((_d(b).abs() if b is not None else 0) + (_d(r).abs() if r is not None else 0) + ref.abs())
    if out16:
        bound = bound + C_H * ref.abs() + 2.0 ** -25
    mut = {k: v + epi for k, v in mut.items()}
    mut.update(_models(extra, ref))
    got = got.to(DEV)
    if where is not None:
        where = where.to(DEV)
        got, ref, bound, mut = got[where], ref[where], bound[where], {k: v[where] for k, v in mut.items()}
    return _check(got, ref, bound, mut, act, what)


def fused_accuracy(mode, got, x, w2, b2, w3, b3, r=None, act=1, what="fused", bound_in=None, slice_=None, models=True,
                   extra=None):
    """conv2 (3x3x3, + b2) -> ReLU -> conv3 (1x1, + b3) -> + r -> act; conv2's bound propagates through |w3|.  bound_in:
    optional per-element error bound of x itself (a conv1 output the kernel computed), carried through w2 in quadrature."""
    lin3, lin1 = (lambda a, v: _conv(a, v, 3)), (lambda a, v: _conv(a, v, 1))
    acc2, bound2, mut2 = _product(mode, lin3, _d(x), _d(w2), slice_, models)
    if bound_in is not None:
        bound2 = bound2 + lin3(_d(bound_in) ** 2, _d(w2) ** 2).sqrt()
    b2, w3, b3 = _d(b2), _d(w3), _d(b3)
    y_pre = acc2 + b2
    y = F.relu(y_pre)
    if mode in ("h3", "h3s"):
        assert y.abs().max().item() < 65504, "inputs violate the fp16 split's range precondition"
    bound_y = bound2 + C_T * (b2.abs() + y_pre.abs())
    acc3, bound3, _ = _product(mode, lin1, y, w3, models=False)
    epi = b3 + (_d(r) if r is not None else 0)
    ref = acc3 + epi
    # the cmid channels' errors are independent roundings, so they add in quadrature through w3 like the products in s2; a sum
    # of |w3| bound_y is sqrt(cmid) looser and cannot reject a tail whose 3x3x3 conv lost its compensation
    bound = bound3 + lin1(bound_y ** 2, w3 ** 2).sqrt() + C_T * (b3.abs() + (_d(r).abs() if r is not None else 0) + ref.abs())
    mut = {k: lin1(F.relu(v + b2), w3) + epi for k, v in mut2.items()}
    mut.update(_models(extra, ref))
    return _check(got.to(DEV), ref, bound, mut, act, what)


def linear_accuracy(mode, got, x, w, b=None, act=1, what="linear", slice_=None, models=True, extra=None):
    """got [M][N] = act(x [M][K] . w [N][K]^T + b)."""
    acc, bound, mut = _product(mode, _gemm, _d(x), _d(w), slice_, models)
    epi = _d(b) if b is not None else torch.zeros_like(acc)
    ref = acc + epi
    bound = bound + C_T * (epi.abs() + ref.abs())
    mut = {k: v + epi for k, v in mut.items()}
    mut.update(_models(extra, ref))
    return _check(got.to(DEV), ref, bound, mut, act, what)


# ------------------------------------------------------------------------------------------------ inputs and launches
def _act(g, shape, kind):
    if kind == "relu":
        return F.relu(torch.randn(shape, generator=g))
    if kind == "signed":
        return torch.randn(shape, generator=g)
    # "wide": magnitudes log-uniform over 2^-10 .. 2^14, some at 6e4 (below the fp16 split's 65504), random signs, half zeros
    mag = torch.exp2(torch.rand(shape, generator=g) * 24 - 10)
    mag = torch.where(torch.rand(shape, generator=g) < 2e-3, torch.full(shape, 6.0e4), mag)
    sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return torch.where(torch.rand(shape, generator=g) < 0.5, torch.zeros(shape), mag * sign)


def _scale(kind):
    return 2.0 ** -12 if kind == "tiny" else 1.0  # tiny weights: fp16-subnormal hi parts; the layer's biases and residuals shrink too


def _weight(g, shape, kind):
    return torch.randn(shape, generator=g) / math.sqrt(math.prod(shape[1:])) * _scale(kind)


def split_pairs(v):
    """fp32 [..., C] -> split-pair fp16 [..., 2 C]: per 32-channel slice 32 hi = fp16(v), then 32 lo = fp16((v - hi) * 2048)."""
    hi = v.half()
    lo = ((v - hi.float()) * 2048.0).half()
    sh = v.shape[:-1] + (v.shape[-1] // 32, 32)
    return torch.stack([hi.reshape(sh), lo.reshape(sh)], -2).reshape(v.shape[:-1] + (2 * v.shape[-1],))


def pack(S, mode, w):
    """w [cout][cin][k][k][k] (a [N][K] weight as [N][K][1][1][1]) -> the layout of `mode`."""
    cout, cin, ks = w.shape[:3]
    K = ks ** 3 * cin
    fn, rows, dt = {"tf32": ("sis3d_pack_conv_weight_tc", 1, torch.float32), "x3": ("sis3d_pack_conv_weight_tc_x3", 2, torch.float32),
                    "f16": ("sis3d_pack_conv_weight_tc_f16", 1, torch.float16), "h3": ("sis3d_pack_conv_weight_tc_h3", 2, torch.float16),
                    "h3s": ("sis3d_pack_conv_weight_tc_h3", 2, torch.float16)}[mode]
    out = torch.empty(rows * cout, K, dtype=dt, device=DEV)
    S.check(getattr(S.lib, fn)(S.ptr(w.contiguous()), cout, cin, ks, S.ptr(out), S.stream()))
    return out


def _tile_list(S, row):
    """Canvas voxels of the crops, and the brick list covering them (sis3d_conv3d_tc_brick)."""
    X, Y, Z = row["dims"]
    bx, by, bz = C.c_int32(), C.c_int32(), C.c_int32()
    S.lib.sis3d_conv3d_tc_brick(1, 3, row["cin"], row["cout"], C.byref(bx), C.byref(by), C.byref(bz))
    mask = torch.zeros(X, Y, Z, dtype=torch.bool)
    tiles, x0 = [], 0
    for s in row["tiles"]:
        mask[x0:x0 + s[0], :s[1], :s[2]] = True
        for i in range(0, s[0], bx.value):
            for j in range(0, s[1], by.value):
                for k in range(0, s[2], bz.value):
                    tiles.append([x0 + i, j, k, x0 + s[0], s[1], s[2], 0, 0])
        x0 += s[0] + 1
    return mask, torch.tensor(tiles, dtype=torch.int32, device=DEV)


class Case:
    """One row on the device: seeded inputs, packed weights, launch() into a fresh NaN-filled output, and the checks."""

    def __init__(self, S, row):
        self.S, self.row = S, row
        g = torch.Generator().manual_seed(zlib.crc32(row["id"].encode()))
        k = row["kind"]
        if k == "linear":
            M, K, N = row["M"], row["K"], row["N"]
            self.x, self.w = _act(g, (M, K), row["x"]), _weight(g, (N, K), row["w"])
            self.b = torch.randn(N, generator=g) * _scale(row["w"])
            self.r, self.written_mask = None, None
            self.ld, self.coff, self.rows, self.cout, self.odims = N, 0, M, N, (M,)
        else:
            X, Y, Z = row["dims"]
            cin, cout = row["cin"], row["cout"]
            ks = row.get("ks", 3)
            self.x = _act(g, (X, Y, Z, cin), row["x"])
            self.where = None
            if row.get("tiles"):
                self.where, self.tiles = _tile_list(S, row)
                self.x = self.x * self.where[..., None]  # zero canvas around the crops
            if k == "conv":
                self.w = _weight(g, (cout, cin, ks, ks, ks), row["w"])
                self.b = torch.randn(cout, generator=g) * _scale(row["w"]) if row["bias"] else None
            else:
                cmid = row["cmid"]
                self.w2, self.b2 = _weight(g, (cmid, cin, 3, 3, 3), row["w"]), torch.randn(cmid, generator=g) * _scale(row["w"])
                self.w3, self.b3 = _weight(g, (cout, cmid, 1, 1, 1), "normal"), torch.randn(cout, generator=g) * _scale(row["w"])
            self.odims = tuple(d // 2 for d in row["dims"]) if ks == 2 else row["dims"]
            self.r = torch.randn(self.odims + (cout,), generator=g) * _scale(row["w"]) if row["res"] else None
            self.ld, self.coff, self.rows, self.cout = cout + 8, 4, math.prod(self.odims), cout
        # what the launch may write: the output slice of every written voxel
        self.written_mask = torch.zeros(self.rows + GUARD, self.ld, dtype=torch.bool, device=DEV)
        vox = slice(None) if getattr(self, "where", None) is None else self.where.reshape(-1).to(DEV)
        self.written_mask[:self.rows][vox, self.coff:self.coff + self.cout] = True
        self._device_operands()

    def _device_operands(self):
        S, row, m = self.S, self.row, self.row["mode"]
        d = lambda t: None if t is None else t.to(DEV).contiguous()
        self.xd, self.bd = d(self.x), d(getattr(self, "b", None))
        if row["kind"] == "linear":
            self.wd = d(self.w) if m == "tf32" else pack(S, m, d(self.w).view(row["N"], row["K"], 1, 1, 1))
            self.nbytes = int(S.lib.sis3d_linear_tc_workspace_bytes(row["M"], row["N"], row["K"]))
            self.ws = torch.empty(self.nbytes, dtype=torch.uint8, device=DEV)
            return
        if row["kind"] == "conv":
            self.wd = pack(S, m, d(self.w))
        else:
            self.w2d, self.w3d = pack(S, m, d(self.w2)), pack(S, m, d(self.w3))
            self.b2d, self.b3d = d(self.b2), d(self.b3)
        if m == "f16":
            self.xd = self.xd.half()
        elif m == "h3s":
            self.xd = split_pairs(self.xd).contiguous()
        self.res_ld, self.res_coff, self.rbuf = 0, 0, None
        if self.r is not None:  # residual from a wider tensor, NaN outside its slice
            self.res_ld, self.res_coff = self.cout + 12, 8
            self.rbuf = torch.full((self.rows, self.res_ld), float("nan"), device=DEV)
            self.rbuf[:, 8:8 + self.cout] = self.r.to(DEV).reshape(self.rows, self.cout)

    def new_out(self):
        return torch.full((self.rows + GUARD, self.ld), float("nan"), device=DEV)

    def launch(self, out):
        S, L, row, m = self.S, self.S.lib, self.row, self.row["mode"]
        P, st = S.ptr, S.stream()
        if row["kind"] == "linear":
            fn = {"tf32": L.sis3d_linear_tc, "x3": L.sis3d_linear_tc_x3, "h3": L.sis3d_linear_tc_h3}[m]
            S.check(fn(P(self.xd), P(self.wd), P(self.bd), P(out), row["M"], row["K"], row["N"], row["act"], P(self.ws),
                       C.c_size_t(self.nbytes), st))
            return
        X, Y, Z = row["dims"]
        res = (P(self.rbuf), self.res_ld, self.res_coff)
        dst = (P(out), self.ld, self.coff, X, Y, Z)
        if row["kind"] == "fused":
            fn = {"tf32": L.sis3d_conv3d_k3_tc_fused, "x3": L.sis3d_conv3d_k3_tc_fused_x3, "h3": L.sis3d_conv3d_k3_tc_fused_h3,
                  "h3s": L.sis3d_conv3d_k3_tc_fused_h3_split}[m]
            S.check(fn(P(self.xd), P(self.w2d), P(self.b2d), P(self.w3d), P(self.b3d), *res, *dst, row["cin"], row["cmid"],
                       row["cout"], row["act"], st))
            return
        shape = (row["cin"], row["cout"], row["ks"])
        tiles = (P(self.tiles), len(self.tiles)) if row["tiles"] else (None, 0)
        if m == "tf32":
            S.check(L.sis3d_conv3d_k3_tc(P(self.xd), P(self.wd), P(self.bd), *res, *dst, *shape, *tiles, row["act"], st))
        elif m == "f16":
            S.check(L.sis3d_conv3d_tc_f16(P(self.xd), P(self.wd), P(self.bd), *res, P(out), None, *dst[1:], *shape, *tiles,
                                          row["act"], st))
        else:
            fn = L.sis3d_conv3d_k3_tc_x3 if m == "x3" else L.sis3d_conv3d_k3_tc_h3
            S.check(fn(P(self.xd), P(self.wd), P(self.bd), *res, *dst, *shape, row["act"], st))

    def written(self, out):
        return out[:self.rows, self.coff:self.coff + self.cout].reshape(self.odims + (self.cout,))

    def check_untouched(self, out):
        assert bool(torch.isnan(out[~self.written_mask]).all()), f"{self.row['id']}: wrote outside its output slice"
        assert bool(torch.isfinite(out[self.written_mask]).all()), f"{self.row['id']}: output voxels left unwritten"

    def accuracy(self, out):
        row, got, what = self.row, self.written(out), self.row["id"]
        if row["kind"] == "linear":
            return linear_accuracy(row["mode"], got, self.x, self.w, self.b, row["act"], what)
        if row["kind"] == "fused":
            return fused_accuracy(row["mode"], got, self.x, self.w2, self.b2, self.w3, self.b3, self.r, row["act"], what)
        return conv_accuracy(row["mode"], got, self.x, self.w, self.b, self.r, row["act"], self.where, what)


def launched_instances(fn, attempts=3):
    """Run fn under the profiler; the conv3d_k3_tc_kernel instances it launched, from the kernel names.  Now and then the
    profiler returns no device events for a region; fn (a deterministic launch) then runs again under a fresh profiler, and
    after `attempts` empty sessions the result is None (nothing to compare)."""
    for _ in range(attempts):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        found = []
        for e in prof.events():
            m = re.search(r"conv3d_k3_tc_kernel<([^>]*)>", e.name)
            if m:
                found.append(parse_inst(m.group(1)))
                continue
            m = re.search(r"conv3d_k3_tc_kernelI((?:L[ib]\d+E)+)E", e.name)  # mangled: Li32E ... Lb0E
            if m:
                v = [int(a) for a in re.findall(r"L[ib](\d+)E", m.group(1))]
                found.append(inst(*v[:-1], bool(v[-1])))
        if found:
            return found
    return None


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.parametrize("row", ROWS, ids=[r["id"] for r in ROWS])
def test_tc_instance_accuracy(S, row, record_property):
    case = Case(S, row)
    a, b = case.new_out(), case.new_out()
    case.launch(a)
    found = launched_instances(lambda: case.launch(b))
    assert found in (None, [row["inst"]]), f"the row does not reach the instance it names: launched {found}"
    record_property("kernel_name_checked", found is not None)
    torch.cuda.synchronize()
    assert torch.equal(_bits(a), _bits(b)), "two launches on the same inputs differ"
    case.check_untouched(a)
    if row["graph"]:  # the production path (SIS3D_CUDA_GRAPH=1) replays captured launches
        gout = case.new_out()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            case.launch(gout)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(gout), _bits(a)), "CUDA-graph replay differs from the eager launch"
    if row["kind"] == "linear":
        rc = {"tf32": S.lib.sis3d_linear_tc, "x3": S.lib.sis3d_linear_tc_x3, "h3": S.lib.sis3d_linear_tc_h3}[row["mode"]](
            S.ptr(case.xd), S.ptr(case.wd), S.ptr(case.bd), S.ptr(a), row["M"], row["K"], row["N"], row["act"], S.ptr(case.ws),
            C.c_size_t(case.nbytes - 1), S.stream())
        assert rc == EWORKSPACE, f"workspace of sis3d_linear_tc_workspace_bytes() - 1 accepted (rc {rc})"
    k, m = case.accuracy(a)
    record_property("kernel_err_over_bound", k)
    record_property("min_model_err_over_bound", m)


_CHILD = """
import sys
sys.path.insert(0, sys.argv[1])
import conftest  # noqa: F401  (puts the package on sys.path)
import torch
import test_gpu_tc_accuracy as T
from lib import _sis3d as S
for row in T.CLUSTER_ROWS:
    case = T.Case(S, row)
    out = case.new_out()
    found = T.launched_instances(lambda: case.launch(out))
    torch.save({"out": out.cpu(), "inst": found}, f"{sys.argv[2]}/{row['id']}.pt")
"""


def test_cluster_instances_equal_single_cta(S, tmp_path, record_property):
    """The CL = 2 instances (2-CTA weight-tile multicast, SIS3D_CLUSTER=1) give the CL = 1 bits and meet the same bound.
    use_cluster() reads the environment once per process, so they run in a child process."""
    env = dict(os.environ, SIS3D_CLUSTER="1")
    p = subprocess.run([sys.executable, "-c", _CHILD, os.path.dirname(os.path.abspath(__file__)), str(tmp_path)], env=env,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    worst = 0.0
    for row in CLUSTER_ROWS:
        case = Case(S, row)
        out = case.new_out()
        found = launched_instances(lambda: case.launch(out))
        assert found in (None, [row["inst"][:7] + (1, row["inst"][8])]), f"{row['id']}: launched {found}"
        child = torch.load(tmp_path / f"{row['id']}.pt")
        assert child["inst"] in (None, [row["inst"]]), f"{row['id']}: child launched {child['inst']}"
        assert torch.equal(_bits(child["out"]), _bits(out.cpu())), f"{row['id']}: CL = 2 differs from CL = 1"
        case.check_untouched(out)
        worst = max(worst, case.accuracy(out)[0])
    record_property("kernel_err_over_bound", worst)
