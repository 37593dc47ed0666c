"""Per-element accuracy of the fp32 CUDA-core kernels against fp64, and bit equality with their host build.

conv3d_igemm_f32 (conv_simt.cu: the narrow geometry / mask-head / classifier convolutions and the split-K linear layer),
mlp_tail_kernel (roi.cu), the sparse back-projection convolution (sparse.cu) and enet_conv2d_kernel (enet2d/enet2d.cu) all
accumulate with fmaf in ascending k order, so each output has the rigorous bound

    |got - ref| <= gamma_n * (sum_k |x_k w_k| + |bias| + |residual|),     gamma_n = n u / (1 - n u),  u = 2^-24

with ref in fp64 and n the chain depth: K + 2 for the convolutions, k_per_split + splits + 1 for the split-K linear layer,
C + 8 for the sparse convolution (the per-tap GEMM, then the combine in tap order).  A sigmoid output adds 1/4 of the
pre-activation bound + 2^-21; PReLU multiplies it by max(1, |slope|) and adds one rounding; ReLU and max add nothing.
mlp_tail keeps its intermediates in shared memory, so its bound is carried through the layers: |W|^T e + gamma (|W|^T (|h| + e)
+ |b|).  Each case also proves the test's power: fp64 models of broken kernels on the same inputs (a 16-wide K chunk, a tap,
a split-K partial, a 32-row weight slab, a view of the back-projection max, a crop border padded with scene data, the
residual's top-left element instead of its 2x2 max) must exceed the bound by 4x somewhere.

The same sources build for the host (tools/cuda_host_emu.py, csrc/enet2d host build), with exact fmaf and no contraction;
the epilogues hold no mul-add nvcc could contract, so on the GPU every output buffer -- including the NaN outside the
written slice -- must equal the host build's bit for bit.  This catches what only a GPU shows (races, async ordering,
grid-stride wrap, atomics order); the fp64 bound catches what both builds share.  The exceptions, bounded instead:

  - act = 2 (sigmoid): expf of the CUDA math library and of the host libm differ by up to 2 ulp, so the GPU output is
    within 2^-21 |host| of the host build's;
  - enet_pool_affine: nvcc contracts `v * scale + shift` into one fma, the host build rounds twice, so the outputs differ
    by at most the rounding of the product (and of the PReLU slope).

Layout: outputs go to NaN-filled buffers wider than the output (channel offset, guard rows); nothing outside the written
slice may change.  Every launch runs twice with identical bits (the sparse convolution numbers voxels with atomics, in a
different order every run), one case per family is replayed from a CUDA graph, and the launched kernels' names (read through
torch.profiler) must match the instances the row names (tests/test_simt_instance_coverage.py keeps the table complete)."""
import ctypes as C
import math
import os
import re
import subprocess
import zlib

import pytest
import torch
import torch.nn.functional as F

from test_gpu_tc_accuracy import POWER, _act, _check, _weight

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
SIG_FLOOR = 2.0 ** -21
GUARD = 3          # guard rows after the last output row
ESUPPORT = -4      # SIS3D_EUNSUPPORTED
NUM_SMS = 132


def gamma(n):
    return n * U / (1 - n * U)


# ------------------------------------------------------------------------------------------------ devices
class Dev:
    """Where a case runs: libsis3d on the GPU, or the host build of the same sources on CPU tensors."""

    def __init__(self, lib3d, lib2d, device, stream=lambda: None):
        self.lib3d, self.lib2d, self.device, self.stream = lib3d, lib2d, device, stream

    @staticmethod
    def ptr(t):
        return None if t is None else C.c_void_p(t.data_ptr())

    def t(self, v):
        return None if v is None else v.to(self.device).contiguous()

    def check(self, rc, what=""):
        assert rc == 0, f"{what} returned {rc}"


def build_enet_emu(out):
    """The host build of enet2d.cu (the recipe of csrc/enet2d/Makefile, plus -ffp-contract=off) at `out`."""
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-sis_b200", "csrc", "enet2d")
    subprocess.check_call(["g++", "-O2", "-std=c++20", "-DSIS3D_HOST_EMU", "-x", "c++", "-fPIC", "-shared", "-pthread",
                           "-ffp-contract=off", f"-I{d}", f"-I{os.path.join(d, '..', '..', '..', 'include')}",
                           "-Wno-unknown-pragmas", "-o", out, os.path.join(d, "enet2d.cu")])
    return C.CDLL(out)


@pytest.fixture(scope="module")
def S():
    from lib import _sis3d
    return _sis3d


@pytest.fixture(scope="module")
def gpu(S):
    return Dev(S.lib, S.lib, DEV, S.stream)


@pytest.fixture(scope="module")
def host(emu_lib, tmp_path_factory):
    return Dev(emu_lib, build_enet_emu(str(tmp_path_factory.mktemp("enet_emu") / "libsis3d_enet_emu.so")), "cpu")


# ------------------------------------------------------------------------------------------------ shared helpers
def _gen(row):
    return torch.Generator().manual_seed(zlib.crc32(row["id"].encode()))


def _nan(shape, device, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=device)


def _raw(t):
    """Bit pattern of a tensor (so that NaN == NaN)."""
    return t.view({torch.float32: torch.int32, torch.float16: torch.int16}.get(t.dtype, t.dtype))


def fmaf_chain_accuracy(got, acc, absum, n, epi=None, act=0, mutants=None, what="fmaf chain"):
    """Assert got == act(acc + epi) within the bound of an fmaf chain of depth n, per element: gamma_n (absum + |epi|), a
    quarter of it + 2^-21 through a sigmoid (act = 2).  acc / absum: fp64 sum_k x_k w_k / sum_k |x_k w_k|.  Returns max err / bound.
    mutants: optional fp64 models (name -> pre-activation output) that must each miss the bound by POWER somewhere; with
    them, returns (max err / bound, smallest model max err / bound)."""
    epi = torch.zeros_like(acc) if epi is None else epi
    bound = gamma(n) * (absum + epi.abs())
    ref = acc + epi
    f = (lambda v: v)
    if act == 2:
        f, bound = torch.sigmoid, bound / 4 + SIG_FLOOR
    elif act == 1:
        f = F.relu
    if mutants is not None:
        return _check(got, f(ref), bound, {k: f(v) for k, v in mutants.items()}, 0, what)
    ref = f(ref)
    e = (got.double().to(ref.device) - ref).abs()
    k = torch.where(e == 0, torch.zeros_like(e), e / bound).max().item()
    assert k <= 1.0, f"{what}: max err/bound {k:.3g}"
    return k


def _chunk_mask(K, j):
    """bool [K]: the 16-wide K chunk j (negative: from the end)."""
    m = torch.zeros(K, dtype=torch.bool)
    n = (K + 15) // 16
    j = j % n
    m[16 * j:16 * j + 16] = True
    return m


def _k_to_w(mask_k, taps, cin):
    """K-order mask (k = tap * cin + c) -> [cin][taps] float mask of the weight layout [cout][cin][taps...]."""
    return mask_k.view(taps, cin).t().double()


KNOWN = ("conv3d_igemm_f32", "splitk_reduce_kernel", "pack_conv_weight_kernel", "maxpool3_vc_kernel", "maxpool3_tiled_kernel",
         "vc_to_ncdhw_kernel", "mlp_tail_kernel", "mask_select_kernel", "sparse_cover_kernel", "sparse_gemm_kernel",
         "sparse_combine_kernel", "feats_transpose_kernel2", "enet_conv2d_kernel", "enet_pack_weight_kernel",
         "enet_pool_affine_kernel", "enet_to_nchw_kernel")


def kernel_id(name):
    """'void sis3d::conv3d_igemm_f32<64, 4>(sis3d::ConvArgs)' or its mangled form -> 'conv3d_igemm_f32<64,4>'."""
    for k in KNOWN:
        i = name.find(k)
        if i < 0:
            continue
        rest = name[i + len(k):]
        m = re.match(r"<([^<>]*)>", rest)
        if m:
            return f"{k}<{','.join(a.strip() for a in m.group(1).split(','))}>"
        m = re.match(r"I((?:L[ib]\d+E)+)E", rest)
        if m:
            args = [("true" if v == "1" else "false") if t == "b" else v for t, v in re.findall(r"L([ib])(\d+)E", m.group(1))]
            return f"{k}<{','.join(args)}>"
        return k
    return None


def launched_kernels(fn, attempts=3):
    """Sorted ids of the libsis3d kernels fn launched, from torch.profiler; None if the profiler saw no kernel at all."""
    for _ in range(attempts):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        found = [kernel_id(e.name) for e in prof.events()]
        found = sorted(f for f in found if f)
        if found:
            return found
    return None


# ------------------------------------------------------------------------------------------------ conv3d_igemm_f32
def conv_inst(cout):
    return "conv3d_igemm_f32<32,2>" if cout <= 32 else "conv3d_igemm_f32<64,4>"


def conv(cin, cout, ks, dims, *, layout="vc", bias=True, res=False, act=1, out16=None, crops=None, canvas=False, x="signed",
         graph=False, emu=True):
    stride, pad = (2, 0) if ks == 2 else (1, 1 if ks == 3 else 0)
    K = ks ** 3 * cin
    path = "fast" if layout == "vc" and cin % 16 == 0 else ("gather" if K <= 128 else "gatherK")
    inst = conv_inst(cout)
    rid = "-".join(str(v) for v in ("conv", "bn" + inst[17:19], path, layout, f"k{ks}", f"{cin}to{cout}",
                                     "x".join(map(str, dims)), f"crops{len(crops)}" if crops else "", "canvas" if canvas else "",
                                     "bias" if bias else "", "res" if res else "", f"act{act}", f"o16{out16}" if out16 else "")
                   if v != "")
    return dict(fam="conv", id=rid, cin=cin, cout=cout, ks=ks, stride=stride, pad=pad, dims=dims, layout=layout, bias=bias,
                res=res, act=act, out16=out16, crops=crops, canvas=canvas, x=x, graph=graph, emu=emu,
                kernels=[inst] * (2 if out16 == "only" else 1))


def _conv3(x, w, stride, pad):
    """VC [X][Y][Z][cin] (fp64) x [cout][cin][k][k][k] -> VC."""
    return F.conv3d(x.permute(3, 0, 1, 2)[None], w, stride=stride, padding=pad)[0].permute(1, 2, 3, 0)


class ConvCase:
    def __init__(self, row):
        g = _gen(row)
        self.row = r = row
        X, Y, Z = r["dims"]
        cin, cout, ks = r["cin"], r["cout"], r["ks"]
        self.scene = _act(g, (X, Y, Z, cin), r["x"])
        self.w = _weight(g, (cout, cin, ks, ks, ks), "normal")
        self.b = torch.randn(cout, generator=g) if r["bias"] else None
        self.regs, m = [], 0
        for c in r["crops"] or [(0, 0, 0, X, Y, Z)]:
            od = tuple((s + 2 * r["pad"] - ks) // r["stride"] + 1 for s in c[3:])
            self.regs.append((c, od, m))
            m += math.prod(od)
        self.m = m
        self.res = torch.randn(m, cout, generator=g) if r["res"] else None
        self.ld, self.coff, self.res_ld, self.res_coff = cout + 8, 4, cout + 12, 8
        self.out_rows = X * Y * Z if r["canvas"] else m
        wm = torch.zeros(self.out_rows + GUARD, self.ld, dtype=torch.bool)
        for rows in self._rows():
            wm[rows, self.coff:self.coff + cout] = True
        self.written_mask = wm

    def _rows(self):
        """Output-buffer rows of each region's voxels, in the region's m order."""
        X, Y, Z = self.row["dims"]
        for c, od, moff in self.regs:
            if self.row["canvas"]:
                idx = torch.arange(X * Y * Z).view(X, Y, Z)
                yield idx[c[0]:c[0] + od[0], c[1]:c[1] + od[1], c[2]:c[2] + od[2]].reshape(-1)
            else:
                yield torch.arange(moff, moff + math.prod(od))

    def operands(self, dev, S):
        r, X, Y, Z = self.row, *self.row["dims"]
        cin, cout, ks = r["cin"], r["cout"], r["ks"]
        o = {"x": dev.t(self.scene if r["layout"] == "vc" else self.scene.permute(3, 0, 1, 2)), "b": dev.t(self.b)}
        o["wp"] = torch.empty(ks ** 3 * cin, (cout + 3) // 4 * 4, device=dev.device)
        wd = dev.t(self.w)
        dev.check(dev.lib3d.sis3d_pack_conv_weight(dev.ptr(wd), cout, cin, ks, dev.ptr(o["wp"]), dev.stream()), "pack")
        o["rbuf"] = None
        if self.res is not None:
            o["rbuf"] = _nan((self.m, self.res_ld), dev.device)
            o["rbuf"][:, self.res_coff:self.res_coff + cout] = self.res.to(dev.device)
        ents = []
        for (c, od, moff) in self.regs:
            vox = (c[0] * Y + c[1]) * Z + c[2]
            e = dict(in_dim=c[3:], out_dim=od, res_off=moff * self.res_ld)
            if r["layout"] == "vc":
                e.update(in_off=vox * cin, in_stride=(Y * Z * cin, Z * cin, cin))
            else:
                e.update(in_off=vox, in_stride=(Y * Z, Z, 1))
            if r["canvas"]:
                e.update(out_off=vox * self.ld, out_stride=(Y * Z * self.ld, Z * self.ld, self.ld))
            else:
                e.update(out_off=moff * self.ld)
            ents.append(e)
        o["regions"], o["tiles"] = S.make_regions(ents, dev.device)
        o["in_sc"] = 1 if r["layout"] == "vc" else X * Y * Z
        return o

    def new_outs(self, dev):
        o = {"out": _nan((self.out_rows + GUARD, self.ld), dev.device)}
        if self.row["out16"]:
            o["out16"] = _nan((self.out_rows + GUARD, self.ld), dev.device, torch.float16)
        return o

    def launch(self, dev, o, outs):
        r, P = self.row, dev.ptr
        calls = [(outs["out"], outs.get("out16"))] if r["out16"] != "only" else [(None, outs["out16"]), (outs["out"], None)]
        for out, out16 in calls:
            dev.check(dev.lib3d.sis3d_conv3d_ex(
                P(o["x"]), C.c_int64(o["in_sc"]), P(o["wp"]), P(o["b"]), P(o["rbuf"]), self.res_ld, self.res_coff, P(out),
                P(out16), self.ld, self.coff, P(o["regions"]), len(self.regs), o["tiles"], r["cin"], r["cout"], r["ks"],
                r["stride"], r["pad"], r["act"], dev.stream()), "sis3d_conv3d_ex")

    def check_layout(self, outs):
        wm = self.written_mask.to(outs["out"].device)
        for k, v in outs.items():
            assert bool(torch.isnan(v[~wm]).all()), f"{k}: written outside the output slice"
            assert bool(torch.isfinite(v[wm]).all()), f"{k}: output left unwritten"
        if "out16" in outs:
            assert torch.equal(_raw(outs["out16"][wm]), _raw(outs["out"][wm].half())), "fp16 twin != fp16(fp32 output)"

    def accuracy(self, outs):
        r = self.row
        cin, cout, ks, st, pad = r["cin"], r["cout"], r["ks"], r["stride"], r["pad"]
        K, taps = ks ** 3 * cin, ks ** 3
        sc = self.scene.to(DEV).double()
        w = self.w.to(DEV).double()
        masks = {"chunk_first": _chunk_mask(K, 0), "chunk_last": _chunk_mask(K, -1)}
        tap = torch.zeros(K, dtype=torch.bool)
        t0 = taps // 2
        tap[t0 * cin:(t0 + 1) * cin] = True
        masks["tap_dropped"] = tap
        wmask = {n: _k_to_w(m, taps, cin).reshape(1, cin, ks, ks, ks).to(DEV) for n, m in masks.items()}
        X, Y, Z = r["dims"]
        got, ref, absum, mut = [], [], [], {n: [] for n in list(wmask) + (["crop_border_scene_data"] if r["crops"] else [])}
        out = outs["out"]
        for (c, od, moff), rows in zip(self.regs, self._rows()):
            x0, y0, z0, sx, sy, sz = c
            crop = sc[x0:x0 + sx, y0:y0 + sy, z0:z0 + sz]
            acc = _conv3(crop, w, st, pad).reshape(-1, cout)
            absum.append(_conv3(crop.abs(), w.abs(), st, pad).reshape(-1, cout))
            ref.append(acc)
            for n, wm in wmask.items():
                mut[n].append(acc - _conv3(crop, w * wm, st, pad).reshape(-1, cout))
            if r["crops"]:  # the crop's zero border replaced by the neighbouring scene voxels
                p = pad
                ext = F.pad(sc.permute(3, 0, 1, 2), (p, p, p, p, p, p)).permute(1, 2, 3, 0)
                ext = ext[x0:x0 + sx + 2 * p, y0:y0 + sy + 2 * p, z0:z0 + sz + 2 * p]
                mut["crop_border_scene_data"].append(_conv3(ext, w, st, 0).reshape(-1, cout))
            got.append(out[rows.to(out.device), self.coff:self.coff + cout])
        got, ref, absum = torch.cat(got), torch.cat(ref), torch.cat(absum)
        mut = {n: torch.cat(v) for n, v in mut.items()}
        epi = torch.zeros_like(ref)
        if self.b is not None:
            epi = epi + self.b.to(DEV).double()
        if self.res is not None:
            epi = epi + self.res.to(DEV).double()
        bound = gamma(K + 2) * (absum + epi.abs())
        act = {0: lambda v: v, 1: F.relu, 2: torch.sigmoid}[r["act"]]
        if r["act"] == 2:
            bound = bound / 4 + SIG_FLOOR
        return _check(got, act(ref + epi), bound, {n: act(v + epi) for n, v in mut.items()}, 0, r["id"])


# crops of one 17 x 11 x 13 scene: different sizes, one of extent 1 along x, interior ones (scene data beyond every face)
CROPS = [(2, 1, 3, 7, 8, 9), (10, 2, 1, 1, 6, 5), (12, 0, 0, 5, 11, 13), (3, 9, 4, 6, 2, 8)]
CONV_ROWS = [
    conv(32, 32, 3, (9, 6, 7), graph=True), conv(16, 64, 3, (13, 5, 7), res=True, act=0),
    conv(128, 64, 3, (6, 5, 7), x="relu"),                                          # K = 3456
    conv(2, 32, 2, (13, 9, 11), layout="ncdhw", bias=False, out16="both"),          # geometry layer 0: odd extents
    conv(2, 64, 3, (7, 9, 5), layout="ncdhw", out16="only"),                        # mask head layer 0
    conv(8, 24, 3, (9, 5, 7), res=True, act=0),                                     # VC gather, K = 216 past the tap table
    conv(32, 128, 3, (6, 5, 4), layout="ncdhw", res=True),                          # NCDHW gather, K = 864, two N blocks
    conv(64, 19, 1, (7, 3, 5), act=2), conv(32, 40, 1, (9, 8, 5), act=2, bias=False),
    conv(32, 64, 2, (9, 7, 11), x="relu"), conv(16, 32, 2, (5, 3, 7), res=True, act=0, out16="both"),
    conv(2, 64, 3, (17, 11, 13), layout="ncdhw", crops=CROPS, canvas=True, res=True, graph=True),   # the mask head's crops
    conv(32, 32, 3, (17, 11, 13), crops=CROPS, bias=False),
    conv(16, 64, 3, (17, 11, 13), crops=CROPS, canvas=True, out16="both"),
    conv(8, 19, 3, (17, 11, 13), crops=CROPS, act=2),
]


# ------------------------------------------------------------------------------------------------ split-K linear layer
def linear_splits(M, N, K):
    """conv_simt.cu linear_splits + the k_per_split rounding of sis3d_linear: (splits, k_per_split)."""
    tiles = -(-M // 64) * -(-N // 64)
    s = max(1, min(K // 64, (2 * NUM_SMS + tiles - 1) // tiles))
    if s == 1:
        return 1, K
    kps = -(-(-(-K // s)) // 16) * 16
    return -(-K // kps), kps


def linear(M, K, N, *, bias=True, act=1, x="signed", graph=False, emu=True):
    s, kps = linear_splits(M, N, K)
    inst = conv_inst(N)
    rid = f"linear-bn{inst[17:19]}-{M}x{K}to{N}-{'split' + str(s) if s > 1 else 'unsplit'}-{x}" + \
        ("-nobias" if not bias else "") + f"-act{act}"
    return dict(fam="linear", id=rid, M=M, K=K, N=N, bias=bias, act=act, x=x, graph=graph, emu=emu, splits=s, kps=kps,
                kernels=sorted([inst] + (["splitk_reduce_kernel"] if s > 1 else [])))


class LinearCase:
    def __init__(self, row):
        g = _gen(row)
        self.row = r = row
        self.x = _act(g, (r["M"], r["K"]), r["x"])
        self.w = _weight(g, (r["N"], r["K"]), "normal")
        self.b = torch.randn(r["N"], generator=g) if r["bias"] else None

    def operands(self, dev, S):
        r = self.row
        o = {"x": dev.t(self.x), "b": dev.t(self.b), "wp": torch.empty(r["K"], (r["N"] + 3) // 4 * 4, device=dev.device)}
        wd = dev.t(self.w.view(r["N"], r["K"], 1, 1, 1))
        dev.check(dev.lib3d.sis3d_pack_conv_weight(dev.ptr(wd), r["N"], r["K"], 1, dev.ptr(o["wp"]), dev.stream()), "pack")
        o["nbytes"] = int(dev.lib3d.sis3d_linear_workspace_bytes(r["M"], r["N"], r["K"]))
        o["ws"] = torch.empty(o["nbytes"], dtype=torch.uint8, device=dev.device)
        return o

    def new_outs(self, dev):
        return {"y": _nan((self.row["M"] * self.row["N"] + GUARD,), dev.device)}

    def launch(self, dev, o, outs):
        r, P = self.row, dev.ptr
        dev.check(dev.lib3d.sis3d_linear(P(o["x"]), P(o["wp"]), P(o["b"]), P(outs["y"]), r["M"], r["K"], r["N"], r["act"],
                                         P(o["ws"]), C.c_size_t(o["nbytes"]), dev.stream()), "sis3d_linear")

    def check_layout(self, outs):
        n = self.row["M"] * self.row["N"]
        assert bool(torch.isfinite(outs["y"][:n]).all()) and bool(torch.isnan(outs["y"][n:]).all())

    def accuracy(self, outs):
        r = self.row
        x, w = self.x.to(DEV).double(), self.w.to(DEV).double()
        acc = x @ w.T
        epi = self.b.to(DEV).double() if self.b is not None else torch.zeros_like(acc)
        K, kps = r["K"], r["kps"]
        masks = {"chunk_first": _chunk_mask(K, 0), "chunk_last": _chunk_mask(K, -1)}
        if r["splits"] > 1:
            sp = torch.zeros(K, dtype=torch.bool)
            sp[:kps] = True
            masks["split_partial_dropped"] = sp
        mut = {n: acc - x[:, m.to(DEV)] @ w[:, m.to(DEV)].T for n, m in masks.items()}
        n = kps + r["splits"] + 1 if r["splits"] > 1 else K + 2
        bound = gamma(n) * (x.abs() @ w.abs().T + epi.abs())
        act = F.relu if r["act"] == 1 else (lambda v: v)
        got = outs["y"][:r["M"] * r["N"]].view(r["M"], r["N"])
        return _check(got, act(acc + epi), bound, {k: act(v + epi) for k, v in mut.items()}, 0, r["id"])


LINEAR_ROWS = [
    linear(1, 256, 32, bias=False, graph=True), linear(7, 64, 5, act=0), linear(200, 1056, 19, x="wide"),
    linear(300, 112, 114), linear(200, 8192, 256, x="wide", emu=False), linear(65, 8192, 64, x="wide", act=0, emu=False),
    linear(130, 512, 66, bias=False, act=0),
]


# ------------------------------------------------------------------------------------------------ mlp_tail
def mlp(R, d1, d2, d3, nc, nb, *, graph=False, emu=True):
    return dict(fam="mlp", id=f"mlp_tail-R{R}-{d1}_{d2}_{d3}-nc{nc}-nb{nb}", R=R, d=(d1, d2, d3), nc=nc, nb=nb, graph=graph,
                emu=emu, kernels=["mlp_tail_kernel"])


def mlp_forward(x, layers, drop=None):
    """fp64 forward of mlp_tail (two ReLU layers, then the class and box heads on the second one's output) from input x and
    layers [(w [N][K], b [N])] x 4, with the fmaf-chain bound carried through the layers.  drop = (layer, k0): that layer's
    weight columns k0..k0+31 zeroed (a broken kernel that skips one 32-row slab).  Returns the flattened [class | box]
    outputs and their bounds."""
    h = x.to(DEV).double()
    e = torch.zeros_like(h)
    outs_, bounds = [], []
    for i, (w, b) in enumerate(layers):
        w, b = w.to(DEV).double().clone(), b.to(DEV).double()
        if drop is not None and drop[0] == i:
            w[:, drop[1]:drop[1] + 32] = 0
        pre = h @ w.T + b
        eb = e @ w.abs().T + gamma(w.shape[1] + 1) * ((h.abs() + e) @ w.abs().T + b.abs())
        if i < 2:
            h, e = F.relu(pre), eb
        else:
            outs_.append(pre)
            bounds.append(eb.expand_as(pre))
    return torch.cat([v.reshape(-1) for v in outs_]), torch.cat([v.reshape(-1) for v in bounds])


class MlpCase:
    def __init__(self, row):
        g = _gen(row)
        self.row = r = row
        d1, d2, d3 = r["d"]
        self.x = F.relu(torch.randn(r["R"], d1, generator=g))
        self.layers = [(_weight(g, (n, k), "normal"), torch.randn(n, generator=g))
                       for k, n in ((d1, d2), (d2, d3), (d3, r["nc"]), (d3, r["nb"]))]

    def operands(self, dev, S):
        o = {"x": dev.t(self.x), "p": []}
        for w, b in self.layers:
            n, k = w.shape
            wp = torch.empty(k, (n + 3) // 4 * 4, device=dev.device)
            wd = dev.t(w.view(n, k, 1, 1, 1))
            dev.check(dev.lib3d.sis3d_pack_conv_weight(dev.ptr(wd), n, k, 1, dev.ptr(wp), dev.stream()), "pack")
            o["p"].append((wp, dev.t(b)))
        return o

    def new_outs(self, dev):
        r = self.row
        return {"cls": _nan(((r["R"] + GUARD) * r["nc"],), dev.device), "box": _nan(((r["R"] + GUARD) * r["nb"],), dev.device)}

    def launch(self, dev, o, outs):
        r, P = self.row, dev.ptr
        (w2, b2), (w3, b3), (wc, bc), (wb, bb) = o["p"]
        d1, d2, d3 = r["d"]
        dev.check(dev.lib3d.sis3d_mlp_tail(P(o["x"]), r["R"], d1, P(w2), P(b2), d2, P(w3), P(b3), d3, P(wc), P(bc), r["nc"],
                                           P(wb), P(bb), r["nb"], P(outs["cls"]), P(outs["box"]), dev.stream()), "mlp_tail")

    def check_layout(self, outs):
        R = self.row["R"]
        for k, n in (("cls", self.row["nc"]), ("box", self.row["nb"])):
            assert bool(torch.isfinite(outs[k][:R * n]).all()) and bool(torch.isnan(outs[k][R * n:]).all()), k

    def accuracy(self, outs):
        """fp64 forward with the bound carried through the layers; broken models drop one 32-row slab of one layer."""
        r = self.row
        L = [(w.to(DEV).double(), b.to(DEV).double()) for w, b in self.layers]
        forward = lambda drop=None: mlp_forward(self.x, L, drop)
        ref, bound = forward()
        d1, d2, d3 = r["d"]
        mut = {"layer2_slab0": forward((0, 0))[0], "layer3_last_slab": forward((1, (d2 - 1) // 32 * 32))[0],
               "cls_slab0": forward((2, 0))[0], "box_slab0": forward((3, 0))[0]}
        got = torch.cat([outs["cls"][:r["R"] * r["nc"]], outs["box"][:r["R"] * r["nb"]]])
        return _check(got, ref, bound, mut, 0, r["id"])


MLP_ROWS = [mlp(203, 256, 256, 256, 19, 114, graph=True), mlp(5, 200, 77, 130, 7, 42), mlp(1, 96, 256, 33, 19, 114),
            mlp(203, 100, 64, 256, 18, 108)]


# ------------------------------------------------------------------------------------------------ sparse back-projection conv
def sparse(C_, cout, dims, views, img, *, n_pairs=None, out16=False, cover=0.3, graph=False, emu=True):
    n_pairs = views if n_pairs is None else n_pairs
    rid = f"sparse-{cout}-C{C_}-{'x'.join(map(str, dims))}-v{views}p{n_pairs}-img{img[0]}x{img[1]}" + ("-o16" if out16 else "")
    return dict(fam="sparse", id=rid, C=C_, cout=cout, dims=dims, views=views, img=img, n_pairs=n_pairs, out16=out16,
                cover=cover, graph=graph, emu=emu,
                kernels=sorted(["feats_transpose_kernel2", "sparse_cover_kernel", f"sparse_gemm_kernel<{cout}>",
                                "sparse_combine_kernel"]))


class SparseCase:
    def __init__(self, row):
        g = _gen(row)
        self.row = r = row
        X, Y, Z = r["dims"]
        V, (iw, ih), Cn = r["views"], r["img"], r["C"]
        self.feats = torch.randn(V, Cn, ih, iw, generator=g)
        n0, hw = X * Y * Z, iw * ih
        pix = torch.randint(0, hw, (V, n0), generator=g, dtype=torch.int64)
        self.pix = torch.where(torch.rand(V, n0, generator=g) < r["cover"], pix, -1).to(torch.int16)
        self.pairs = torch.stack([torch.randperm(V, generator=g), torch.randperm(V, generator=g)], 1).to(torch.int32)
        self.w = _weight(g, (r["cout"], Cn, 2, 2, 2), "normal")
        self.out_ld, self.coff = r["cout"] + 12, 8
        self.n1 = (X // 2) * (Y // 2) * (Z // 2)

    def operands(self, dev, S):
        r = self.row
        o = {"feats": dev.t(self.feats), "pix": dev.t(self.pix), "pairs": dev.t(self.pairs),
             "np": dev.t(torch.tensor([r["n_pairs"]], dtype=torch.int32)),
             "wp": torch.empty(8 * r["C"], r["cout"], device=dev.device)}
        wd = dev.t(self.w)
        dev.check(dev.lib3d.sis3d_pack_conv_weight(dev.ptr(wd), r["cout"], r["C"], 2, dev.ptr(o["wp"]), dev.stream()), "pack")
        o["nbytes"] = int(dev.lib3d.sis3d_backproject_conv_k2s2_workspace_bytes(*r["dims"], r["cout"]))
        o["ws"] = torch.empty(o["nbytes"], dtype=torch.uint8, device=dev.device)
        return o

    def new_outs(self, dev):
        r = self.row
        (iw, ih) = r["img"]
        o = {"out": _nan((self.n1 + GUARD, self.out_ld), dev.device), "feats_t": _nan((r["views"], iw * ih, r["C"]), dev.device)}
        if r["out16"]:
            o["out16"] = _nan((self.n1 + GUARD, self.out_ld), dev.device, torch.float16)
        return o

    def launch(self, dev, o, outs, checked=True):
        r, P = self.row, dev.ptr
        (iw, ih) = r["img"]
        rc = dev.lib3d.sis3d_backproject_conv_k2s2_ex(
            P(o["feats"]), P(outs["feats_t"]), P(o["pix"]), P(o["pairs"]), P(o["np"]), r["views"], r["C"], iw, ih,
            *r["dims"], P(o["wp"]), r["cout"], P(outs["out"]), P(outs.get("out16")), self.out_ld, self.coff, P(o["ws"]),
            C.c_size_t(o["nbytes"]), dev.stream())
        if checked:
            dev.check(rc, "sis3d_backproject_conv_k2s2_ex")
        return rc

    def check_layout(self, outs):
        wm = torch.zeros(self.n1 + GUARD, self.out_ld, dtype=torch.bool, device=outs["out"].device)
        wm[:self.n1, self.coff:self.coff + self.row["cout"]] = True
        for k in ("out", "out16"):
            if k in outs:
                assert bool(torch.isnan(outs[k][~wm]).all()) and bool(torch.isfinite(outs[k][wm]).all()), k
        if "out16" in outs:
            assert torch.equal(_raw(outs["out16"][wm]), _raw(outs["out"][wm].half())), "fp16 twin != fp16(fp32 output)"
        assert torch.equal(outs["feats_t"], self.feats.to(outs["out"].device).flatten(2).transpose(1, 2))

    def imageft(self, skip=None):
        """fp64 back-projected volume VC [X][Y][Z][C]: max over the paired views (0 where a view does not cover the voxel)."""
        r = self.row
        X, Y, Z = r["dims"]
        f = self.feats.to(DEV).double().flatten(2)           # [V][C][hw]
        pix = self.pix.to(DEV).long()
        best = None
        for p in range(min(r["n_pairs"], r["views"])):
            if p == skip:
                continue
            fi, mi = int(self.pairs[p, 0]), int(self.pairs[p, 1])
            px = pix[mi]
            v = torch.where(px[None] >= 0, f[fi][:, px.clamp(min=0)], torch.zeros((), dtype=torch.float64, device=DEV))
            best = v if best is None else torch.maximum(best, v)
        return best.view(-1, Z, Y, X).permute(3, 2, 1, 0)     # lin = (z * Y + y) * X + x

    def accuracy(self, outs):
        r = self.row
        w = self.w.to(DEV).double()
        x = self.imageft()
        cout = r["cout"]
        acc = _conv3(x, w, 2, 0).reshape(-1, cout)
        bound = gamma(r["C"] + 8) * _conv3(x.abs(), w.abs(), 2, 0).reshape(-1, cout)
        tm = torch.zeros(1, 1, 2, 2, 2, dtype=torch.float64, device=DEV)
        tm[..., 1, 1, 1] = 1
        mut = {"view_left_out": _conv3(self.imageft(skip=0), w, 2, 0).reshape(-1, cout),
               "tap_dropped": acc - _conv3(x, w * tm, 2, 0).reshape(-1, cout)}
        got = outs["out"][:self.n1, self.coff:self.coff + cout]
        return _check(got, acc, bound, mut, 1, r["id"])


SPARSE_ROWS = [
    sparse(16, 32, (13, 9, 11), 3, (8, 6), out16=True, graph=True), sparse(128, 64, (12, 7, 9), 5, (10, 8), n_pairs=3),
    sparse(16, 64, (9, 11, 7), 70, (4, 3), cover=0.02),                   # 70 pairs: past the 64 staged in shared memory
    sparse(128, 32, (33, 17, 25), 4, (12, 9), out16=True),
    sparse(16, 64, (71, 61, 65), 3, (16, 12), cover=0.05, emu=False),      # grid-stride wrap of the cover and combine passes
]


# ------------------------------------------------------------------------------------------------ ENet conv
def enet_inst(N, Ho, Wo, cin, cout, nchw):
    vec = not nchw and cin % 4 == 0
    bn = 16 if cout <= 16 else (32 if cout <= 32 else 64)
    nt = -(-cout // bn)
    m = N * Ho * Wo
    half = bn < 64 and -(-m // (4096 // bn)) * nt < 2 * NUM_SMS
    return f"enet_conv2d_kernel<{bn},{'true' if vec else 'false'},{2 if half else 4}>"


def enet(N, H, W, cin, cout, k, *, stride=1, dil=1, nchw=False, bias=True, slope=True, res=None, res_c=None, coff=0,
         res_odd=(0, 0), graph=False, emu=True):
    """res_odd: extra (rows, columns) of a pooled residual, whose floor-mode 2x2 max-pool leaves them out."""
    kh, kw = k
    py, px = (kh - 1) // 2 * dil, (kw - 1) // 2 * dil
    Ho, Wo = (H + 2 * py - dil * (kh - 1) - 1) // stride + 1, (W + 2 * px - dil * (kw - 1) - 1) // stride + 1
    inst = enet_inst(N, Ho, Wo, cin, cout, nchw)
    res_c = (res_c or cout) if res else 0
    rid = "-".join(str(v) for v in ("enet", inst[19:-1].replace(",", "_"), f"n{N}", f"{H}x{W}", f"{cin}to{cout}", f"k{kh}x{kw}",
                                     f"s{stride}" if stride > 1 else "", f"d{dil}" if dil > 1 else "", "nchw" if nchw else "",
                                     res or "", f"resc{res_c}" if res and res_c < cout else "", f"coff{coff}" if coff else "",
                                     "odd{}x{}".format(*res_odd) if any(res_odd) else "",
                                     "" if slope else "noprelu") if v != "")
    return dict(fam="enet", id=rid, N=N, H=H, W=W, cin=cin, cout=cout, kh=kh, kw=kw, stride=stride, dil=dil, py=py, px=px,
                Ho=Ho, Wo=Wo, nchw=nchw, bias=bias, slope=slope, res=res, res_c=res_c, coff=coff, res_odd=res_odd, graph=graph, emu=emu,
                kernels=[inst])


class EnetConv(C.Structure):
    """struct sis3d_enet_conv (include/sis3d_enet.h)."""
    _fields_ = [("inp", C.c_void_p), ("in_sn", C.c_int64), ("in_sy", C.c_int64), ("in_sx", C.c_int64), ("in_sc", C.c_int64),
                ("w", C.c_void_p), ("bias", C.c_void_p), ("slope", C.c_void_p), ("res", C.c_void_p), ("out", C.c_void_p),
                ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("cin", C.c_int32), ("Ho", C.c_int32), ("Wo", C.c_int32),
                ("cout", C.c_int32), ("ldw", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("stride", C.c_int32),
                ("pad_y", C.c_int32), ("pad_x", C.c_int32), ("dil", C.c_int32), ("out_ld", C.c_int32), ("out_coff", C.c_int32),
                ("res_ld", C.c_int32), ("res_c", C.c_int32), ("res_pool", C.c_int32), ("res_h", C.c_int16),
                ("res_w", C.c_int16)]


def enet_conv_accuracy(got, acc, absum, K, epi, slope=None, mutants=None, operand_err=0.0, what="enet conv"):
    """Assert got == prelu(acc + epi, slope) for one sis3d_enet_conv2d output within the bound of its fmaf chain,
    gamma_(K+2) (absum + |epi|) (+ operand_err: the caller's own rounding of the operands, e.g. BatchNorm folded into the
    weights in fp32), carried through the PReLU: times max(1, |slope|), plus one rounding of the product.  mutants: fp64
    models (name -> pre-activation output, or (pre-activation output, slope) for a model with another PReLU slope), each
    must miss the bound by POWER somewhere.  Returns (max err / bound, smallest model max err / bound)."""
    pre_bound = gamma(K + 2) * (absum + epi.abs()) + operand_err
    ref = acc + epi
    mutants = {n: v if isinstance(v, tuple) else (v, slope) for n, v in (mutants or {}).items()}
    if slope is None:
        return _check(got, ref, pre_bound, {n: v for n, (v, _) in mutants.items()}, 0, what)
    pr = lambda v, s: torch.where(v >= 0, v, v * s)
    bound = pre_bound * slope.abs().clamp(min=1.0) + U * pr(ref, slope).abs()
    return _check(got, pr(ref, slope), bound, {n: pr(v, s) for n, (v, s) in mutants.items()}, 0, what)


class EnetCase:
    def __init__(self, row):
        g = _gen(row)
        self.row = r = row
        self.x = torch.randn(r["N"], r["cin"], r["H"], r["W"], generator=g)      # NCHW
        self.w = _weight(g, (r["cout"], r["cin"], r["kh"], r["kw"]), "normal")
        self.b = torch.randn(r["cout"], generator=g) if r["bias"] else None
        self.slope = torch.rand(r["cout"], generator=g) * 0.5 if r["slope"] else None
        self.res = None
        if r["res"]:
            f = 2 if r["res"] == "pool" else 1
            self.res = torch.randn(r["N"], f * r["Ho"] + r["res_odd"][0], f * r["Wo"] + r["res_odd"][1], r["res_c"], generator=g)
        self.m = r["N"] * r["Ho"] * r["Wo"]
        self.out_ld = r["coff"] + r["cout"] + 4
        self.res_ld = r["res_c"] + 4

    def operands(self, dev, S):
        r = self.row
        o = {"x": dev.t(self.x if r["nchw"] else self.x.permute(0, 2, 3, 1)), "b": dev.t(self.b), "slope": dev.t(self.slope)}
        o["wp"] = torch.empty(r["kh"] * r["kw"] * r["cin"], (r["cout"] + 3) // 4 * 4, device=dev.device)
        wd = dev.t(self.w)
        dev.check(dev.lib2d.sis3d_enet_pack_weight(dev.ptr(wd), r["cout"], r["cin"], r["kh"], r["kw"], dev.ptr(o["wp"]),
                                                   dev.stream()), "enet pack")
        o["res"] = None
        if self.res is not None:
            o["res"] = _nan(self.res.shape[:3] + (self.res_ld,), dev.device)
            o["res"][..., :r["res_c"]] = self.res.to(dev.device)
        return o

    def new_outs(self, dev):
        return {"out": _nan((self.m + GUARD, self.out_ld), dev.device)}

    def launch(self, dev, o, outs):
        r, P = self.row, dev.ptr
        H, W, cin = r["H"], r["W"], r["cin"]
        st = (cin * H * W, W, 1, H * W) if r["nchw"] else (H * W * cin, W * cin, cin, 1)
        a = EnetConv(P(o["x"]), *st, P(o["wp"]), P(o["b"]), P(o["slope"]), P(o["res"]), P(outs["out"]), r["N"], H, W, cin,
                     r["Ho"], r["Wo"], r["cout"], o["wp"].shape[1], r["kh"], r["kw"], r["stride"], r["py"], r["px"], r["dil"],
                     self.out_ld, r["coff"], self.res_ld, r["res_c"], 1 if r["res"] == "pool" else 0,
                     *(self.res.shape[1:3] if self.res is not None else (0, 0)))
        dev.check(dev.lib2d.sis3d_enet_conv2d(C.byref(a), dev.stream()), "sis3d_enet_conv2d")

    def check_layout(self, outs):
        wm = torch.zeros(self.m + GUARD, self.out_ld, dtype=torch.bool, device=outs["out"].device)
        wm[:self.m, self.row["coff"]:self.row["coff"] + self.row["cout"]] = True
        assert bool(torch.isnan(outs["out"][~wm]).all()) and bool(torch.isfinite(outs["out"][wm]).all())

    def accuracy(self, outs):
        r = self.row
        x, w = self.x.to(DEV).double(), self.w.to(DEV).double()
        cin, kh, kw, cout = r["cin"], r["kh"], r["kw"], r["cout"]

        def cv(a, b):
            y = F.conv2d(a, b, stride=r["stride"], padding=(r["py"], r["px"]), dilation=r["dil"])
            return y.permute(0, 2, 3, 1).reshape(-1, cout)

        acc, absum = cv(x, w), cv(x.abs(), w.abs())
        K, taps = kh * kw * cin, kh * kw
        tap = torch.zeros(K, dtype=torch.bool)
        t0 = taps // 2
        tap[t0 * cin:(t0 + 1) * cin] = True
        masks = {"chunk_first": _chunk_mask(K, 0), "chunk_last": _chunk_mask(K, -1), "tap_dropped": tap}
        mut = {n: acc - cv(x, w * _k_to_w(m, taps, cin).reshape(1, cin, kh, kw).to(DEV)) for n, m in masks.items()}
        bias = self.b.to(DEV).double() if self.b is not None else torch.zeros(cout, dtype=torch.float64, device=DEV)

        def residual(rr):  # [N][Ho][Wo][res_c] -> [m][cout], zero beyond res_c
            full = torch.zeros(self.m, cout, dtype=torch.float64, device=DEV)
            full[:, :r["res_c"]] = rr.reshape(-1, r["res_c"])
            return full

        res, pool_models = torch.zeros_like(acc), {}
        if self.res is not None:
            rr = self.res.to(DEV).double()
            if r["res"] == "pool":
                pool = lambda t: F.max_pool2d(t.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
                pool_models["res_pool_top_left"] = residual(rr[:, :2 * r["Ho"]:2, :2 * r["Wo"]:2])
                if any(r["res_odd"]):  # the residual addressed as if it were [N][2Ho][2Wo]
                    pool_models["res_pool_even_extent"] = residual(pool(rr.reshape(-1)[:self.m * 4 * r["res_c"]].reshape(
                        r["N"], 2 * r["Ho"], 2 * r["Wo"], r["res_c"])))
                rr = pool(rr)
            res = residual(rr)
        epi = bias + res
        mut = {n: v + epi for n, v in mut.items()}
        mut.update({n: acc + bias + v for n, v in pool_models.items()})
        got = outs["out"][:self.m, r["coff"]:r["coff"] + cout]
        slope = self.slope.to(DEV).double() if self.slope is not None else None
        return enet_conv_accuracy(got, acc, absum, K, epi, slope, mut, what=r["id"])


ENET_ROWS = [
    enet(2, 32, 41, 16, 16, (3, 3), dil=2, res="res", graph=True),                  # <16, vec, 2>
    enet(1, 130, 520, 4, 13, (3, 3), coff=3),                                       # <16, vec, 4>
    enet(2, 64, 82, 3, 13, (3, 3), stride=2, nchw=True, slope=False),               # <16, nchw, 2>: ENet's first conv
    enet(2, 128, 264, 3, 16, (3, 3), nchw=True),                                    # <16, nchw, 4>
    enet(2, 17, 23, 64, 32, (5, 1), res="res", res_c=24),                           # <32, vec, 2>, K = 320
    enet(1, 128, 264, 16, 32, (1, 5), bias=False),                                  # <32, vec, 4>
    enet(2, 21, 19, 8, 24, (3, 3), dil=4, nchw=True, res="res", res_c=16, coff=4),  # <32, nchw, 2>
    enet(1, 128, 264, 3, 32, (3, 3)),                                               # <32, cin % 4 != 0, 4>
    enet(2, 16, 21, 128, 64, (3, 3), res="pool", coff=4),                           # <64, vec, 4>, K = 1152 past the tap table
    enet(2, 19, 25, 64, 128, (3, 3), dil=8, res="pool", res_c=96),                  # two N blocks, K = 576
    enet(2, 40, 41, 65, 64, (3, 3), dil=16, nchw=True),                             # <64, nchw, 4>, K = 585
    enet(3, 24, 33, 32, 32, (3, 3), stride=2, res="pool"),
    enet(3, 15, 21, 64, 128, (2, 2), stride=2, res="pool", res_c=64, res_odd=(1, 1)),  # ENet's down-sampling conv1 shape,
]                                                                                          # floor-mode pool of an odd skip


# ------------------------------------------------------------------------------------------------ exact kernels
def exact(kind, **kw):
    rid = f"exact-{kind}-" + "-".join(f"{k}{'x'.join(map(str, v)) if isinstance(v, tuple) else v}" for k, v in kw.items()
                                       if k not in ("graph", "emu"))
    kernels = {"maxpool3": None, "pool_affine": ["enet_pool_affine_kernel"], "to_nchw": ["enet_to_nchw_kernel"],
               "vc_to_ncdhw": ["vc_to_ncdhw_kernel"], "pack3d": ["pack_conv_weight_kernel"],
               "pack2d": ["enet_pack_weight_kernel"], "mask_select": ["mask_select_kernel"]}[kind]
    if kind == "maxpool3":
        kernels = ["maxpool3_tiled_kernel" if kw["C"] % 16 == 0 else "maxpool3_vc_kernel"]
    return dict(fam="exact", kind=kind, id=rid, graph=kw.pop("graph", False), emu=kw.pop("emu", True), kernels=kernels, **kw)


class ExactCase:
    """Kernels without arithmetic (or, for enet_pool_affine, one affine + PReLU): compared with == (bitwise)."""

    def __init__(self, row):
        g = _gen(row)
        self.row = r = row
        k = r["kind"]
        if k == "maxpool3":
            self.x = torch.randn(*r["dims"], r["C"], generator=g)
        elif k == "pool_affine":
            self.x = torch.randn(r["N"], r["C"], r["H"], r["W"], generator=g)
            self.aff = [torch.randn(r["C"], generator=g), torch.randn(r["C"], generator=g), torch.rand(r["C"], generator=g)]
        elif k == "to_nchw":
            self.x = torch.randn(r["N"] * r["P"], r["ld"], generator=g)
        elif k == "vc_to_ncdhw":
            self.x = torch.randn(r["nvox"], r["C"], generator=g)
        elif k in ("pack3d", "pack2d"):
            self.x = torch.randn(r["shape"], generator=g)
        else:
            sizes = list(r["sizes"])
            self.offs = torch.tensor([0] + sizes).cumsum(0)
            self.total = int(self.offs[-1])
            q = torch.randint(-8, 9, (self.total, r["ncls"]), generator=g).float() / 16   # 0.5 = thresh exactly, often
            self.x = q + torch.randn(self.total, r["ncls"], generator=g) * (torch.rand(self.total, 1, generator=g) < 0.5)
            self.cls = torch.randint(0, r["ncls"], (len(sizes),), generator=g, dtype=torch.int32)

    def operands(self, dev, S):
        o = {"x": dev.t(self.x)}
        if self.row["kind"] == "pool_affine":
            o["aff"] = [dev.t(a) for a in self.aff]
        if self.row["kind"] == "mask_select":
            o["offs"], o["cls"] = dev.t(self.offs), dev.t(self.cls)
        return o

    def out_shape(self):
        r = self.row
        return {"maxpool3": lambda: (math.prod(r["dims"]) + GUARD, 2 * r["C"]),
                "pool_affine": lambda: (r["N"] * (r["H"] // 2) * (r["W"] // 2) + GUARD, r["C"] + 5),
                "to_nchw": lambda: (r["N"] * r["C"] + GUARD, r["P"]), "vc_to_ncdhw": lambda: (r["C"] + GUARD, r["nvox"]),
                "pack3d": lambda: (r["shape"][2] ** 3 * r["shape"][1] + GUARD, (r["shape"][0] + 3) // 4 * 4),
                "pack2d": lambda: (r["shape"][2] * r["shape"][3] * r["shape"][1] + GUARD, (r["shape"][0] + 3) // 4 * 4),
                "mask_select": lambda: (self.total + GUARD,)}[r["kind"]]()

    def new_outs(self, dev):
        o = {"out": _nan(self.out_shape(), dev.device)}
        if self.row["kind"] == "mask_select":
            o["bits"] = torch.full((self.total + GUARD,), 7, dtype=torch.uint8, device=dev.device)
        return o

    def launch(self, dev, o, outs):
        r, P, k, st = self.row, dev.ptr, self.row["kind"], dev.stream()
        x, out = P(o["x"]), P(outs["out"])
        if k == "maxpool3":
            dev.check(dev.lib3d.sis3d_maxpool3(x, out, 2 * r["C"], r["C"], *r["dims"], r["C"], st))
        elif k == "pool_affine":
            N, Cn, H, W = self.x.shape
            dev.check(dev.lib2d.sis3d_enet_pool_affine(x, C.c_int64(Cn * H * W), C.c_int64(W), C.c_int64(1), C.c_int64(H * W), N, H,
                                                       W, Cn, *[P(a) for a in o["aff"]], out, Cn + 5, 5, st))
        elif k == "to_nchw":
            dev.check(dev.lib2d.sis3d_enet_to_nchw(x, r["ld"], r["coff"], r["N"], C.c_int64(r["P"]), r["C"], out, st))
        elif k == "vc_to_ncdhw":
            dev.check(dev.lib3d.sis3d_vc_to_ncdhw(x, out, C.c_int64(r["nvox"]), r["C"], st))
        elif k == "pack3d":
            co, ci, ks = r["shape"][:3]
            dev.check(dev.lib3d.sis3d_pack_conv_weight(x, co, ci, ks, out, st))
        elif k == "pack2d":
            co, ci, kh, kw = r["shape"]
            dev.check(dev.lib2d.sis3d_enet_pack_weight(x, co, ci, kh, kw, out, st))
        else:
            dev.check(dev.lib3d.sis3d_mask_select(x, P(o["offs"]), P(o["cls"]), len(r["sizes"]), r["ncls"], C.c_int64(r["hint"]),
                                                  C.c_float(0.5), out, P(outs["bits"]), st))

    def expected(self, device):
        """The written slice (row slice, column slice) and its exact value."""
        r, k = self.row, self.row["kind"]
        x = self.x.to(device)
        if k == "maxpool3":
            C_ = r["C"]
            v = F.max_pool3d(x.permute(3, 0, 1, 2)[None], 3, 1, 1)[0].permute(1, 2, 3, 0).reshape(-1, C_)
            return (slice(0, v.shape[0]), slice(C_, 2 * C_)), v
        if k == "pool_affine":
            sc, sh, sl = [a.to(device) for a in self.aff]
            v = F.max_pool2d(x, 2).permute(0, 2, 3, 1).reshape(-1, r["C"]) * sc + sh  # value checked against fp64 in accuracy()
            return (slice(0, v.shape[0]), slice(5, 5 + r["C"])), torch.where(v >= 0, v, v * sl)
        if k == "to_nchw":
            v = x.view(r["N"], r["P"], r["ld"])[..., r["coff"]:r["coff"] + r["C"]].transpose(1, 2).reshape(-1, r["P"])
            return (slice(0, v.shape[0]), slice(None)), v
        if k == "vc_to_ncdhw":
            return (slice(0, r["C"]), slice(None)), x.t()
        if k == "pack3d":
            co, ci, ks = r["shape"][:3]
            v = F.pad(x.reshape(co, ci, ks ** 3).permute(2, 1, 0).reshape(-1, co), (0, (-co) % 4))
            return (slice(0, v.shape[0]), slice(None)), v
        if k == "pack2d":
            co, ci, kh, kw = r["shape"]
            v = F.pad(x.reshape(co, ci, kh * kw).permute(2, 1, 0).reshape(-1, co), (0, (-co) % 4))
            return (slice(0, v.shape[0]), slice(None)), v
        crop = torch.repeat_interleave(torch.arange(len(r["sizes"])), torch.tensor(r["sizes"])).to(device)
        v = x.gather(1, self.cls.to(device).long()[crop][:, None])[:, 0]
        return (slice(0, self.total),), v

    def check_layout(self, outs):
        out = outs["out"]
        sl, v = self.expected(out.device)
        wm = torch.zeros(out.shape, dtype=torch.bool, device=out.device)
        wm[sl] = True
        assert bool(torch.isnan(out[~wm]).all()), "written outside the output slice"
        assert bool(torch.isfinite(out[wm]).all()), "output left unwritten"
        if "bits" in outs:
            b = outs["bits"]
            assert torch.equal(b[:self.total], (v >= 0.5).to(torch.uint8)) and bool((b[self.total:] == 7).all())

    def accuracy(self, outs):
        sl, v = self.expected(outs["out"].device)
        got = outs["out"][sl].reshape(v.shape)
        if self.row["kind"] == "pool_affine":  # one fma: within one rounding of the fp64 value
            r = self.row
            sc, sh, sl_ = [a.to(got.device).double() for a in self.aff]
            p = F.max_pool2d(self.x.to(got.device).double(), 2).permute(0, 2, 3, 1).reshape(-1, r["C"])
            pre = p * sc + sh
            ref = torch.where(pre >= 0, pre, pre * sl_)
            bound = U * ((p * sc).abs() + pre.abs()) * torch.clamp(sl_, min=1) + U * ref.abs()
            e = (got.double() - ref).abs()
            assert bool((e <= bound).all()), f"pool_affine: max err/bound {(e / bound).max().item():.3g}"
            return (e / bound).nan_to_num(0.0).max().item(), float("inf")
        assert torch.equal(_raw(got), _raw(v)), f"{self.row['id']}: differs from the exact result"
        return 0.0, float("inf")


EXACT_ROWS = [
    exact("maxpool3", C=64, dims=(9, 5, 7), graph=True), exact("maxpool3", C=16, dims=(17, 8, 3)),
    exact("maxpool3", C=8, dims=(6, 9, 11)), exact("maxpool3", C=4, dims=(90, 80, 76)),           # 547200 > 2112 * 256
    exact("pool_affine", N=2, C=3, H=64, W=82), exact("pool_affine", N=9, C=3, H=256, W=328, emu=False),  # 566784: wraps
    exact("to_nchw", N=2, P=37 * 41, C=19, ld=24, coff=3), exact("vc_to_ncdhw", nvox=777, C=45),
    exact("pack3d", shape=(66, 128, 3, 3, 3)), exact("pack3d", shape=(66, 256, 3, 3, 3)),          # 470016 > 1056 * 256
    exact("pack2d", shape=(16, 3, 3, 3)), exact("pack2d", shape=(128, 256, 3, 3)),                # 294912: wraps
    exact("mask_select", sizes=(5, 0, 130, 0, 1, 64), ncls=19, hint=200),
    exact("mask_select", sizes=(0, 40000, 0, 120000, 3, 150001), ncls=7, hint=1000, emu=False),   # 310004 > 1056 * 256
]

CASES = {"conv": ConvCase, "linear": LinearCase, "mlp": MlpCase, "sparse": SparseCase, "enet": EnetCase, "exact": ExactCase}
ROWS = CONV_ROWS + LINEAR_ROWS + MLP_ROWS + SPARSE_ROWS + ENET_ROWS + EXACT_ROWS


# ------------------------------------------------------------------------------------------------ the checks
def host_tolerance(case, key, h):
    """Allowed |GPU - host| per element of output `key` (host values h) for the rows whose two builds cannot agree in bits
    (module docstring); None: bit equality."""
    row = case.row
    if row["fam"] == "conv" and row["act"] == 2:
        return SIG_FLOOR * h.abs()
    if row.get("kind") == "pool_affine":  # the rounding of the product (times the slope), and one of the output
        p = F.max_pool2d(case.x.double(), 2).permute(0, 2, 3, 1).reshape(-1, row["C"])
        sc, sl = case.aff[0].double(), case.aff[2].double()
        tol = torch.zeros(h.shape, dtype=torch.float64)
        tol[:p.shape[0], 5:] = U * (p * sc).abs() * torch.clamp(sl, min=1) + 2 * U * h[:p.shape[0], 5:].double().abs()
        return tol
    return None


def compare_with_host(case, outs, host, S):
    """Run the case on the host build and compare every output buffer; returns the number of elements that differ."""
    ho = case.new_outs(host)
    case.launch(host, case.operands(host, S), ho)
    differ = 0
    for k, v in outs.items():
        h, g = ho[k], v.cpu()
        tol = None if k == "bits" else host_tolerance(case, k, h)
        ne = int((_raw(g) != _raw(h)).sum())
        if tol is None:
            assert ne == 0, f"{k}: the GPU and the host build differ in {ne} elements"
        else:
            assert torch.equal(torch.isnan(g), torch.isnan(h)), f"{k}: NaN pattern differs from the host build"
            fin = torch.isfinite(h)
            e = (g.double() - h.double()).abs()
            assert bool((e[fin] <= tol[fin]).all()), f"{k}: the GPU differs from the host build by more than the allowed " \
                f"rounding ({(e[fin] / tol[fin]).nan_to_num(posinf=1e9).max().item():.3g}x)"
        differ += ne
    return differ


def run_row(row, dev, S, host=None, record=lambda k, v: None):
    case = CASES[row["fam"]](row)
    o = case.operands(dev, S)
    a, b = case.new_outs(dev), case.new_outs(dev)
    case.launch(dev, o, a)
    if dev.device == "cuda":
        found = launched_kernels(lambda: case.launch(dev, o, b))
        if found is not None:  # the template instances exactly; the profiler may miss an untemplated helper kernel
            inst = lambda ks: sorted(k for k in ks if "<" in k)
            assert inst(found) == inst(row["kernels"]) and set(found) <= set(row["kernels"]), \
                f"the row does not reach the kernels it names: launched {found}"
        record("kernels_launched", found)
        torch.cuda.synchronize()
    else:
        case.launch(dev, o, b)
    for k in a:
        assert torch.equal(_raw(a[k]), _raw(b[k])), f"{k}: two launches on the same inputs differ"
    case.check_layout(a)
    if row["graph"] and dev.device == "cuda":
        gout = case.new_outs(dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            case.launch(dev, o, gout)
        graph.replay()
        torch.cuda.synchronize()
        for k in a:
            assert torch.equal(_raw(gout[k]), _raw(a[k])), f"{k}: CUDA-graph replay differs from the eager launch"
    if host is not None and row["emu"]:
        record("elements_differing_from_host_build", compare_with_host(case, a, host, S))
    k, m = case.accuracy(a)
    record("kernel_err_over_bound", k)
    record("min_model_err_over_bound", m)
    return k, m


@pytest.mark.parametrize("row", ROWS, ids=[r["id"] for r in ROWS])
def test_simt_kernel_accuracy(S, gpu, host, row, record_property):
    run_row(row, gpu, S, host, record_property)


def test_sparse_conv_refuses_before_launching(S, gpu):
    """A channel count whose staged operands exceed shared memory is refused before anything is launched: the scratch
    transpose and the workspace keep their contents and the launch counter does not move."""
    row = sparse(512, 64, (6, 5, 7), 2, (4, 3))
    case = SparseCase(row)
    o = case.operands(gpu, S)
    o["ws"] = _nan((o["nbytes"] // 4 + 1,), DEV)
    outs = case.new_outs(gpu)
    before = {k: v.clone() for k, v in outs.items()}
    torch.cuda.synchronize()
    n0 = S.launch_count()
    rc = case.launch(gpu, o, outs, checked=False)
    torch.cuda.synchronize()
    assert rc == ESUPPORT
    assert S.launch_count() == n0
    assert bool(torch.isnan(o["ws"]).all())
    for k, v in outs.items():
        assert torch.equal(_raw(v), _raw(before[k])), k
