"""CPU: wiring of the work-in-progress ENet executor (lib/nets/enet.py) -- strides, paddings, output sizes, residual /
pooled-skip hookup, weight packing order, channel slices -- checked against the reference features by substituting a numpy
model of the C contract declared in csrc/enet2d/sis3d_enet.h for the CUDA library.  (The CUDA kernels themselves have not
run on a GPU yet; this test pins everything above them.)"""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden
from lib.nets.enet import EnetEncoder, _Conv


def _arr(ptr, n):
    return np.ctypeslib.as_array((C.c_float * int(n)).from_address(int(ptr if not hasattr(ptr, "value") else ptr.value)))


class _NumpyEnetLib:
    """The documented behaviour of libsis3d_enet.so, on host memory."""

    def __init__(self):
        self.packed_shapes = {}

    def sis3d_enet_pack_weight(self, w, cout, cin, kh, kw, packed, stream):
        ldw = (cout + 3) // 4 * 4
        src = _arr(w, cout * cin * kh * kw).reshape(cout, cin, kh * kw)
        dst = _arr(packed, kh * kw * cin * ldw).reshape(kh * kw, cin, ldw)
        dst[:] = 0
        dst[:, :, :cout] = np.transpose(src, (2, 1, 0))  # k = (ky*kw + kx)*cin + c
        return 0

    def sis3d_enet_conv2d(self, args, stream):
        a = C.cast(args, C.POINTER(_Conv)).contents
        N, H, W, cin, Ho, Wo, cout = a.N, a.H, a.W, a.cin, a.Ho, a.Wo, a.cout
        span = (N - 1) * a.in_sn + (H - 1) * a.in_sy + (W - 1) * a.in_sx + (cin - 1) * a.in_sc + 1
        flat = _arr(a.inp, span)
        x = np.lib.stride_tricks.as_strided(flat, (N, H, W, cin), tuple(4 * s for s in (a.in_sn, a.in_sy, a.in_sx, a.in_sc)))
        w = _arr(a.w, a.kh * a.kw * cin * a.ldw).reshape(a.kh, a.kw, cin, a.ldw)[..., :cout]
        acc = np.zeros((N, Ho, Wo, cout), dtype=np.float64)
        for ky in range(a.kh):
            for kx in range(a.kw):
                iy = np.arange(Ho) * a.stride - a.pad_y + ky * a.dil
                ix = np.arange(Wo) * a.stride - a.pad_x + kx * a.dil
                vy, vx = (iy >= 0) & (iy < H), (ix >= 0) & (ix < W)
                patch = np.zeros((N, Ho, Wo, cin), dtype=np.float64)
                patch[:, np.ix_(vy, vx)[0], np.ix_(vy, vx)[1]] = x[:, iy[vy]][:, :, ix[vx]]
                acc += patch @ w[ky, kx].astype(np.float64)
        if a.bias:
            acc += _arr(a.bias, cout)
        if a.res:
            rh, rw = (a.res_h, a.res_w) if a.res_h or a.res_w else ((2 * Ho, 2 * Wo) if a.res_pool else (Ho, Wo))
            r = _arr(a.res, N * rh * rw * a.res_ld).reshape(N, rh, rw, a.res_ld)[..., :a.res_c]
            if a.res_pool:  # floor-mode 2x2/2 max-pool: [2Ho | 2Ho + 1][2Wo | 2Wo + 1] -> [Ho][Wo]
                assert rh in (2 * Ho, 2 * Ho + 1) and rw in (2 * Wo, 2 * Wo + 1)
                acc[..., :a.res_c] += r[:, :2 * Ho, :2 * Wo].reshape(N, Ho, 2, Wo, 2, a.res_c).max(axis=(2, 4))
            else:
                assert (rh, rw) == (Ho, Wo)
                acc[..., :a.res_c] += r
        if a.slope:
            sl = _arr(a.slope, cout)
            acc = np.where(acc >= 0, acc, acc * sl)
        out = _arr(a.out, N * Ho * Wo * a.out_ld).reshape(N, Ho, Wo, a.out_ld)
        out[..., a.out_coff:a.out_coff + cout] = acc.astype(np.float32)
        return 0

    def sis3d_enet_pool_affine(self, inp, sn, sy, sx, sc, N, H, W, Cn, scale, shift, slope, out, out_ld, out_coff, stream):
        span = (N - 1) * sn + (H - 1) * sy + (W - 1) * sx + (Cn - 1) * sc + 1
        x = np.lib.stride_tricks.as_strided(_arr(inp, span), (N, H, W, Cn), tuple(4 * s for s in (sn, sy, sx, sc)))
        p = x[:, :H // 2 * 2, :W // 2 * 2].reshape(N, H // 2, 2, W // 2, 2, Cn).max(axis=(2, 4))
        v = p * _arr(scale, Cn) + _arr(shift, Cn)
        v = np.where(v >= 0, v, v * _arr(slope, Cn))
        _arr(out, N * (H // 2) * (W // 2) * out_ld).reshape(N, H // 2, W // 2, out_ld)[..., out_coff:out_coff + Cn] = v
        return 0

    def sis3d_enet_to_nchw(self, inp, ld, coff, N, P, Cn, out, stream):
        P = int(P.value if hasattr(P, "value") else P)
        x = _arr(inp, N * P * ld).reshape(N, P, ld)[..., coff:coff + Cn]
        _arr(out, N * Cn * P).reshape(N, Cn, P)[:] = np.transpose(x, (0, 2, 1))
        return 0


def test_executor_wiring_reproduces_reference_features():
    g = load_golden("enet_encoder.npz")
    params = [torch.from_numpy(g[k]) for k in sorted(k for k in g if k.startswith("p"))]
    enc = EnetEncoder(params, "cpu", lib=_NumpyEnetLib())
    x = torch.from_numpy(np.random.default_rng(int(g["seed"])).standard_normal((1, 3, 256, 328)).astype(np.float32))
    y = enc(x)
    ref = torch.from_numpy(g["features"])
    assert y.shape == ref.shape
    assert float((y - ref).abs().max()) < 2e-4 and float((y - ref).norm() / ref.norm()) < 2e-6


def _emu_lib():
    import os
    import subprocess
    from conftest import ROOT
    d = os.path.join(ROOT, "3d-sis_b200", "csrc", "enet2d")
    subprocess.check_call(["make", "-C", d, "emu"], stdout=subprocess.DEVNULL)
    return C.CDLL(os.path.join(ROOT, "3d-sis_b200", "lib", "libsis3d_enet_emu.so"))


def _golden_params():
    g = load_golden("enet_encoder.npz")
    return [torch.from_numpy(g[k]) for k in sorted(k for k in g if k.startswith("p"))]


def test_cuda_source_under_host_emulation_matches_the_contract_model():
    """The SAME enet2d.cu that nvcc compiles for sm_90a, compiled for the host (csrc/enet2d/host_emu.h: one CUDA block =
    blockDim std::threads meeting at a barrier for __syncthreads) and driven by the executor: checks the kernels' index
    arithmetic, tap tables, shared-memory staging, epilogues and packing on a small image against the numpy contract model
    and the torch program -- everything short of running on the GPU itself."""
    from lib.nets import enet_program as E
    emu = _emu_lib()
    params = _golden_params()
    x = torch.from_numpy(np.random.default_rng(5).standard_normal((2, 3, 48, 72)).astype(np.float32))
    y_emu = EnetEncoder(params, "cpu", lib=emu)(x)
    y_model = EnetEncoder(params, "cpu", lib=_NumpyEnetLib())(x)
    with torch.no_grad():
        y_ref = E.run_program(E.compile_enet(params), x)
    assert y_emu.shape == y_ref.shape == (2, 128, 6, 9)
    assert float((y_emu - y_model).abs().max()) < 1e-4
    assert float((y_emu - y_ref).abs().max()) < 2e-4 and float((y_emu - y_ref).norm() / y_ref.norm()) < 1e-5


@pytest.mark.parametrize("hw", [(44, 76), (50, 72)], ids=["44x76", "50x72"])
def test_host_emulation_pools_odd_skips_in_floor_mode(hw):
    """Images whose half (50 rows: 25 at the first down-sampling bottleneck) or quarter (44 x 76: 11 x 19 at the second)
    is odd: the pooled skip drops the last row / column as the reference's floor-mode MaxPool2d does, and the
    down-sampling conv (2x2, stride 2) reads the same rows, so every later feature still matches the torch program."""
    from lib.nets import enet_program as E
    params = _golden_params()
    x = torch.from_numpy(np.random.default_rng(6).standard_normal((2, 3) + hw).astype(np.float32))
    y_emu = EnetEncoder(params, "cpu", lib=_emu_lib())(x)
    y_model = EnetEncoder(params, "cpu", lib=_NumpyEnetLib())(x)
    with torch.no_grad():
        y_ref = E.run_program(E.compile_enet(params), x)
    assert y_emu.shape == y_ref.shape == (2, 128, hw[0] // 8, hw[1] // 8)
    assert float((y_model - y_ref).abs().max()) < 2e-4
    assert float((y_emu - y_ref).abs().max()) < 2e-4 and float((y_emu - y_ref).norm() / y_ref.norm()) < 1e-5


class _CountingLib(_NumpyEnetLib):
    def __init__(self):
        super().__init__()
        self.calls = 0

    def __getattribute__(self, name):
        if name.startswith("sis3d_enet_") and name != "sis3d_enet_pack_weight":
            object.__setattr__(self, "calls", object.__getattribute__(self, "calls") + 1)
        return object.__getattribute__(self, name)


@pytest.mark.parametrize("hw", [(255, 328), (256, 327), (47, 72)], ids=["255x328", "256x327", "47x72"])
def test_encoder_refuses_odd_image_sizes_before_launching(hw):
    """The initial block concatenates a 3x3/s2 conv (ceil(H/2) rows) with a 2x2/s2 max-pool (floor(H/2) rows), which the
    reference cannot do for an odd H or W: the executor refuses such images before its first launch."""
    lib = _CountingLib()
    enc = EnetEncoder(_golden_params(), "cpu", lib=lib)
    with pytest.raises(ValueError, match="even H and W"):
        enc(torch.zeros((1, 3) + hw))
    assert lib.calls == 0


def test_conv_refuses_a_residual_extent_it_cannot_pool():
    """sis3d_enet_conv2d takes the residual's height and width: Ho x Wo, or 2Ho | 2Ho + 1 by 2Wo | 2Wo + 1 for the pooled
    skip; any other extent is an invalid argument (-1), refused before a launch."""
    emu = _emu_lib()
    Ho, Wo, cin, cout = 3, 4, 4, 8
    x = np.zeros((1, Ho, Wo, cin), np.float32)
    w = np.zeros((cin, cout), np.float32)
    out = np.full((1, Ho, Wo, cout), 7.0, np.float32)
    res = np.zeros((1, 2 * Ho + 2, 2 * Wo + 2, cout), np.float32)
    p = lambda a: a.ctypes.data

    def run(pool, rh, rw):
        a = _Conv(inp=p(x), in_sn=Ho * Wo * cin, in_sy=Wo * cin, in_sx=cin, in_sc=1, w=p(w), res=p(res), out=p(out), N=1, H=Ho,
                  W=Wo, cin=cin, Ho=Ho, Wo=Wo, cout=cout, ldw=cout, kh=1, kw=1, stride=1, dil=1, out_ld=cout, res_ld=cout,
                  res_c=cout, res_pool=pool, res_h=rh, res_w=rw)
        return emu.sis3d_enet_conv2d(C.byref(a), None)

    for pool, rh, rw in ((0, Ho + 1, Wo), (0, Ho, Wo - 1), (1, 2 * Ho - 1, 2 * Wo), (1, 2 * Ho, 2 * Wo + 2), (1, 2 * Ho + 2, 2 * Wo),
                         (1, 0, 2 * Wo), (0, Ho, 0)):
        assert run(pool, rh, rw) == -1, (pool, rh, rw)
    assert bool((out == 7.0).all())
    # 0 x 0: the extent of callers that predate res_h / res_w (Ho x Wo, or 2Ho x 2Wo pooled)
    for pool, rh, rw in ((0, Ho, Wo), (1, 2 * Ho, 2 * Wo), (1, 2 * Ho + 1, 2 * Wo + 1), (0, 0, 0), (1, 0, 0)):
        assert run(pool, rh, rw) == 0, (pool, rh, rw)
    assert bool((out == 0.0).all())


def test_conv_struct_keeps_its_layout():
    """res_h / res_w took the place of the trailing int32 `reserved`: the struct keeps its size and every other offset, so a
    caller built against the earlier layout (reserved = 0) still runs, with the even residual extent it assumed."""
    assert C.sizeof(_Conv) == 160
    assert _Conv.res_pool.offset == 152 and _Conv.res_h.offset == 156 and _Conv.res_w.offset == 158
