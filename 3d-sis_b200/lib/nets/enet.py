"""ENet encoder executor over the sis3d_enet_* entry points of libsis3d.so (SURVEY row f2; reference: lib/nets/enet.py:130-590,
create_enet_for_3d :697-715; lib/nets/network.py:199-213 is where the features enter the 3-D network).

`Network` builds one when cfg.USE_IMAGES and not cfg.USE_IMAGES_GT, from the `image_enet_fixed.*` / `image_enet_trainable.*`
entries of its state_dict (same names as the reference), so raw images [n,3,H,W] (even H and W; cfg.IMAGE_SHAPE, 256x328 by
default) are a valid input of the hot path.  The host side (lib/nets/enet_program.py: BatchNorm folding into a flat conv
program) is checked on the CPU against the unmodified reference; the kernels against tests/golden/enet_encoder.npz on the
GPU (tests/test_gpu_enet.py) and launch by launch against fp64 (tests/test_gpu_enet_stage.py).

Every bottleneck is three (asymmetric: four) launches of one fp32 implicit-GEMM kernel with bias / residual / PReLU fused in
the epilogue; the down-sampling skip (floor-mode 2x2 max-pool + zero channel padding) is read inside the last conv's epilogue."""
from __future__ import annotations

import ctypes as C

import torch

from lib.nets.enet_program import compile_enet


class _Conv(C.Structure):
    _fields_ = [("inp", C.c_void_p), ("in_sn", C.c_int64), ("in_sy", C.c_int64), ("in_sx", C.c_int64), ("in_sc", C.c_int64),
                ("w", C.c_void_p), ("bias", C.c_void_p), ("slope", C.c_void_p), ("res", C.c_void_p), ("out", C.c_void_p),
                ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("cin", C.c_int32), ("Ho", C.c_int32), ("Wo", C.c_int32),
                ("cout", C.c_int32), ("ldw", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("stride", C.c_int32),
                ("pad_y", C.c_int32), ("pad_x", C.c_int32), ("dil", C.c_int32), ("out_ld", C.c_int32), ("out_coff", C.c_int32),
                ("res_ld", C.c_int32), ("res_c", C.c_int32), ("res_pool", C.c_int32), ("res_h", C.c_int16),
                ("res_w", C.c_int16)]


class EnetEncoder:
    def __init__(self, params, device, lib=None):
        """lib: object with the four sis3d_enet_* entry points (default: libsis3d.so).  tests/test_enet_executor.py passes a
        numpy model of the C contract (include/sis3d_enet.h) with device='cpu' to check this executor's wiring without a GPU."""
        self.dev = torch.device(device)
        self._S = None
        if lib is None:
            if self.dev.type != "cuda":
                raise RuntimeError("libsis3d.so operates on CUDA memory (no CPU fallback)")
            from lib import _sis3d as S  # raises loudly when the library is missing
            lib, self._S = S.lib, S
        self.lib = lib
        self.ops = []
        stream = self._stream()
        for op in compile_enet([p.float().cpu() for p in params]):
            if op[0] == "conv":
                _, w, b, stride, pad, dil, slope, src, dst = op
                cout, cin, kh, kw = w.shape
                wd = w.contiguous().to(self.dev)
                packed = torch.empty(kh * kw * cin, (cout + 3) // 4 * 4, device=self.dev)
                self._check(self.lib.sis3d_enet_pack_weight(C.c_void_p(wd.data_ptr()), cout, cin, kh, kw, C.c_void_p(packed.data_ptr()),
                                                            stream))
                self.ops.append(dict(kind="conv", w=packed, bias=b.contiguous().to(self.dev),
                                     slope=None if slope is None else slope.contiguous().to(self.dev), cout=cout, cin=cin, kh=kh,
                                     kw=kw, stride=stride, pad=pad, dil=dil))
            elif op[0] == "affine_prelu":
                self.ops.append(dict(kind="affine", scale=op[1].contiguous().to(self.dev), shift=op[2].contiguous().to(self.dev),
                                     slope=op[3].contiguous().to(self.dev)))
            elif op[0] == "add_prelu":
                self.ops.append(dict(kind="add", slope=op[3].contiguous().to(self.dev), cout=op[5]))
            elif op[0] == "pool":
                self.ops.append(dict(kind="pool"))
        if self.dev.type == "cuda":
            torch.cuda.current_stream().synchronize()

    def _stream(self):
        if self._S is not None:
            return self._S.stream()  # honours the stream slot pinned by the scene loop
        return C.c_void_p(torch.cuda.current_stream().cuda_stream) if self.dev.type == "cuda" else None

    @staticmethod
    def _check(rc):
        if rc != 0:
            raise RuntimeError(f"libsis3d ENet call failed (code {rc})")

    def _conv(self, op, x, strides, n, h, w, out, out_ld, out_coff, res=None, res_c=0, res_ld=0, res_pool=0, slope=None):
        a = _Conv()
        a.inp, (a.in_sn, a.in_sy, a.in_sx, a.in_sc) = x.data_ptr(), strides
        a.w, a.bias = op["w"].data_ptr(), op["bias"].data_ptr()
        sl = slope if slope is not None else op["slope"]
        a.slope = sl.data_ptr() if sl is not None else None
        a.res = res.data_ptr() if res is not None else None
        a.out = out.data_ptr()
        ho = (h + 2 * op["pad"][0] - op["dil"] * (op["kh"] - 1) - 1) // op["stride"] + 1
        wo = (w + 2 * op["pad"][1] - op["dil"] * (op["kw"] - 1) - 1) // op["stride"] + 1
        a.N, a.H, a.W, a.cin, a.Ho, a.Wo, a.cout, a.ldw = n, h, w, op["cin"], ho, wo, op["cout"], op["w"].shape[1]
        a.kh, a.kw, a.stride, a.pad_y, a.pad_x, a.dil = op["kh"], op["kw"], op["stride"], op["pad"][0], op["pad"][1], op["dil"]
        a.out_ld, a.out_coff, a.res_ld, a.res_c, a.res_pool = out_ld, out_coff, res_ld, res_c, res_pool
        if res is not None:
            a.res_h, a.res_w = res.shape[1], res.shape[2]  # the pooled skip's input may have an odd height / width
        self._check(self.lib.sis3d_enet_conv2d(C.byref(a), self._stream()))
        return ho, wo

    def __call__(self, images):
        """images: float32 CUDA [n,3,H,W] (normalised RGB) -> features [n,128,H/8,W/8] (NCHW, as network.py:199-213 expects)."""
        if images.dim() == 4 and max(images.shape[2:]) > 65534:  # the residual extents are int16 in sis3d_enet_conv
            raise ValueError(f"ENet encoder: images up to 65534 x 65534 pixels, got {tuple(images.shape)}")
        if images.dim() != 4 or images.shape[1] != 3 or images.shape[2] % 2 or images.shape[3] % 2:
            # the initial block concatenates a 3x3/s2 conv (ceil(H/2) rows) with a 2x2/s2 max-pool (floor(H/2) rows): the
            # reference cannot run an odd height or width, and here the conv would write past the pooled half's rows
            raise ValueError(f"ENet encoder: images must be [n, 3, H, W] with even H and W, got {tuple(images.shape)}")
        x_img = images.to(self.dev, torch.float32).contiguous()
        n, _, H, W = x_img.shape
        ops = iter(self.ops)
        nhwc = lambda t, c: (t.shape[1] * t.shape[2] * c, t.shape[2] * c, c, 1)
        # initial block: conv 3->13 || pool + affine + PReLU, both writing their channel slice of the 16-channel tensor
        op = next(ops)
        h, w = H // 2, W // 2
        x = torch.empty(n, h, w, 16, device=self.dev)
        self._conv(op, x_img, (3 * H * W, W, 1, H * W), n, H, W, x, 16, 0)
        next(ops)  # pool
        af = next(ops)
        self._check(self.lib.sis3d_enet_pool_affine(C.c_void_p(x_img.data_ptr()), 3 * H * W, W, 1, H * W, n, H, W, 3,
                                                    C.c_void_p(af["scale"].data_ptr()), C.c_void_p(af["shift"].data_ptr()),
                                                    C.c_void_p(af["slope"].data_ptr()), C.c_void_p(x.data_ptr()), 16, 13, self._stream()))
        c = 16
        pending = []
        for op in ops:  # bottlenecks: conv1, conv2 (or the 1x5 / 5x1 pair), conv3 [+ pool] + add_prelu
            if op["kind"] != "add":
                pending.append(op)
                continue
            convs = [o for o in pending if o["kind"] == "conv"]
            down = any(o["kind"] == "pool" for o in pending)
            pending = []
            mid = convs[0]["cout"]
            y = torch.empty(n, h // (2 if down else 1), w // (2 if down else 1), mid, device=self.dev)
            hh, ww = self._conv(convs[0], x, nhwc(x, c), n, h, w, y, mid, 0)
            for cv in convs[1:-1]:
                y2 = torch.empty_like(y)
                self._conv(cv, y, nhwc(y, mid), n, hh, ww, y2, mid, 0)
                y = y2
            cout = op["cout"]
            xn = torch.empty(n, hh, ww, cout, device=self.dev)
            self._conv(convs[-1], y, nhwc(y, mid), n, hh, ww, xn, cout, 0, res=x, res_c=c, res_ld=c, res_pool=1 if down else 0,
                       slope=op["slope"])
            x, c, h, w = xn, cout, hh, ww
        out = torch.empty(n, c, h, w, device=self.dev)
        self._check(self.lib.sis3d_enet_to_nchw(C.c_void_p(x.data_ptr()), c, 0, n, C.c_int64(h * w), c, C.c_void_p(out.data_ptr()),
                                                self._stream()))
        return out
