"""ctypes binding of libsis3d.so (C ABI declared in include/sis3d.h).

PyTorch is used for device memory, streams and torch.distributed only; every kernel on the hot path
lives in libsis3d.so.  There is NO fallback: if the library is missing the import fails loudly, and
every wrapper raises on CPU tensors.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsis3d.so")


class Sis3dError(RuntimeError):
    pass


if not os.path.exists(_LIB_PATH):
    raise ImportError(f"{_LIB_PATH} not found: build it with `python __graft_entry__.py build` "
                      "(or `make -C 3d-sis_b200/csrc`); there is no CPU/PyTorch fallback for the hot path")
lib = C.CDLL(_LIB_PATH)


class Region(C.Structure):
    """struct sis3d_region (include/sis3d.h)."""
    _fields_ = [("in_off", C.c_int64), ("out_off", C.c_int64), ("res_off", C.c_int64),
                ("in_dim", C.c_int32 * 3), ("out_dim", C.c_int32 * 3), ("in_stride", C.c_int64 * 3),
                ("out_stride", C.c_int64 * 3), ("tile_begin", C.c_int32), ("pad_", C.c_int32)]


class RpnLevel(C.Structure):
    """struct sis3d_rpn_level (include/sis3d.h)."""
    _fields_ = [("cls", C.c_void_p), ("deltas", C.c_void_p), ("anchor_sizes", C.c_void_p),
                ("grid", C.c_int32 * 3), ("num_anchors", C.c_int32), ("cls_mode", C.c_int32), ("cls_ld", C.c_int32),
                ("deltas_ld", C.c_int32), ("pad_", C.c_int32)]


class MaskPlan(C.Structure):
    """struct sis3d_mask_plan (include/sis3d.h)."""
    _fields_ = [("n_kept", C.c_int32), ("canvas", C.c_int32 * 3), ("n_tiles_tc", C.c_int32), ("tiles_first", C.c_int32),
                ("tiles_last", C.c_int32), ("tiles_mid", C.c_int32), ("total_voxels", C.c_int64), ("off_first", C.c_int64),
                ("off_last", C.c_int64), ("off_rest", C.c_int64), ("off_offs", C.c_int64), ("off_cls", C.c_int64),
                ("off_kept", C.c_int64), ("off_sizes", C.c_int64), ("bytes", C.c_int64)]


class MaskStage(C.Structure):
    """struct sis3d_mask_stage (include/sis3d.h)."""
    _fields_ = [("scene", C.c_void_p), ("X", C.c_int32), ("Y", C.c_int32), ("Z", C.c_int32), ("ncls", C.c_int32),
                ("math", C.c_int32), ("reserved", C.c_int32), ("w_first", C.c_void_p), ("w_last", C.c_void_p),
                ("w_mid", C.c_void_p * 4), ("tables", C.c_void_p), ("canvas", C.c_void_p), ("canvas_bytes", C.c_size_t),
                ("canvas32", C.c_void_p), ("canvas32_bytes", C.c_size_t), ("masks", C.c_void_p), ("bits", C.c_void_p),
                ("bits_host", C.c_void_p), ("thresh", C.c_float), ("reserved2", C.c_int32)]


class MaskColorPlan(C.Structure):
    """struct sis3d_mask_color_plan (include/sis3d.h)."""
    _fields_ = [("off_crops", C.c_int64), ("off_g2c", C.c_int64), ("off_last128", C.c_int64), ("off_c0", C.c_int64),
                ("off_c128", C.c_int64), ("bytes", C.c_int64)]


class MaskStageColor(C.Structure):
    """struct sis3d_mask_stage_color (include/sis3d.h)."""
    _fields_ = [("scene", C.c_void_p), ("X", C.c_int32), ("Y", C.c_int32), ("Z", C.c_int32), ("ncls", C.c_int32),
                ("math", C.c_int32), ("only_images", C.c_int32), ("w_geom_first", C.c_void_p), ("w_geom_last", C.c_void_p),
                ("w_geom_mid", C.c_void_p * 4), ("w_color_first", C.c_void_p), ("w_color_mid", C.c_void_p * 4),
                ("w_color_last", C.c_void_p), ("w_combine", C.c_void_p), ("w_combine_last", C.c_void_p), ("feats_t", C.c_void_p),
                ("pix", C.c_void_p), ("pairs", C.c_void_p), ("n_pairs", C.c_void_p), ("n_views", C.c_int32), ("hw", C.c_int32),
                ("crop_in", C.c_void_p), ("tables", C.c_void_p), ("canvas", C.c_void_p), ("canvas_bytes", C.c_size_t),
                ("canvas32", C.c_void_p), ("canvas32_bytes", C.c_size_t), ("masks", C.c_void_p), ("bits", C.c_void_p),
                ("bits_host", C.c_void_p), ("thresh", C.c_float), ("reserved", C.c_int32)]


REGION_BYTES = C.sizeof(Region)
TILE_M = 64

# every exported symbol of include/sis3d.h (checked by tests/test_abi.py)
SYMBOLS = ["sis3d_strerror", "sis3d_version", "sis3d_launch_count", "sis3d_nms_workspace_bytes", "sis3d_nms",
           "sis3d_roi_pool_fwd", "sis3d_roi_pool_levels", "sis3d_view_params_host", "sis3d_project_map", "sis3d_project_compact",
           "sis3d_project_compact_workspace_bytes", "sis3d_backproject_pairs", "sis3d_project_scatter_lists",
           "sis3d_backproject_max", "sis3d_backproject_conv_k2s2_workspace_bytes", "sis3d_backproject_conv_k2s2",
           "sis3d_pack_conv_weight", "sis3d_conv3d", "sis3d_maxpool3",
           "sis3d_vc_to_ncdhw", "sis3d_pack_conv_weight_tc_f16", "sis3d_cast_f16", "sis3d_conv3d_tc_f16", "sis3d_conv3d_ex",
           "sis3d_backproject_conv_k2s2_ex", "sis3d_linear_workspace_bytes", "sis3d_linear", "sis3d_linear_tc_supported", "sis3d_linear_tc_workspace_bytes", "sis3d_linear_tc", "sis3d_mlp_tail", "sis3d_pack_conv_weight_tc", "sis3d_conv3d_k3_tc_supported", "sis3d_conv3d_tc_brick", "sis3d_conv3d_k3_tc",
           "sis3d_conv3d_k3_tc_fused_supported", "sis3d_conv3d_k3_tc_fused",
           "sis3d_rpn_workspace_bytes", "sis3d_rpn_proposals", "sis3d_detect_decode", "sis3d_mask_plan_build", "sis3d_mask_stage_launch", "sis3d_memcpy_async",
           "sis3d_mask_color_plan_build", "sis3d_mask_color_gather", "sis3d_mask_color_feats_t", "sis3d_mask_stage_color_launch",
           "sis3d_mask_select", "sis3d_pack_conv_weight_tc_x3", "sis3d_conv3d_k3_tc_x3", "sis3d_conv3d_k3_tc_fused_x3",
           "sis3d_linear_tc_x3", "sis3d_pack_conv_weight_tc_h3", "sis3d_conv3d_k3_tc_h3", "sis3d_conv3d_k3_tc_fused_h3",
           "sis3d_linear_tc_h3", "sis3d_chunk_decode", "sis3d_conv3d_k1_tc_h3_split", "sis3d_conv3d_k3_tc_fused_h3_split", "sis3d_mask_overlap",
           "sis3d_instance_paint", "sis3d_vertex_instance_overlap", "sis3d_segment_gt_slots", "sis3d_voxel_mesh_count",
           "sis3d_voxel_mesh",
           "sis3d_ply_ascii_lengths", "sis3d_ply_ascii"]
# include/sis3d_enet.h
SYMBOLS_ENET = ["sis3d_enet_pack_weight", "sis3d_enet_conv2d", "sis3d_enet_pool_affine", "sis3d_enet_to_nchw"]

lib.sis3d_strerror.restype = C.c_char_p
lib.sis3d_launch_count.restype = C.c_int64
lib.sis3d_nms_workspace_bytes.restype = C.c_size_t
lib.sis3d_rpn_workspace_bytes.restype = C.c_size_t
lib.sis3d_linear_workspace_bytes.restype = C.c_size_t
lib.sis3d_linear_tc_workspace_bytes.restype = C.c_size_t
lib.sis3d_backproject_conv_k2s2_workspace_bytes.restype = C.c_size_t
lib.sis3d_project_compact_workspace_bytes.restype = C.c_size_t


def check(rc: int, what: str = ""):
    if rc != 0:
        raise Sis3dError(f"libsis3d {what} failed: {lib.sis3d_strerror(rc).decode()} (code {rc})")


def ptr(t):
    """Device pointer of a CUDA tensor (or None)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise Sis3dError("libsis3d operates on CUDA tensors only (no CPU fallback)")
    return C.c_void_p(t.data_ptr())


_pinned_stream = [None]


def stream():
    """cudaStream_t of torch's current stream (cached while a Network stream slot is active: the lookup costs ~15 us)."""
    s = _pinned_stream[0]
    return s if s is not None else C.c_void_p(torch.cuda.current_stream().cuda_stream)


def pin_stream(handle):
    """Fix the stream handle returned by stream() (None = look it up on every call).  Returns the previous value."""
    old = _pinned_stream[0]
    _pinned_stream[0] = handle
    return old


def launch_count() -> int:
    return int(lib.sis3d_launch_count())


def f32(x):
    return C.c_float(float(x))


import numpy as _np

REGION_DTYPE = _np.dtype({"names": ["in_off", "out_off", "res_off", "in_dim", "out_dim", "in_stride", "out_stride", "tile_begin", "pad_"],
                          "formats": ["<i8", "<i8", "<i8", ("<i4", 3), ("<i4", 3), ("<i8", 3), ("<i8", 3), "<i4", "<i4"],
                          "offsets": [0, 8, 16, 24, 36, 48, 72, 96, 100], "itemsize": 104})


def regions_array(in_off, out_off, in_dim, out_dim, in_stride, out_stride=None):
    """Vectorised builder of a sis3d_region table (numpy structured array matching the C struct) + tile count."""
    n = len(in_off)
    a = _np.zeros(n, dtype=REGION_DTYPE)
    a["in_off"], a["out_off"] = in_off, out_off
    a["in_dim"], a["out_dim"], a["in_stride"] = in_dim, out_dim, in_stride
    if out_stride is not None:
        a["out_stride"] = out_stride
    m = _np.prod(_np.asarray(out_dim, dtype=_np.int64).reshape(n, 3), axis=1)
    t = (m + TILE_M - 1) // TILE_M
    a["tile_begin"] = _np.concatenate([[0], _np.cumsum(t)[:-1]])
    return a, int(t.sum())


def make_regions(entries, device):
    """entries: list of dict(in_off,out_off,res_off,in_dim,out_dim,in_stride) -> (device uint8 tensor, n_tiles)."""
    arr = (Region * len(entries))()
    tiles = 0
    for i, e in enumerate(entries):
        r = arr[i]
        r.in_off, r.out_off, r.res_off = int(e["in_off"]), int(e["out_off"]), int(e.get("res_off", 0))
        for k in range(3):
            r.in_dim[k], r.out_dim[k], r.in_stride[k] = int(e["in_dim"][k]), int(e["out_dim"][k]), int(e["in_stride"][k])
            r.out_stride[k] = int(e["out_stride"][k]) if "out_stride" in e else 0
        r.tile_begin = tiles
        m = int(e["out_dim"][0]) * int(e["out_dim"][1]) * int(e["out_dim"][2])
        tiles += (m + TILE_M - 1) // TILE_M
    host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
    return host.to(device), tiles
