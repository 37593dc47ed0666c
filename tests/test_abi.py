"""CPU-only: the C-ABI library loads and exports every symbol include/sis3d.h declares."""
import os
import re

from conftest import ROOT


def test_header_symbols_exported():
    from lib import _sis3d as S
    hdr = open(os.path.join(ROOT, "include", "sis3d.h")).read()
    declared = set(re.findall(r"\b(sis3d_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    missing = [s for s in sorted(declared) if not hasattr(S.lib, s)]
    assert not missing, f"declared in sis3d.h but not exported by libsis3d.so: {missing}"
    assert set(S.SYMBOLS) <= declared
    assert S.lib.sis3d_version() >= 100
    assert S.lib.sis3d_strerror(-3).decode() == "workspace too small"


def test_enet_header_symbols_exported():
    from lib import _sis3d as S
    hdr = open(os.path.join(ROOT, "include", "sis3d_enet.h")).read()
    declared = set(re.findall(r"\b(sis3d_enet_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(S.SYMBOLS_ENET)
    assert not [s for s in sorted(declared) if not hasattr(S.lib, s)]


def test_enet_state_dict_contract():
    """USE_IMAGES_GT=False: the 2-D encoder's parameters and BatchNorm buffers appear under the reference's state_dict names
    (lib/nets/enet_keys.py, generated from the unmodified reference) with the reference's shapes, in its order."""
    from lib.nets.enet_keys import ENET_KEYS
    from lib.utils.config import cfg, cfg_from_file, cfg_reset
    cfg_reset()
    cfg_from_file(os.path.join(ROOT, "3d-sis_b200", "experiments", "cfgs", "ScanNet", "rpn_class_mask_5.yml"))
    cfg.NUM_CLASSES, cfg.USE_IMAGES, cfg.USE_IMAGES_GT = 19, True, False
    from lib.nets import backbones
    net = getattr(backbones, cfg.NET)()
    net.init_modules()
    sd = net.state_dict()
    enet_keys = [k for k in sd if k.startswith("image_enet_")]
    assert enet_keys == [k[0] for k in ENET_KEYS]
    for name, shape, kind, dt in ENET_KEYS:
        want = (int(cfg.NUM_2D_CLASSES),) + tuple(shape[1:]) if name.startswith("image_enet_classification") else tuple(shape)
        assert tuple(sd[name].shape) == want, name
    assert len(net._enet_names) == 429  # encoder tensors the kernels consume (no num_batches_tracked, no classifier)
    cfg_reset()


def test_region_struct_layout():
    from lib import _sis3d as S
    assert S.REGION_BYTES == 104  # 3*8 + 3*4 + 3*4 + 3*8 + 3*8 + 4 + 4


def test_no_cpu_fallback():
    import pytest
    import torch
    from lib import _sis3d as S
    from lib.layer_utils.nms_wrapper import nms
    with pytest.raises(S.Sis3dError):
        nms(torch.zeros(4, 6), 0.5)


def test_state_dict_contract():
    """Parameter names/shapes equal the reference's state_dict (SURVEY 8b)."""
    import sis3d_synth as synth
    from lib.utils.config import cfg, cfg_from_file, cfg_reset
    cfg_reset()
    cfg_from_file(os.path.join(ROOT, "3d-sis_b200", "experiments", "cfgs", "ScanNet", "rpn_class_mask_5.yml"))
    cfg.NUM_CLASSES, cfg.USE_IMAGES_GT = 19, True
    from lib.nets import backbones
    net = backbones.ScanNet_Backbone()
    net.init_modules()
    want = synth.param_shapes()
    got = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    assert got == dict(want)


def test_host_side_queries_and_argument_checks():
    """Pure host entry points answer without a GPU: capability queries, brick shapes, workspace sizes, EINVAL on nulls."""
    import ctypes as C
    from lib import _sis3d as S
    L = S.lib
    # wgmma conv support matrix (cin % 32 == 0, cout in {32, 64, 128k})
    assert [L.sis3d_conv3d_k3_tc_supported(ci, co) for ci, co in ((32, 32), (64, 64), (128, 256), (2, 64), (32, 19), (48, 64))] \
        == [1, 1, 1, 0, 0, 0]
    # fused bottleneck tails: (cmid, cout) in {(32,32), (32,64), (64,128)}
    assert [L.sis3d_conv3d_k3_tc_fused_supported(*t) for t in ((32, 32, 32), (32, 32, 64), (64, 64, 128), (32, 32, 128), (2, 32, 32))] \
        == [1, 1, 1, 0, 0]
    assert L.sis3d_linear_tc_supported(8192, 256) == 1 and L.sis3d_linear_tc_supported(100, 256) == 0
    bx, by, bz = C.c_int32(), C.c_int32(), C.c_int32()
    L.sis3d_conv3d_tc_brick(0, 3, 64, 64, C.byref(bx), C.byref(by), C.byref(bz))
    assert (bx.value, by.value, bz.value) == (8, 2, 8)          # whole volumes
    L.sis3d_conv3d_tc_brick(1, 3, 64, 64, C.byref(bx), C.byref(by), C.byref(bz))
    assert (bx.value, by.value, bz.value) == (4, 4, 8)          # ragged tile lists of the mask head
    assert bx.value * by.value * bz.value == 128
    levels = (S.RpnLevel * 2)()
    for lv, A in zip(levels, (3, 11)):
        lv.grid[0], lv.grid[1], lv.grid[2], lv.num_anchors = 24, 12, 24, A
    for fn, args in ((L.sis3d_nms_workspace_bytes, (400,)), (L.sis3d_rpn_workspace_bytes, (levels, 2, 400)),
                     (L.sis3d_linear_workspace_bytes, (200, 256, 8192)), (L.sis3d_linear_tc_workspace_bytes, (200, 256, 8192))):
        assert 0 < fn(*args) < (1 << 31)
    assert L.sis3d_rpn_workspace_bytes(None, 2, 400) == 0 and L.sis3d_rpn_workspace_bytes(levels, 99, 400) == 0
    # argument validation happens before any CUDA call
    assert L.sis3d_nms(None, 4, C.c_float(0.5), None, None, None, None) == -1
    assert L.sis3d_maxpool3(None, None, 64, 0, 4, 4, 4, 64, None) == -1
    assert L.sis3d_conv3d_k3_tc_fused(None, None, None, None, None, None, 0, 0, None, 64, 0, 8, 8, 8, 32, 32, 64, 1, None) == -1
    assert L.sis3d_mask_stage_launch(None, None, None, None) == -1
    assert L.sis3d_memcpy_async(None, None, C.c_size_t(16), 1, None) == -1
    assert L.sis3d_view_params_host(None, None, None, None, 1, 1, C.c_double(1), C.c_double(1), C.c_double(0), C.c_double(0), 41, 32,
                                    C.c_double(0.1), C.c_double(4.0), 8, 8, 8, None) == -1


def test_zero_and_negative_sizes_are_rejected():
    """cin / cout / K / N / M <= 0: the support predicates say no, the workspace queries return 0 and the entry points return
    SIS3D_EINVAL -- before any division by the tile or chunk count (an integer division by zero kills the caller's process,
    so the calls run in a child)."""
    import subprocess
    import sys
    code = """
import ctypes as C, sys
sys.path[:0] = sys.argv[1:]
from lib import _sis3d as S
L = S.lib
out = []
for a, b in ((0, 32), (32, 0), (-32, 64), (64, -128), (0, 0)):
    out += [L.sis3d_conv3d_k3_tc_supported(a, b), L.sis3d_linear_tc_supported(a, b)]
    out += [L.sis3d_conv3d_k3_tc_fused_supported(min(a, b), 32, 32), L.sis3d_conv3d_k3_tc_fused_supported(32, a, b)]
for m, n, k in ((0, 32, 1024), (-1, 32, 1024), (8, 0, 1024), (8, -128, 1024), (8, 32, 0), (8, 32, -32)):
    out += [L.sis3d_linear_tc_workspace_bytes(m, n, k), L.sis3d_linear_workspace_bytes(m, n, k)]
p = C.c_void_p(16)  # never dereferenced: the size checks come first
for m, k, n in ((8, 0, 32), (8, 1024, 0), (0, 1024, 32), (8, -32, 32)):
    for fn in (L.sis3d_linear_tc, L.sis3d_linear_tc_x3, L.sis3d_linear_tc_h3):
        out.append(fn(p, p, None, p, m, k, n, 0, p, C.c_size_t(1 << 20), None) + 1)
for cin, cout in ((0, 32), (32, 0), (-32, 32)):
    for fn in (L.sis3d_conv3d_k3_tc_x3, L.sis3d_conv3d_k3_tc_h3):
        out.append(fn(p, p, None, None, 0, 0, p, 32, 0, 4, 4, 4, cin, cout, 3, 1, None) + 1)
    out.append(L.sis3d_conv3d_k3_tc(p, p, None, None, 0, 0, p, 32, 0, 4, 4, 4, cin, cout, 3, None, 0, 1, None) + 1)
    out.append(L.sis3d_conv3d_tc_f16(p, p, None, None, 0, 0, p, None, 32, 0, 4, 4, 4, cin, cout, 3, None, 0, 1, None) + 1)
    out.append(L.sis3d_conv3d_k3_tc_fused_h3(p, p, None, p, None, None, 0, 0, p, 32, 0, 4, 4, 4, cin, 32, cout, 1, None) + 1)
print("nonzero", [i for i, v in enumerate(out) if v])
"""
    p = subprocess.run([sys.executable, "-c", code, os.path.join(ROOT, "3d-sis_b200"), ROOT], capture_output=True, text=True,
                       timeout=120)
    assert p.returncode == 0, f"child died (exit {p.returncode}): {p.stderr[-2000:]}"
    assert p.stdout.split("\n")[-2] == "nonzero []", p.stdout
