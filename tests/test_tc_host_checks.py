"""Return codes of the tensor-core conv / fused / GEMM / fp16 entry points (3d-sis_b200/csrc/conv_tc.cu) for rejected
arguments, including which code wins when several apply.

The CPU table holds only arguments rejected before the driver's tensor-map encoder is looked up, so no row touches the
device or a pointer: the pointers are aligned fake addresses, never dereferenced.  Codes decided after that lookup (a linear
workspace below the documented size, an fp16 row width the kernel has no form for, an empty tile list) are in the
gpu-marked test at the end."""
import ctypes as C

import pytest

OK, EINVAL, EWORKSPACE, EUNSUPPORTED = 0, -1, -3, -4

P, I, Z = C.c_void_p, C.c_int, C.c_size_t
CONV = [("in", P), ("w", P), ("bias", P), ("res", P), ("res_ld", I), ("res_coff", I), ("out", P), ("out_ld", I),
        ("out_coff", I), ("X", I), ("Y", I), ("Z", I), ("cin", I), ("cout", I), ("ks", I)]
CONV_TAIL = [("act", I), ("stream", P)]
TILES = [("tiles", P), ("n_tiles", I)]
FUSED = [("in", P), ("w", P), ("bias2", P), ("w3", P), ("bias3", P), ("res", P), ("res_ld", I), ("res_coff", I), ("out", P),
         ("out_ld", I), ("out_coff", I), ("X", I), ("Y", I), ("Z", I), ("cin", I), ("cmid", I), ("cout", I), ("act", I),
         ("stream", P)]
LINEAR = [("x", P), ("w", P), ("bias", P), ("y", P), ("M", I), ("K", I), ("N", I), ("act", I), ("ws", P), ("ws_bytes", Z),
          ("stream", P)]
SPLIT = [("in", P), ("w", P), ("bias", P), ("out_split", P), ("X", I), ("Y", I), ("Z", I), ("cin", I), ("cout", I), ("act", I),
         ("stream", P)]
F16 = [("in", P), ("w", P), ("bias", P), ("res", P), ("res_ld", I), ("res_coff", I), ("out", P), ("out16", P), ("out_ld", I),
       ("out_coff", I), ("X", I), ("Y", I), ("Z", I), ("cin", I), ("cout", I), ("ks", I)] + TILES + CONV_TAIL

ENTRY = {  # entry point -> (signature, family)
    "sis3d_conv3d_k3_tc": (CONV + TILES + CONV_TAIL, "conv"),
    "sis3d_conv3d_k3_tc_x3": (CONV + CONV_TAIL, "conv"),
    "sis3d_conv3d_k3_tc_h3": (CONV + CONV_TAIL, "conv"),
    "sis3d_conv3d_k1_tc_h3_split": (SPLIT, "split"),
    "sis3d_conv3d_k3_tc_fused": (FUSED, "fused"),
    "sis3d_conv3d_k3_tc_fused_x3": (FUSED, "fused"),
    "sis3d_conv3d_k3_tc_fused_h3": (FUSED, "fused"),
    "sis3d_conv3d_k3_tc_fused_h3_split": (FUSED, "fused"),
    "sis3d_linear_tc": (LINEAR, "linear"),
    "sis3d_linear_tc_x3": (LINEAR, "linear"),
    "sis3d_linear_tc_h3": (LINEAR, "linear"),
    "sis3d_conv3d_tc_f16": (F16, "f16"),
}

_ptrs = iter(range(0x10000000, 0x20000000, 0x100000))
BASE = {  # arguments every check accepts: distinct 16-byte-aligned fake pointers, a supported layer
    "in": next(_ptrs), "w": next(_ptrs), "w3": next(_ptrs), "bias": next(_ptrs), "bias2": next(_ptrs), "bias3": next(_ptrs),
    "res": next(_ptrs), "out": next(_ptrs), "out16": next(_ptrs), "out_split": next(_ptrs), "x": next(_ptrs), "y": next(_ptrs),
    "ws": next(_ptrs), "tiles": None, "stream": None,
    "res_ld": 64, "res_coff": 0, "out_ld": 64, "out_coff": 0, "X": 8, "Y": 8, "Z": 8, "cin": 64, "cmid": 32, "cout": 64, "ks": 3,
    "n_tiles": 0, "act": 1, "M": 8, "K": 64, "N": 64, "ws_bytes": 1 << 40,
}
TILE_LIST = next(_ptrs)

ALL = ("conv", "split", "fused", "linear", "f16")
CONVS = ("conv", "split", "fused", "f16")
# (case id, families or entry points it applies to, argument changes, expected code); "+4" offsets a pointer by 4 bytes
CASES = [
    ("null_in", ("conv", "split", "fused", "f16"), {"in": None}, EINVAL),
    ("null_w", CONVS, {"w": None}, EINVAL),
    ("null_w3", ("fused",), {"w3": None}, EINVAL),
    ("null_out", ("conv", "fused"), {"out": None}, EINVAL),
    ("null_out_split", ("split",), {"out_split": None}, EINVAL),
    ("null_out32_and_out16", ("f16",), {"out": None, "out16": None}, EINVAL),
    ("null_x", ("linear",), {"x": None}, EINVAL),
    ("null_w_linear", ("linear",), {"w": None}, EINVAL),
    ("null_y", ("linear",), {"y": None}, EINVAL),
    ("null_workspace", ("linear",), {"ws": None}, EINVAL),
    ("X0", CONVS, {"X": 0}, EINVAL),
    ("Y_negative", CONVS, {"Y": -1}, EINVAL),
    ("Z0", CONVS, {"Z": 0}, EINVAL),
    ("cin0", CONVS, {"cin": 0}, EINVAL),
    ("cout0", CONVS, {"cout": 0}, EINVAL),
    ("cmid0", ("fused",), {"cmid": 0}, EINVAL),
    ("M0", ("linear",), {"M": 0}, EINVAL),
    ("K_negative", ("linear",), {"K": -32}, EINVAL),
    ("N0", ("linear",), {"N": 0}, EINVAL),
    ("ks0", ("conv", "f16"), {"ks": 0}, EINVAL),
    ("ks4", ("conv", "f16"), {"ks": 4}, EINVAL),
    ("ks2_f16", ("f16",), {"ks": 2}, EINVAL),
    ("ks2_extent1", ("conv",), {"ks": 2, "Y": 1}, EINVAL),
    ("ks2_tiles", ("sis3d_conv3d_k3_tc",), {"ks": 2, "tiles": TILE_LIST, "n_tiles": 4}, EINVAL),
    ("ks2_tiles_unsupported_cin", ("sis3d_conv3d_k3_tc",), {"ks": 2, "tiles": TILE_LIST, "n_tiles": 4, "cin": 48}, EINVAL),
    ("cin48", ("conv", "split", "fused", "f16"), {"cin": 48}, EUNSUPPORTED),
    ("cout48", ("conv", "f16"), {"cout": 48}, EUNSUPPORTED),
    ("cout96", ("conv", "f16"), {"cout": 96}, EUNSUPPORTED),
    ("cout48_split", ("split",), {"cout": 48}, EINVAL),  # the split-pair output needs whole 32-channel slices, checked first
    ("cout96_split", ("split",), {"cout": 96}, EUNSUPPORTED),
    ("cmid32_cout128", ("fused",), {"cmid": 32, "cout": 128}, EUNSUPPORTED),
    ("cmid64_cout64", ("fused",), {"cmid": 64, "cout": 64}, EUNSUPPORTED),
    ("cmid48", ("fused",), {"cmid": 48}, EUNSUPPORTED),
    ("K48", ("linear",), {"K": 48}, EUNSUPPORTED),
    ("N96", ("linear",), {"N": 96}, EUNSUPPORTED),
    ("in_misaligned", ("conv", "split", "fused", "f16"), {"in": "+4"}, EINVAL),
    ("w_misaligned", ALL, {"w": "+4"}, EINVAL),
    ("w3_misaligned", ("fused",), {"w3": "+4"}, EINVAL),
    ("out_misaligned", ("conv", "fused", "f16"), {"out": "+4"}, EINVAL),
    ("out16_misaligned", ("f16",), {"out16": "+4"}, EINVAL),
    ("out_split_misaligned", ("split",), {"out_split": "+4"}, EINVAL),
    ("x_misaligned", ("linear",), {"x": "+4"}, EINVAL),
    ("workspace_misaligned", ("linear",), {"ws": "+4"}, EINVAL),
    ("misaligned_unsupported", ("conv", "fused", "f16"), {"in": "+4", "cout": 48}, EUNSUPPORTED),
    ("misaligned_unsupported_linear", ("linear",), {"x": "+4", "N": 48}, EUNSUPPORTED),
    ("null_unsupported", CONVS, {"w": None, "cin": 48}, EINVAL),
    ("null_unsupported_linear", ("linear",), {"w": None, "K": 48}, EINVAL),
    ("out_ld_odd", ("conv", "fused", "f16"), {"out_ld": 66}, EINVAL),
    ("out_coff_odd", ("conv", "fused", "f16"), {"out_coff": 2}, EINVAL),
    ("res_ld_odd", ("conv", "fused", "f16"), {"res_ld": 6}, EINVAL),
    ("res_coff_odd", ("conv", "fused", "f16"), {"res_coff": 1}, EINVAL),
    ("ld_odd_unsupported", ("conv", "fused", "f16"), {"out_ld": 66, "cin": 48}, EUNSUPPORTED),
    ("f16_cin96_misaligned", ("f16",), {"cin": 96, "out16": "+4"}, EINVAL),
    ("f16_cin96_ld_odd", ("f16",), {"cin": 96, "res_coff": 2}, EINVAL),
]


@pytest.fixture(scope="module")
def lib():
    from lib import _sis3d as S
    return C.CDLL(S.lib._name)  # a handle of its own: the argtypes set here do not leak into lib._sis3d


def call(lib, name, changes, base=BASE):
    sig, _ = ENTRY[name]
    fn = getattr(lib, name)
    fn.argtypes = [t for _, t in sig]
    fn.restype = C.c_int
    args = []
    for arg, _ in sig:
        v = changes.get(arg, base[arg])
        args.append(base[arg] + 4 if v == "+4" else v)
    return fn(*args)


def rows():
    for cid, fams, changes, code in CASES:
        for name, (sig, fam) in ENTRY.items():
            if fam in fams or name in fams:
                assert set(changes) <= {a for a, _ in sig}, (cid, name)
                yield pytest.param(name, changes, code, id=f"{name}-{cid}")


@pytest.mark.parametrize("name,changes,code", list(rows()))
def test_rejected_arguments(lib, name, changes, code):
    assert call(lib, name, changes) == code


def test_every_entry_point_has_rows():
    assert {p.values[0] for p in rows()} == set(ENTRY)


@pytest.mark.gpu
def test_codes_after_the_encoder_lookup(lib):
    """Decided after the driver's tensor-map encoder is found: no row launches a kernel or touches its fake pointers."""
    from lib import _sis3d as S
    need = S.lib.sis3d_linear_tc_workspace_bytes(BASE["M"], BASE["N"], BASE["K"])
    assert need > 0
    for name in ("sis3d_linear_tc", "sis3d_linear_tc_x3", "sis3d_linear_tc_h3"):  # the documented size, in every mode
        assert call(lib, name, {"ws_bytes": need - 1}) == EWORKSPACE, name
        assert call(lib, name, {"ws_bytes": 0, "K": 48}) == EUNSUPPORTED, name  # the shape check comes first
    # fp16 rows are 32 channels or a multiple of 64
    assert call(lib, "sis3d_conv3d_tc_f16", {"cin": 96}) == EUNSUPPORTED
    assert call(lib, "sis3d_conv3d_tc_f16", {"cin": 160, "ks": 1}) == EUNSUPPORTED
    # an empty tile list is a successful call that launches nothing (its tensor maps are encoded first, on real memory)
    import torch
    buf = torch.zeros(1 << 20, device="cuda")
    real = {k: (buf.data_ptr() if isinstance(v, int) and 0x10000000 <= v < 0x20000000 else v) for k, v in BASE.items()}
    n0 = S.launch_count()
    for name in ("sis3d_conv3d_k3_tc", "sis3d_conv3d_tc_f16"):
        assert call(lib, name, {"tiles": buf.data_ptr(), "n_tiles": 0}, real) == OK, name
    torch.cuda.synchronize()
    assert S.launch_count() == n0
