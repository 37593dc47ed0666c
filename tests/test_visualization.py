"""CPU: the result visualisation tools (tools/visualization.py, tools/scannet_benchmark/visualize_benchmark.py and
proj_label.py) with csrc/ply.cu and csrc/eval.cu compiled for the host by tools/cuda_host_emu.py.

- the golden sets of oracle/make_golden_visualization.py (the reference's own tools): every file byte for byte, the
  palette, and write_bbox's cylinder vertices to <= 2 ulp;
- the device formatter against Python's '{:f}' / '{:d}' on more than 10^6 values (ties, one ulp either side, tiny
  negatives, +-0, subnormals, nan / inf, integers to 2^63), values >= 2^64 through the host route;
- sis3d_voxel_mesh + the formatter against oracle/ply_writer.py on seeded volumes, in one slab and in many;
- the departures listed in the tools' docstrings, and the argument checks of every new entry point."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_golden_visualization as G  # noqa: E402  (the seeded inputs; no reference code involved)
import ply_writer as W  # noqa: E402

GOLDEN = "visualization_reference.npz"
CPU = torch.device("cpu")


@pytest.fixture(scope="module")
def ply_emu_lib(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import cuda_host_emu
    out = str(tmp_path_factory.mktemp("emu_ply") / "libsis3d_ply_emu.so")
    cuda_host_emu.build(out, [os.path.join(ROOT, "3d-sis_b200", "csrc", f) for f in ("eval.cu", "ply.cu")])
    lib = C.CDLL(out)
    lib.sis3d_strerror.restype = C.c_char_p
    return lib


@pytest.fixture
def host_ply(monkeypatch, ply_emu_lib):
    """lib._sis3d pointed at the emulated library, accepting host tensors; the tools' default device is the CPU."""
    from lib import _sis3d as S
    from tools import visualization as V
    monkeypatch.setattr(S, "lib", ply_emu_lib)
    monkeypatch.setattr(S, "ptr", lambda t: None if t is None else C.c_void_p(t.data_ptr()))
    monkeypatch.setattr(S, "stream", lambda: None)
    monkeypatch.setattr(V, "_device", lambda device=None: CPU)
    return S


def golden_bytes(g, key):
    return g[key].tobytes()


# ------------------------------------------------------------------------------------------------------------ golden
@pytest.mark.parametrize("mode", ["results", "result"])
def test_result_folders_equal_reference(host_ply, tmp_path, mode):
    from tools import visualization as V
    g = load_golden(GOLDEN)
    scenes = G.result_scenes()
    G.write_result_scenes(scenes, str(tmp_path))
    V.main(["--path", str(tmp_path), "--mode", mode])
    inputs = {os.path.join(s, n) for s, files in scenes.items() for n in files}
    written = sorted(os.path.relpath(os.path.join(d, f), tmp_path) for d, _, fs in os.walk(tmp_path) for f in fs)
    written = [w for w in written if w not in inputs]
    assert written == list(g["res_files"])
    for rel in written:
        got = (tmp_path / rel).read_bytes()
        assert got == golden_bytes(g, "res__" + rel.replace(os.sep, "__")), rel


def test_slabs_do_not_change_result_files(host_ply, tmp_path):
    """The same files when every file is written in slabs of 1500 lines (several slabs per file, both buffers in turn)."""
    from tools import visualization as V
    g = load_golden(GOLDEN)
    G.write_result_scenes(G.result_scenes(), str(tmp_path))
    V.visualize_results(str(tmp_path), slab_lines=1500)
    for rel in g["res_files"]:
        assert (tmp_path / rel).read_bytes() == golden_bytes(g, "res__" + rel.replace(os.sep, "__")), rel


def test_benchmark_visualisation_equals_reference(host_ply, tmp_path):
    from tools.scannet_benchmark import visualize_benchmark as VB
    g = load_golden(GOLDEN)
    res, scans, out = tmp_path / "res", tmp_path / "scans", tmp_path / "out"
    G.write_benchmark_inputs(G.benchmark_scenes(), str(res), str(scans))
    VB.main(["--result_dir", str(res), "--output_dir", str(out), "--scan_path", str(scans)])
    assert sorted(os.listdir(out)) == list(g["bench_files"])
    for name in g["bench_files"]:
        assert (out / name).read_bytes() == golden_bytes(g, "bench__" + name), name


def test_proj_label_equals_reference(tmp_path):
    from tools.scannet_benchmark import proj_label
    g = load_golden(GOLDEN)
    G.write_benchmark_inputs(G.benchmark_scenes(), str(tmp_path), str(tmp_path / "scans_unused"))
    shutil.rmtree(tmp_path / "scans_unused")
    proj_label.main(["--pred_path", str(tmp_path)])
    names = sorted(k[len("proj__"):] for k in g if k.startswith("proj__"))
    assert names == sorted(f for f in os.listdir(tmp_path) if f.endswith(".txt"))
    for name in names:
        assert (tmp_path / name).read_bytes() == golden_bytes(g, "proj__" + name), name


def test_palette_equals_reference():
    from tools import visualization as V
    g = load_golden(GOLDEN)
    assert np.array_equal(np.array(V.create_color_palette(), np.int64), g["palette"])
    assert np.array_equal(W.PALETTE, g["palette"])


@pytest.mark.parametrize("key", list(G.BBOX_SETS))
def test_bbox_cylinders_equal_reference(key):
    from tools import visualization as V
    g = load_golden(GOLDEN)
    v, c, f = V.write_bbox(G.BBOX_SETS[key](), None)
    want = g[f"bbox_{key}_verts"]
    assert v.shape == want.shape
    assert np.array_equal(np.isnan(v), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.isnan(want).any() or key != "f32"  # the flat box's zero-length edges give nan
    ulp = np.abs(v[ok] - want[ok]) / np.spacing(np.maximum(np.abs(want[ok]), np.finfo(np.float64).tiny))
    assert ulp.max() <= 2, ulp.max()
    assert np.array_equal(c, g[f"bbox_{key}_colors"])
    assert np.array_equal(f, g[f"bbox_{key}_faces"])


# ------------------------------------------------------------------------------------------------------------ formatter
def formatter_values(seed=3):
    """>= 10^6 float64 values with every case the formatter has to get right."""
    rng = np.random.default_rng(seed)
    ties = (2 * rng.integers(-2 ** 40, 2 ** 40, 120000) + 1) / 128.0  # odd multiples of 2^-7: v * 10^6 ends in .5 exactly
    ties = np.concatenate([ties, [122.0703125, -122.0703125, 2 ** -7, 3 * 2 ** -7, -2 ** -7]])
    near = np.concatenate([np.nextafter(ties, np.inf), np.nextafter(ties, -np.inf)])
    tiny = np.concatenate([-rng.uniform(0, 1e-6, 20000), rng.uniform(0, 1e-6, 20000),
                           [-1e-7, -4.9999999e-7, -5e-7, -5.0000001e-7, 5e-7, -0.0, 0.0, 1e-300, -1e-300]])
    sub = np.concatenate([rng.integers(1, 2 ** 52, 10000).view(np.float64), -rng.integers(1, 2 ** 52, 10000).view(np.float64),
                          [5e-324, -5e-324, 2.2250738585072014e-308, -2.2250738585072009e-308]])
    special = np.array([np.nan, -np.nan, np.inf, -np.inf, np.float64(2 ** 64) - 2048, -(np.float64(2 ** 64) - 2048),
                        2.0 ** 53, 2.0 ** 53 + 2, 2.0 ** 63, -2.0 ** 63, 999999.9999995, 0.9999995, -0.9999995, 0.0000005])
    ints = rng.integers(-2 ** 62, 2 ** 62, 100000).astype(np.float64)
    uniform = rng.uniform(-1e4, 1e4, 400000)
    small = rng.uniform(-1, 1, 100000) * 10.0 ** rng.integers(-8, 3, 100000)
    bits = (rng.integers(0, 2 ** 52, 100000) | (rng.integers(0, 1087, 100000) << 52)).view(np.float64)  # any |v| < 2^64
    v = np.concatenate([ties, near, tiny, sub, special, ints, uniform, small, bits, -bits[:40000]])
    return v[: len(v) // 3 * 3]


def test_formatter_equals_python_format(host_ply, tmp_path):
    from tools import visualization as V
    v = formatter_values()
    assert v.size >= 10 ** 6
    rng = np.random.default_rng(4)
    n = v.size // 3
    cols = rng.integers(-2 ** 63, 2 ** 63 - 1, (n, 3), dtype=np.int64, endpoint=True)
    cols[:6] = [[0, -1, 1], [2 ** 63 - 1, -2 ** 63, 10], [9, 99, 999], [255, 16320, 24480], [-10, -99, 100], [7, 0, 0]]
    faces = rng.integers(0, 2 ** 63 - 1, (n // 4, 3), dtype=np.int64, endpoint=True)
    faces[0] = [0, 9, 2 ** 63 - 1]
    path = tmp_path / "f.ply"
    V.write_ply(v.reshape(-1, 3), None, faces, str(path), slab_lines=400000)  # colours None: 0 0 0
    text = path.read_bytes()
    head = V.PLY_HEADER.format(n, len(faces)).encode()
    assert text[:len(head)] == head
    want = "".join("{:f} {:f} {:f} 0 0 0\n".format(*r) for r in v.reshape(-1, 3).tolist())
    want += "".join("3 {:d} {:d} {:d}\n".format(*r) for r in faces.tolist())
    assert text[len(head):] == want.encode()
    # integers in the colour columns: through the lengths / write passes directly
    lines = device_lines(host_ply, v.reshape(-1, 3)[:50000], cols[:50000], np.zeros((0, 3), np.int64))
    assert lines == "".join("{:f} {:f} {:f} {:d} {:d} {:d}\n".format(*a, *b) for a, b in
                            zip(v.reshape(-1, 3)[:50000].tolist(), cols[:50000].tolist())).encode()


def device_lines(S, verts, colors, faces, expect_big=0):
    """sis3d_ply_ascii_lengths + sis3d_ply_ascii on host arrays (the emulated library) -> the text."""
    vt = torch.from_numpy(np.ascontiguousarray(verts, np.float64).reshape(-1))
    ct = torch.from_numpy(np.ascontiguousarray(colors, np.int64).reshape(-1))
    ft = torch.from_numpy(np.ascontiguousarray(faces, np.int64).reshape(-1))
    nv, nf = len(verts), len(faces)
    n = nv + nf
    offs = torch.zeros(n + 2, dtype=torch.int64)
    scratch = torch.zeros(max((n + 2047) // 2048, 1), dtype=torch.int64)
    args = (S.ptr(vt) if nv else None, S.ptr(ct) if nv else None, C.c_int64(nv), S.ptr(ft) if nf else None, C.c_int64(nf),
            C.c_int64(0), C.c_int64(n))
    assert S.lib.sis3d_ply_ascii_lengths(*args, S.ptr(offs), S.ptr(scratch), None) == 0
    assert int(offs[n + 1]) == expect_big
    if expect_big:
        return None
    out = torch.zeros(max(int(offs[n]), 1), dtype=torch.uint8)
    assert S.lib.sis3d_ply_ascii(*args, S.ptr(offs), S.ptr(out), None) == 0
    return out.numpy()[:int(offs[n])].tobytes()


def test_values_from_2_64_take_the_host_route(host_ply, tmp_path):
    from tools import visualization as V
    big = np.array([[2.0 ** 64, 1.0, 2.0], [-1e300, 0.5, -2.0 ** 70], [1.0, 2.0, 3.0]])
    assert device_lines(host_ply, big, np.zeros((3, 3), np.int64), np.zeros((0, 3), np.int64), expect_big=2) is None
    assert device_lines(host_ply, big[2:], np.zeros((1, 3), np.int64), np.zeros((0, 3), np.int64)) == b"1.000000 2.000000 3.000000 0 0 0\n"
    path = tmp_path / "big.ply"
    verts = np.concatenate([np.tile([[1.25, -0.0, 7.0]], (5, 1)), big, np.tile([[3.0, 4.0, 5.0]], (5, 1))])
    V.write_ply(verts, None, [[0, 1, 2]], str(path), slab_lines=4)  # slabs with and without a big value
    assert path.read_bytes() == W.ply_text(verts, None, [[0, 1, 2]])


# ------------------------------------------------------------------------------------------------------------ voxel mesh
@pytest.mark.parametrize("seed, dims, slab", [(0, (7, 5, 3), 1 << 24), (1, (33, 17, 9), 1 << 24), (2, (64, 32, 48), 1 << 24),
                                              (3, (64, 32, 48), 5000), (4, (20, 3, 40), 250)])
def test_voxel_mesh_equals_oracle(host_ply, tmp_path, seed, dims, slab):
    from tools import visualization as V
    rng = np.random.default_rng(seed)
    vol = np.where(rng.random(dims) < 0.25, rng.integers(-3, 100, dims), 0).astype(np.int64)
    vol[0, 0, 0], vol[-1, -1, -1] = 1, 43
    path = tmp_path / "m.ply"
    n = V.write_mask(vol, str(path), slab_lines=slab)
    assert n == int((vol > 0).sum())
    assert path.read_bytes() == W.ply_text(*W.mask_mesh(vol))


def test_write_mask_float_volume(host_ply, tmp_path):
    """Float labels as the reference treats them: drawn when > 0, palette[int(v % 41)] (nan never drawn)."""
    from tools import visualization as V
    rng = np.random.default_rng(7)
    vol = np.where(rng.random((9, 8, 7)) < 0.4, rng.uniform(-5, 90, (9, 8, 7)), 0.0)
    vol[1, 1, 1], vol[2, 2, 2], vol[3, 3, 3] = np.nan, 0.25, 41.0
    V.write_mask(vol, str(tmp_path / "f.ply"))
    assert (tmp_path / "f.ply").read_bytes() == W.ply_text(*W.mask_mesh(vol))


def test_painted_masks_equal_oracle(host_ply, tmp_path):
    """First nonzero class wins; class 0 leaves voxels to later boxes; negative classes claim without drawing; a larger
    mask is cropped; .5 corners round half to even."""
    from tools import visualization as V
    rng = np.random.default_rng(8)
    dims = (30, 20, 25)
    boxes, masks = [], []
    for b in range(12):
        lo = rng.integers(0, 15, 3) + rng.choice([0.0, 0.5, 0.4], 3)
        hi = np.minimum(lo + rng.integers(1, 10, 3) + rng.choice([0.0, 0.5], 3), dims)
        boxes.append(np.concatenate([lo, hi]))
        ext = np.maximum(np.rint(hi) - np.rint(lo), 0).astype(int)
        masks.append(G._mask(rng, tuple(ext + (1 if b % 4 == 0 else 0))))
    boxes = np.array(boxes, np.float32)
    classes = np.array([3, 0, 45, -2, 7, 0, 12, 3.9, 41, 80, 1, 2], np.float32)
    V.write_painted_masks(dims, boxes, masks, classes, str(tmp_path / "p.ply"))
    want = W.ply_text(*W.mask_mesh(W.paint_masks(dims, boxes, masks, classes)))
    assert (tmp_path / "p.ply").read_bytes() == want


# ------------------------------------------------------------------------------------------------------------ departures
def test_non_directories_are_skipped_in_sorted_order(host_ply, tmp_path, capsys):
    """The reference calls np.load on every entry and crashes on a file; here files are skipped."""
    from tools import visualization as V
    g = load_golden(GOLDEN)
    G.write_result_scenes(G.result_scenes(), str(tmp_path))
    (tmp_path / "README.txt").write_text("not a scene\n")
    visited = []
    orig = V.visualize_result_folder
    V.visualize_result_folder = lambda d, *a, **k: (visited.append(os.path.basename(d)), orig(d, *a, **k))
    try:
        V.main(["--path", str(tmp_path), "--mode", "results"])
    finally:
        V.visualize_result_folder = orig
    assert visited == sorted(G.result_scenes())
    for rel in g["res_files"]:
        assert (tmp_path / rel).read_bytes() == golden_bytes(g, "res__" + rel.replace(os.sep, "__")), rel


def test_other_modes_write_nothing(host_ply, tmp_path):
    from tools import visualization as V
    G.write_result_scenes(G.result_scenes(), str(tmp_path))
    before = sorted(os.listdir(tmp_path / "scene0000_00"))
    V.main(["--path", str(tmp_path), "--mode", "npy"])
    assert sorted(os.listdir(tmp_path / "scene0000_00")) == before


def test_benchmark_scene_without_instances_writes_the_mesh(host_ply, tmp_path):
    """The reference's np.concatenate raises for a scene with no instances; here the aligned mesh is written alone."""
    from tools.scannet_benchmark import visualize_benchmark as VB
    from tools.scannet_benchmark import utils as U
    scenes = G.benchmark_scenes()
    res, scans, out = tmp_path / "res", tmp_path / "scans", tmp_path / "out"
    G.write_benchmark_inputs(scenes, str(res), str(scans))
    name = sorted(scenes)[1]
    (res / (name + ".txt")).write_text("")
    VB.main(["--result_dir", str(res), "--output_dir", str(out), "--scan_path", str(scans)])
    pts = U.read_mesh_vertices(str(scans / name / (name + "_vh_clean_2.ply")))
    faces = U.read_mesh_faces(str(scans / name / (name + "_vh_clean_2.ply")))
    aligned = VB.coords_multiplication(scenes[name]["align"], pts)
    colors = np.zeros_like(pts) + np.array([64, 64, 96])
    assert (out / (name + ".ply")).read_bytes() == W.ply_text(aligned, colors, faces)
    assert b"16320 16320 24480\n" in (out / (name + ".ply")).read_bytes()


def test_read_ply_needs_only_xyz_and_faces(tmp_path):
    """The reference's read_ply unpacks exactly x y z red green blue alpha; here any vertex properties are accepted."""
    from tools import visualization as V
    from tools.scannet_benchmark import utils as U
    rng = np.random.default_rng(2)
    verts = rng.uniform(-1, 1, (40, 3)).astype(np.float32)
    faces = [[i, (i + 1) % 40, (i + 2) % 40] + ([(i + 3) % 40] if i % 3 == 0 else []) for i in range(30)]
    head = ("ply\nformat ascii 1.0\nelement vertex 40\nproperty float nx\nproperty float x\nproperty float y\n"
            "property float z\nproperty int label\nelement face 30\nproperty list uchar int vertex_indices\nend_header\n")
    with open(tmp_path / "a.ply", "w") as f:
        f.write(head)
        for i, v in enumerate(verts):
            f.write(f"0.5 {float(v[0])!r} {float(v[1])!r} {float(v[2])!r} {i}\n")
        for t in faces:
            f.write(f"{len(t)} " + " ".join(map(str, t)) + "\n")
    p, t, c = V.read_ply(str(tmp_path / "a.ply"))
    assert np.array_equal(p, verts) and c is None
    assert np.array_equal(t, np.array([f[:3] for f in faces]))
    G.write_ascii_mesh(str(tmp_path / "b.ply"), verts, faces)
    p, t, c = V.read_ply(str(tmp_path / "b.ply"))
    assert np.array_equal(p, verts) and c.shape == (40, 3)
    assert np.array_equal(t, np.array([f[:3] for f in faces]))


@pytest.mark.parametrize("fmt", ["binary_little_endian", "binary_big_endian", "ascii"])
def test_read_mesh_faces_binary_and_ascii(tmp_path, fmt):
    import make_golden_scannet_eval as SE
    from tools.scannet_benchmark import utils as U
    rng = np.random.default_rng(5)
    verts = rng.uniform(-1, 1, (30, 3)).astype(np.float32)
    faces = rng.integers(0, 30, (25, 3))
    SE.write_ply(str(tmp_path / "m.ply"), verts, fmt, faces)
    assert np.array_equal(U.read_mesh_faces(str(tmp_path / "m.ply")), faces)
    assert np.array_equal(U.read_mesh_vertices(str(tmp_path / "m.ply")), verts)


def test_loadtxt_and_byte_parser_agree(tmp_path):
    from tools.scannet_benchmark import visualize_benchmark as VB
    m = (np.random.default_rng(1).random(500) < 0.3).astype(np.int64)
    np.savetxt(tmp_path / "a.txt", m, fmt="%d")
    np.savetxt(tmp_path / "b.txt", m.astype(np.float64))
    for name in ("a.txt", "b.txt"):
        got = VB.load_mask(str(tmp_path / name))
        assert got.dtype == np.float64 and np.array_equal(got, np.loadtxt(tmp_path / name))


def test_no_cuda_device_is_an_error(tmp_path):
    """Without a CUDA device (and without the emulated library) the launch raises: there is no CPU path."""
    from lib import _sis3d as S
    from tools import visualization as V
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(S.Sis3dError, match="no CPU fallback"):
        V.write_mask(np.ones((2, 2, 2), np.int64), str(tmp_path / "x.ply"))


# ------------------------------------------------------------------------------------------------------------ arguments
def test_argument_checks(ply_emu_lib):
    lib = ply_emu_lib
    buf = (C.c_int64 * 64)()
    d = (C.c_double * 64)()
    i32 = (C.c_int32 * 64)()
    i64 = lambda v: C.c_int64(v)
    EINVAL = -1
    # sis3d_voxel_mesh_count
    assert lib.sis3d_voxel_mesh_count(i32, None, 0, -1, 2, 2, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh_count(i32, None, -1, 2, 2, 2, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh_count(None, None, 0, 2, 2, 2, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh_count(i32, None, 0, 2, 2, 2, None, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh_count(i32, None, 0, 2, 2, 2, buf, None, None) == EINVAL
    assert lib.sis3d_voxel_mesh_count(None, None, 0, 0, 2, 2, buf, buf, None) == 0
    # sis3d_voxel_mesh
    assert lib.sis3d_voxel_mesh(i32, None, 0, 2, -2, 2, buf, buf, i64(0), i64(1), d, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh(i32, None, 0, 2, 2, 2, buf, buf, i64(-1), i64(1), d, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh(i32, None, 0, 2, 2, 2, buf, buf, i64(3), i64(1), d, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh(None, None, 0, 2, 2, 2, buf, buf, i64(0), i64(1), d, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh(i32, None, 0, 2, 2, 2, None, buf, i64(0), i64(1), d, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh(i32, None, 0, 2, 2, 2, buf, None, i64(0), i64(1), d, buf, buf, None) == EINVAL
    assert lib.sis3d_voxel_mesh(i32, None, 0, 2, 2, 2, buf, None, i64(0), i64(0), d, buf, buf, None) == 0
    # sis3d_ply_ascii_lengths / sis3d_ply_ascii
    for f, tail in ((lib.sis3d_ply_ascii_lengths, (buf, buf)), (lib.sis3d_ply_ascii, (buf, C.create_string_buffer(64)))):
        assert f(d, buf, i64(-1), buf, i64(1), i64(0), i64(0), *tail, None) == EINVAL
        assert f(d, buf, i64(1), buf, i64(-1), i64(0), i64(0), *tail, None) == EINVAL
        assert f(d, buf, i64(1), buf, i64(1), i64(1), i64(0), *tail, None) == EINVAL
        assert f(d, buf, i64(1), buf, i64(1), i64(-1), i64(1), *tail, None) == EINVAL
        assert f(d, buf, i64(1), buf, i64(1), i64(0), i64(3), *tail, None) == EINVAL
        assert f(None, buf, i64(1), buf, i64(1), i64(0), i64(2), *tail, None) == EINVAL
        assert f(d, None, i64(1), buf, i64(1), i64(0), i64(2), *tail, None) == EINVAL
        assert f(d, buf, i64(1), None, i64(1), i64(0), i64(2), *tail, None) == EINVAL
        assert f(None, None, i64(1), buf, i64(1), i64(1), i64(2), *tail, None) == 0  # faces only: no vertex arrays needed
    assert lib.sis3d_ply_ascii_lengths(d, buf, i64(1), buf, i64(1), i64(0), i64(2), None, buf, None) == EINVAL
    assert lib.sis3d_ply_ascii_lengths(d, buf, i64(1), buf, i64(1), i64(0), i64(2), buf, None, None) == EINVAL
    assert lib.sis3d_ply_ascii(d, buf, i64(1), buf, i64(1), i64(0), i64(2), None, C.create_string_buffer(64), None) == EINVAL
    assert lib.sis3d_ply_ascii(d, buf, i64(1), buf, i64(1), i64(0), i64(2), buf, None, None) == EINVAL
