"""CPU: the ScanNet instance benchmark on the host and, under host emulation, through the vertex-transfer kernels.

- tools/scannet_benchmark/evaluate_semantic_instance.py against the reference's own evaluator
  (tests/golden/scannet_instance_eval_reference.npz, recorded by oracle/make_golden_scannet_eval.py from seeded inputs that
  are regenerated here): AP arrays with nan in the same places, stdout and CSV byte for byte;
- the PLY reader, vox2mesh.py's command line, and the chain vox2mesh CLI -> evaluator against the reference chain;
- sis3d_instance_paint / sis3d_vertex_instance_overlap (csrc/eval.cu compiled for the host by tools/cuda_host_emu.py)
  against vox2mesh.paint_instances / vertex_labels / np.bincount, and evaluate_predictions.py's fused route against the
  file route and the reference chain."""
import contextlib
import ctypes as C
import io
import os
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_golden_scannet_eval as G  # noqa: E402  (the seeded inputs; no reference code involved)

GOLDEN = "scannet_instance_eval_reference.npz"


def run_quiet(f, *a):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        r = f(*a)
    return r, buf.getvalue()


def check_against_golden(g, key, ap, stdout, csv):
    assert np.array_equal(ap, g[key + "_ap"], equal_nan=True), key
    assert stdout == str(g[key + "_stdout"]), key
    assert csv == str(g[key + "_csv"]), key


def file_route_text(tmp, key):
    from tools.scannet_benchmark import evaluate_semantic_instance as E
    pred, gt = str(tmp / "pred"), str(tmp / "gt")
    G.write_text_set(G.TEXT_SETS[key](), pred, gt)
    (ap, avgs), out = run_quiet(E.main, ["--pred_path", pred, "--gt_path", gt])
    with open(os.path.join(pred, E.RESULT_FILE)) as f:
        return ap, avgs, out, f.read(), pred, gt


@pytest.mark.parametrize("key", list(G.TEXT_SETS))
def test_text_sets_equal_reference(tmp_path, key):
    g = load_golden(GOLDEN)
    ap, avgs, out, csv, _, _ = file_route_text(tmp_path, key)
    check_against_golden(g, key, ap, out, csv)
    assert avgs["all_ap"] == g[key + "_all_ap"] or (np.isnan(avgs["all_ap"]) and np.isnan(g[key + "_all_ap"]))


def test_handmade_set_takes_every_branch():
    """The hand-made set reaches the branches it was made for: the empty-curve line, a class with GT only, classes with
    neither."""
    g = load_golden(GOLDEN)
    ap = g["text_hand_ap"]
    assert "\n\n\n" in str(g["text_hand_stdout"]).split("scans processed: 3")[1]  # print('') of the empty curve
    from tools.scannet_benchmark.evaluate_semantic_instance import CLASS_LABELS
    sofa, desk = CLASS_LABELS.index("sofa"), CLASS_LABELS.index("desk")
    assert (ap[0, desk] == 0).all() and (ap[0, sofa] == 0).all()
    assert np.isnan(ap[0, CLASS_LABELS.index("bed")]).all()


def test_scene_order_does_not_change_the_result(tmp_path):
    from tools.scannet_benchmark import evaluate_semantic_instance as E
    for key in ("text_hand", "text_rand0"):
        d = tmp_path / key
        ap, _, out, csv, pred, gt = file_route_text(d, key)
        names = sorted(f for f in os.listdir(pred) if f.endswith(".txt") and f != E.RESULT_FILE)[::-1]
        other = str(d / "reversed.csv")
        (ap2, _), out2 = run_quiet(E.evaluate, [os.path.join(pred, n) for n in names], [os.path.join(gt, n) for n in names],
                                   pred, other)
        assert np.array_equal(ap, ap2, equal_nan=True)
        assert out == out2 and open(other).read() == csv


def test_missing_gt_and_malformed_lines_exit(tmp_path, capsys):
    from tools.scannet_benchmark import evaluate_semantic_instance as E
    pred, gt = tmp_path / "pred", tmp_path / "gt"
    pred.mkdir(), gt.mkdir()
    with pytest.raises(SystemExit) as e:
        E.main(["--pred_path", str(pred), "--gt_path", str(gt)])
    assert e.value.code == 2 and "No result files found." in capsys.readouterr().err
    (pred / "scene0000_00.txt").write_text("predicted_masks/a.txt 3\n")
    with pytest.raises(SystemExit) as e:
        E.main(["--pred_path", str(pred), "--gt_path", str(gt)])
    assert e.value.code == 2 and "does not match any gt file" in capsys.readouterr().err
    (gt / "scene0000_00.txt").write_text("0\n0\n")
    with pytest.raises(SystemExit) as e:
        E.main(["--pred_path", str(pred), "--gt_path", str(gt)])
    assert e.value.code == -1 and "Expected (per line)" in capsys.readouterr().err
    (pred / "scene0000_00.txt").write_text("../outside.txt 3 0.5\n")
    with pytest.raises(SystemExit) as e:
        E.main(["--pred_path", str(pred), "--gt_path", str(gt)])
    assert e.value.code == -1 and "points outside of prediction path" in capsys.readouterr().err


# ------------------------------------------------------------------------------------------------------------ PLY
@pytest.mark.parametrize("fmt", ["binary_little_endian", "binary_big_endian", "ascii"])
def test_ply_reader(tmp_path, fmt):
    from tools.scannet_benchmark.utils import read_mesh_vertices
    rng = np.random.default_rng(3)
    v = rng.normal(size=(257, 3)).astype(np.float32)
    p = str(tmp_path / "m.ply")
    G.write_ply(p, v, fmt, faces=np.stack([np.arange(10), np.arange(1, 11), np.arange(2, 12)], 1))
    got = read_mesh_vertices(p)
    assert got.dtype == np.float32 and np.array_equal(got, v)


def test_ply_reader_element_before_vertex_and_extra_properties(tmp_path):
    from tools.scannet_benchmark.utils import read_mesh_vertices
    head = ("ply\nformat binary_little_endian 1.0\nelement camera 2\nproperty double a\nproperty list uchar short l\n"
            "element vertex 3\nproperty uchar red\nproperty double z\nproperty float x\nproperty short q\nproperty float y\n"
            "end_header\n")
    cam = b"".join(np.float64(i).tobytes() + bytes([2]) + np.array([7, 8], "<i2").tobytes() for i in range(2))
    dt = np.dtype([("red", "u1"), ("z", "<f8"), ("x", "<f4"), ("q", "<i2"), ("y", "<f4")])
    v = np.zeros(3, dt)
    v["x"], v["y"], v["z"] = [1, 2, 3], [4, 5, 6], [7.5, 8.5, 9.5]
    p = tmp_path / "m.ply"
    p.write_bytes(head.encode() + cam + v.tobytes())
    assert read_mesh_vertices(str(p)).tolist() == [[1, 4, 7.5], [2, 5, 8.5], [3, 6, 9.5]]


@pytest.mark.parametrize("header, match", [
    ("plx\nformat ascii 1.0\nelement vertex 0\nproperty float x\nend_header\n", "magic"),
    ("ply\nformat binary_middle_endian 1.0\nelement vertex 0\nend_header\n", "format"),
    ("ply\nelement vertex 0\nproperty float x\nproperty float y\nproperty float z\nend_header\n", "no format"),
    ("ply\nformat ascii 1.0\nelement vertex 0\nproperty float x\nproperty float y\nproperty float z\n", "end_header"),
    ("ply\nformat ascii 1.0\nelement face 0\nproperty list uchar int i\nend_header\n", "no vertex"),
    ("ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nend_header\n0 0\n", "'z'"),
    ("ply\nformat ascii 1.0\nelement vertex 1\nproperty quad x\nend_header\n", "malformed PLY property"),
    ("ply\nformat ascii 1.0\nproperty float x\nend_header\n", "before any element"),
    ("ply\nformat ascii 1.0\nelement vertex x\nend_header\n", "element line"),
    ("ply\nformat binary_little_endian 1.0\nelement vertex 1\nproperty float x\nproperty float y\nproperty float z\n"
     "property list uchar int n\nend_header\n", "list property inside the vertex"),
    ("ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\nproperty float z\n"
     "end_header\n" + "\0" * 12, "ends inside"),
])
def test_ply_reader_rejects(tmp_path, header, match):
    from tools.scannet_benchmark.utils import read_mesh_vertices
    p = tmp_path / "bad.ply"
    p.write_bytes(header.encode("latin-1"))
    with pytest.raises(ValueError, match=match):
        read_mesh_vertices(str(p))


# ------------------------------------------------------------------------------------------------------------ chain
def write_chain(tmp, key, ply_fmt="binary_little_endian"):
    dirs = {k: str(tmp / k) for k in ("results", "scans", "frames", "gt", "bench")}
    chain = G.CHAIN_SETS[key]()
    G.write_chain_inputs(chain, dirs["results"], dirs["scans"], dirs["frames"], dirs["gt"], ply_fmt)
    return chain, dirs


def file_route_chain(dirs):
    """vox2mesh.py's CLI, then evaluate_semantic_instance.py's: -> (ap, stdout of the evaluator, CSV text)."""
    from tools.scannet_benchmark import evaluate_semantic_instance as E
    from tools.scannet_benchmark import vox2mesh as V
    run_quiet(V.main, ["--pred_dir", dirs["results"], "--output_dir", dirs["bench"], "--scan_path", dirs["scans"],
                       "--frames", dirs["frames"]])
    (ap, _), out = run_quiet(E.main, ["--pred_path", dirs["bench"], "--gt_path", dirs["gt"]])
    with open(os.path.join(dirs["bench"], E.RESULT_FILE)) as f:
        return ap, out, f.read()


def fused_route_chain(dirs, tmp):
    from tools.scannet_benchmark import evaluate_predictions as F
    out_file = str(tmp / "fused" / "result.csv")
    os.makedirs(os.path.dirname(out_file), exist_ok=True)
    (ap, _), out = run_quiet(F.main, ["--pred_dir", dirs["results"], "--scan_path", dirs["scans"], "--frames",
                                      dirs["frames"], "--gt_path", dirs["gt"], "--output_file", out_file])
    with open(out_file) as f:
        return ap, out, f.read()


@pytest.mark.parametrize("key", list(G.CHAIN_SETS))
def test_vox2mesh_cli_then_evaluator_equal_reference_chain(tmp_path, key):
    _, dirs = write_chain(tmp_path, key)
    check_against_golden(load_golden(GOLDEN), key, *file_route_chain(dirs))


@pytest.mark.parametrize("ply_fmt", ["binary_little_endian", "ascii"])
def test_vox2mesh_cli_equals_export(tmp_path, ply_fmt):
    from tools.scannet_benchmark import utils
    from tools.scannet_benchmark import vox2mesh as V
    chain, dirs = write_chain(tmp_path, "chain1", ply_fmt)
    os.makedirs(os.path.join(dirs["results"], "scene9999_00"))  # a result folder without a mesh is skipped
    (_, out) = run_quiet(V.main, ["--pred_dir", dirs["results"], "--output_dir", dirs["bench"], "--scan_path", dirs["scans"],
                                  "--frames", dirs["frames"]])
    assert out.splitlines() == ["0/4", "1/4", "2/4", "3/4"]
    assert sorted(os.listdir(dirs["bench"])) == ["predicted_masks"] + [s + ".txt" for s in sorted(chain)]
    want = tmp_path / "want"
    for s, c in chain.items():
        verts = utils.read_mesh_vertices(os.path.join(dirs["scans"], s, s + "_vh_clean_2.ply"))
        assert np.array_equal(verts, c["verts"])
        V.export(verts, V.load_matrix(os.path.join(dirs["frames"], s, "world2grid.txt")),
                 V.load_pred(os.path.join(dirs["results"], s)), str(want), s)
    for root, _, files in os.walk(want):
        for f in files:
            rel = os.path.relpath(os.path.join(root, f), want)
            assert open(os.path.join(dirs["bench"], rel), "rb").read() == open(os.path.join(want, rel), "rb").read(), rel
    assert len(os.listdir(os.path.join(dirs["bench"], "predicted_masks"))) == sum(1 for _ in os.scandir(want / "predicted_masks"))


# ------------------------------------------------------------------------------------------------------------ kernels
@pytest.fixture(scope="module")
def eval_emu_lib(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import cuda_host_emu
    out = str(tmp_path_factory.mktemp("emu_scannet") / "libsis3d_eval_emu.so")
    cuda_host_emu.build(out, [os.path.join(ROOT, "3d-sis_b200", "csrc", "eval.cu")])
    lib = C.CDLL(out)
    lib.sis3d_strerror.restype = C.c_char_p
    return lib


@pytest.fixture
def host_eval(monkeypatch, eval_emu_lib):
    """lib._sis3d pointed at the emulated library, accepting host tensors."""
    from lib import _sis3d as S
    monkeypatch.setattr(S, "lib", eval_emu_lib)
    monkeypatch.setattr(S, "ptr", lambda t: None if t is None else C.c_void_p(t.data_ptr()))
    monkeypatch.setattr(S, "stream", lambda: None)
    return S


def seeded_kernel_case(seed, dims=(60, 30, 50), n_box=12, n_vert=4000):
    """Boxes with masks (some larger than their box, one empty box, one box painting the value 0.0), vertices around them
    and outside the canvas, and GT ids.  Vertex grid coordinates stay >= 0.1 voxel away from half-integers."""
    rng = np.random.default_rng(seed)
    box, masks = [], []
    for b in range(n_box):
        lo = np.array([rng.integers(0, d - 12) for d in dims]) + rng.choice([0.0, 0.5, -0.5, 0.3], 3)
        lo = np.maximum(lo, 0)
        hi = lo + rng.integers(1, 12, 3) + rng.choice([0.0, 0.5, 0.4], 3)
        if b == 4:
            hi[1] = lo[1]  # empty box: skipped
        box.append(np.concatenate([lo, hi]))
        shape = tuple(np.maximum(np.rint(hi).astype(int) - np.rint(lo).astype(int), 0) + (1 if rng.random() < 0.3 else 0))
        masks.append(np.where(rng.random(shape) < 0.6, rng.choice([1.0, 0.3, -2.0], shape), 0.0).astype(np.float32))
    cls = rng.integers(1, 19, n_box)
    conf = rng.uniform(0.02, 0.99, n_box)
    cls[0], conf[0] = 0, 0.01  # box 0 paints 0 * 100 + 0 + 0.01 - 0.01 == 0.0: nothing
    w2g = np.eye(4)
    w2g[:3, :3] = np.array([[0, 21.333333333333332, 0], [21.333333333333332, 0, 0], [0, 0, -21.333333333333332]])
    w2g[:3, 3] = [3.25, -1.5, dims[2] - 2.0]
    g = np.concatenate([rng.integers(-3, np.array(dims) + 3, (n_vert, 3))]).astype(np.float64)
    grid = g + rng.uniform(-0.4, 0.4, g.shape)
    verts = ((grid - w2g[:3, 3]) @ np.linalg.inv(w2g[:3, :3]).T).astype(np.float32)
    gt = rng.choice([0, 7, 3001, 3002, 5001, 25001, 1001], n_vert)
    return dict(box=np.array(box, np.float32), cls=cls, conf=conf, masks=masks, w2g=w2g, verts=verts, gt=gt, dims=dims)


def check_kernels_against_host(c):
    """owner == paint_instances' first box, per-vertex box == vertex_labels, hist == np.bincount, first vertex == first
    labelled index.  -> number of vertices whose box differs between host and device."""
    from tools.scannet_benchmark import evaluate_predictions as F
    from tools.scannet_benchmark import vox2mesh as V
    dims = c["dims"]
    values = F.box_values(c["cls"], c["conf"])
    bits, offs, ibox, lo, ext = F.pack_boxes(c["box"], values, c["masks"], dims)
    uniq, slot = np.unique(c["gt"], return_inverse=True)
    hist, first, vbox = F.vertex_instance_overlap(c["verts"], c["w2g"], slot.astype(np.int32), len(uniq), bits, offs, ibox,
                                                  lo, ext, dims, want_vertex_box=True)
    scene = V.paint_instances(c["box"], c["cls"], c["conf"], c["masks"], dims)
    value, valid = V.vertex_labels(c["verts"], c["w2g"], scene)
    # the value a vertex sees identifies its box: the boxes' values are distinct here
    assert len(set(values.tolist())) == len(values)
    want_box = np.full(len(value), -1)
    for b, v in enumerate(values):
        want_box[valid & (value == v)] = b
    assert (valid.sum() > 0) and (want_box >= 0).sum() == valid.sum()
    mismatches = int((vbox != want_box).sum())
    print(f"{len(vbox)} vertices, {int(valid.sum())} labelled, host/device label disagreements: {mismatches}")
    want_hist = np.zeros_like(hist)
    np.add.at(want_hist, (want_box[valid], slot[valid]), 1)
    assert np.array_equal(hist, want_hist)
    for b in range(len(values)):
        idx = np.nonzero(want_box == b)[0]
        assert first[b] == (idx[0] if len(idx) else F.NO_VERTEX)
    return mismatches, scene, bits, offs, ibox, lo, ext, values


def check_owner_volume(scene, bits, offs, ibox, lo, ext, values):
    """The owner volume read back through the paint kernel alone, against the painted canvas."""
    import torch
    from lib import _sis3d as S
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (bits if len(bits) else np.zeros(1, np.uint8), offs, ibox)]
    owner = torch.full((int(np.prod(ext)),), -7, dtype=torch.int32, device=dev)
    S.check(S.lib.sis3d_instance_paint(S.ptr(t[0]), S.ptr(t[1]), S.ptr(t[2]), len(offs), *[int(v) for v in lo],
                                       *[int(v) for v in ext], S.ptr(owner), S.stream()), "instance_paint")
    own = owner.cpu().numpy().reshape(tuple(int(v) for v in ext))
    sub = scene[lo[0]:lo[0] + ext[0], lo[1]:lo[1] + ext[1], lo[2]:lo[2] + ext[2]]
    want = np.full(sub.shape, -1)
    for b, v in enumerate(values):  # distinct values: the painted value names the box
        if v != 0:
            want[sub == v] = b
    assert np.array_equal(own, want)
    outside = scene.copy()
    outside[lo[0]:lo[0] + ext[0], lo[1]:lo[1] + ext[1], lo[2]:lo[2] + ext[2]] = 0
    assert not outside.any()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kernels_equal_host_emulated(host_eval, seed):
    mism, *rest = check_kernels_against_host(seeded_kernel_case(seed))
    assert mism == 0
    check_owner_volume(*rest)


def test_pack_boxes_follows_vox2mesh_rules():
    from tools.scannet_benchmark import evaluate_predictions as F
    from tools.scannet_benchmark import vox2mesh as V
    box = np.array([[0, 0, 0, 2, 2, 2], [1, 1, 1, 3, 3, 3]], np.float32)
    vals = np.array([1.5, 101.5])
    with pytest.raises(IndexError, match="mask 1 is smaller"):
        F.pack_boxes(box, vals, [np.ones((2, 2, 2)), np.ones((2, 2, 1))], (8, 8, 8))
    with pytest.raises(IndexError, match="mask 1 is smaller"):  # as paint_instances
        V.paint_instances(box, [1, 1], [0.5, 0.5], [np.ones((2, 2, 2)), np.ones((2, 2, 1))], (8, 8, 8))
    with pytest.raises(IndexError, match="box 1 leaves"):
        F.pack_boxes(box, vals, [np.ones((2, 2, 2))] * 2, (8, 8, 2))
    bits, offs, ibox, lo, ext = F.pack_boxes(box, vals, [np.full((3, 2, 2), 0.3), np.ones((2, 2, 2))], (8, 8, 8))
    assert bits.tolist() == [1] * 16 and offs.tolist() == [0, 8] and lo.tolist() == [0, 0, 0] and ext.tolist() == [3, 3, 3]
    bits, offs, ibox, lo, ext = F.pack_boxes(box, np.array([0.0, 101.5]), [np.ones((2, 2, 2))] * 2, (8, 8, 8))  # value 0.0
    assert ibox[0].tolist() == [0] * 6 and lo.tolist() == [1, 1, 1] and ext.tolist() == [2, 2, 2]


def test_kernel_argument_checks(host_eval):
    L = host_eval.lib
    buf = (C.c_int64 * 8)()
    i32 = (C.c_int32 * 8)()
    assert L.sis3d_instance_paint(None, None, None, -1, 0, 0, 0, 1, 1, 1, i32, None) == -1
    assert L.sis3d_instance_paint(None, None, None, 0, 0, 0, 0, -1, 1, 1, i32, None) == -1
    assert L.sis3d_instance_paint(None, None, None, 1, 0, 0, 0, 1, 1, 1, i32, None) == -1  # boxes without masks
    assert L.sis3d_instance_paint(None, None, None, 0, 0, 0, 0, 1, 1, 1, None, None) == -1  # no owner volume
    assert L.sis3d_instance_paint(None, None, None, 0, 0, 0, 0, 0, 1, 1, None, None) == 0  # nothing to do
    assert L.sis3d_instance_paint(None, None, None, 0, 0, 0, 0, 2, 2, 2, i32, None) == 0
    assert list(i32) == [-1] * 8  # no box: nothing owned
    ov = L.sis3d_vertex_instance_overlap
    f32, f64 = (C.c_float * 3)(), (C.c_double * 16)()
    assert ov(None, -1, None, None, 0, 0, 0, 0, 0, 0, 4, 4, 4, None, 0, 0, None, None, None, None) == -1
    assert ov(f32, 1, None, None, 0, 0, 0, 0, 0, 0, 4, 4, 4, i32, 1, 0, None, None, None, None) == -1  # no world2grid
    assert ov(f32, 1, f64, None, 0, 0, 0, 1, 1, 1, 4, 4, 4, i32, 1, 0, None, None, None, None) == -1  # no owner volume
    assert ov(f32, 1, f64, i32, 0, 0, 0, 1, 1, 1, 4, 4, 4, None, 1, 0, None, None, None, None) == -1  # no GT slots
    assert ov(f32, 1, f64, i32, 0, 0, 0, 1, 1, 1, 4, 4, 4, i32, 1, 1, buf, None, None, None) == -1  # no first_vertex
    assert ov(f32, 1, f64, i32, 0, 0, 0, 1, 1, 1, 4, 4, 4, i32, 1, 1, None, i32, None, None) == -1  # no hist
    assert ov(f32, 1, f64, i32, 0, 0, 0, 1, 1, 1, -4, 4, 4, i32, 1, 1, buf, i32, None, None) == -1  # negative canvas
    assert ov(None, 0, None, None, 0, 0, 0, 0, 0, 0, 4, 4, 4, None, 0, 0, None, None, None, None) == 0


def test_real_library_exports_the_entry_points():
    from lib import _sis3d as S
    assert S.lib.sis3d_instance_paint(None, None, None, -1, 0, 0, 0, 0, 0, 0, None, None) == -1
    assert S.lib.sis3d_vertex_instance_overlap(None, -1, None, None, 0, 0, 0, 0, 0, 0, 0, 0, 0, None, 0, 0, None, None, None,
                                               None) == -1


def test_fused_route_without_device_raises():
    import torch
    from lib import _sis3d as S
    from tools.scannet_benchmark import evaluate_predictions as F
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(S.Sis3dError):
        F.vertex_instance_overlap(np.zeros((1, 3), np.float32), np.eye(4), np.zeros(1, np.int32), 1, np.zeros(0, np.uint8),
                                  np.zeros(0, np.int64), np.zeros((0, 6), np.int32), np.zeros(3, int), np.zeros(3, int))


# ------------------------------------------------------------------------------------------------------------ fused route
@pytest.mark.parametrize("key", list(G.CHAIN_SETS))
def test_fused_route_equals_file_route_and_reference_emulated(host_eval, tmp_path, key):
    _, dirs = write_chain(tmp_path, key)
    fused = fused_route_chain(dirs, tmp_path)
    check_against_golden(load_golden(GOLDEN), key, *fused)
    ap, out, csv = file_route_chain(dirs)
    assert np.array_equal(ap, fused[0], equal_nan=True) and out == fused[1] and csv == fused[2]


def test_fused_route_scene_selection(host_eval, tmp_path, capsys):
    from tools.scannet_benchmark import evaluate_predictions as F
    chain, dirs = write_chain(tmp_path, "chain0")
    os.makedirs(os.path.join(dirs["results"], "scene9999_00"))  # no mesh: not a scene
    args = ["--pred_dir", dirs["results"], "--scan_path", dirs["scans"], "--frames", dirs["frames"], "--gt_path", dirs["gt"],
            "--output_file", str(tmp_path / "r.csv")]
    run_quiet(F.main, args)
    os.remove(os.path.join(dirs["gt"], "scene0001_00.txt"))
    with pytest.raises(SystemExit) as e:
        F.main(args)
    assert e.value.code == 2 and "Result file scene0001_00.txt does not match any gt file" in capsys.readouterr().err
