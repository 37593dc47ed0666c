"""GPU: the result visualisation tools through the real libsis3d (csrc/ply.cu, csrc/eval.cu) on the device.

- the golden sets of oracle/make_golden_visualization.py byte for byte;
- the formatter against Python's '{:f}' / '{:d}' on the CPU suite's 10^6 values;
- a 208x48x160 result folder with 100 kept masks and GT, a 150k-vertex benchmark mesh with 60 instances, and the folders
  lib.model.trainval.test writes from synthetic chunks, against oracle/ply_writer.py (sha1 of every file)."""
import hashlib
import os
import pickle
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, "oracle"))
import make_golden_visualization as G  # noqa: E402
import ply_writer as W  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = "visualization_reference.npz"


def sha1(b):
    return hashlib.sha1(b).hexdigest()


def host_result_files(d):
    """{file name: bytes} of one result folder from oracle/ply_writer.py and the host cylinders (pinned by the golden)."""
    from tools import visualization as V
    ld = lambda f: np.load(os.path.join(d, f)) if os.path.exists(os.path.join(d, f)) else None
    pk = lambda f: pickle.load(open(os.path.join(d, f), "rb")) if os.path.exists(os.path.join(d, f)) else None
    scene = ld("scene.npy")
    out = {"scene.ply": W.ply_text(*W.mask_mesh(scene))}
    box, cls, masks, index = ld("pred_box.npy"), ld("pred_class.npy"), pk("pred_mask"), pk("pred_mask_index")
    box = box[:, :6][index]
    cls = cls[index]
    out["pred_bbox.ply"] = W.ply_text(*V.bbox_cylinders(np.concatenate([box, cls[:, None]], 1)))
    out["pred_mask.ply"] = W.ply_text(*W.mask_mesh(W.paint_masks(scene.shape, box, masks, cls)))
    gb, gc, gm = ld("gt_box.npy"), ld("gt_class.npy"), pk("gt_mask")
    if gb is not None:
        out["gt_bbox.ply"] = W.ply_text(*V.bbox_cylinders(np.concatenate([gb[:, :6], gc[:, None]], 1)))
        out["gt_mask.ply"] = W.ply_text(*W.mask_mesh(W.paint_masks(scene.shape, gb[:, :6], gm, gc)))
    return out


def check_folder(d):
    for name, want in host_result_files(d).items():
        with open(os.path.join(d, name), "rb") as f:
            assert sha1(f.read()) == sha1(want), (d, name)


def test_golden_sets_on_device(tmp_path):
    from tools import visualization as V
    from tools.scannet_benchmark import visualize_benchmark as VB
    g = load_golden(GOLDEN)
    res = tmp_path / "res"
    G.write_result_scenes(G.result_scenes(), str(res))
    V.main(["--path", str(res), "--mode", "results"])
    for rel in g["res_files"]:
        assert (res / rel).read_bytes() == g["res__" + rel.replace(os.sep, "__")].tobytes(), rel
    b, scans, out = tmp_path / "b", tmp_path / "scans", tmp_path / "out"
    G.write_benchmark_inputs(G.benchmark_scenes(), str(b), str(scans))
    VB.main(["--result_dir", str(b), "--output_dir", str(out), "--scan_path", str(scans)])
    for name in g["bench_files"]:
        assert (out / name).read_bytes() == g["bench__" + name].tobytes(), name


def test_formatter_on_device(tmp_path):
    from tools import visualization as V
    from test_visualization import formatter_values
    v = formatter_values().reshape(-1, 3)
    rng = np.random.default_rng(4)
    cols = rng.integers(-2 ** 63, 2 ** 63 - 1, v.shape, dtype=np.int64, endpoint=True)
    path = tmp_path / "f.ply"
    V.write_ply(v, cols / 255.0, None, str(path))
    got = path.read_bytes()
    c255 = (cols / 255.0 * 255).astype(np.int64)
    want = V.PLY_HEADER.format(len(v), 0) + "".join("{:f} {:f} {:f} {:d} {:d} {:d}\n".format(*a, *c)
                                                   for a, c in zip(v.tolist(), c255.tolist()))
    assert got == want.encode()


def large_result_folder(d, seed=0, dims=(208, 48, 160), n_box=120, n_keep=100):
    rng = np.random.default_rng(seed)
    os.makedirs(d, exist_ok=True)
    np.save(os.path.join(d, "scene.npy"), (rng.random(dims) < 0.12).astype(np.int64))
    lo = rng.integers(0, np.array(dims) - 24, (n_box, 3)) + rng.choice([0.0, 0.5, 0.3], (n_box, 3))
    hi = np.minimum(lo + rng.integers(4, 24, (n_box, 3)) + rng.choice([0.0, 0.5], (n_box, 3)), dims)
    box = np.concatenate([lo, hi], 1).astype(np.float32)
    keep = np.zeros(n_box, bool)
    keep[rng.permutation(n_box)[:n_keep]] = True
    ext = lambda b: tuple(int(v) for v in np.maximum(np.rint(b[3:6]) - np.rint(b[:3]), 0))
    masks = [(rng.random(ext(b)) < 0.6).astype(np.float32) for b, k in zip(box, keep) if k]
    np.save(os.path.join(d, "pred_box.npy"), box)
    np.save(os.path.join(d, "pred_class.npy"), rng.integers(1, 19, n_box).astype(np.int64))
    pickle.dump(masks, open(os.path.join(d, "pred_mask"), "wb"))
    pickle.dump([bool(k) for k in keep], open(os.path.join(d, "pred_mask_index"), "wb"))
    gbox = np.floor(box[:40]).astype(np.float32)
    np.save(os.path.join(d, "gt_box.npy"), gbox)
    np.save(os.path.join(d, "gt_class.npy"), rng.integers(1, 19, 40).astype(np.float32))
    pickle.dump([(rng.random(ext(b)) < 0.7).astype(np.float32) for b in gbox], open(os.path.join(d, "gt_mask"), "wb"))


def test_large_result_folder_equals_oracle(tmp_path):
    from tools import visualization as V
    d = str(tmp_path / "scene0000_00")
    large_result_folder(d)
    V.visualize_results(str(tmp_path))
    check_folder(d)


def test_large_benchmark_mesh_equals_host_writer(tmp_path):
    from tools.scannet_benchmark import visualize_benchmark as VB
    from tools import visualization as V
    import make_golden_scannet_eval as SE
    rng = np.random.default_rng(1)
    n, scene = 150000, "scene0500_00"
    verts = rng.uniform(0, 8, (n, 3)).astype(np.float32)
    faces = rng.integers(0, n, (2 * n, 3))
    os.makedirs(tmp_path / "scans" / scene)
    SE.write_ply(str(tmp_path / "scans" / scene / (scene + "_vh_clean_2.ply")), verts, "binary_little_endian", faces)
    align = np.eye(4)
    align[:3, 3] = [-4.0, -4.0, 0.25]
    with open(tmp_path / "scans" / scene / (scene + ".txt"), "w") as f:
        f.write("axisAlignment = " + " ".join(repr(float(v)) for v in align.reshape(-1)) + "\n")
    res = tmp_path / "res"
    os.makedirs(res / "pred_mask")
    masks = []
    with open(res / (scene + ".txt"), "w") as f:
        for i in range(60):
            m = np.zeros(n, np.int64)
            a = int(rng.integers(0, n - 6000))
            m[a:a + int(rng.integers(500, 6000))] = 1
            np.savetxt(res / "pred_mask" / f"{i:03d}.txt", m, fmt="%d")
            f.write(f"pred_mask/{i:03d}.txt {int(rng.integers(0, 19))} 0.9\n")
            masks.append(m)
    VB.main(["--result_dir", str(res), "--output_dir", str(tmp_path / "out"), "--scan_path", str(tmp_path / "scans")])
    pts = VB.coords_multiplication(align, verts)
    colors = np.zeros_like(verts) + np.array([64, 64, 96])
    boxes = []
    for i, m in enumerate(masks):
        idx = m.nonzero()[0]
        r, g, b = V.create_color_palette()[(i + 1) % 41]
        colors[idx] = [r / 255.0, g / 255.0, b / 255.0]
        boxes.append(np.concatenate([pts[idx].min(0), pts[idx].max(0), [i + 1]]))
    bv, bc, bf = V.bbox_cylinders(np.array(boxes))
    want = W.ply_text(np.concatenate([pts, bv]), np.concatenate([colors, bc]), np.concatenate([faces, bf + n]))
    assert sha1((tmp_path / "out" / (scene + ".ply")).read_bytes()) == sha1(want)


def test_test_mode_results_visualised_end_to_end(tmp_path):
    import sis3d_synth as synth
    from lib.model import trainval
    from tools import visualization as V
    c = synth.CASES["odd_45x27x41"]
    net, cfg = synth.make_net(c, keep_debug=False, math="exact")
    torch.save({k: v.detach().cpu().clone() for k, v in net.state_dict().items()}, str(tmp_path / "step_1.pth"))
    paths, provider = synth.write_chunks(str(tmp_path), c, (202, 7, 8))
    cfg.TEST_FILELIST = paths
    cfg.TEST_SAVE_DIR = str(tmp_path / "results")
    assert trainval.test(SimpleNamespace(output_dir=str(tmp_path), step=1, num_workers=0), view_provider=provider) == len(paths)
    V.main(["--path", cfg.TEST_SAVE_DIR, "--mode", "results"])
    folders = sorted(os.listdir(cfg.TEST_SAVE_DIR))
    assert len(folders) == len(paths)
    for s in folders:
        check_folder(os.path.join(cfg.TEST_SAVE_DIR, s))
