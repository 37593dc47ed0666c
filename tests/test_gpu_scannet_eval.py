"""GPU: the ScanNet benchmark's vertex-transfer kernels (sis3d_instance_paint, sis3d_vertex_instance_overlap in csrc/eval.cu)
against vox2mesh's host painting and lookup, inside a CUDA graph, at a real scene size, and evaluate_predictions.py end to end
against the two-step file route on the output of the benchmark mode."""
import ctypes as C
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import load_golden
from test_scannet_eval import (GOLDEN, G, check_against_golden, check_kernels_against_host, check_owner_volume,
                               file_route_chain, fused_route_chain, seeded_kernel_case, write_chain)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kernels_equal_host_on_device(seed):
    mism, *rest = check_kernels_against_host(seeded_kernel_case(seed))
    assert mism == 0
    check_owner_volume(*rest)


def test_real_size_scene():
    """208x48x160 with 100 boxes and ~150k vertices; vertex grid coordinates stay >= 0.1 voxel from half-integers, so the
    host's BLAS product and the device's fixed-order fp64 rows pick the same voxel.  The disagreement count is printed."""
    mism, *rest = check_kernels_against_host(seeded_kernel_case(5, dims=(208, 48, 160), n_box=100, n_vert=150000))
    assert mism == 0
    check_owner_volume(*rest)


@pytest.mark.parametrize("key", list(G.CHAIN_SETS))
def test_fused_route_on_device(tmp_path, key):
    _, dirs = write_chain(tmp_path, key)
    fused = fused_route_chain(dirs, tmp_path)
    check_against_golden(load_golden(GOLDEN), key, *fused)
    ap, out, csv = file_route_chain(dirs)
    assert np.array_equal(ap, fused[0], equal_nan=True) and out == fused[1] and csv == fused[2]


def test_graph_capture_equals_eager():
    from lib import _sis3d as S
    from tools.scannet_benchmark import evaluate_predictions as F
    c = seeded_kernel_case(1)
    values = F.box_values(c["cls"], c["conf"])
    bits, offs, ibox, lo, ext = F.pack_boxes(c["box"], values, c["masks"], c["dims"])
    uniq, slot = np.unique(c["gt"], return_inverse=True)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = [dev(c["verts"]), dev(c["w2g"].astype(np.float64)), dev(slot.astype(np.int32)), dev(offs), dev(ibox), dev(bits)]
    n_vert, n_box, n_slot = len(c["verts"]), len(offs), len(uniq)
    n_owner = int(np.prod(ext))

    def launch(owner, res, stream):
        h = C.c_void_p(stream.cuda_stream)
        S.check(S.lib.sis3d_instance_paint(S.ptr(t[5]), S.ptr(t[3]), S.ptr(t[4]), n_box, *[int(v) for v in lo],
                                           *[int(v) for v in ext], S.ptr(owner), h), "instance_paint")
        first = res[n_box * n_slot:n_box * n_slot + n_box].view(torch.int32)
        vbox = res[n_box * n_slot + n_box:].view(torch.int32)
        S.check(S.lib.sis3d_vertex_instance_overlap(
            S.ptr(t[0]), n_vert, S.ptr(t[1]), S.ptr(owner), *[int(v) for v in lo], *[int(v) for v in ext], *c["dims"],
            S.ptr(t[2]), n_slot, n_box, S.ptr(res), S.ptr(first), S.ptr(vbox), h), "vertex_instance_overlap")

    size = n_box * n_slot + n_box + n_vert
    eager_owner = torch.full((n_owner,), -7, dtype=torch.int32, device="cuda")
    eager = torch.full((size,), -7, dtype=torch.int64, device="cuda")
    launch(eager_owner, eager, torch.cuda.current_stream())
    owner = torch.full_like(eager_owner, -7)
    replayed = torch.full_like(eager, -7)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch(owner, replayed, torch.cuda.current_stream())
    torch.cuda.synchronize()
    assert (replayed == -7).all() and (owner == -7).all()  # captured, not run
    graph.replay()
    graph.replay()  # the graph initialises its own outputs: a second replay gives the same counts
    torch.cuda.synchronize()
    assert torch.equal(eager_owner, owner) and torch.equal(eager, replayed)
    hist, first, _ = F.vertex_instance_overlap(c["verts"], c["w2g"], slot.astype(np.int32), n_slot, bits, offs, ibox, lo, ext,
                                               c["dims"])
    e = eager.cpu().numpy()
    assert np.array_equal(e[:n_box * n_slot].reshape(n_box, n_slot), hist)
    assert np.array_equal(e[n_box * n_slot:n_box * n_slot + n_box].view(np.int32)[:n_box], first)


def test_benchmark_mode_end_to_end(tmp_path):
    """trainval.benchmark on synthetic chunks, then synthetic meshes, world2grid.txt and GT ids around its kept boxes: the
    fused tool prints the same stdout and writes the same CSV as vox2mesh.py followed by evaluate_semantic_instance.py."""
    import sis3d_synth as synth
    from lib.model import trainval
    c = synth.CASES["odd_45x27x41"]
    net, cfg = synth.make_net(c, keep_debug=False, math="exact")
    torch.save({k: v.detach().cpu().clone() for k, v in net.state_dict().items()}, str(tmp_path / "step_1.pth"))
    chunks = tmp_path / "chunks"
    chunks.mkdir()
    paths, provider = synth.write_chunks(str(chunks), c, (202, 7, 8, 9, 10, 11))
    cfg.TEST_FILELIST = paths
    dirs = {k: str(tmp_path / k) for k in ("results", "scans", "frames", "gt", "bench")}
    cfg.TEST_SAVE_DIR = dirs["results"]
    args = SimpleNamespace(output_dir=str(tmp_path), step=1, num_workers=0)
    assert trainval.benchmark(args, view_provider=provider) == len(paths)
    rng = np.random.default_rng(9)
    scenes = sorted(os.listdir(dirs["results"]))
    assert len(scenes) == len(paths)
    n_kept = 0
    os.makedirs(dirs["gt"])
    for s in scenes:
        d = os.path.join(dirs["results"], s)
        keep = np.asarray(pickle.load(open(os.path.join(d, "pred_mask_index"), "rb")), bool)
        box = np.load(os.path.join(d, "pred_box.npy"))[keep, :6]
        cls = np.load(os.path.join(d, "pred_class.npy"))[keep]
        n_kept += len(box)
        g = [rng.integers(0, c["dims"], (3000, 3))]
        for b in box:  # vertices around every kept box
            g.append(rng.integers(np.floor(b[:3]).astype(int) - 1, np.ceil(b[3:]).astype(int) + 1, (300, 3)))
        g = np.concatenate(g).astype(np.float64)
        gi = g.astype(np.int64)
        gt = np.zeros(len(g), np.int64)
        for k, b in enumerate(box):
            inside = np.all((gi >= np.rint(b[:3])) & (gi < np.rint(b[3:])), axis=1) & (gt == 0)
            label = int(cls[k]) if 1 <= cls[k] <= 18 and rng.random() < 0.8 else int(rng.integers(1, 19))
            gt[inside] = label * 1000 + k + 1
        w2g = np.eye(4)
        w2g[:3, :3] *= 1 / G.VOXEL
        w2g[:3, 3] = rng.uniform(-2, 2, 3)
        grid = g + rng.uniform(-0.4, 0.4, g.shape)
        verts = ((grid - w2g[:3, 3]) * G.VOXEL).astype(np.float32)
        os.makedirs(os.path.join(dirs["scans"], s))
        G.write_ply(os.path.join(dirs["scans"], s, s + "_vh_clean_2.ply"), verts)
        os.makedirs(os.path.join(dirs["frames"], s))
        G.write_world2grid(os.path.join(dirs["frames"], s, "world2grid.txt"), w2g)
        np.savetxt(os.path.join(dirs["gt"], s + ".txt"), gt, fmt="%d")
    assert n_kept > 0
    ap, out, csv = file_route_chain(dirs)
    exported = sum(len(open(os.path.join(dirs["bench"], s + ".txt")).read().splitlines()) for s in scenes)
    assert exported > 0
    fused = fused_route_chain(dirs, tmp_path)
    assert out == fused[1] and csv == fused[2] and np.array_equal(ap, fused[0], equal_nan=True)
    print(f"{len(scenes)} scenes, {n_kept} kept boxes, {exported} exported instances")
    print(out)
