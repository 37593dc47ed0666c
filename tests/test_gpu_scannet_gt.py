"""GPU: ScanNet GT from the annotation files on the device (sis3d_segment_gt_slots in csrc/eval.cu): the export tool
against the unmodified reference's files, the kernel against its numpy restatement and, at a real scan size, against the
reference's per-vertex loop, inside a CUDA graph, and evaluate_predictions.py without --gt_path against the file route,
on the golden chains and end to end on the output of the benchmark mode."""
import ctypes as C
import gc
import os
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from test_scannet_gt import GG, SLOT_CASES, check_chain, check_export_against_golden, check_slots, file_route_exported, \
    fused_from_annotations, slot_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("task", ["instance", "label"])
@pytest.mark.parametrize("key", GG.EXPORT_SETS)
def test_export_equals_reference_on_device(tmp_path, key, task):
    check_export_against_golden(tmp_path, key, task)


@pytest.mark.parametrize("case", list(SLOT_CASES))
def test_kernel_slots_equal_numpy_on_device(case):
    check_slots(case)


@pytest.mark.parametrize("key", GG.CHAIN_SETS)
def test_fused_from_annotations_on_device(tmp_path, key):
    check_chain(tmp_path, key)


def test_real_size_scan(tmp_path):
    """300k vertices, ~5k segments, 100 objects: the device's per-vertex ids equal the reference-style loop's and the
    numpy restatement's, vertex for vertex; the slot counts equal np.unique's."""
    from tools.scannet_benchmark import annotations as A
    from tools.scannet_benchmark import evaluate_predictions as F
    from tools.scannet_benchmark import utils
    p = GG.write_export_inputs("exp_rand0", str(tmp_path / "maps"))
    lm = utils.read_label_mapping(p["tsv"])
    lm2 = utils.read_label_mapping(p["csv"], label_from="nyu40id", label_to="mappedIdConsecutive", delimiter=",")
    cats = ["chair", "table", "office chair", "couch", "desk", "wall", "bed", "kitchen cabinet", "trash can"]
    _, seg, groups = GG.random_scan(np.random.default_rng(17), 300000, 5000, 100, cats)
    GG.write_scan(str(tmp_path / "scans"), "scene0000_00", np.zeros((len(seg), 3), np.float32), seg, groups)
    d = str(tmp_path / "scans" / "scene0000_00")
    agg, segf = os.path.join(d, "scene0000_00.aggregation.json"), os.path.join(d, "scene0000_00_vh_clean_2.0.010000.segs.json")
    gt = A.read_scene_gt(agg, segf, lm, lm2, "instance", "scene0000_00")
    assert len(gt.seg_ids) > 150 and len(gt.slot_ids) > 50
    slot, count = F.segment_gt_slots(gt)
    want = GG.loop_export_ids(*A.read_aggregation(agg), A.read_segmentation(segf, "s"), lm, lm2, "instance")
    got = gt.slot_ids[slot]
    assert int((got != want).sum()) == 0
    assert np.array_equal(slot, A.gt_ids_host(gt)[1])
    u, c = np.unique(want, return_counts=True)
    assert np.array_equal(gt.slot_ids[count > 0], u) and np.array_equal(count[count > 0], c)


def release(graph):
    """Destroy a captured graph now rather than whenever the cyclic GC gets to it: a CUDA graph torn down later, in the
    middle of another test's torch.profiler session, costs that session kernel records."""
    graph.reset()
    gc.collect()
    torch.cuda.synchronize()


def test_graph_replay_equals_eager():
    from lib import _sis3d as S
    gt = slot_case(*SLOT_CASES["many_slots"])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = [dev(gt.seg_index), dev(gt.seg_ids), dev(gt.seg_slot)]
    n_vert, n_seg, n_slot = len(gt.seg_index), len(gt.seg_ids), len(gt.slot_ids)

    def launch(slot, count, stream):
        S.check(S.lib.sis3d_segment_gt_slots(S.ptr(t[0]), n_vert, S.ptr(t[1]), S.ptr(t[2]), n_seg, n_slot, S.ptr(slot),
                                             S.ptr(count), C.c_void_p(stream.cuda_stream)), "segment_gt_slots")
    outs = []
    for _ in range(2):  # two eager launches
        slot = torch.full((n_vert,), -7, dtype=torch.int32, device="cuda")
        count = torch.full((n_slot,), -7, dtype=torch.int64, device="cuda")
        launch(slot, count, torch.cuda.current_stream())
        outs.append((slot, count))
    slot = torch.full((n_vert,), -7, dtype=torch.int32, device="cuda")
    count = torch.full((n_slot,), -7, dtype=torch.int64, device="cuda")
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch(slot, count, torch.cuda.current_stream())
    torch.cuda.synchronize()
    assert (slot == -7).all() and (count == -7).all()  # captured, not run
    graph.replay()
    graph.replay()  # the call initialises its counts: a second replay gives the same
    torch.cuda.synchronize()
    for a, b in ((outs[0], outs[1]), (outs[0], (slot, count))):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert int(count.sum()) == n_vert
    release(graph)


def test_fused_graph_replay_equals_eager():
    """The fused sequence from annotations (segment slots, paint, overlap) captured in one CUDA graph: replay equals the
    eager call, and two eager calls give identical bits."""
    from lib import _sis3d as S
    from test_scannet_eval import seeded_kernel_case
    from tools.scannet_benchmark import annotations as A
    from tools.scannet_benchmark import evaluate_predictions as F
    c = seeded_kernel_case(1)
    rng = np.random.default_rng(3)
    n_vert = len(c["verts"])
    seg_ids = np.sort(rng.choice(np.arange(0, 2 ** 31 - 1, 9973), 1500, replace=False)).astype(np.int32)
    seg_index = seg_ids[rng.integers(0, len(seg_ids), n_vert)]
    table = np.sort(rng.choice(seg_ids, 1100, replace=False))
    ids = rng.choice([3001, 3002, 5001, 7, 25001, 1001] + list(range(1, 1500)), len(table))
    slot_ids = np.unique(np.concatenate([[0], ids]))
    gt = A.SegmentGT(seg_index, table, np.searchsorted(slot_ids, ids).astype(np.int32), slot_ids, "")
    values = F.box_values(c["cls"], c["conf"])
    bits, offs, ibox, lo, ext = F.pack_boxes(c["box"], values, c["masks"], c["dims"])
    eager = [F.vertex_instance_overlap(c["verts"], c["w2g"], None, 0, bits, offs, ibox, lo, ext, c["dims"],
                                       want_vertex_box=True, segment_gt=gt) for _ in range(2)]
    for a, b in zip(*eager):
        assert np.array_equal(a, b)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = [dev(c["verts"]), dev(c["w2g"].astype(np.float64)), dev(seg_index), dev(offs), dev(ibox), dev(bits), dev(table),
         dev(gt.seg_slot)]
    n_box, n_slot = len(offs), len(slot_ids)
    owner = torch.full((int(np.prod(ext)),), -7, dtype=torch.int32, device="cuda")
    slots = torch.full((n_vert,), -7, dtype=torch.int32, device="cuda")
    res = torch.full((n_box * n_slot + n_box + n_vert + n_slot,), -7, dtype=torch.int64, device="cuda")
    hist, first = res[:n_box * n_slot], res[n_box * n_slot:n_box * n_slot + n_box].view(torch.int32)
    vbox = res[n_box * n_slot + n_box:n_box * n_slot + n_box + n_vert].view(torch.int32)
    count = res[n_box * n_slot + n_box + n_vert:]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        h = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        S.check(S.lib.sis3d_segment_gt_slots(S.ptr(t[2]), n_vert, S.ptr(t[6]), S.ptr(t[7]), len(table), n_slot, S.ptr(slots),
                                             S.ptr(count), h), "segment_gt_slots")
        S.check(S.lib.sis3d_instance_paint(S.ptr(t[5]), S.ptr(t[3]), S.ptr(t[4]), n_box, *[int(v) for v in lo],
                                           *[int(v) for v in ext], S.ptr(owner), h), "instance_paint")
        S.check(S.lib.sis3d_vertex_instance_overlap(
            S.ptr(t[0]), n_vert, S.ptr(t[1]), S.ptr(owner), *[int(v) for v in lo], *[int(v) for v in ext], *c["dims"],
            S.ptr(slots), n_slot, n_box, S.ptr(hist), S.ptr(first), S.ptr(vbox), h), "vertex_instance_overlap")
    torch.cuda.synchronize()
    assert (res == -7).all()  # captured, not run
    graph.replay()
    graph.replay()  # the calls initialise their own outputs: a second replay gives the same
    torch.cuda.synchronize()
    r = res.cpu().numpy()
    want_hist, want_first, want_vbox, want_count = eager[0]
    assert np.array_equal(r[:n_box * n_slot].reshape(n_box, n_slot), want_hist)
    assert np.array_equal(first.cpu().numpy()[:n_box], want_first) and np.array_equal(vbox.cpu().numpy()[:n_vert], want_vbox)
    assert np.array_equal(count.cpu().numpy(), want_count) and int(want_count.sum()) == n_vert
    assert np.array_equal(slots.cpu().numpy(), A.gt_ids_host(gt)[1])
    release(graph)


def test_benchmark_mode_end_to_end(tmp_path):
    """trainval.benchmark on synthetic chunks, then synthetic meshes, world2grid.txt and annotation files around its kept
    boxes: evaluate_predictions.py without --gt_path prints the same stdout and writes the same CSV as the export tool,
    vox2mesh.py and evaluate_semantic_instance.py in turn."""
    import sis3d_synth as synth
    from lib.model import trainval
    G = GG.G
    c = synth.CASES["odd_45x27x41"]
    net, cfg = synth.make_net(c, keep_debug=False, math="exact")
    torch.save({k: v.detach().cpu().clone() for k, v in net.state_dict().items()}, str(tmp_path / "step_1.pth"))
    chunks = tmp_path / "chunks"
    chunks.mkdir()
    paths, provider = synth.write_chunks(str(chunks), c, (202, 7, 8, 9, 10, 11))
    cfg.TEST_FILELIST = paths
    p = {k: str(tmp_path / k) for k in ("results", "scans", "frames")}
    cfg.TEST_SAVE_DIR = p["results"]
    args = SimpleNamespace(output_dir=str(tmp_path), step=1, num_workers=0)
    assert trainval.benchmark(args, view_provider=provider) == len(paths)
    rng = np.random.default_rng(9)
    scenes = sorted(os.listdir(p["results"]))
    n_kept = n_objects = 0
    for s in scenes:
        d = os.path.join(p["results"], s)
        keep = np.asarray(pickle.load(open(os.path.join(d, "pred_mask_index"), "rb")), bool)
        box = np.load(os.path.join(d, "pred_box.npy"))[keep, :6]
        cls = np.load(os.path.join(d, "pred_class.npy"))[keep]
        n_kept += len(box)
        g = [rng.integers(0, c["dims"], (3000, 3))]
        for b in box:  # vertices around every kept box
            g.append(rng.integers(np.floor(b[:3]).astype(int) - 1, np.ceil(b[3:]).astype(int) + 1, (300, 3)))
        g = np.concatenate(g).astype(np.float64)
        w2g = np.eye(4)
        w2g[:3, :3] *= 1 / G.VOXEL
        w2g[:3, 3] = rng.uniform(-2, 2, 3)
        verts = ((g + rng.uniform(-0.4, 0.4, g.shape) - w2g[:3, 3]) * G.VOXEL).astype(np.float32)
        seg, groups = GG.annotate_chain_scene(rng, dict(verts=verts, w2g=w2g, box=box, cls=cls))
        n_objects += len(groups)
        GG.write_scan(p["scans"], s, verts, seg, groups)
        os.makedirs(os.path.join(p["frames"], s))
        G.write_world2grid(os.path.join(p["frames"], s, "world2grid.txt"), w2g)
    assert n_kept > 0 and n_objects > 0
    p["filelist"], p["tsv"], p["csv"] = (str(tmp_path / f) for f in ("filelist.txt", "labels.tsv", "nyu40.csv"))
    (tmp_path / "filelist.txt").write_text("".join(s + "\n" for s in scenes))
    (tmp_path / "labels.tsv").write_text(GG.label_tsv())
    (tmp_path / "nyu40.csv").write_text(GG.label_csv(False))
    ap, out, csv = file_route_exported(p, tmp_path)
    fused = fused_from_annotations(p, tmp_path)
    assert out == fused[1] and csv == fused[2] and np.array_equal(ap, fused[0], equal_nan=True)
    print(f"{len(scenes)} scenes, {n_kept} kept boxes, {n_objects} GT objects")
    print(out)
