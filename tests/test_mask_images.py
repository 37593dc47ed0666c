"""CPU: the colour-aware mask head (MASK_USE_IMAGES, MASK_ONLY_IMAGES) against the unmodified reference
(tests/golden/mask_images_reference.npz, written by oracle/make_golden_mask_images.py), and its crop gather.

- the product model's mask head has the reference's state_dict keys and shapes, in its order, under both switches;
- the two combinations the reference cannot run are refused before any parameter is declared, and the reference failed on both;
- the oracle's forward (oracle/port_mask_images.py) equals the reference on every case;
- the colour planner's tables (sis3d_mask_color_plan_build, host code of libsis3d) describe every crop of both stage layouts;
- the gather (csrc/mask_color.cu), built for the host (tools/cuda_host_emu.py), equals the oracle's back-projected volume
  at every crop voxel bit for bit (fp16 rounding of it on the fp16 canvas), and writes nothing else: killed views, views that
  see nothing, crops on every scene face, extent-1 crops and adjacent crops whose one-voxel slab stays zero."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import sis3d_synth as synth
from conftest import ROOT, load_golden
from lib import _sis3d as S
from lib.layer_utils import projection as P
from lib.utils.config import cfg, cfg_from_file, cfg_reset

GOLDEN = "mask_images_reference.npz"
FORWARD = ("use_96x48x96", "only_96x48x96", "killed_45x27x41", "enet_45x27x41", "gt_45x27x41", "oimg_45x27x41",
           "suncg_40x24x40")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def case_inputs(g, tag):
    """(case dict, data, views) of a golden case: views["feats"] are the raw images when the case has them, and the killed
    views see nothing within PROJ_DEPTH_MAX."""
    dims = tuple(int(v) for v in g[f"{tag}_dims"])
    seed, n_img = int(g[f"{tag}_seed"]), int(g[f"{tag}_n_img"])
    cfgname = str(g[f"{tag}_cfgname"])
    c = dict(cfgname=cfgname, dims=dims, n_img=n_img, seed=seed, use_images=True, use_mask=True)
    data, boxes = synth.make_scene(seed, dims)
    from oracle import port
    views = synth.make_views(seed, dims, n_img, boxes, intrinsic=np.array(port.make_cfg(cfgname).INTRINSIC, dtype=np.float32))
    for k in g[f"{tag}_killed"]:
        views["depths"][int(k)][:] = 9.0
    s = int(g[f"{tag}_images_seed"])
    if s >= 0:
        views["feats"] = np.random.default_rng(s).standard_normal((n_img, 3, 256, 328)).astype(np.float32)
    return c, data, views


def case_weights(port, g, tag):
    ocfg = port.make_cfg(str(g[f"{tag}_cfgname"]))
    gt = bool(int(g[f"{tag}_gt"]))
    w = synth.make_weights(seed=0, net=ocfg.NET, use_images=True, num_classes=ocfg.NUM_CLASSES,
                           a1=0 if gt else ocfg.NUM_ANCHORS_LEVEL1, a2=0 if gt else ocfg.NUM_ANCHORS_LEVEL2, use_mask=True,
                           only_images=bool(int(g[f"{tag}_only_images_backbone"])), mask_images=str(g[f"{tag}_mask_images"]))
    return ocfg, {k: v for k, v in w.items() if not (gt and k.startswith("classifier_"))}


def oracle_forward(port, g, tag):
    from oracle import port_mask_images
    c, data, views = case_inputs(g, tag)
    ocfg, w = case_weights(port, g, tag)
    if int(g[f"{tag}_images_seed"]) >= 0:
        from test_only_images import enet_params
        with torch.no_grad():
            views = dict(views, feats=port.enet_encoder(enet_params(), torch.from_numpy(views["feats"])).numpy())
    only = str(g[f"{tag}_mask_images"]) == "only"
    if int(g[f"{tag}_gt"]):
        return port_mask_images.forward_gt_rois(ocfg, w, data, views, g[f"{tag}_gt_box"], only), w
    return port_mask_images.forward(ocfg, w, data, views, only, bool(int(g[f"{tag}_only_images_backbone"]))), w


@pytest.fixture
def scannet_cfg():
    def make(**over):
        cfg_reset()
        cfg_from_file(os.path.join(ROOT, "3d-sis_b200", "experiments", "cfgs", "ScanNet", "rpn_class_mask_5.yml"))
        cfg.NUM_CLASSES = 19
        cfg.USE_IMAGES_GT, cfg.USE_MASK = True, True
        for k, v in over.items():
            cfg[k] = v
        from lib.nets import backbones
        return getattr(backbones, cfg.NET)()
    yield make
    cfg_reset()


@pytest.mark.parametrize("mode", ["use", "only"])
def test_state_dict_equals_reference(golden, scannet_cfg, mode):
    net = scannet_cfg(USE_IMAGES=True, MASK_USE_IMAGES=True, MASK_ONLY_IMAGES=mode == "only")
    net.init_modules()
    got = [(k, tuple(v.shape)) for k, v in net.state_dict().items() if k.startswith("mask_backbone.")]
    want = [(str(k), tuple(int(v) for v in s)) for k, s in zip(golden[f"sd_{mode}_keys"], golden[f"sd_{mode}_shapes"])]
    assert got == want  # names, shapes and order
    d = dict(got)
    assert d["mask_backbone.geometry.10.weight"] == (64, 64, 1, 1, 1) and d["mask_backbone.color.0.weight"] == (64, 128, 3, 3, 3)
    assert d["mask_backbone.color.10.weight"][0] == (19 if mode == "only" else 64)
    assert d["mask_backbone.combine.0.weight"] == (128, 128, 3, 3, 3) and d["mask_backbone.combine.2.weight"] == (19, 128, 1, 1, 1)
    assert net.mask_backbone.colour and net.mask_backbone.only_images == (mode == "only")
    w = synth.make_weights(seed=0, use_images=True, num_classes=19, a1=3, a2=11, use_mask=True, mask_images=mode)
    assert [(k, tuple(v.shape)) for k, v in w.items() if k.startswith("mask_backbone.")] == want
    # the switches are read when the head is built: a net built colour-aware stays so
    cfg.MASK_USE_IMAGES = cfg.MASK_ONLY_IMAGES = False
    assert net._mask_colour() and net.mask_backbone.only_images == (mode == "only")


@pytest.mark.parametrize("over,what,key", [
    (dict(USE_IMAGES=False, MASK_USE_IMAGES=True), "MASK_USE_IMAGES with USE_IMAGES=False", "refused_no_images"),
    (dict(USE_IMAGES=True, MASK_USE_IMAGES=False, MASK_ONLY_IMAGES=True), "MASK_ONLY_IMAGES without MASK_USE_IMAGES",
     "refused_only_without_use")])
def test_refused_combinations(golden, scannet_cfg, over, what, key):
    m = scannet_cfg(**over)
    with pytest.raises(NotImplementedError, match=what):
        m.init_modules()
    assert not list(m.parameters()) and not list(m.buffers()), "parameters were declared before the refusal"
    assert str(golden[key]).split(":")[0].endswith("Error"), golden[key]  # the unmodified reference failed here


def test_switches_off_leave_the_mask_head_unchanged(scannet_cfg):
    net = scannet_cfg(USE_IMAGES=True)
    net.init_modules()
    keys = [k for k in net.state_dict() if k.startswith("mask_backbone.")]
    assert keys == [f"mask_backbone.geometry.{i}.weight" for i in (0, 2, 4, 6, 8, 10)]
    assert not net._mask_colour()


@pytest.mark.parametrize("tag", FORWARD)
def test_oracle_equals_reference(oracle, golden, tag):
    g, k = golden, tag + "_"
    out, _ = oracle_forward(oracle, g, tag)
    assert list(g[k + "killing_inds"]) == out["killing_inds"]
    sub = np.asarray(out["imageft"], dtype=np.float32).reshape(-1)[::int(g["step_imageft"])]
    if int(g[k + "images_seed"]) < 0:
        assert np.array_equal(sub, g[k + "imageft_sub"])  # exact: copy / max
    else:
        np.testing.assert_allclose(sub, g[k + "imageft_sub"], atol=1e-4)
    np.testing.assert_allclose(out["rois"].numpy(), g[k + "rois"], atol=1e-3)
    assert np.array_equal(np.asarray(out["cls_pred"]), g[k + "cls_pred"])
    np.testing.assert_allclose(np.asarray(out["cls_prob"]), g[k + "cls_prob"], atol=1e-5)
    np.testing.assert_allclose(out["pred_box"], g[k + "pred_box"], atol=1e-3)
    assert np.array_equal(out["mask_keep"], g[k + "keep"])
    assert np.array_equal(out["mask_crops"], g[k + "crops"])
    assert len(out["mask_pred"]) == int(g[k + "n_masks"]) > 0
    for j, i in enumerate(np.nonzero(out["mask_keep"])[0]):
        m = out["mask_pred"][j][0].numpy()
        c = int(g[k + "cls_pred"][i])
        np.testing.assert_allclose(m[c].reshape(-1)[::int(g["step_mask_cls"])], g[k + f"mask_{j}_cls_sub"], atol=1e-5)
        np.testing.assert_allclose(m.reshape(-1)[::int(g["step_mask_allcls"])], g[k + f"mask_{j}_allcls_sub"], atol=1e-5)
        assert abs(int((m[c] > 0.5).sum()) - int(g[k + f"mask_{j}_cls_on"])) <= 1


def test_golden_cases_cover_the_ask(golden):
    g = golden
    assert list(g["killed_45x27x41_killing_inds"]) == [1]
    assert int(g["enet_45x27x41_images_seed"]) >= 0
    assert int(g["gt_45x27x41_gt"]) == 1 and int(g["oimg_45x27x41_only_images_backbone"]) == 1
    for tag in FORWARD:
        assert int(g[f"{tag}_n_masks"]) >= 2, tag  # several crops per case
    faces = 0
    for tag in FORWARD:
        dims = g[f"{tag}_dims"]
        crops = g[f"{tag}_crops"][g[f"{tag}_keep"]]
        faces += int(((crops[:, :3] == 0) | (crops[:, 3:] == dims)).any(1).sum())
    assert faces > 0, "no kept crop on a scene face"
    assert [int(g[f"loop_test_{s}_written"]) for s in range(int(g["loop_n_scenes"]))] == [1] * int(g["loop_n_scenes"])
    # the reference's loops hand the mask head `[]` for the image features: the fixture's loop set crops the forward's own
    assert str(g["loop_refused"]).startswith("TypeError: conv3d()") and "list" in str(g["loop_refused"])
    assert os.path.getsize(os.path.join(ROOT, "tests", "golden", GOLDEN)) <= 1 << 20


# ---------------------------------------------------------------- planner and gather (host builds of the shipped code)
def det_table(crops):
    """[n, 16] detection rows keeping `crops` (x0, y0, z0, x1, y1, z1), with one dropped row between them."""
    rows = []
    for c in crops:
        r = np.zeros(16, np.float32)
        r[8], r[9:15], r[7] = 1.0, c, 3
        rows.append(r)
        rows.append(np.zeros(16, np.float32))  # keep flag off: not planned
    return np.stack(rows)


HOST_LIB = S.lib  # the planners are host code of libsis3d itself (no device needed)


def plans(det, dims, canvas):
    plan, cplan = S.MaskPlan(), S.MaskColorPlan()
    blob = np.zeros(1 << 20, np.uint8)
    args = (C.c_void_p(det.ctypes.data), det.shape[0])
    assert HOST_LIB.sis3d_mask_plan_build(*args, *dims, 19, int(canvas), C.c_void_p(blob.ctypes.data), C.c_size_t(blob.size),
                                          C.byref(plan)) == 0
    assert HOST_LIB.sis3d_mask_color_plan_build(*args, C.byref(plan), C.c_void_p(blob.ctypes.data), C.c_size_t(blob.size),
                                                C.byref(cplan)) == 0
    return plan, cplan, blob


def regions(blob, off, n):
    return np.frombuffer(blob[off:off + n * S.REGION_BYTES].tobytes(), dtype=S.REGION_DTYPE)


DIMS = (36, 22, 32)
CROPS = np.array([[0, 0, 0, 5, 4, 6],              # corner: the x, y and z = 0 faces
                  [5, 3, 2, 9, 9, 10],             # adjacent to the first along x
                  [30, 18, 26, 36, 22, 32],        # the x, y and z = max faces
                  [10, 0, 0, 11, 22, 32],          # extent 1 in x, the whole y and z
                  [12, 7, 31, 20, 8, 32],          # extent 1 in y and z, on the z = max face
                  [0, 10, 5, 36, 12, 9]], np.int64)  # the whole x extent


@pytest.mark.parametrize("canvas", [False, True])
def test_color_plan_tables(canvas):
    det = det_table(CROPS)
    plan, cplan, blob = plans(det, DIMS, canvas)
    nk = int(plan.n_kept)
    assert nk == len(CROPS) and cplan.off_crops >= plan.bytes and cplan.bytes <= blob.size
    crops = blob[cplan.off_crops:cplan.off_crops + 32 * nk].view(np.int32).reshape(nk, 8)
    ext = CROPS[:, 3:] - CROPS[:, :3]
    xoff = np.concatenate([[0], np.cumsum(ext[:, 0] + 1)[:-1]])
    assert np.array_equal(crops[:, :3], CROPS[:, :3]) and np.array_equal(crops[:, 3:6], ext)
    assert np.array_equal(crops[:, 6], xoff) and not crops[:, 7].any()
    offs = blob[plan.off_offs:plan.off_offs + 8 * (nk + 1)].view(np.int64)
    last, g2c, l128 = regions(blob, plan.off_last, nk), regions(blob, cplan.off_g2c, nk), regions(blob, cplan.off_last128, nk)
    cy, cz = int(plan.canvas[1]), int(plan.canvas[2])
    for j in range(nk):
        w, h, l = ext[j]
        assert tuple(g2c[j]["in_dim"]) == tuple(g2c[j]["out_dim"]) == (w, h, l) == tuple(l128[j]["out_dim"])
        assert g2c[j]["tile_begin"] == l128[j]["tile_begin"] == last[j]["tile_begin"]
        assert l128[j]["out_off"] == last[j]["out_off"] == offs[j] * 19 and not l128[j]["out_stride"].any()
        if canvas:
            assert tuple(g2c[j]["in_stride"]) == (cy * cz * 64, cz * 64, 64) and g2c[j]["in_off"] == xoff[j] * cy * cz * 64
            assert tuple(g2c[j]["out_stride"]) == (cy * cz * 128, cz * 128, 128) and g2c[j]["out_off"] == xoff[j] * cy * cz * 128
            assert tuple(l128[j]["in_stride"]) == (cy * cz * 128, cz * 128, 128) and l128[j]["in_off"] == xoff[j] * cy * cz * 128
        else:
            assert tuple(g2c[j]["in_stride"]) == (h * l * 64, l * 64, 64) and g2c[j]["in_off"] == offs[j] * 64
            assert g2c[j]["out_off"] == offs[j] * 128 and not g2c[j]["out_stride"].any()
            assert tuple(l128[j]["in_stride"]) == (h * l * 128, l * 128, 128) and l128[j]["in_off"] == offs[j] * 128
            c0, c128 = regions(blob, cplan.off_c0, nk)[j], regions(blob, cplan.off_c128, nk)[j]
            assert c0["in_off"] == c128["in_off"] == offs[j] * 128 and c0["out_off"] == offs[j] * 64
            assert c128["out_off"] == offs[j] * 128 and tuple(c0["in_stride"]) == tuple(c128["in_stride"]) == tuple(l128[j]["in_stride"])
    # a blob too small for the colour tables is reported, with the size it needs
    small = np.zeros(int(plan.bytes), np.uint8)
    p2, c2 = S.MaskPlan(), S.MaskColorPlan()
    S.check(S.lib.sis3d_mask_plan_build(C.c_void_p(det.ctypes.data), det.shape[0], *DIMS, 19, int(canvas),
                                        C.c_void_p(small.ctypes.data), C.c_size_t(small.size), C.byref(p2)))
    assert S.lib.sis3d_mask_color_plan_build(C.c_void_p(det.ctypes.data), det.shape[0], C.byref(p2), C.c_void_p(small.ctypes.data),
                                             C.c_size_t(small.size), C.byref(c2)) == -3 and c2.bytes == cplan.bytes


@pytest.fixture(scope="module")
def gather_lib(tmp_path_factory):
    """csrc/mask_color.cu and csrc/project.cu (maps, pairs, the dense back-projection) built for the host."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import cuda_host_emu
    out = str(tmp_path_factory.mktemp("emu_color") / "libsis3d_color_emu.so")
    cuda_host_emu.build(out, [os.path.join(ROOT, "3d-sis_b200", "csrc", f) for f in ("project.cu", "mask_color.cu")])
    lib = C.CDLL(out)
    lib.sis3d_strerror.restype = C.c_char_p
    return lib


@pytest.fixture
def emu(monkeypatch, gather_lib):
    monkeypatch.setattr(S, "lib", gather_lib)
    monkeypatch.setattr(S, "ptr", lambda t: None if t is None else C.c_void_p(t.data_ptr()))
    monkeypatch.setattr(S, "stream", lambda: None)
    return S


def gather(S_, feats_t, pix, pairs, n_pairs, n_img, plan, cplan, blob, layout, dims):
    nk, total = int(plan.n_kept), int(plan.total_voxels)
    crops = torch.from_numpy(blob[cplan.off_crops:cplan.off_crops + 32 * nk].view(np.int32).copy())
    offs = torch.from_numpy(blob[plan.off_offs:plan.off_offs + 8 * (nk + 1)].view(np.int64).copy())
    cx, cy, cz = (int(v) for v in plan.canvas)
    if layout == 0:
        out = torch.full((total, 128), 7.0)  # every row is written
    else:
        out = torch.zeros(cx, cy, cz, 128, dtype=torch.float16 if layout == 2 else torch.float32)
    S_.check(S_.lib.sis3d_mask_color_gather(S_.ptr(feats_t), S_.ptr(pix), S_.ptr(pairs), S_.ptr(n_pairs), n_img, 128, 41 * 32,
                                            *dims, S_.ptr(crops), S_.ptr(offs), nk, C.c_int64(total), cy, cz, layout, S_.ptr(out),
                                            None), "mask_color_gather")
    return out, offs.numpy()


VIEW_ROWS = {  # row -> (seed, n_img, views that see nothing, views dropped by killing_inds through the host pairing)
    "views": (202, 3, (), ()),
    "blind_view": (202, 3, (1,), ()),
    "killed_view": (303, 4, (), (2,)),
}


@pytest.mark.parametrize("row", list(VIEW_ROWS))
@pytest.mark.parametrize("layout", [0, 1, 2])
def test_gather_equals_oracle_volume_emulated(oracle, emu, row, layout):
    seed, n_img, blind, killed = VIEW_ROWS[row]
    ocfg = oracle.make_cfg("scannet")
    _, boxes = synth.make_scene(seed, DIMS)
    v = synth.make_views(seed, DIMS, n_img, boxes)
    for k in blind:
        v["depths"][k][:] = 9.0
    intr = ocfg.INTRINSIC
    vp = P._view_params_torch(intr, (41, 32), ocfg.PROJ_DEPTH_MIN, ocfg.PROJ_DEPTH_MAX, DIMS, torch.from_numpy(v["poses"]),
                              torch.from_numpy(v["world2grid"]))
    pix, counts = P.project_maps(vp, torch.from_numpy(v["depths"]).contiguous(), (intr[0][0], intr[1][1], intr[0][2], intr[1][2]),
                                 (ocfg.PROJ_DEPTH_MIN, ocfg.PROJ_DEPTH_MAX, ocfg.VOXEL_SIZE), DIMS, 41, 32)
    feats = torch.from_numpy(v["feats"]).contiguous()
    if killed:  # the reference calling convention: every map is real here, and killing_inds skips by position
        pl = [(k, k) for k in range(n_img) if k not in killed]
        pairs = torch.tensor([x for p in pl for x in p] + [0] * (3 * n_img - 2 * len(pl)), dtype=torch.int32)
        n_pairs = torch.tensor([len(pl)], dtype=torch.int32)
        want = None
        for k in range(n_img):
            if k not in killed:
                cur = P.backproject(feats[k:k + 1], pix[k:k + 1], torch.zeros(3, dtype=torch.int32),
                                    torch.ones(1, dtype=torch.int32), DIMS, 41, 32)
                want = cur if want is None else torch.maximum(want, cur)
        want = want.permute(3, 0, 1, 2)[None]
    else:
        pairs, n_pairs = torch.empty(3 * n_img, dtype=torch.int32), torch.empty(1, dtype=torch.int32)
        emu.check(emu.lib.sis3d_backproject_pairs(emu.ptr(counts), n_img, emu.ptr(pairs), emu.ptr(n_pairs), None))
        want, kill = oracle.backproject_views(ocfg, v["feats"], v["depths"], v["poses"], v["world2grid"], DIMS)
        assert set(blind) <= set(kill)
    feats_t = torch.empty(n_img, 41 * 32, 128)
    emu.check(emu.lib.sis3d_mask_color_feats_t(emu.ptr(feats), n_img, 128, 41 * 32, emu.ptr(feats_t), None))
    assert torch.equal(feats_t, feats.reshape(n_img, 128, -1).transpose(1, 2))
    vol = want[0].permute(1, 2, 3, 0)  # [X, Y, Z, 128]
    assert 0 < float((vol != 0).float().mean()) < 0.5
    plan, cplan, blob = plans(det_table(CROPS), DIMS, layout != 0)
    out, offs = gather(emu, feats_t, pix, pairs, n_pairs, n_img, plan, cplan, blob, layout, DIMS)
    ext = CROPS[:, 3:] - CROPS[:, :3]
    xoff = np.concatenate([[0], np.cumsum(ext[:, 0] + 1)[:-1]])
    written = torch.zeros(out.shape[:-1], dtype=torch.bool) if layout else None
    for j, c in enumerate(CROPS):
        ref = vol[c[0]:c[3], c[1]:c[4], c[2]:c[5]]
        if layout == 0:
            got = out[offs[j]:offs[j + 1]].reshape(ref.shape)
        else:
            w, h, l = ext[j]
            got = out[xoff[j]:xoff[j] + w, :h, :l]
            written[xoff[j]:xoff[j] + w, :h, :l] = True
        if layout == 2:
            ref = ref.half()
        assert torch.equal(got, ref), (row, layout, j)
    if layout:  # outside the crops -- the slabs between them and the rows past a crop's own h, l -- nothing was written
        assert not out[~written].any()
