"""GPU: the colour-aware mask head (MASK_USE_IMAGES, MASK_ONLY_IMAGES) on the ragged mask stage.

- golden parity with the unmodified reference (tests/golden/mask_images_reference.npz): integer outputs bit-exact in the
  default mode; masks within 1e-3 of the fixture, checked by teacher-forcing the reference's detections in every math mode;
- the gather: every crop's 128 channels equal the dense back-projected volume (sis3d_backproject_max on the same maps) bit
  for bit, on the sparse and the dense back-projection routes, from features and from raw images through ENet, eager and on
  graph replay (which must gather what the eager forward gathers: the maps outlive the captured graph's own use of them);
- the layers: on all three mask routes the stage's output is within the fp64 bound of tests/test_gpu_mask_stage.py carried
  through every layer of both stacks, the concatenation and combine, and fp64 models of broken compositions miss it by POWER;
- the scene loop: forward_pipelined equals forward bit for bit over scenes of changing shape and view count, with detected
  and with ground-truth RoIs; run_scenes writes byte-identical files synchronously and pipelined, equal to the reference's
  loops, with the reference's mask mAP; a default and a colour-aware net in one process give what each gives alone;
- scale: a 208x48x160 scene with whole-scene ground-truth boxes runs the 128-channel canvas at its largest."""
import ctypes as C
import filecmp
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sis3d_synth as synth
from conftest import load_golden
from lib import _sis3d as S
from lib.layer_utils import projection as proj
from lib.nets.network import Network
from test_gpu_mask_stage import F16_FLOOR, U16, _prop
from test_gpu_simt_accuracy import SIG_FLOOR, gamma
from test_gpu_tc_accuracy import C_1X, C_T, POWER
from test_mask_images import FORWARD, GOLDEN, case_inputs, det_table
from test_only_images import enet_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROUTE_MODE = {0: "fp32", 1: "tf32", 2: "exact"}  # mask route -> a math mode that reaches it


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def make_color_net(mask_images="use", math="exact", enet=False, keep_debug=False, gt_rois=None, only_images=False,
                   cfgname="scannet"):
    """The colour-aware product Network with the weights the fixture's reference model loaded; enet=True declares the 2-D
    encoder (USE_IMAGES_GT = False) with the parameters of tests/golden/enet_encoder.npz."""
    c = dict(cfgname=cfgname, use_images=True, use_mask=True)
    net, cfg = synth.make_net(c, keep_debug=keep_debug, math=math, gt_rois=gt_rois, only_images=only_images,
                              mask_images=mask_images)
    if not enet:
        return net, cfg
    sd3d = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    del net
    cfg.USE_IMAGES_GT = False
    from lib.nets import backbones
    torch.manual_seed(1234)
    net = getattr(backbones, cfg.NET)()
    net.init_modules()
    sd = net.state_dict()
    for n, p in zip(net._enet_names, enet_params(), strict=True):
        sd[n] = p
    sd.update(sd3d)
    net.load_state_dict(sd, strict=True)
    net._keep_debug = keep_debug
    net.set_conv_math(math)
    return net, cfg


def case_net(g, tag, math="exact", keep_debug=False):
    net, cfg = make_color_net(str(g[f"{tag}_mask_images"]), math, enet=int(g[f"{tag}_images_seed"]) >= 0, keep_debug=keep_debug,
                              gt_rois=False if int(g[f"{tag}_gt"]) else None,
                              only_images=bool(int(g[f"{tag}_only_images_backbone"])), cfgname=str(g[f"{tag}_cfgname"]))
    c, data, views = case_inputs(g, tag)
    blobs = synth.make_blobs(c, data, views)
    if int(g[f"{tag}_gt"]):
        blobs["gt_box"] = [torch.from_numpy(g[f"{tag}_gt_box"])]
    return net, cfg, blobs


def check_masks(masks, g, tag):
    k = tag + "_"
    assert len(masks) == int(g[k + "n_masks"])
    pc = g[k + "cls_pred"][g[k + "keep"]]
    worst = 0.0
    for j, m in enumerate(masks):
        m = m[0].cpu().numpy()
        worst = max(worst, float(np.abs(m[pc[j]].reshape(-1)[::int(g["step_mask_cls"])] - g[k + f"mask_{j}_cls_sub"]).max()),
                    float(np.abs(m.reshape(-1)[::int(g["step_mask_allcls"])] - g[k + f"mask_{j}_allcls_sub"]).max()))
    assert worst < 1e-3, f"{tag}: masks differ from the reference's by {worst:.3g}"
    return worst


@pytest.mark.parametrize("tag", FORWARD)
def test_golden_default_mode(golden, tag):
    g, k = golden, tag + "_"
    net, _, blobs = case_net(g, tag)
    for rep in range(3):  # eager on first sight, then captured and replayed
        P = net.forward(blobs, "TEST", None)
        det = P["detections_host"]
        assert np.array_equal(P["cls_pred"].cpu().numpy(), g[k + "cls_pred"])
        assert np.array_equal(det[:, 8] > 0.5, g[k + "keep"])
        assert np.array_equal(det[:, 9:15].astype(np.int64), g[k + "crops"])
        check_masks(P["mask_pred"][0], g, tag)
    if not int(g[k + "gt"]):
        assert net._replayed_kernels > 0


def teacher_forced(net, blobs, g, tag):
    """The mask stage on the reference's detections (keep flags, crops, classes), with the scene's own colour sources."""
    k = tag + "_"
    keep, crops, cls = g[k + "keep"], g[k + "crops"], g[k + "cls_pred"]
    det = np.zeros((len(keep), 16), np.float32)
    det[:, 7], det[:, 8], det[:, 9:15] = cls, keep, crops
    net._ensure_packed()
    dims = tuple(int(v) for v in blobs["data"].shape[2:])
    with torch.no_grad():
        src = net._color_sources(blobs, None, dims, torch.device(DEV), net._fused_inputs(blobs, dims))
        scene = blobs["data"].to(DEV, torch.float32).contiguous()
        masks = net._mask_branch(scene, det, len(det), None, src)
    torch.cuda.synchronize()
    return masks


@pytest.mark.parametrize("math", list(Network.MATH_MODES))
@pytest.mark.parametrize("tag", FORWARD)
def test_golden_masks_teacher_forced(golden, tag, math):
    net, _, blobs = case_net(golden, tag, math)
    worst = check_masks(teacher_forced(net, blobs, golden, tag), golden, tag)
    print(f"{tag} {math}: worst mask difference {worst:.3g}")


# ------------------------------------------------------------------------------------------------ the gather
def _dense(src, dims):
    """The dense back-projected volume of the stage's own colour sources (sis3d_backproject_max), VC [X, Y, Z, 128]."""
    n, hw, Cn = src["feats_t"].shape
    feats = src["feats_t"].transpose(1, 2).contiguous().view(n, Cn, 32, 41)
    return proj.backproject(feats, src["pix"], src["pairs"], src["n_pairs"], dims, 41, 32)


def gathered(net, det, dims, src):
    """Every kept crop's gathered colour input (compact layout), and the crop list."""
    plan, cplan, stage = net._mask_plan(det, det.shape[0], *dims, 19, False, torch.device(DEV), True)
    nk, total = int(plan.n_kept), int(plan.total_voxels)
    host = stage.numpy()
    crops = torch.from_numpy(host[cplan.off_crops:cplan.off_crops + 32 * nk].view(np.int32).reshape(nk, 8).copy())
    offs = torch.from_numpy(host[plan.off_offs:plan.off_offs + 8 * (nk + 1)].view(np.int64).copy())
    crops_d, offs_d = crops.to(DEV), offs.to(DEV)
    out = torch.full((total, 128), float("nan"), device=DEV)
    S.check(S.lib.sis3d_mask_color_gather(S.ptr(src["feats_t"]), S.ptr(src["pix"]), S.ptr(src["pairs"]), S.ptr(src["n_pairs"]),
                                          int(src["n_views"]), 128, int(src["hw"]), *dims, S.ptr(crops_d), S.ptr(offs_d), nk,
                                          C.c_int64(total), 1, 1, 0, S.ptr(out), S.stream()), "gather")
    torch.cuda.synchronize()
    return out, crops.numpy(), offs.numpy()


class GatherSpy:
    """Wraps a net's colour mask stage: before each call, gathers every kept crop on its own and checks it against the dense
    volume of the same sources; records the gathered crops."""

    def __init__(self, net):
        self.net, self.seen = net, []
        orig = net._mask_branch_color

        def spy(scene, det, n, extras, color):
            dims = tuple(int(v) for v in scene.shape[2:])
            torch.cuda.synchronize()
            out, crops, offs = gathered(net, np.ascontiguousarray(det[:n], np.float32), dims, color)
            vol = _dense(color, dims)
            for j, c in enumerate(crops):
                ref = vol[c[0]:c[0] + c[3], c[1]:c[1] + c[4], c[2]:c[2] + c[5]].reshape(-1, 128)
                assert torch.equal(out[offs[j]:offs[j + 1]], ref), f"crop {j} {c[:6]}: gather differs from the dense volume"
            self.seen.append((out.cpu(), crops, vol.cpu() if net._keep_debug else None))
            return orig(scene, det, n, extras, color)

        net.__dict__["_mask_branch_color"] = spy


@pytest.mark.parametrize("sparse", [True, False])
@pytest.mark.parametrize("tag", ["use_96x48x96", "enet_45x27x41", "killed_45x27x41"])
def test_gather_equals_dense_volume(golden, tag, sparse):
    net, _, blobs = case_net(golden, tag, keep_debug=not sparse)
    net._sparse_color = sparse
    spy = GatherSpy(net)
    net._use_graph = False
    net.forward(blobs, "TEST", None)
    eager = spy.seen[-1]
    assert len(eager[1]) == int(golden[f"{tag}_n_masks"]) > 0
    if not sparse:  # keep_debug: the static stage's own dense volume, the one the reference crops
        assert torch.equal(eager[2], net._imageft_vc.cpu())
    net._use_graph, net._keep_debug = True, False
    for _ in range(3):
        net.forward(blobs, "TEST", None)
        assert torch.equal(spy.seen[-1][0], eager[0]), "graph replay gathered other features than the eager forward"
    assert net._replayed_kernels > 0


# ------------------------------------------------------------------------------------------------ the layers against fp64
def _layer(x, e, w, tc, relu, store16):
    pad = w.shape[2] // 2
    y = F.conv3d(x, w, padding=pad)
    p = _prop(e, w)
    ax = x.abs() + e
    if tc:
        loc = C_1X * F.conv3d(ax * ax, w * w, padding=pad).sqrt() + C_T * (y.abs() + p)
    else:
        loc = gamma(w[0].numel() + 2) * F.conv3d(ax, w.abs(), padding=pad)
    e = p + loc
    if relu:
        y = F.relu(y)
    if store16:
        e = e + U16 * (y.abs() + e) + F16_FLOOR
    return y, e


def _stack(x, e, W, prefix, route, first_tc):
    for i, idx in enumerate((0, 2, 4, 6, 8)):
        tc = route > 0 and (i > 0 or first_tc)
        x, e = _layer(x, e, W[f"{prefix}.{idx}"], tc, True, route == 2 and i < 4)
    return _layer(x, e, W[f"{prefix}.10"], False, False, route == 2)


def reference(xs, xi, W, route, only, model=None):
    """fp64 output and bound of one crop: xs [1,2,w,h,l] scene window, xi [1,128,w,h,l] colour window (or, for the slab
    model, [1,128,w+2,h,l] with the neighbours' slices at x = 0 and w + 1)."""
    ei = (U16 * xi.abs() + F16_FLOOR) if route == 2 else torch.zeros_like(xi)
    if xi.shape[2] != xs.shape[2]:  # the slab model: colour.0 reads real data in its x padding
        w0 = W["color.0"]
        y = F.conv3d(F.pad(xi, (1, 1, 1, 1, 0, 0)), w0)
        x, e = F.relu(y), torch.zeros_like(y)
        for i, idx in enumerate((2, 4, 6, 8)):
            x, e = _layer(x, e, W[f"color.{idx}"], route > 0, True, False)
        col, ec = _layer(x, e, W["color.10"], False, False, False)
    else:
        col, ec = _stack(xi, ei, W, "color", route, True)
    if only:
        if model == "geometry_run_under_only":
            g, _ = _stack(xs, torch.zeros_like(xs), W, "geometry", route, False)
            col = col + g[:, :col.shape[1]]
        return torch.sigmoid(col), ec / 4 + SIG_FLOOR
    geo, eg = _stack(xs, torch.zeros_like(xs), W, "geometry", route, False)
    if model == "relu_after_geometry_1x1":
        geo = F.relu(geo)
    cat = torch.cat([col, geo] if model == "swapped_halves" else [geo, col], 1)
    x, e = _layer(cat, torch.cat([eg, ec], 1), W["combine.0"], route > 0, model != "combine_without_relu", False)
    y, e = _layer(x, e, W["combine.2"], False, False, False)
    return torch.sigmoid(y), e / 4 + SIG_FLOOR


MODELS = ("swapped_halves", "relu_after_geometry_1x1", "combine_without_relu", "crop_window_off_by_one", "last_view_not_max",
          "killed_view_counted", "neighbour_features_in_slab", "geometry_run_under_only")
ONLY_MODELS = {"crop_window_off_by_one", "last_view_not_max", "killed_view_counted", "neighbour_features_in_slab",
               "geometry_run_under_only"}


def _volume(src, dims, pairs=None):
    s = dict(src)
    if pairs is not None:
        s["pairs"] = torch.tensor(sum(([a, b] for a, b in pairs), []) + [0] * (3 * int(src["n_views"]) - 2 * len(pairs)),
                                  dtype=torch.int32, device=DEV)
        s["n_pairs"] = torch.tensor([len(pairs)], dtype=torch.int32, device=DEV)
    return _dense(s, dims).permute(3, 0, 1, 2)[None].double()


def _win(v, x0, y0, z0, w, h, l):
    """Window of an NCDHW volume with zeros outside it."""
    X, Y, Z = v.shape[2:]
    out = v.new_zeros(v.shape[0], v.shape[1], w, h, l)
    xa, ya, za = max(x0, 0), max(y0, 0), max(z0, 0)
    xb, yb, zb = min(x0 + w, X), min(y0 + h, Y), min(z0 + l, Z)
    if xa < xb and ya < yb and za < zb:
        out[:, :, xa - x0:xb - x0, ya - y0:yb - y0, za - z0:zb - z0] = v[:, :, xa:xb, ya:yb, za:zb]
    return out


LAYER_ROWS = {  # row -> the golden case giving the scene, views and (but for the edge row) crops
    "bench_crops": "use_96x48x96",
    "edge_crops": "use_96x48x96",     # EDGE_CROPS
    "killed_view": "killed_45x27x41",  # view 1 sees nothing: the reference's pairing then keeps view 0 alone
}
EDGE_CROPS = np.array([[0, 0, 0, 12, 8, 14],          # the x, y and z = 0 faces
                       [12, 5, 4, 20, 17, 22],        # adjacent to the first along x
                       [84, 36, 80, 96, 48, 96],      # the x, y and z = max faces
                       [40, 0, 0, 41, 48, 96],        # extent 1 in x, the whole y and z
                       [44, 20, 95, 60, 21, 96],      # extent 1 in y and z, on the z = max face
                       [0, 24, 40, 96, 30, 52]], np.int64)  # the whole x extent


def _row(golden, rid):
    tag = LAYER_ROWS[rid]
    c, data, views = case_inputs(golden, tag)
    if rid == "edge_crops":
        det = det_table(EDGE_CROPS)
        det[:, 7] = np.arange(len(det)) % 19
        return synth.make_blobs(c, data, views), det
    det = np.zeros((len(golden[tag + "_keep"]), 16), np.float32)
    det[:, 7], det[:, 8], det[:, 9:15] = golden[tag + "_cls_pred"], golden[tag + "_keep"], golden[tag + "_crops"]
    return synth.make_blobs(c, data, views), det


@pytest.mark.parametrize("only", [False, True])
@pytest.mark.parametrize("route", [0, 1, 2])
@pytest.mark.parametrize("rid", list(LAYER_ROWS))
def test_layers_against_fp64(golden, rid, route, only):
    blobs, det = _row(golden, rid)
    net, _ = make_color_net("only" if only else "use", ROUTE_MODE[route])
    assert net.MASK_ROUTES.index(net._mask_math) == route
    with torch.no_grad():
        p = dict(net.named_parameters())
        # the head without the synthetic model's gain: logits where the sigmoid is not saturated
        p["mask_backbone." + ("color.10" if only else "combine.2") + ".weight"].mul_(0.125)
        if not only:  # nor the geometry half's: its rounding would otherwise hide what the colour half gets wrong
            p["mask_backbone.geometry.10.weight"].mul_(0.125)
    dims = tuple(int(v) for v in blobs["data"].shape[2:])
    net._ensure_packed()
    with torch.no_grad():
        src = net._color_sources(blobs, None, dims, torch.device(DEV), net._fused_inputs(blobs, dims))
        scene = blobs["data"].to(DEV, torch.float32).contiguous()
        masks = net._mask_branch(scene, det, len(det), None, src)
    torch.cuda.synchronize()
    W = {k[len("mask_backbone."):-len(".weight")]: v.detach().double() for k, v in net.state_dict().items()
         if k.startswith("mask_backbone.")}
    vol = _volume(src, dims)
    np_ = int(src["n_pairs"].item())
    pr = [tuple(p) for p in src["pairs"][:2 * np_].view(-1, 2).tolist()]
    alt = {"last_view_not_max": _volume(src, dims, pr[-1:])} if len(pr) > 1 else {}
    naive = [(v, v) for v in range(int(src["n_views"]))]
    if pr != naive:  # a view without a projection counted after all: every view paired with its own map
        alt["killed_view_counted"] = _volume(src, dims, naive)
    sd = scene.double()
    kept = det[det[:, 8] > 0.5]
    cr = [(int(d[9]), int(d[10]), int(d[11]), int(d[12] - d[9]), int(d[13] - d[10]), int(d[14] - d[11])) for d in kept]
    worst, ratio = 0.0, {}
    for j, (c, m) in enumerate(zip(cr, masks)):
        xs, xi = _win(sd, *c), _win(vol, *c)
        ref, bound = reference(xs, xi, W, route, only)
        got = m.double()
        worst = max(worst, float(((got - ref).abs() / bound).max()))
        for name in MODELS:
            if only and name not in ONLY_MODELS or not only and name == "geometry_run_under_only":
                continue
            if name in ("last_view_not_max", "killed_view_counted"):
                if name not in alt:
                    continue
                mref, _ = reference(xs, _win(alt[name], *c), W, route, only)
            elif name == "crop_window_off_by_one":
                mref, _ = reference(xs, _win(vol, c[0] + 1, *c[1:]), W, route, only)
            elif name == "neighbour_features_in_slab":  # no zero slab: the canvas neighbours' edge slices pad the crop
                if len(cr) < 2:
                    continue
                ext = vol.new_zeros(1, 128, c[3] + 2, c[4], c[5])
                ext[:, :, 1:-1] = xi
                for k, last in ((j - 1, True), (j + 1, False)):  # the previous crop's last slice, the next crop's first
                    if 0 <= k < len(cr):
                        n_ = cr[k]
                        h, l = min(c[4], n_[4]), min(c[5], n_[5])
                        x = n_[0] + n_[3] - 1 if last else n_[0]
                        ext[:, :, 0 if last else -1, :h, :l] = vol[:, :, x, n_[1]:n_[1] + h, n_[2]:n_[2] + l]
                mref, _ = reference(xs, ext, W, route, only)
            else:
                mref, _ = reference(xs, xi, W, route, only, model=name)
            ratio[name] = max(ratio.get(name, 0.0), float(((got - mref).abs() / bound).max()))
    print(f"{rid} route {route} only={only}: worst err/bound {worst:.3g}; model ratios "
          + ", ".join(f"{k} {v:.3g}" for k, v in ratio.items()))
    assert worst <= 1.0, f"{rid} route {route}: err/bound {worst:.3g}"
    for name, r in ratio.items():
        assert r >= POWER, f"{rid} route {route}: the model '{name}' is within {r:.3g} of the bound"
    if not only:
        assert {"swapped_halves", "relu_after_geometry_1x1", "combine_without_relu"} <= set(ratio)
    assert {"crop_window_off_by_one", "neighbour_features_in_slab"} <= set(ratio)
    assert ("killed_view_counted" if rid == "killed_view" else "last_view_not_max") in ratio


# ------------------------------------------------------------------------------------------------ the scene loop
def _snap(P):
    masks = P["mask_pred"][0]
    return dict(det=P["detections_host"].copy(), cls_prob=P["cls_prob"].clone(), masks=[m.clone() for m in masks],
                bits=P["mask_bits_host"].copy() if "mask_bits_host" in P else None)


def _same(a, b):
    return (np.array_equal(a["det"].view(np.int32), b["det"].view(np.int32)) and torch.equal(a["cls_prob"], b["cls_prob"])
            and len(a["masks"]) == len(b["masks"])
            and all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a["masks"], b["masks"])))


def _loop_blobs(k, gt=False):
    dims, n_img = (40 + 8 * (k % 3), 24 + 4 * (k % 2), 40 + 4 * (k % 4)), 1 + k % 5
    data, boxes = synth.make_scene(800 + k, dims)
    b = synth.make_blobs(dict(use_images=True), data, synth.make_views(800 + k, dims, n_img, boxes))
    if gt:
        rng = np.random.default_rng(k)
        b["gt_box"] = [torch.from_numpy(np.concatenate([boxes, rng.integers(0, 19, (len(boxes), 1))], 1).astype(np.float32))]
    return b


@pytest.mark.parametrize("mode", ["use", "only"])
def test_pipelined_equals_forward(mode):
    blobs = [_loop_blobs(k) for k in range(6)]
    seq = [blobs[i] for i in (0, 1, 2, 3, 4, 5, 1, 0, 3, 2, 5, 4, 0, 1)]
    net, _ = make_color_net(mode)
    net._use_graph = False
    eager = [_snap(net.forward(b, "TEST", None)) for b in seq]
    net._use_graph = True
    sync = [_snap(net.forward(b, "TEST", None)) for b in seq]
    assert net._replayed_kernels > 0
    got = [(b, _snap(P)) for b, P in net.forward_pipelined(iter(seq))]
    assert len(got) == len(seq) and all(a[0] is b for a, b in zip(got, seq))
    for k, (e, s, (_, p)) in enumerate(zip(eager, sync, got)):
        assert _same(e, s), f"scene {k}: graph replay differs from eager"
        assert _same(s, p), f"scene {k}: pipelined differs from forward"
    assert sum(len(s["masks"]) for s in sync) > 10


def test_gt_rois_pipelined_equals_forward():
    """Ground-truth RoIs: the scene runs the projection maps and pairs (no backbone, RPN or classifier) before its stage."""
    blobs = [_loop_blobs(k, gt=True) for k in range(6)]
    seq = blobs + blobs[::-1]
    net, _ = make_color_net("use", gt_rois=False)
    sync = [_snap(net.forward(b, "TEST", None)) for b in seq]
    got = [_snap(P) for _, P in net.forward_pipelined(iter(seq))]
    for k, (s, p) in enumerate(zip(sync, got)):
        assert _same(s, p), f"scene {k}: pipelined differs from forward"
    assert net._replayed_kernels == 0 and sum(len(s["masks"]) for s in sync) > 10


def test_two_nets_in_one_process():
    blobs = [_loop_blobs(k) for k in range(4)]
    alone = {}
    for mode in (None, "use"):
        net, _ = make_color_net(mode)
        alone[mode] = [_snap(net.forward(b, "TEST", None)) for b in blobs + blobs]
        del net
    default, _ = make_color_net(None)
    colour, _ = make_color_net("use")
    for i, b in enumerate(blobs + blobs):
        assert _same(_snap(default.forward(b, "TEST", None)), alone[None][i]), f"default net, scene {i}"
        assert _same(_snap(colour.forward(b, "TEST", None)), alone["use"][i]), f"colour-aware net, scene {i}"
    for net, want in ((default, alone[None]), (colour, alone["use"])):
        for i, (_, P) in enumerate(net.forward_pipelined(iter(blobs))):
            assert _same(_snap(P), want[i])


def test_mask_backbone_forward_on_a_dense_crop(golden):
    """MaskBackbone.forward(scene, imageft) -- the reference's signature -- on a crop of the dense volume equals the stage's
    own result for that crop."""
    tag = "use_96x48x96"
    for route in (0, 1, 2):
        net, _, blobs = case_net(golden, tag, ROUTE_MODE[route])
        masks = teacher_forced(net, blobs, golden, tag)
        dims = tuple(int(v) for v in blobs["data"].shape[2:])
        with torch.no_grad():
            src = net._color_sources(blobs, None, dims, torch.device(DEV), net._fused_inputs(blobs, dims))
        vol = _dense(src, dims).permute(3, 0, 1, 2)[None]
        scene = blobs["data"].to(DEV)
        crops = golden[tag + "_crops"][golden[tag + "_keep"]]
        for j in (0, len(crops) - 1):
            x0, y0, z0, x1, y1, z1 = (int(v) for v in crops[j])
            m = net.mask_backbone(scene[:, :, x0:x1, y0:y1, z0:z1], vol[:, :, x0:x1, y0:y1, z0:z1])
            torch.testing.assert_close(m, masks[j], atol=1e-5, rtol=0)
        with pytest.raises(S.Sis3dError, match="image-feature crop"):
            net.mask_backbone(scene[:, :, :4, :4, :4], None)


def _gt_masks(g, s):
    bits = np.unpackbits(g[f"loop_{s}_gt_bits"])
    out, o = [], 0
    for b in g[f"loop_{s}_gt_box"]:
        ext = tuple(int(v) for v in np.rint(b[3:6]).astype(int) - np.rint(b[0:3]).astype(int))
        n = int(np.prod(ext))
        out.append(bits[o:o + n].reshape(ext).astype(np.uint8))
        o += n
    return out


@pytest.mark.parametrize("mode", ["test", "benchmark"])
def test_run_scenes_matches_the_reference_loops(golden, tmp_path, mode):
    from lib.model.trainval import SceneEvaluator, run_scenes
    g = golden
    dims, n_img = tuple(int(v) for v in g["loop_dims"]), int(g["loop_n_img"])
    scenes = []
    for s in range(int(g["loop_n_scenes"])):
        data, boxes = synth.make_scene(int(g[f"loop_{s}_seed"]), dims)
        b = synth.make_blobs(dict(use_images=True), data, synth.make_views(int(g[f"loop_{s}_seed"]), dims, n_img, boxes))
        b["id"], b["gt_box"], b["gt_mask"] = [str(g[f"loop_{s}_id"])], [torch.from_numpy(g[f"loop_{s}_gt_box"])], [_gt_masks(g, s)]
        scenes.append(b)
    lines = {}
    for drv in ("pipelined", "sync"):
        net, _ = make_color_net("use")
        ev = SceneEvaluator() if mode == "test" else None
        assert run_scenes(net, iter(scenes), str(tmp_path / drv), pipelined=drv == "pipelined", evaluator=ev) == len(scenes)
        lines[drv] = ev.summary() if ev is not None else None
    if mode == "test":
        assert lines["pipelined"] == lines["sync"] == str(g["loop_test_printed"]).split("\n")
    for s in range(len(scenes)):
        d = {m: tmp_path / m / str(g[f"loop_{s}_id"]) for m in ("pipelined", "sync")}
        names = sorted(os.listdir(d["sync"]))
        assert names == sorted(os.listdir(d["pipelined"]))
        for f in names:
            assert filecmp.cmp(d["sync"] / f, d["pipelined"] / f, shallow=False), f"scene {s}: {f} differs"
        k = f"loop_{mode}_{s}_"
        assert int(g[k + "written"]) == 1
        ld = lambda f: np.load(d["sync"] / (f + ".npy"))
        assert ld("pred_class").dtype == g[k + "pred_class"].dtype and np.array_equal(ld("pred_class"), g[k + "pred_class"])
        np.testing.assert_allclose(ld("pred_conf"), g[k + "pred_conf"], atol=1e-4)
        np.testing.assert_allclose(ld("pred_box"), g[k + "pred_box"], atol=2e-3)
        assert pickle.load(open(d["sync"] / "pred_mask_index", "rb")) == [bool(v) for v in g[k + "pred_mask_index"]]
        pm = pickle.load(open(d["sync"] / "pred_mask", "rb"))
        assert [m.shape for m in pm] == [tuple(v) for v in g[k + "pred_mask_shapes"]]
        if pm:
            got = np.concatenate([m.reshape(-1) != 0 for m in pm])
            want = np.unpackbits(g[k + "pred_mask_bits"])[:got.size].astype(bool)
            assert (got != want).mean() < 1e-3, f"scene {s}: {(got != want).sum()} of {got.size} mask voxels differ"


# ------------------------------------------------------------------------------------------------ scale
SCALE_BOXES = 12  # whole-scene boxes: the fp16 route's canvases then take about 20 GB


@pytest.mark.parametrize("math", ["exact", "tf32"])
def test_whole_scene_boxes_at_208x48x160(math):
    dims = (208, 48, 160)
    data, boxes = synth.make_scene(909, dims)
    views = synth.make_views(909, dims, 40, boxes)
    b = synth.make_blobs(dict(use_images=True), data, views)
    gt = np.zeros((SCALE_BOXES, 7), np.float32)
    gt[:, 3:6], gt[:, 6] = dims, np.arange(SCALE_BOXES) % 19
    net, _ = make_color_net("use", math, gt_rois=False)
    b1 = dict(b, gt_box=[torch.from_numpy(gt[:1])])
    one = net.forward(b1, "TEST", None)["mask_pred"][0][0].clone()
    P = net.forward(dict(b, gt_box=[torch.from_numpy(gt)]), "TEST", None)
    masks = P["mask_pred"][0]
    assert len(masks) == SCALE_BOXES and tuple(masks[0].shape[2:]) == dims
    assert torch.isfinite(one).all() and 0.0 < float(one.mean()) < 1.0
    for j, m in enumerate(masks):  # the same crop at every canvas position: the same bricks, the same bits
        assert torch.equal(m, one), f"box {j} differs from the scene's single-box result"
