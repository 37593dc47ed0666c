"""CPU: the image-only ScanNet backbone (ONLY_IMAGES = USE_IMAGES = True) against the unmodified reference
(tests/golden/only_images_reference.npz, written by oracle/make_golden_only_images.py).

- the product model's state_dict has the reference's keys and shapes (no geometry1, a 128-channel colour stack, a 128-input
  geometry2.0), and the reference's state_dict loads into it with strict=True;
- the two neighbouring combinations the reference cannot run (SUNCG_Backbone with ONLY_IMAGES; ScanNet_Backbone with
  ONLY_IMAGES and USE_IMAGES = False) are refused before any parameter is declared, and the reference failed on both;
- the oracle's image-only forward (oracle/port_only_images.py) equals the reference on every case: integer outputs exactly, floats to the bars of
  tests/test_oracle_golden.py."""
import os

import numpy as np
import pytest
import torch

import sis3d_synth as synth
from conftest import ROOT, load_golden
from lib.utils.config import cfg, cfg_from_file, cfg_reset

GOLDEN = "only_images_reference.npz"
FORWARD = ("cfg2_96x48x96", "killed_45x27x41", "scene_88x44x88", "enet_45x27x41")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def enet_params():
    g = load_golden("enet_encoder.npz")
    return [torch.from_numpy(g[k]) for k in sorted(k for k in g if k.startswith("p"))]


def case_inputs(g, tag):
    """(case dict, data, views) of a golden case: views["feats"] are the raw images when the case has them, and the killed
    views see nothing within PROJ_DEPTH_MAX."""
    dims = tuple(int(v) for v in g[f"{tag}_dims"])
    seed, n_img = int(g[f"{tag}_seed"]), int(g[f"{tag}_n_img"])
    c = dict(cfgname="scannet", dims=dims, n_img=n_img, seed=seed, use_images=True, use_mask=True)
    data, boxes = synth.make_scene(seed, dims)
    views = synth.make_views(seed, dims, n_img, boxes)
    for k in g[f"{tag}_killed"]:
        views["depths"][int(k)][:] = 9.0
    s = int(g[f"{tag}_images_seed"])
    if s >= 0:
        views["feats"] = np.random.default_rng(s).standard_normal((n_img, 3, 256, 328)).astype(np.float32)
    return c, data, views


def step(g, name):
    """Stride of the fixture's samples of `name` (imageft, level, rpn_prob, mask_cls, mask_allcls)."""
    return int(g[f"step_{name}"])


def stats_close(t, want, rel):
    """[sum, sum |.|, max, min] of a whole tensor against the fixture's, each within rel * sum |.|."""
    a = np.asarray(t, dtype=np.float64).reshape(-1)
    got = np.array([a.sum(), np.abs(a).sum(), a.max(), a.min()])
    return bool((np.abs(got - want) <= rel * want[1]).all())


def oracle_forward(port, g, tag):
    from oracle import port_only_images
    c, data, views = case_inputs(g, tag)
    ocfg = port.make_cfg("scannet")
    w = synth.make_weights(seed=0, net=ocfg.NET, use_images=True, num_classes=ocfg.NUM_CLASSES, a1=ocfg.NUM_ANCHORS_LEVEL1,
                           a2=ocfg.NUM_ANCHORS_LEVEL2, use_mask=True, only_images=True)
    if int(g[f"{tag}_images_seed"]) >= 0:
        with torch.no_grad():
            views = dict(views, feats=port.enet_encoder(enet_params(), torch.from_numpy(views["feats"])).numpy())
    return port_only_images.forward(ocfg, w, data, views), w


def _ncdhw_sub(t, step):
    return np.asarray(t, dtype=np.float32).reshape(-1)[::step]


@pytest.fixture
def scannet_cfg():
    def make(net="ScanNet", **over):
        cfg_reset()
        cfg_from_file(os.path.join(ROOT, "3d-sis_b200", "experiments", "cfgs", net, "rpn_class_mask_5.yml"))
        cfg.NUM_CLASSES = 26 if net == "SUNCG" else 19
        cfg.USE_IMAGES_GT = True  # the 3-D model alone: no 2-D encoder declared
        for k, v in over.items():
            cfg[k] = v
        from lib.nets import backbones
        return getattr(backbones, cfg.NET)()
    yield make
    cfg_reset()


def test_state_dict_equals_reference(golden, scannet_cfg):
    net = scannet_cfg(USE_IMAGES=True, ONLY_IMAGES=True)
    net.init_modules()
    sd = net.state_dict()
    want = {str(k): tuple(int(v) for v in s if v) for k, s in zip(golden["sd_keys"], golden["sd_shapes"])}
    got = {k: tuple(v.shape) for k, v in sd.items()}
    assert got == want
    assert not any(k.startswith("geometry1.") for k in got)
    assert got["color.4.weight"] == (128, 64, 2, 2, 2) and got["color.6.conv3.weight"] == (128, 32, 1, 1, 1)
    assert got["geometry2.0.weight"] == (128, 128, 3, 3, 3)
    ref = {k: torch.full(s, 0.5) for k, s in want.items()}
    assert not net.load_state_dict(ref, strict=True).missing_keys
    assert [op[:2] for op in net.SPEC["color"]] == [("k2s2", 0), ("bneck", 2), ("pool", 3), ("k2s2", 4), ("bneck", 6),
                                                    ("pool", 7)]
    assert set(net.SPEC) == {"color", "geometry2"}
    # the synthetic weights of the image-only model are keyed and shaped like it
    w = synth.make_weights(seed=0, use_images=True, num_classes=19, a1=3, a2=11, use_mask=True, only_images=True)
    assert {k: tuple(v.shape) for k, v in w.items()} == got


@pytest.mark.parametrize("net,over,what", [
    ("SUNCG", dict(USE_IMAGES=True, ONLY_IMAGES=True), "SUNCG_Backbone with ONLY_IMAGES"),
    ("ScanNet", dict(USE_IMAGES=False, ONLY_IMAGES=True), "ScanNet_Backbone with ONLY_IMAGES and USE_IMAGES=False")])
def test_refused_combinations(golden, scannet_cfg, net, over, what):
    m = scannet_cfg(net, **over)
    with pytest.raises(NotImplementedError, match=what):
        m.init_modules()
    assert not list(m.parameters()) and not list(m.buffers()), "parameters were declared before the refusal"
    key = "refused_suncg" if net == "SUNCG" else "refused_no_images"
    assert str(golden[key]).split(":")[0].endswith("Error"), golden[key]  # the unmodified reference failed here


def test_suncg_without_images_ignores_only_images(scannet_cfg):
    """As in the reference (backbones.py:124, 148-153), ONLY_IMAGES without USE_IMAGES leaves SUNCG_Backbone's program as it
    is."""
    a = scannet_cfg("SUNCG", USE_IMAGES=False, ONLY_IMAGES=True)
    a.init_modules()
    b = scannet_cfg("SUNCG", USE_IMAGES=False, ONLY_IMAGES=False)
    b.init_modules()
    assert a.SPEC == b.SPEC and {k: v.shape for k, v in a.state_dict().items()} == {k: v.shape for k, v in b.state_dict().items()}


@pytest.mark.parametrize("tag", FORWARD)
def test_oracle_equals_reference(oracle, golden, tag):
    g, k = golden, tag + "_"
    out, _ = oracle_forward(oracle, g, tag)
    assert list(g[k + "killing_inds"]) == out["killing_inds"]
    if int(g[k + "images_seed"]) < 0:
        assert np.array_equal(_ncdhw_sub(out["imageft"], step(g, "imageft")), g[k + "imageft_sub"])  # exact: copy / max
    else:  # the 2-D encoder: fp32 convolutions in another order
        np.testing.assert_allclose(_ncdhw_sub(out["imageft"], step(g, "imageft")), g[k + "imageft_sub"], atol=1e-4)
    for lvl in (1, 2):
        assert out[f"level{lvl}"].shape[1] == 128
        np.testing.assert_allclose(_ncdhw_sub(out[f"level{lvl}"], step(g, "level")), g[k + f"level{lvl}_sub"], atol=1e-4,
                                   rtol=1e-4)
        assert stats_close(out[f"level{lvl}"], g[k + f"level{lvl}_stats"], 1e-5), f"level {lvl}: whole-tensor moments"
        np.testing.assert_allclose(_ncdhw_sub(out[f"rpn_prob_level{lvl}"], step(g, "rpn_prob")), g[k + f"rpn_prob_sub_l{lvl}"],
                                   atol=2e-6)
    assert out["rois"].shape == g[k + "rois"].shape
    np.testing.assert_allclose(out["rois"].numpy(), g[k + "rois"], atol=1e-3)
    np.testing.assert_allclose(out["roi_scores"].numpy().reshape(-1), g[k + "roi_scores"].reshape(-1), atol=2e-6)
    assert np.array_equal(out["level_inds"].numpy(), g[k + "level_inds"])
    np.testing.assert_allclose(out["cls_prob"].numpy(), g[k + "cls_prob"], atol=1e-5)
    assert np.array_equal(out["cls_pred"].numpy(), g[k + "cls_pred"])
    np.testing.assert_allclose(out["bbox_pred"].numpy(), g[k + "bbox_pred"], atol=1e-5)
    np.testing.assert_allclose(out["pred_box"], g[k + "pred_box"], atol=1e-3)
    assert np.array_equal(out["mask_keep"], g[k + "keep"])
    assert np.array_equal(out["mask_crops"], g[k + "crops"])
    assert len(out["mask_pred"]) == int(g[k + "n_masks"]) > 0
    for j, i in enumerate(np.nonzero(out["mask_keep"])[0]):
        m = out["mask_pred"][j][0].numpy()
        np.testing.assert_allclose(m[int(g[k + "cls_pred"][i])].reshape(-1)[::step(g, "mask_cls")], g[k + f"mask_{j}_cls_sub"],
                                   atol=1e-5)
        np.testing.assert_allclose(m.reshape(-1)[::step(g, "mask_allcls")], g[k + f"mask_{j}_allcls_sub"], atol=1e-5)
        assert abs(int((m[int(g[k + "cls_pred"][i])] > 0.5).sum()) - int(g[k + f"mask_{j}_cls_on"])) <= 1


def test_golden_cases_cover_the_ask(golden):
    g = golden
    assert list(g["killed_45x27x41_killing_inds"]) == [1]
    assert int(g["enet_45x27x41_images_seed"]) >= 0
    assert [int(g[f"loop_test_{s}_written"]) for s in range(int(g["loop_n_scenes"]))] == [1] * int(g["loop_n_scenes"])
