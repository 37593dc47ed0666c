"""Inference drivers with the reference's entry points `test(args)` / `benchmark(args)`
(lib/model/trainval.py:75-93, SolverWrapper.test 769-941, .benchmark 634-767).

Per scene: forward (the mask head runs ONCE -- the reference runs it in forward and again in the
driver, trainval.py:882-897), then the on-disk results the ScanNet tooling consumes
(trainval.py:839-845, 909-911): pred_class.npy, pred_conf.npy, pred_box.npy, scene.npy, pickled pred_mask /
pred_mask_index.  Class-specific decode, clipping, confidence and degenerate-box filtering were already
done on the device (csrc/roi.cu detect_decode_kernel) and arrive in one [n,16] table.
Training (`train`) is out of scope of the GPU inference path.
"""
from __future__ import annotations

import os
import pickle
import time

import numpy as np
import torch

from lib.datasets.dataset import Dataset, collate_fn
from lib.utils.config import cfg


def scene_key(scene_id):
    return os.path.basename(str(scene_id))[:12]


def detections_from_predictions(net_or_predictions):
    """-> pred_class int64[n], pred_conf float64[n], pred_box float32[n,6], keep bool[n] (trainval.py:825-858)."""
    P = getattr(net_or_predictions, "_predictions", net_or_predictions)
    det = P["detections_host"]
    return det[:, 7].astype(np.int64), det[:, 6].astype(np.float64), det[:, 0:6].astype(np.float32), det[:, 8] > 0.5


def save_scene_results(out_dir, scene_id, blobs, net_or_predictions):
    """Result files of one scene from `net._predictions` (synchronous forward) or the dict the scene loop yields."""
    P = getattr(net_or_predictions, "_predictions", net_or_predictions)
    d = os.path.join(out_dir, scene_key(scene_id))
    os.makedirs(d, exist_ok=True)
    pred_class, pred_conf, pred_box, keep = detections_from_predictions(P)
    np.save(os.path.join(d, "pred_class"), pred_class)
    np.save(os.path.join(d, "pred_conf"), pred_conf)
    np.save(os.path.join(d, "pred_box"), pred_box)
    np.save(os.path.join(d, "scene"), np.where(blobs["data"][0, 0].cpu().numpy() <= 1, 1, 0))
    if cfg.USE_MASK:
        masks = []
        if keep.any():  # the thresholded predicted-class channels (csrc/roi.cu mask_select_kernel): already on the host when the
            # scene loop produced them, else one D2H
            bits = P["mask_bits_host"] if "mask_bits_host" in P else P["mask_bits"].cpu().numpy()
            offs, sizes = P["mask_offsets"], P["mask_sizes"]
            for j in range(len(sizes)):
                masks.append(bits[int(offs[j]):int(offs[j + 1])].reshape(tuple(int(v) for v in sizes[j])).astype(np.float32))
        with open(os.path.join(d, "pred_mask"), "wb") as f:
            pickle.dump(masks, f)
        with open(os.path.join(d, "pred_mask_index"), "wb") as f:
            pickle.dump([bool(k) for k in keep], f)
    return d


class SceneEvaluator:
    """Box and mask mAP of test mode (SolverWrapper.test, trainval.py:775-776, 844-845, 847-921, 926-941), fed one scene at
    a time by run_scenes.  The box IoU and the matching run on the host.  The mask overlaps are counted on the device from
    the mask stage's thresholded bits (lib.utils.evaluation.launch_mask_overlap); the counts of a scene are collected when
    the next scene is added, so the scene loop never waits for them."""

    def __init__(self):
        from lib.utils.evaluation import DetectionMAP
        self.box = DetectionMAP(cfg.NUM_CLASSES, ignore_class=[0], overlap_threshold=cfg.MAP_THRESH)
        self.mask = DetectionMAP(cfg.NUM_CLASSES, ignore_class=[0], overlap_threshold=cfg.MAP_THRESH)
        self._pending = None

    def add(self, scene_dir, blobs, P):
        """One scene: writes gt_class.npy / gt_box.npy (and the pickled gt_mask) beside its predictions, accumulates the box
        mAP of the kept detections and queues the mask overlaps of the kept masks."""
        from lib.utils.evaluation import launch_mask_overlap, pack_masks
        gt = blobs["gt_box"][0].numpy()
        gt_box, gt_class = gt[:, 0:6], gt[:, 6]
        np.save(os.path.join(scene_dir, "gt_class"), gt_class)
        np.save(os.path.join(scene_dir, "gt_box"), gt_box)
        pred_class, pred_conf, pred_box, keep = detections_from_predictions(P)
        self.box.evaluate(pred_box[keep], pred_class[keep], pred_conf[keep], gt_box, gt_class)
        if not cfg.USE_MASK:
            return
        gt_mask = blobs["gt_mask"][0]
        with open(os.path.join(scene_dir, "gt_mask"), "wb") as f:
            pickle.dump(gt_mask, f)
        dims = tuple(int(v) for v in blobs["data"].shape[2:])  # the reference's net._scene_info
        gb, go, gbox = pack_masks(gt_mask, gt_box, dims, "GT")
        det = P["detections_host"]
        if "mask_bits" in P:  # crop i of the packed bits sits at the crop bounds of kept detection i (columns 9-14)
            job = launch_mask_overlap(P["mask_bits"], P["mask_offsets"], det[keep][:, 9:15], gb, go, gbox)
        else:                 # no kept detection
            job = launch_mask_overlap(np.zeros(0, np.uint8), np.zeros(0, np.int64), np.zeros((0, 6), np.int32), gb, go, gbox)
        self._collect()
        self._pending = (job, pred_class[keep], pred_conf[keep], gt_class)

    def _collect(self):
        if self._pending is not None:
            job, pred_class, pred_conf, gt_class = self._pending
            self._pending = None
            self.mask.evaluate_overlaps(pred_class, pred_conf, job.result(), gt_class)

    def summary(self):
        """Collects the last scene and returns the lines test mode prints (trainval.py:929-941)."""
        from lib.utils.evaluation import summary_lines
        self._collect()
        lines = []
        if cfg.USE_CLASS:
            self.box.finalize()
            lines += summary_lines("CLASSIFICATION", self.box, int(cfg.NUM_CLASSES))
        if cfg.USE_MASK:
            self.mask.finalize()
            lines += summary_lines("mask", self.mask, int(cfg.NUM_CLASSES))
        return lines


def run_scenes(net, data_loader, out_dir, skip_existing=False, pipelined=True, evaluator=None):
    """The scene loop of SolverWrapper.test / .benchmark (trainval.py:787-911).  pipelined=True drives it through
    Network.forward_pipelined (several scenes in flight, results read back asynchronously); blobs that carry precomputed
    projection index lists (the reference's calling convention) go through the synchronous forward.  An `evaluator`
    (SceneEvaluator) is handed every scene after its result files are written."""
    os.makedirs(out_dir, exist_ok=True)
    t0 = time.time()
    done = 0

    def todo():
        for blobs in data_loader:
            if skip_existing and os.path.isdir(os.path.join(out_dir, scene_key(blobs["id"][0]))):  # trainval.py:647-653
                continue
            yield blobs
    it = todo()
    if pipelined:
        first = next(it, None)
        if first is not None and "proj_ind_3d" not in first:
            import itertools
            for blobs, P in net.forward_pipelined(itertools.chain([first], it)):
                d = save_scene_results(out_dir, blobs["id"][0], blobs, P)
                if evaluator is not None:
                    evaluator.add(d, blobs, P)
                done += 1
            it = iter(())
        elif first is not None:
            import itertools
            it = itertools.chain([first], it)
    for blobs in it:
        net.forward(blobs, "TEST", None)
        d = save_scene_results(out_dir, blobs["id"][0], blobs, net)
        if evaluator is not None:
            evaluator.add(d, blobs, net._predictions)
        done += 1
    torch.cuda.synchronize()
    print("It took {:.3f}s for test on whole scenes".format(time.time() - t0))
    return done


def _build(args, mode, view_provider=None):
    from lib.nets import backbones
    filelist = cfg.TEST_FILELIST
    workers = getattr(args, "num_workers", 0)
    dataset = Dataset(filelist, mode, view_provider=view_provider, device_decode=(workers == 0))
    if workers == 0:
        # files are read + parsed a few scenes ahead in a background thread; the voxel block is decoded on the device
        from lib.datasets.prefetch import Prefetcher
        loader = (collate_fn([item]) for item in Prefetcher((dataset[i] for i in range(len(dataset))), depth=6))
    else:
        loader = torch.utils.data.DataLoader(dataset, batch_size=1, shuffle=False, num_workers=workers, collate_fn=collate_fn)
    net = getattr(backbones, cfg.NET)()
    net.init_modules()
    ckpt = os.path.join(args.output_dir, "step_{}.pth".format(args.step))
    net.load_state_dict(torch.load(ckpt, map_location="cpu"), strict=False)
    return net, loader


def test(args, view_provider=None, pipelined=True):
    """Every scene's result files plus gt_class.npy, gt_box.npy and the pickled gt_mask, then the reference's box and mask
    mAP summary (trainval.py:926-941) on stdout."""
    net, loader = _build(args, "test", view_provider)
    ev = SceneEvaluator()
    done = run_scenes(net, loader, cfg.TEST_SAVE_DIR, pipelined=pipelined, evaluator=ev)
    for line in ev.summary():
        print(line)
    return done


def benchmark(args, view_provider=None):
    net, loader = _build(args, "benchmark", view_provider)
    return run_scenes(net, loader, cfg.TEST_SAVE_DIR, skip_existing=True)


def train(args):
    raise NotImplementedError("training is out of scope of the GPU inference hot path (SURVEY section 8)")
