"""Per-vertex GT files of ScanNet scans for the instance benchmark, from ScanNet's annotations (reference:
tools/scannet_benchmark/export_train_mesh_for_evaluation.py; lines cited per function).

    python export_train_mesh_for_evaluation.py --scan_path SCANS --filelist LIST --output_dir GT
        --label_map_file scannetv2-labels.combined.tsv --label_map_file2 nyu40labels_scannet.csv --type instance|label

Every folder `<scene>` of scan_path that is a line of the filelist is exported to `<output_dir>/<scene>.txt`: one '%d' line
per mesh vertex, `label * 1000 + instance` (uint32) for --type instance, the consecutive label id for --type label, 0 for
an unannotated vertex -- the files evaluate_semantic_instance.py --gt_path reads.  The rules are resolved per segment on
the host (annotations.py, which documents them and the departures); sis3d_segment_gt_slots (csrc/eval.cu) assigns every
vertex its segment's GT id on the device, the same kernel evaluate_predictions.py uses when it reads the annotations
itself.  The mesh is read as the reference reads it, so a scan without `<scene>_vh_clean_2.ply` fails.  There is no CPU
path: without a CUDA device the launch raises.
"""
from __future__ import annotations

import argparse
import os
import sys

if __package__:
    from . import annotations, utils
    from .evaluate_predictions import segment_gt_slots
else:  # run as a script
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
    from tools.scannet_benchmark import annotations, utils
    from tools.scannet_benchmark.evaluate_predictions import segment_gt_slots

TASK_TYPES = {"label", "instance"}


def export(mesh_file, agg_file, seg_file, label_map_file, label_map_file2, type, output_file):
    """export_train_mesh_for_evaluation.py:73-96: one scan's GT file."""
    label_map = utils.read_label_mapping(label_map_file, label_from="raw_category", label_to="nyu40id")
    label_map2 = utils.read_label_mapping(label_map_file2, label_from="nyu40id", label_to="mappedIdConsecutive", delimiter=",")
    utils.read_mesh_vertices(mesh_file)
    scene = os.path.basename(os.path.dirname(os.path.abspath(agg_file)))
    gt = annotations.read_scene_gt(agg_file, seg_file, label_map, label_map2, type, scene)
    gt_slot, _ = segment_gt_slots(gt)
    utils.export_ids(output_file, gt.slot_ids[gt_slot])


def main(argv=None):
    """export_train_mesh_for_evaluation.py:28-36, 99-109: a scene is exported when `scene + '\\n'` is one of the
    filelist's lines as readlines() returns them, in os.listdir order."""
    parser = argparse.ArgumentParser()
    parser.add_argument("--scan_path", required=True, help="path to scannet scene (e.g., data/ScanNet/v2")
    parser.add_argument("--filelist", required=True, help="path to scannet scene txt file (e.g., datagen/fileLists/scannetv2_val.txt")
    parser.add_argument("--output_dir", required=True, help="output file")
    parser.add_argument("--label_map_file", required=True, help="path to scannetv2-labels.combined.tsv")
    parser.add_argument("--label_map_file2", required=True, help="path to nyu40labels_scannet.csv")
    parser.add_argument("--type", required=True, help="task type [label or instance]")
    opt = parser.parse_args(argv)
    assert opt.type in TASK_TYPES
    with open(opt.filelist) as f:
        filelist = f.readlines()
    for scan_name in os.listdir(opt.scan_path):
        if scan_name + "\n" not in filelist:
            continue
        print(scan_name)
        scan = os.path.join(opt.scan_path, scan_name)
        export(os.path.join(scan, scan_name + "_vh_clean_2.ply"), os.path.join(scan, scan_name + ".aggregation.json"),
               os.path.join(scan, scan_name + "_vh_clean_2.0.010000.segs.json"), opt.label_map_file, opt.label_map_file2,
               opt.type, os.path.join(opt.output_dir, scan_name + ".txt"))


if __name__ == "__main__":
    main()
