"""ScanNet semantic-instance evaluation: AP, AP50 and AP25 for each of the 18 benchmark classes (reference:
tools/scannet_benchmark/evaluate_semantic_instance.py, adapted there from the CityScapes evaluation; lines cited per
function).

    python evaluate_semantic_instance.py --pred_path DIR --gt_path DIR [--output_file FILE]

`pred_path` holds one `<scene>.txt` per scene, each line `<relative mask path> <label id> <confidence>`, the masks holding one
0/1 line per mesh vertex (what vox2mesh.py writes).  `gt_path` holds `<scene>.txt` with one instance id per vertex
(`label * 1000 + instance`; ids below 1000 are unlabelled groups).  The table is printed to stdout and written as CSV to
`output_file` (default `pred_path/semantic_instance_evaluation.txt`).  Numbers, table and CSV equal the reference's.

The matching works on counts: per prediction, the number of its vertices carrying each GT id (`assign_instances`).  Here they
come from the mask files; evaluate_predictions.py obtains the same counts on the GPU, straight from the voxel predictions, and
feeds them to the same functions.

Departures from the reference, none of which changes a number:
- numpy 2: builtin `float` / `bool` for the removed `np.float` / `np.bool`, and `np.isin` for `np.in1d`.
- Malformed prediction lines and masks outside `pred_path` are reported through `utils.print_error` (stderr, exit -1); the
  reference meant to, but calls an undefined `util` and dies with NameError.
- Scenes are evaluated in sorted order, not `os.listdir` order.  The AP does not depend on the order: tied scores are
  resolved through `np.unique`'s first index of each tie group, and the greedy-assignment keys are unique per scene.
- Arguments are parsed in `main()`, and the evaluation parameters are module constants, so the functions can be imported.
"""
from __future__ import annotations

import argparse
import os
import sys
from copy import deepcopy

import numpy as np

if __package__:
    from . import utils
else:  # run as a script
    import utils

# ---------- labels (evaluate_semantic_instance.py:56-63)
CLASS_LABELS = ["cabinet", "bed", "chair", "sofa", "table", "door", "window", "bookshelf", "picture", "counter", "desk",
                "curtain", "refrigerator", "shower curtain", "toilet", "sink", "bathtub", "otherfurniture"]
VALID_CLASS_IDS = np.array([1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18])
ID_TO_LABEL = {VALID_CLASS_IDS[i]: CLASS_LABELS[i] for i in range(len(VALID_CLASS_IDS))}
LABEL_TO_ID = {CLASS_LABELS[i]: VALID_CLASS_IDS[i] for i in range(len(VALID_CLASS_IDS))}

# ---------- evaluation parameters (evaluate_semantic_instance.py:64-72)
OVERLAPS = np.append(np.arange(0.5, 0.95, 0.05), 0.25)  # this exact expression: the thresholds are its float64 values
MIN_REGION_SIZES = np.array([100])                      # [vertices]
DISTANCE_THRESHES = np.array([float("inf")])            # [m]
DISTANCE_CONFS = np.array([-float("inf")])

RESULT_FILE = "semantic_instance_evaluation.txt"


# ------------------------------------------------------------------------------------------------------------ matching
def assign_instances(gt_uniq, gt_counts, preds):
    """GT <-> prediction association of one scene (evaluate_semantic_instance.py:258-313), from counts.

    gt_uniq / gt_counts: `np.unique(gt_ids, return_counts=True)` of the scene's per-vertex GT ids.  preds: (filename,
    label_id, confidence, hist) in prediction-file order, where hist[k] is the number of the prediction's vertices whose GT
    id is gt_uniq[k].  -> (gt2pred, pred2gt) as the reference builds them."""
    gt2pred = deepcopy(utils.get_instances(gt_uniq, VALID_CLASS_IDS, CLASS_LABELS, ID_TO_LABEL, gt_counts))
    for label in gt2pred:
        for gt in gt2pred[label]:
            gt["matched_pred"] = []
    pred2gt = {label: [] for label in CLASS_LABELS}
    slot = {int(i): k for k, i in enumerate(gt_uniq.tolist())}
    void = ~np.isin(gt_uniq // 1000, VALID_CLASS_IDS)  # id 0 and groups included: 0 is not a valid class
    n_pred = 0
    for filename, label_id, conf, hist in preds:
        if label_id not in ID_TO_LABEL:
            continue
        label_name = ID_TO_LABEL[label_id]
        hist = np.asarray(hist)
        num = int(hist.sum())
        if num < MIN_REGION_SIZES[0]:  # dropped before it gets a pred_id
            continue
        pred = {"filename": filename, "pred_id": n_pred, "label_id": label_id, "vert_count": num, "confidence": conf,
                "void_intersection": int(hist[void].sum())}
        matched_gt = []
        for gt in gt2pred[label_name]:
            inter = int(hist[slot[gt["instance_id"]]])
            if inter > 0:
                gt_copy, pred_copy = gt.copy(), pred.copy()
                gt_copy["intersection"] = pred_copy["intersection"] = inter
                matched_gt.append(gt_copy)
                gt["matched_pred"].append(pred_copy)
        pred["matched_gt"] = matched_gt
        n_pred += 1
        pred2gt[label_name].append(pred)
    return gt2pred, pred2gt


def assign_instances_for_scan(pred_file, gt_file, pred_path):
    """evaluate_semantic_instance.py:248-313: the association of one scene from its prediction and GT text files."""
    try:
        pred_info = utils.read_instance_prediction_file(pred_file, pred_path)
    except Exception as e:
        utils.print_error("unable to load " + pred_file + ": " + str(e))
    try:
        gt_ids = utils.load_ids(gt_file)
    except Exception as e:
        utils.print_error("unable to load " + gt_file + ": " + str(e))
    gt_uniq, gt_inv, gt_counts = np.unique(gt_ids, return_inverse=True, return_counts=True)

    def preds():
        for mask_file, info in pred_info.items():
            if info["label_id"] not in ID_TO_LABEL:  # the mask of an invalid label is never read
                continue
            mask = utils.load_ids(mask_file)
            if len(mask) != len(gt_ids):
                utils.print_error("wrong number of lines in " + mask_file + "(%d) vs #mesh vertices (%d), please double check "
                                  "and/or re-download the mesh" % (len(mask), len(gt_ids)))
            yield mask_file, info["label_id"], info["conf"], np.bincount(gt_inv[mask != 0], minlength=len(gt_uniq))
    return assign_instances(gt_uniq, gt_counts, preds())


def _precision_recall_ap(y_true, y_score, hard_false_negatives):
    """The AP of one class at one threshold (evaluate_semantic_instance.py:173-219)."""
    order = np.argsort(y_score)
    y_score_sorted, y_true_sorted = y_score[order], y_true[order]
    cumsum = np.cumsum(y_true_sorted)
    _, unique_indices = np.unique(y_score_sorted, return_index=True)  # one point per distinct score, first of its tie group
    n_points = len(unique_indices) + 1
    n_examples = len(y_score_sorted)
    if len(cumsum):
        n_true = cumsum[-1]
    else:  # predictions and GT exist, but nothing survived: the reference prints an empty line here and the AP is 0
        print("")
    precision, recall = np.zeros(n_points), np.zeros(n_points)
    cumsum = np.append(cumsum, 0)  # so that index -1 reads 0 for the first point
    for k, first in enumerate(unique_indices):
        before = cumsum[first - 1]
        tp = n_true - before
        fp = n_examples - first - tp
        fn = before + hard_false_negatives
        precision[k] = float(tp) / (tp + fp)
        recall[k] = float(tp) / (tp + fn)
    precision[-1], recall[-1] = 1.0, 0.0  # the artificial first point of the curve
    padded = np.append(np.append(recall[0], recall), 0.0)
    return np.dot(precision, np.convolve(padded, [-0.5, 0, 0.5], "valid"))


def evaluate_matches(matches):
    """AP [distance thresholds, classes, overlaps] (evaluate_semantic_instance.py:75-226).  Per threshold, every GT walks its
    matched predictions in prediction-file order and takes the first unvisited one above the threshold (strict >); a
    second one above it becomes a false positive carrying the lower of the two scores.  Unmatched predictions are false
    positives unless more than `overlap` of their vertices are void, group or small-GT vertices."""
    ap = np.zeros((1, len(CLASS_LABELS), len(OVERLAPS)), float)
    min_region_size, dist_thresh, dist_conf = MIN_REGION_SIZES[0], DISTANCE_THRESHES[0], DISTANCE_CONFS[0]
    for oi, th in enumerate(OVERLAPS):
        visited = {p["filename"]: False for m in matches.values() for label in CLASS_LABELS for p in m["pred"][label]
                   if "filename" in p}
        for li, label in enumerate(CLASS_LABELS):
            y_true, y_score = np.empty(0), np.empty(0)
            hard_fn = 0
            has_gt = has_pred = False
            for m in matches.values():
                preds = m["pred"][label]
                gts = [gt for gt in m["gt"][label] if gt["instance_id"] >= 1000 and gt["vert_count"] >= min_region_size
                       and gt["med_dist"] <= dist_thresh and gt["dist_conf"] >= dist_conf]
                has_gt |= bool(gts)
                has_pred |= bool(preds)
                cur_true = np.ones(len(gts))
                cur_score = np.ones(len(gts)) * (-float("inf"))
                cur_match = np.zeros(len(gts), dtype=bool)
                for gi, gt in enumerate(gts):
                    found = False
                    for pred in gt["matched_pred"]:
                        if visited[pred["filename"]]:
                            continue
                        overlap = float(pred["intersection"]) / (gt["vert_count"] + pred["vert_count"] - pred["intersection"])
                        if overlap > th:
                            conf = pred["confidence"]
                            if cur_match[gi]:  # a second match: the lower score is a false positive
                                hi_s, lo_s = max(cur_score[gi], conf), min(cur_score[gi], conf)
                                cur_score[gi] = hi_s
                                cur_true = np.append(cur_true, 0)
                                cur_score = np.append(cur_score, lo_s)
                                cur_match = np.append(cur_match, True)
                            else:
                                found = True
                                cur_match[gi] = True
                                cur_score[gi] = conf
                                visited[pred["filename"]] = True
                    if not found:
                        hard_fn += 1
                cur_true, cur_score = cur_true[cur_match], cur_score[cur_match]
                for pred in preds:
                    if any(float(gt["intersection"]) / (gt["vert_count"] + pred["vert_count"] - gt["intersection"]) > th
                           for gt in pred["matched_gt"]):
                        continue
                    ignore = pred["void_intersection"]
                    for gt in pred["matched_gt"]:
                        if gt["instance_id"] < 1000:  # group
                            ignore += gt["intersection"]
                        if gt["vert_count"] < min_region_size or gt["med_dist"] > dist_thresh or gt["dist_conf"] < dist_conf:
                            ignore += gt["intersection"]  # small GT
                    if float(ignore) / pred["vert_count"] <= th:
                        cur_true = np.append(cur_true, 0)
                        cur_score = np.append(cur_score, pred["confidence"])
                y_true, y_score = np.append(y_true, cur_true), np.append(y_score, cur_score)
            if has_gt and has_pred:
                ap[0, li, oi] = _precision_recall_ap(y_true, y_score, hard_fn)
            elif has_gt:
                ap[0, li, oi] = 0.0
            else:
                ap[0, li, oi] = float("nan")
    return ap


def compute_averages(aps):
    """evaluate_semantic_instance.py:228-245: nanmean over classes x overlaps without 0.25 (and at 0.5, 0.25); per class,
    np.average."""
    o50 = np.where(np.isclose(OVERLAPS, 0.5))
    o25 = np.where(np.isclose(OVERLAPS, 0.25))
    all_but25 = np.where(np.logical_not(np.isclose(OVERLAPS, 0.25)))
    avgs = {"all_ap": np.nanmean(aps[0, :, all_but25]), "all_ap_50%": np.nanmean(aps[0, :, o50]),
            "all_ap_25%": np.nanmean(aps[0, :, o25]), "classes": {}}
    for li, label in enumerate(CLASS_LABELS):
        avgs["classes"][label] = {"ap": np.average(aps[0, li, all_but25]), "ap50%": np.average(aps[0, li, o50]),
                                  "ap25%": np.average(aps[0, li, o25])}
    return avgs


# ------------------------------------------------------------------------------------------------------------ output
def print_results(avgs):
    """The table (evaluate_semantic_instance.py:316-351)."""
    width = 64
    print("")
    print("#" * width)
    print("{:<15}".format("what") + ":" + "{:>15}".format("AP") + "{:>15}".format("AP_50%") + "{:>15}".format("AP_25%"))
    print("#" * width)
    for label in CLASS_LABELS:
        c = avgs["classes"][label]
        print("{:<15}".format(label) + ":" + "".join("{:>15.3f}".format(c[k]) for k in ("ap", "ap50%", "ap25%")))
    print("-" * width)
    print("{:<15}".format("average") + ":" + "".join("{:>15.3f}".format(avgs[k]) for k in ("all_ap", "all_ap_50%", "all_ap_25%")))
    print("")


def write_result_file(avgs, filename):
    """The CSV (evaluate_semantic_instance.py:354-364)."""
    with open(filename, "w") as f:
        f.write(",".join(["class", "class id", "ap", "ap50", "ap25"]) + "\n")
        for i, label in enumerate(CLASS_LABELS):
            c = avgs["classes"][label]
            f.write(",".join(str(x) for x in [label, VALID_CLASS_IDS[i], c["ap"], c["ap50%"], c["ap25%"]]) + "\n")


def finish(matches, output_file):
    """AP, averages, table and CSV of a `{scene key: {"gt": gt2pred, "pred": pred2gt}}` dict -> (ap, avgs)."""
    ap = evaluate_matches(matches)
    avgs = compute_averages(ap)
    print_results(avgs)
    write_result_file(avgs, output_file)
    return ap, avgs


def evaluate(pred_files, gt_files, pred_path, output_file):
    """evaluate_semantic_instance.py:367-385 -> (ap, avgs)."""
    print("evaluating", len(pred_files), "scans...")
    matches = {}
    for i in range(len(pred_files)):
        gt2pred, pred2gt = assign_instances_for_scan(pred_files[i], gt_files[i], pred_path)
        matches[os.path.abspath(gt_files[i])] = {"gt": gt2pred, "pred": pred2gt}
        sys.stdout.write("\rscans processed: {}".format(i + 1))
        sys.stdout.flush()
    print("")
    return finish(matches, output_file)


def main(argv=None):
    """evaluate_semantic_instance.py:45-52, 388-401."""
    parser = argparse.ArgumentParser()
    parser.add_argument("--pred_path", required=True, help="path to directory of predicted .txt files")
    parser.add_argument("--gt_path", required=True, help="path to directory of gt .txt files")
    parser.add_argument("--output_file", default="", help="output file [default: pred_path/semantic_instance_evaluation.txt]")
    opt = parser.parse_args(argv)
    if opt.output_file == "":
        opt.output_file = os.path.join(opt.pred_path, RESULT_FILE)
    names = sorted(f for f in os.listdir(opt.pred_path) if f.endswith(".txt") and f != RESULT_FILE)
    if not names:
        utils.print_error("No result files found.", user_fault=True)
    gt_files = []
    for name in names:
        gt_file = os.path.join(opt.gt_path, name)
        if not os.path.isfile(gt_file):
            utils.print_error("Result file {} does not match any gt file".format(name), user_fault=True)
        gt_files.append(gt_file)
    return evaluate([os.path.join(opt.pred_path, n) for n in names], gt_files, opt.pred_path, opt.output_file)


if __name__ == "__main__":
    main()
