"""Class ids of benchmark predictions -> ScanNet's NYU40 ids, before a benchmark submission (the reference's
tools/scannet_benchmark/proj_label.py).

    python tools/scannet_benchmark/proj_label.py --pred_path RESULTS

Every file of RESULTS (not its subfolders) is rewritten in place: the second word of each line, the class id 0-18 of
3D-SIS's 18-class set, becomes its NYU40 id, and each line's words are joined by single spaces.  Files are visited in
sorted order.  Runs on the host only.
"""
from __future__ import annotations

import argparse
import os

# proj_label.py:4-24 of the reference
MAPPING = {0: 0, 1: 3, 2: 4, 3: 5, 4: 6, 5: 7, 6: 8, 7: 9, 8: 10, 9: 11, 10: 12, 11: 14, 12: 16, 13: 24, 14: 28, 15: 33,
           16: 34, 17: 36, 18: 39}


def project_file(path):
    with open(path) as f:
        lines = f.readlines()
    out = []
    for line in lines:
        words = line.split()
        words[1] = str(MAPPING[int(words[1])])
        out.append(" ".join(words) + "\n")
    with open(path, "w") as f:
        f.writelines(out)


def main(argv=None):
    parser = argparse.ArgumentParser()
    parser.add_argument("--pred_path", default="./ScanNet_Benchmark_Result")
    opt = parser.parse_args(argv)
    for name in sorted(os.listdir(opt.pred_path)):
        if os.path.isdir(os.path.join(opt.pred_path, name)):
            continue
        print(name)
        project_file(os.path.join(opt.pred_path, name))


if __name__ == "__main__":
    main()
