"""File helpers of the ScanNet instance benchmark (reference: tools/scannet_benchmark/utils.py; lines cited per function).

Only what the evaluator, vox2mesh's command line and the GT export need: per-vertex id files, label maps, instance
prediction files, GT instances, and the vertex positions of a PLY mesh.  The reference reads meshes with `plyfile`; `read_mesh_vertices` here parses the PLY
header itself, so nothing beyond numpy is needed.
"""
from __future__ import annotations

import csv
import os
import sys

import numpy as np


def print_error(message, user_fault=False):
    """utils.py:19-23: the message on stderr, then exit status 2 for a user error, -1 otherwise."""
    sys.stderr.write("ERROR: " + str(message) + "\n")
    sys.exit(2 if user_fault else -1)


def represents_int(s):
    """utils.py:26-31: whether int(s) succeeds."""
    try:
        int(s)
        return True
    except ValueError:
        return False


def read_label_mapping(filename, label_from="raw_category", label_to="nyu40id", delimiter="\t"):
    """utils.py:33-43: `{row[label_from]: int(row[label_to])}` over the rows of a delimited file with a header row; a later
    duplicate row wins.  When the first key represents an int, every key is converted with int()."""
    assert os.path.isfile(filename)
    mapping = {}
    with open(filename) as f:
        for row in csv.DictReader(f, delimiter=delimiter):
            mapping[row[label_from]] = int(row[label_to])
    if represents_int(list(mapping.keys())[0]):
        mapping = {int(k): v for k, v in mapping.items()}
    return mapping


def export_ids(filename, ids):
    """utils.py:57-60: one '%d' line per id."""
    with open(filename, "w") as f:
        f.write("".join("%d\n" % i for i in np.asarray(ids).tolist()))


def load_ids(filename):
    """utils.py:63-66: one integer per line -> int64 array."""
    with open(filename) as f:
        return np.array(f.read().splitlines(), dtype=np.int64)


def read_instance_prediction_file(filename, pred_path):
    """utils.py:150-170: `{abs mask path: {"label_id": int(float(label)), "conf": float(score)}}`, in line order.

    The reference's checks for a malformed line and for a mask outside `pred_path` call an undefined `util` and die with
    NameError; here they report the reference's message through print_error, as intended."""
    with open(filename) as f:
        lines = f.read().splitlines()
    info = {}
    root = os.path.abspath(pred_path)
    for line in lines:
        parts = line.split(" ")
        if len(parts) != 3:
            print_error("invalid instance prediction file. Expected (per line): [rel path prediction] [label id prediction] "
                        "[confidence prediction]")
        if os.path.isabs(parts[0]):
            print_error("invalid instance prediction file. First entry in line must be a relative path")
        mask_file = os.path.abspath(os.path.join(os.path.dirname(filename), parts[0]))
        if os.path.commonprefix([mask_file, root]) != root:
            print_error("predicted mask {} in prediction text file {} points outside of prediction path.".format(mask_file, filename))
        info[mask_file] = {"label_id": int(float(parts[1])), "conf": float(parts[2])}
    return info


class Instance:
    """utils.py:107-148: one GT instance; its label is `instance_id // 1000`."""

    def __init__(self, instance_id, vert_count):
        self.instance_id = int(instance_id)
        self.label_id = int(self.instance_id // 1000)
        self.vert_count = int(vert_count)
        self.med_dist = -1
        self.dist_conf = 0.0

    def to_dict(self):
        return {"instance_id": self.instance_id, "label_id": self.label_id, "vert_count": self.vert_count,
                "med_dist": self.med_dist, "dist_conf": self.dist_conf}


def get_instances(ids, class_ids, class_labels, id2label, counts=None):
    """utils.py:173-184: `{label name: [instance dict, ...]}` over the nonzero `np.unique(ids)` whose label is a valid class,
    in ascending id order.  `counts` (the matching np.unique counts) saves recounting when the caller has them."""
    if counts is None:
        uniq, counts = np.unique(ids, return_counts=True)
    else:
        uniq = ids
    instances = {label: [] for label in class_labels}
    valid = set(int(c) for c in class_ids)
    for i, n in zip(uniq.tolist(), np.asarray(counts).tolist()):
        if i == 0:
            continue
        inst = Instance(i, n)
        if inst.label_id in valid:
            instances[id2label[inst.label_id]].append(inst.to_dict())
    return instances


# ------------------------------------------------------------------------------------------------------------------ PLY
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def _parse_ply_header(f, filename):
    """-> (format, [(element name, count, [(property name, type | ("list", count type, item type))])]) with `f` positioned at
    the first byte after `end_header`."""
    if f.readline().rstrip(b"\r\n") != b"ply":
        raise ValueError(f"{filename}: not a PLY file (no 'ply' magic line)")
    fmt, elements = None, []
    while True:
        raw = f.readline()
        if not raw:
            raise ValueError(f"{filename}: PLY header has no end_header")
        words = raw.decode("ascii", errors="replace").split()
        if not words or words[0] in ("comment", "obj_info"):
            continue
        if words[0] == "end_header":
            break
        if words[0] == "format":
            if len(words) != 3 or words[1] not in ("ascii", "binary_little_endian", "binary_big_endian"):
                raise ValueError(f"{filename}: unsupported PLY format line {raw!r}")
            fmt = words[1]
        elif words[0] == "element":
            if len(words) != 3 or not words[2].isdigit():
                raise ValueError(f"{filename}: malformed PLY element line {raw!r}")
            elements.append((words[1], int(words[2]), []))
        elif words[0] == "property":
            if not elements:
                raise ValueError(f"{filename}: PLY property before any element")
            if words[1:2] == ["list"]:
                if len(words) != 5 or words[2] not in _PLY_TYPES or words[3] not in _PLY_TYPES:
                    raise ValueError(f"{filename}: malformed PLY list property {raw!r}")
                elements[-1][2].append((words[4], ("list", _PLY_TYPES[words[2]], _PLY_TYPES[words[3]])))
            else:
                if len(words) != 3 or words[1] not in _PLY_TYPES:
                    raise ValueError(f"{filename}: malformed PLY property {raw!r}")
                elements[-1][2].append((words[2], _PLY_TYPES[words[1]]))
        else:
            raise ValueError(f"{filename}: unknown PLY header line {raw!r}")
    if fmt is None:
        raise ValueError(f"{filename}: PLY header has no format line")
    return fmt, elements


def _skip_binary_element(f, count, props, endian, filename):
    if all(not isinstance(t, tuple) for _, t in props):
        f.seek(count * int(np.dtype([(n, endian + t) for n, t in props]).itemsize), os.SEEK_CUR)
        return
    for _ in range(count):  # list properties (faces): each row says how long it is
        for _, t in props:
            if isinstance(t, tuple):
                b = f.read(np.dtype(t[1]).itemsize)
                if len(b) != np.dtype(t[1]).itemsize:
                    raise ValueError(f"{filename}: PLY data ends inside an element")
                n = int(np.frombuffer(b, endian + t[1])[0])
                f.seek(n * np.dtype(t[2]).itemsize, os.SEEK_CUR)
            else:
                f.seek(np.dtype(t).itemsize, os.SEEK_CUR)


def read_mesh_vertices(filename):
    """utils.py:69-78: the `vertex` element's x, y, z as float32 [N, 3].

    Reads ascii, binary_little_endian and binary_big_endian PLY files with any other vertex properties (ScanNet's meshes carry
    `red green blue alpha` uchar) and any elements before or after `vertex`.  Raises ValueError for anything else: a
    malformed header, no vertex element or no x / y / z, a list property inside `vertex` of a binary file, or a file that
    ends early."""
    if not os.path.isfile(filename):
        raise FileNotFoundError(filename)
    with open(filename, "rb") as f:
        fmt, elements = _parse_ply_header(f, filename)
        names = [e[0] for e in elements]
        if "vertex" not in names:
            raise ValueError(f"{filename}: PLY file has no vertex element")
        _, count, props = elements[names.index("vertex")]
        pnames = [n for n, _ in props]
        for axis in ("x", "y", "z"):
            if axis not in pnames:
                raise ValueError(f"{filename}: PLY vertex element has no '{axis}' property")
        if fmt == "ascii":
            return _read_ascii_vertices(f, elements, filename)
        endian = "<" if fmt == "binary_little_endian" else ">"
        if any(isinstance(t, tuple) for _, t in props):
            raise ValueError(f"{filename}: list property inside the vertex element of a binary PLY file is not supported")
        for name, n, p in elements:
            if name == "vertex":
                break
            _skip_binary_element(f, n, p, endian, filename)
        dt = np.dtype([(n, endian + t) for n, t in props])
        buf = f.read(count * dt.itemsize)
        if len(buf) != count * dt.itemsize:
            raise ValueError(f"{filename}: PLY data ends inside the vertex element")
        data = np.frombuffer(buf, dt, count)
    out = np.zeros((count, 3), np.float32)
    out[:, 0], out[:, 1], out[:, 2] = data["x"], data["y"], data["z"]
    return out


def read_mesh_faces(filename):
    """The first three vertex ids of every row of the `face` element's first property, int64 [M, 3] (what the reference's
    visualization.read_ply takes: `face[0][0..2]`, tools/visualization.py:71-72).  Quads and longer polygons give their
    first three ids.  A file without a face element gives [0, 3].  Raises ValueError when that property is not a list,
    when a row has fewer than three ids, or when the file ends early."""
    if not os.path.isfile(filename):
        raise FileNotFoundError(filename)
    with open(filename, "rb") as f:
        fmt, elements = _parse_ply_header(f, filename)
        names = [e[0] for e in elements]
        if "face" not in names:
            return np.zeros((0, 3), np.int64)
        at = names.index("face")
        _, count, props = elements[at]
        if not props or not isinstance(props[0][1], tuple):
            raise ValueError(f"{filename}: the first property of the PLY face element is not a list")
        if fmt == "ascii":
            lines = f.read().decode("ascii", errors="replace").splitlines()
            row = sum(e[1] for e in elements[:at])
            if row + count > len(lines):
                raise ValueError(f"{filename}: PLY data ends inside the face element")
            out = np.zeros((count, 3), np.int64)
            for i in range(count):
                words = lines[row + i].split()
                if len(words) < 4 or int(words[0]) < 3:
                    raise ValueError(f"{filename}: PLY face {i} has fewer than three vertex ids")
                out[i] = [int(w) for w in words[1:4]]
            return out
        endian = "<" if fmt == "binary_little_endian" else ">"
        for name, n, p in elements[:at]:
            _skip_binary_element(f, n, p, endian, filename)
        _, ct, it = props[0][1]
        csize = np.dtype(ct).itemsize
        if len(props) == 1 and count > 0:  # one list per row: uniform rows (all triangles) are read as one array
            start = f.tell()
            head = f.read(csize)
            if len(head) == csize:
                k = int(np.frombuffer(head, endian + ct)[0])
                dt = np.dtype([("n", endian + ct), ("i", endian + it, (k,))])
                rest = f.read(count * dt.itemsize - csize)
                if k >= 3 and len(rest) == count * dt.itemsize - csize:
                    rows = np.frombuffer(head + rest, dt, count)
                    if (rows["n"] == k).all():
                        return rows["i"][:, :3].astype(np.int64)
            f.seek(start)
        out = np.zeros((count, 3), np.int64)
        for i in range(count):
            for j, (_, t) in enumerate(props):
                if isinstance(t, tuple):
                    b = f.read(np.dtype(t[1]).itemsize)
                    if len(b) != np.dtype(t[1]).itemsize:
                        raise ValueError(f"{filename}: PLY data ends inside the face element")
                    n = int(np.frombuffer(b, endian + t[1])[0])
                    b = f.read(n * np.dtype(t[2]).itemsize)
                    if len(b) != n * np.dtype(t[2]).itemsize:
                        raise ValueError(f"{filename}: PLY data ends inside the face element")
                    if j == 0:
                        if n < 3:
                            raise ValueError(f"{filename}: PLY face {i} has fewer than three vertex ids")
                        out[i] = np.frombuffer(b, endian + t[2], 3)
                elif len(f.read(np.dtype(t).itemsize)) != np.dtype(t).itemsize:
                    raise ValueError(f"{filename}: PLY data ends inside the face element")
        return out


def _read_ascii_vertices(f, elements, filename):
    lines = f.read().decode("ascii", errors="replace").splitlines()
    row = 0
    for name, count, props in elements:
        if name != "vertex":
            row += count
            continue
        cols = [n for n, _ in props]
        if any(isinstance(t, tuple) for _, t in props):  # a list inside vertex: take x, y, z only if they precede it
            last = max(cols.index(a) for a in ("x", "y", "z"))
            if any(isinstance(t, tuple) for _, t in props[:last + 1]):
                raise ValueError(f"{filename}: list property before x / y / z in the vertex element is not supported")
        if row + count > len(lines):
            raise ValueError(f"{filename}: PLY data ends inside the vertex element")
        out = np.zeros((count, 3), np.float32)
        ix = [cols.index(a) for a in ("x", "y", "z")]
        for v in range(count):
            words = lines[row + v].split()
            if len(words) <= max(ix):
                raise ValueError(f"{filename}: PLY vertex line {v} has {len(words)} values")
            out[v] = [float(words[i]) for i in ix]
        return out
    raise ValueError(f"{filename}: PLY file has no vertex element")
