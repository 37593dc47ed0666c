"""PLY meshes of test-mode results (the reference's tools/visualization.py, lines cited per function).

    python tools/visualization.py --path RESULTS --mode results

For every result folder `<scene>` under RESULTS, in the folder itself:
- scene.ply: a cube per voxel of scene.npy with a value > 0;
- pred_roi.ply: the cylinder edges of the boxes in pred_roi.npy, when that file exists;
- pred_bbox.ply: the cylinder edges of pred_box.npy's boxes, coloured by pred_class.npy (the kept boxes
  pred_box[pred_mask_index] when the mask files exist);
- pred_mask.ply: the cubes of the kept masks painted into a volume of scene.npy's shape (first mask wins, corners rounded
  half to even, a voxel set where the mask is != 0, a mask larger than its box cropped to the box), coloured by class;
- gt_bbox.ply and gt_mask.ply in the same way from gt_box.npy / gt_class.npy / gt_mask, when test mode wrote them.
Each file is byte for byte what the reference writes (visualization.py:399-503).

The work runs through libsis3d (csrc/ply.cu): the masks are painted by sis3d_instance_paint, the cubes are numbered and
emitted by sis3d_voxel_mesh, and every text line is formatted by sis3d_ply_ascii.  A file is written in slabs of at most
`slab_lines` lines: while the host writes one slab to the file, the GPU formats the next and copies it to pinned memory, so
device memory stays bounded for any scene.  The bounding-box cylinders are computed on the host with numpy, in the
reference's dtypes.  There is no CPU path: without a CUDA device the first launch raises.

Departures from the reference, none of which changes a file it can write:
- `--mode results` (the spelling the reference's README documents) works as `--mode result`; the reference tests only
  'result' and silently writes nothing for 'results'.  `--mode data` (training chunks) is not provided.
- Folders are visited in sorted order and entries that are not directories are skipped; the reference calls np.load on
  them and crashes.
- read_ply needs only the vertices' x, y, z and the face list; the reference needs exactly `x y z red green blue alpha`.
  Its colours come back as float64 [N, 3] when the file has red / green / blue, else None.
- With pred_box.npy but no pred_class.npy the boxes are coloured as class 1, as the GT branch does; the reference's
  `np.oneos_like` there raises AttributeError.
"""
from __future__ import annotations

import argparse
import ctypes as C
import math
import os
import pickle
import sys
import time

import numpy as np
import torch

if __package__:
    from .scannet_benchmark import utils as mesh_io
else:  # run as a script
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    from tools.scannet_benchmark import utils as mesh_io

from lib import _sis3d as S
from lib.utils.evaluation import pack_masks

SLAB_LINES = 1 << 24  # text lines per slab: at most ~1.2 GB of device buffers (inputs and text) per slab
SCAN_TILE = 2048  # SIS3D_PLY_SCAN_TILE

# write_ply's header (visualization.py:85-96), including the space after "ply"
PLY_HEADER = ("ply \nformat ascii 1.0\nelement vertex {:d}\nproperty float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face {:d}\n"
              "property list uchar uint vertex_indices\nend_header\n")


def create_color_palette():
    """The NYU40 / ScanNet label colours (visualization.py:15-58): entry i is label i's colour, entry 0 black."""
    return [(0, 0, 0), (174, 199, 232), (152, 223, 138), (31, 119, 180), (255, 187, 120), (188, 189, 34), (140, 86, 75),
            (255, 152, 150), (214, 39, 40), (197, 176, 213), (148, 103, 189), (196, 156, 148), (23, 190, 207),
            (178, 76, 76), (247, 182, 210), (66, 188, 102), (219, 219, 141), (140, 57, 197), (202, 185, 52),
            (51, 176, 203), (200, 54, 131), (92, 193, 61), (78, 71, 183), (172, 114, 82), (255, 127, 14), (91, 163, 138),
            (153, 98, 156), (140, 153, 101), (158, 218, 229), (100, 125, 154), (178, 127, 135), (120, 185, 128),
            (146, 111, 194), (44, 160, 44), (112, 128, 144), (96, 207, 209), (227, 119, 194), (213, 92, 176),
            (94, 106, 211), (82, 84, 163), (100, 85, 144)]


def palette_written():
    """int64 [41, 3]: what write_ply writes for each palette entry, int(c / 255.0 * 255)."""
    return (np.array(create_color_palette(), np.float64) / 255.0 * 255).astype(np.int64)


def read_ply(ply_file):
    """-> (points float32 [N, 3], indices int64 [M, 3], colors float64 [N, 3] or None) (visualization.py:61-76)."""
    points = mesh_io.read_mesh_vertices(ply_file)
    indices = mesh_io.read_mesh_faces(ply_file)
    colors = None
    with open(ply_file, "rb") as f:
        fmt, elements = mesh_io._parse_ply_header(f, ply_file)
    props = dict(next((e[2] for e in elements if e[0] == "vertex"), []))
    if all(c in props for c in ("red", "green", "blue")) and not any(isinstance(t, tuple) for t in props.values()):
        with open(ply_file, "rb") as f:
            mesh_io._parse_ply_header(f, ply_file)
            colors = _vertex_columns(f, fmt, elements, ("red", "green", "blue"), ply_file)
    return points, indices, colors


def _vertex_columns(f, fmt, elements, names, filename):
    for name, count, props in elements:
        if name == "vertex":
            break
    cols = [n for n, _ in props]
    if fmt == "ascii":
        skip = sum(e[1] for e in elements[:[e[0] for e in elements].index("vertex")])
        rows = f.read().decode("ascii", errors="replace").splitlines()[skip:skip + count]
        data = np.array([r.split() for r in rows], np.float64).reshape(count, len(cols))
        return data[:, [cols.index(n) for n in names]]
    endian = "<" if fmt == "binary_little_endian" else ">"
    for e in elements:
        if e[0] == "vertex":
            break
        mesh_io._skip_binary_element(f, e[1], e[2], endian, filename)
    dt = np.dtype([(n, endian + t) for n, t in props])
    data = np.frombuffer(f.read(count * dt.itemsize), dt, count)
    return np.stack([data[n].astype(np.float64) for n in names], 1)


# ------------------------------------------------------------------------------------------------------ the formatter
def _device(device=None):
    if device is not None:
        return torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


def format_lines_host(verts, colors, faces):
    """write_ply's body lines (visualization.py:97-100) formatted by Python: the route for a slab with a coordinate of
    magnitude >= 2^64, which the device formatter does not handle."""
    out = ["{:f} {:f} {:f} {:d} {:d} {:d}\n".format(*v, *c) for v, c in zip(np.asarray(verts).tolist(), np.asarray(colors).tolist())]
    out += ["3 {:d} {:d} {:d}\n".format(*t) for t in np.asarray(faces).tolist()]
    return "".join(out).encode("ascii")


class PlyWriter:
    """One ASCII PLY file: the header on the host, the body formatted on the device one slab at a time.

    format() takes device arrays of one slab (vertices, then faces; at most `slab_lines` lines) and writes their text: the
    lengths pass, one read-back of the slab's byte count, the write pass and an asynchronous copy into one of two pinned
    buffers.  The previous slab's buffer is written to the file while the device works on this one.  `stats`, when given,
    collects CUDA event pairs per phase ('format', 'd2h') and the seconds spent in file writes ('file_write_s')."""

    def __init__(self, output_file, n_vert, n_face, device=None, stats=None):
        self.dev = _device(device)
        self.cuda = self.dev.type == "cuda"
        self.stats = stats
        self.f = open(output_file, "wb")
        self._write(PLY_HEADER.format(n_vert, n_face).encode("ascii"))
        self.offsets = self.scratch = self.text = None
        self.host = [None, None]
        self.turn = 0
        self.pending = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        try:
            if exc[0] is None:
                self._flush()
        finally:
            self.f.close()

    def _write(self, data):
        t = time.perf_counter()
        self.f.write(data)
        if self.stats is not None:
            self.stats["file_write_s"] = self.stats.get("file_write_s", 0.0) + time.perf_counter() - t

    def _flush(self):
        if self.pending is not None:
            buf, n, done = self.pending
            if done is not None:
                done.synchronize()
            self._write(memoryview(buf.numpy())[:n])
            self.pending = None

    def _event(self):
        if self.cuda and self.stats is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            return e
        return None

    def _grow(self, t, n, dtype, pinned=False):
        if t is not None and t.numel() >= n:
            return t
        if pinned:
            return torch.empty(max(n, 1), dtype=dtype, pin_memory=self.cuda)
        return torch.empty(max(n, 1), dtype=dtype, device=self.dev)

    def format(self, verts, colors, n_vert, faces, n_face):
        n = n_vert + n_face
        if n == 0:
            return
        h = S.stream() if self.cuda else None
        self.offsets = self._grow(self.offsets, n + 2, torch.int64)
        self.scratch = self._grow(self.scratch, (n + SCAN_TILE - 1) // SCAN_TILE, torch.int64)
        args = (S.ptr(verts), S.ptr(colors), C.c_int64(n_vert), S.ptr(faces), C.c_int64(n_face), C.c_int64(0), C.c_int64(n))
        e0 = self._event()
        S.check(S.lib.sis3d_ply_ascii_lengths(*args, S.ptr(self.offsets), S.ptr(self.scratch), h), "ply_ascii_lengths")
        e1 = self._event()
        nbytes, n_big = self.offsets[n:n + 2].tolist()  # waits for this slab's lengths and the previous slab's copy
        if n_big:
            self._flush()
            nv = (verts[:3 * n_vert].view(-1, 3).cpu().numpy(), colors[:3 * n_vert].view(-1, 3).cpu().numpy()) if n_vert \
                else (np.zeros((0, 3)), np.zeros((0, 3), np.int64))
            fc = faces[:3 * n_face].view(-1, 3).cpu().numpy() if n_face else np.zeros((0, 3), np.int64)
            self._write(format_lines_host(nv[0], nv[1], fc))
            return
        self.text = self._grow(self.text, nbytes, torch.uint8)
        e2 = self._event()
        S.check(S.lib.sis3d_ply_ascii(*args, S.ptr(self.offsets), S.ptr(self.text), h), "ply_ascii")
        e3 = self._event()
        buf = self.host[self.turn] = self._grow(self.host[self.turn], nbytes, torch.uint8, pinned=True)
        buf[:nbytes].copy_(self.text[:nbytes], non_blocking=self.cuda)
        done = None
        if self.cuda:
            done = torch.cuda.Event(enable_timing=self.stats is not None)
            done.record()
        if self.stats is not None and self.cuda:
            self.stats.setdefault("format", []).extend([(e0, e1), (e2, e3)])
            self.stats.setdefault("d2h", []).append((e3, done))
        self._flush()
        self.pending = (buf, nbytes, done)
        self.turn ^= 1


def event_ms(pairs):
    """Total milliseconds of (start, end) CUDA event pairs (after the work has finished)."""
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in pairs)


# ------------------------------------------------------------------------------------------------------------ writers
def write_ply(verts, colors, indices, output_file, slab_lines=SLAB_LINES, device=None, stats=None):
    """visualization.py:78-101: vertices (x, y, z as '{:f}'), colours written as int(c * 255) and triangles (the first
    three ids of each row of `indices`).  colors None writes 0 0 0; indices None writes no faces."""
    verts = np.asarray(verts, np.float64)
    verts = verts.reshape(-1, 3) if verts.size == 0 else verts[:, :3]
    colors = np.zeros_like(verts) if colors is None else np.asarray(colors)
    colors = np.zeros((0, 3)) if colors.size == 0 else colors[:, :3]
    if len(colors) != len(verts):
        raise ValueError(f"{len(verts)} vertices but {len(colors)} colours")
    with np.errstate(invalid="ignore"):
        cint = (colors * 255).astype(np.int64)  # int(): truncation toward zero
    faces = np.asarray([] if indices is None else indices)
    faces = np.zeros((0, 3), np.int64) if faces.size == 0 else faces[:, :3].astype(np.int64)
    slab = max(int(slab_lines), 1)
    with PlyWriter(output_file, len(verts), len(faces), device, stats) as w:
        for a in range(0, len(verts), slab):
            v = torch.from_numpy(np.ascontiguousarray(verts[a:a + slab]).reshape(-1)).to(w.dev)
            c = torch.from_numpy(np.ascontiguousarray(cint[a:a + slab]).reshape(-1)).to(w.dev)
            w.format(v, c, len(v) // 3, None, 0)
        for a in range(0, len(faces), slab):
            fc = torch.from_numpy(np.ascontiguousarray(faces[a:a + slab]).reshape(-1)).to(w.dev)
            w.format(None, None, 0, fc, len(fc) // 3)


def write_voxel_mesh(labels, dims, output_file, lut=None, slab_lines=SLAB_LINES, device=None, stats=None):
    """The cubes of a device int32 label volume [X][Y][Z] (or of lut[labels] for a device int32 lut), as write_mask writes
    them: occupied voxels (label > 0) counted and numbered on the device, then emitted and formatted in slabs of at most
    `slab_lines` face lines.  -> number of cubes."""
    dev = labels.device
    cuda = dev.type == "cuda"
    h = S.stream() if cuda else None
    X, Y, Z = (int(d) for d in dims)
    n_rows = Y * Z
    n_lut = 0 if lut is None else int(lut.numel())
    rows = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
    scratch = torch.empty(max((n_rows + SCAN_TILE - 1) // SCAN_TILE, 1), dtype=torch.int64, device=dev)
    palette = torch.from_numpy(palette_written().reshape(-1)).to(dev)
    e0 = torch.cuda.Event(enable_timing=True) if cuda and stats is not None else None
    if e0 is not None:
        e0.record()
    S.check(S.lib.sis3d_voxel_mesh_count(S.ptr(labels), S.ptr(lut), n_lut, X, Y, Z, S.ptr(rows), S.ptr(scratch), h),
            "voxel_mesh_count")
    n_occ = int(rows[n_rows].item())
    per = max(1, int(slab_lines) // 12)  # cubes per slab: 12 face lines each
    m = min(per, max(n_occ, 1))
    vbuf = torch.empty(24 * m, dtype=torch.float64, device=dev)
    cbuf = torch.empty(24 * m, dtype=torch.int64, device=dev)
    fbuf = torch.empty(36 * m, dtype=torch.int64, device=dev)

    def mesh(k0, k1, v, c, f):
        a = torch.cuda.Event(enable_timing=True) if e0 is not None else None
        if a is not None:
            a.record()
        S.check(S.lib.sis3d_voxel_mesh(S.ptr(labels), S.ptr(lut), n_lut, X, Y, Z, S.ptr(rows), S.ptr(palette), C.c_int64(k0),
                                       C.c_int64(k1), S.ptr(v), S.ptr(c), S.ptr(f), h), "voxel_mesh")
        if a is not None:
            b = torch.cuda.Event(enable_timing=True)
            b.record()
            stats.setdefault("mesh", []).append((a, b))

    with PlyWriter(output_file, 8 * n_occ, 12 * n_occ, dev, stats) as w:
        for k0 in range(0, n_occ, per):
            k1 = min(k0 + per, n_occ)
            mesh(k0, k1, vbuf, cbuf, None)
            w.format(vbuf, cbuf, 8 * (k1 - k0), None, 0)
        for k0 in range(0, n_occ, per):
            k1 = min(k0 + per, n_occ)
            mesh(k0, k1, None, None, fbuf)
            w.format(None, None, 0, fbuf, 12 * (k1 - k0))
    return n_occ


def label_codes(values):
    """Values -> int32 codes with the same drawing: 0 where value > 0 fails, else int(value % 41) + 41 (so code > 0 and
    code % 41 is the palette entry write_mask picks, visualization.py:315-318)."""
    v = np.asarray(values)
    with np.errstate(invalid="ignore"):
        return np.where(v > 0, (v % 41).astype(np.int64) + 41, 0).astype(np.int32)


def write_mask(mask, output_file, slab_lines=SLAB_LINES, device=None, stats=None):
    """visualization.py:263-324: a cube (8 vertices, 12 triangles) for every voxel of the [X, Y, Z] volume with a value
    > 0, visited z outermost and x innermost, coloured by palette[int(value % 41)]."""
    mask = np.asarray(mask)
    if mask.ndim != 3:
        raise ValueError(f"write_mask takes a 3-D volume, not shape {mask.shape}")
    dev = _device(device)
    labels = torch.from_numpy(np.ascontiguousarray(label_codes(mask)).reshape(-1)).to(dev)
    return write_voxel_mesh(labels, mask.shape, output_file, None, slab_lines, dev, stats)


def write_painted_masks(dims, boxes, masks, classes, output_file, slab_lines=SLAB_LINES, device=None, stats=None):
    """The mask branch of visualization.py:444-459 / 488-503: every box's mask (voxels != 0) painted at its corners rounded
    half to even into a volume of shape `dims`, a voxel keeping the first nonzero class painted into it (class truncated
    to an integer; classes None paints 1), then write_mask of that volume.  A mask larger than its box is cropped to it;
    a smaller mask or a box leaving the volume raises ValueError."""
    boxes = np.asarray(boxes, np.float64).reshape(-1, 6)
    n = len(boxes)
    cls = np.ones(n, np.int64) if classes is None else np.asarray(classes).reshape(-1)[:n].astype(np.int64)
    ib = np.rint(boxes)
    ib[:, 3:] = np.maximum(ib[:, 3:], ib[:, :3])  # an inverted box paints nothing, as range(min, max) is empty
    ext = (ib[:, 3:] - ib[:, :3]).astype(np.int64)
    # a class that truncates to 0 leaves its voxels free for later boxes (the reference tests mask_scene == 0)
    use = [b for b in range(n) if cls[b] != 0 and ext[b].prod() > 0]
    if len(masks) < n and any(b >= len(masks) for b in use):
        raise ValueError(f"{len(masks)} masks for {n} boxes")
    parts = [np.asarray(masks[b])[:ext[b, 0], :ext[b, 1], :ext[b, 2]] != 0 for b in use]
    bits, offs, ibox = pack_masks(parts, ib[use], tuple(int(d) for d in dims), "mask")
    dev = _device(device)
    h = S.stream() if dev.type == "cuda" else None
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).to(dev)
    bits_d, offs_d, box_d, lut = to(bits), to(offs), to(ibox), to(label_codes(cls[use]))
    X, Y, Z = (int(d) for d in dims)
    owner = torch.empty(max(X * Y * Z, 1), dtype=torch.int32, device=dev)
    S.check(S.lib.sis3d_instance_paint(S.ptr(bits_d), S.ptr(offs_d), S.ptr(box_d), len(use), 0, 0, 0, X, Y, Z, S.ptr(owner),
                                       h), "instance_paint")
    return write_voxel_mesh(owner, (X, Y, Z), output_file, lut, slab_lines, dev, stats)


# ------------------------------------------------------------------------------------------------------------ cylinders
_STACKS = _SLICES = 10
_RADIUS = 0.02
_EDGES = np.array([(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)])
# get_bbox_verts' corners (visualization.py:172-181): 1 = the box's max on that axis
_CORNER_HI = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)], bool)
# create_cylinder_mesh's ring positions (cos, sin of i2 * 2.0 * pi / slices, Python's math) and triangles (139-148)
_RING = np.array([[_RADIUS * math.cos(i2 * 2.0 * math.pi / _SLICES), _RADIUS * math.sin(i2 * 2.0 * math.pi / _SLICES)]
                  for i2 in range(_SLICES)])
_CYL_FACES = np.array([t for i in range(_STACKS) for i2 in range(_SLICES) for t in (
    ((i + 1) * _SLICES + i2, i * _SLICES + i2, i * _SLICES + (i2 + 1) % _SLICES),
    ((i + 1) * _SLICES + i2, i * _SLICES + (i2 + 1) % _SLICES, (i + 1) * _SLICES + (i2 + 1) % _SLICES))], np.int64)
_CYL_VERTS = (_STACKS + 1) * _SLICES


def _length(v):
    """compute_length_vec3 (visualization.py:111-112) over rows: squares summed in v's dtype, sqrt in float64."""
    return np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2]).astype(np.float64))


def _rotation(axis, c, s, t):
    """rotation() of visualization.py:114-132 over rows, in the dtype the operands give (float32, or float64 axes)."""
    axis = axis / _length(axis).astype(axis.dtype)[:, None]
    x, y, z = axis[:, 0], axis[:, 1], axis[:, 2]
    one = axis.dtype.type(1)
    rot = np.zeros((len(axis), 3, 3))
    rot[:, 0, 0] = one + t * (x * x - one)
    rot[:, 0, 1] = z * s + t * x * y
    rot[:, 0, 2] = -y * s + t * x * z
    rot[:, 1, 0] = -z * s + t * x * y
    rot[:, 1, 1] = one + t * (y * y - one)
    rot[:, 1, 2] = x * s + t * y * z
    rot[:, 2, 0] = y * s + t * x * z
    rot[:, 2, 1] = -x * s + t * y * z
    rot[:, 2, 2] = one + t * (z * z - one)
    return rot


def bbox_cylinders(bbox):
    """The meshes write_bbox draws (visualization.py:103-227), vectorised over every edge of every box with the reference's
    dtypes: corners in the boxes' dtype, the edge vector and rotation in float32 (float64 for the axis of an edge along -z),
    the transform and vertices in float64.  A zero-length edge gives nan vertices, as in the reference.
    -> (verts float64 [12 * 110 * n, 3], colors float64 [same, 3] = palette / 255.0, faces int64 [12 * 200 * n, 3])."""
    B = np.asarray(bbox)
    if B.size == 0:
        return np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3), np.int64)
    B = B.reshape(-1, B.shape[-1])
    n = len(B)
    corners = np.where(_CORNER_HI[None], B[:, None, 3:6], B[:, None, 0:3])  # [n, 8, 3], the boxes' dtype
    p0 = corners[:, _EDGES[:, 0]].reshape(-1, 3)
    p1 = corners[:, _EDGES[:, 1]].reshape(-1, 3)
    diff = (p1 - p0).astype(np.float32)
    height = _length(diff)
    with np.errstate(invalid="ignore", divide="ignore"):
        vb = diff / height.astype(np.float32)[:, None]
        va = np.array([0, 0, 1], np.float32)
        axis = np.cross(vb, va)
        dot = vb[:, 0] * va[0] + vb[:, 1] * va[1] + vb[:, 2] * va[2]
        angle = np.arccos(np.clip(dot, np.float32(-1), np.float32(1)))
        turn = angle != 0
        flip = turn & (_length(axis) == 0)  # an edge along -z: axis [1, 0, 0] in float64 (va[0] is 0)
        c, s = np.cos(angle), np.sin(angle)
        t = np.float32(1.0) - c
        rot = np.broadcast_to(np.eye(3), (len(diff), 3, 3)).copy()
        k = turn & ~flip
        if k.any():
            rot[k] = _rotation(axis[k], c[k], s[k], t[k])
        if flip.any():
            ax = np.zeros((int(flip.sum()), 3))
            ax[:, 0] = 1.0
            rot[flip] = _rotation(ax, c[flip].astype(np.float64), s[flip].astype(np.float64), t[flip].astype(np.float64))
    trans = 0.0 + p0.astype(np.float64)
    stack = np.arange(_STACKS + 1, dtype=np.float64)
    pz = (height[:, None] * stack[None]) / _STACKS  # height * i / stacks
    px = np.broadcast_to(_RING[None, None, :, 0], (len(diff), _STACKS + 1, _SLICES))
    py = np.broadcast_to(_RING[None, None, :, 1], (len(diff), _STACKS + 1, _SLICES))
    pz = np.broadcast_to(pz[:, :, None], (len(diff), _STACKS + 1, _SLICES))
    r = rot[:, None, None]
    out = np.empty((len(diff), _STACKS + 1, _SLICES, 3))
    for a in range(3):  # np.dot(transform, [x, y, z, 1.0]), row by row, then / 1.0
        out[..., a] = r[..., a, 0] * px + r[..., a, 1] * py + r[..., a, 2] * pz + trans[:, None, None, a]
    verts = out.reshape(-1, 3)
    pal = np.array(create_color_palette(), np.float64)[(B[:, 6] % 41).astype(np.int64)] / 255.0
    colors = np.repeat(pal, 12 * _CYL_VERTS, axis=0)
    faces = (_CYL_FACES[None] + _CYL_VERTS * np.arange(12 * n)[:, None, None]).reshape(-1, 3)
    return verts, colors, faces


def write_bbox(bbox, output_file=None, slab_lines=SLAB_LINES, device=None, stats=None):
    """visualization.py:103-227: twelve cylinders (radius 0.02, 10 stacks x 10 slices) per box [x0 y0 z0 x1 y1 z1 label],
    coloured by palette[int(label % 41)].  Without output_file -> (verts, colors, indices) arrays."""
    verts, colors, faces = bbox_cylinders(bbox)
    if output_file is None:
        return verts, colors, faces
    write_ply(verts, colors, faces, output_file, slab_lines, device, stats)


# ------------------------------------------------------------------------------------------------------ result folders
def _load(loader, path):
    """The reference's `try: ... except: flag = False` around each result file (visualization.py:407-479)."""
    try:
        return loader(path)
    except Exception:
        return None


def _unpickle(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def visualize_result_folder(d, slab_lines=SLAB_LINES, device=None, stats=None):
    """The files the reference writes into one result folder (visualization.py:403-503)."""
    kw = dict(slab_lines=slab_lines, device=device, stats=stats)
    scene = np.load(os.path.join(d, "scene.npy"))
    write_mask(scene, os.path.join(d, "scene.ply"), **kw)
    first6 = lambda p: np.load(p)[:, :6]
    pred_roi = _load(first6, os.path.join(d, "pred_roi.npy"))
    pred_box = _load(first6, os.path.join(d, "pred_box.npy"))
    pred_class = _load(np.load, os.path.join(d, "pred_class.npy"))
    pred_mask = None
    try:  # kept boxes and classes only when every mask file loads (visualization.py:426-433)
        masks = _unpickle(os.path.join(d, "pred_mask"))
        index = _unpickle(os.path.join(d, "pred_mask_index"))
        pred_box = pred_box[index]
        pred_class = pred_class[index]
        pred_mask = masks
    except Exception:
        pass
    if pred_roi is not None:
        write_bbox(np.concatenate([pred_roi, np.ones_like(pred_roi)[:, 0:1]], 1), os.path.join(d, "pred_roi.ply"), **kw)
    if pred_box is not None:
        label = np.expand_dims(pred_class, 1) if pred_class is not None else np.ones_like(pred_box)[:, 0:1]
        write_bbox(np.concatenate([pred_box, label], 1), os.path.join(d, "pred_bbox.ply"), **kw)
    if pred_mask is not None:
        write_painted_masks(scene.shape, pred_box, pred_mask, pred_class, os.path.join(d, "pred_mask.ply"), **kw)
    gt_box = _load(first6, os.path.join(d, "gt_box.npy"))
    gt_class = _load(np.load, os.path.join(d, "gt_class.npy"))
    gt_mask = _load(_unpickle, os.path.join(d, "gt_mask"))
    if gt_box is not None:
        label = np.expand_dims(gt_class, 1) if gt_class is not None else np.ones_like(gt_box)[:, 0:1]
        write_bbox(np.concatenate([gt_box, label], 1), os.path.join(d, "gt_bbox.ply"), **kw)
        if gt_mask is not None:
            write_painted_masks(scene.shape, gt_box, gt_mask, gt_class, os.path.join(d, "gt_mask.ply"), **kw)


def visualize_results(path, slab_lines=SLAB_LINES, device=None, stats=None):
    """Every result folder under `path`, in sorted order; entries that are not directories are skipped."""
    for scene in sorted(os.listdir(path)):
        if os.path.isdir(os.path.join(path, scene)):
            visualize_result_folder(os.path.join(path, scene), slab_lines, device, stats)


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description="3D-SIS")
    parser.add_argument("--path", type=str, default="../results/")
    parser.add_argument("--mode", type=str, default="npy")
    return parser.parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    print("Called with args:")
    print(args)
    if args.mode in ("result", "results"):
        visualize_results(args.path)


if __name__ == "__main__":
    main()
