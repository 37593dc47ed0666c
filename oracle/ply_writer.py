"""oracle/ply_writer.py -- TEST INFRASTRUCTURE ONLY: the reference's ASCII PLY writers restated in plain Python and numpy, to
check the GPU route (tools/visualization.py) at sizes the golden file cannot hold.

- write_ply: tools/visualization.py:78-101 of the reference (header with its "ply " line, one str.format per line);
- mask_mesh / write_mask: 263-324 (a cube per voxel with value > 0, z outermost, x innermost; corners fl(c - 0.05) and
  fl(c + 0.95); palette[int(value % 41)] / 255.0);
- paint_masks: the mask branches of 444-459 / 488-503 (int(round()) corners, first nonzero class wins, mask != 0).
The cube loop is vectorised with numpy (np.nonzero over the volume transposed to z, y, x order); the text is formatted one
line at a time with the same format strings, so its bytes are what the reference writes.  The palette is the published
NYU40 / ScanNet label colour table (tests/golden/visualization_reference.npz pins it).
"""
from __future__ import annotations

import numpy as np

PALETTE = np.array([
    (0, 0, 0), (174, 199, 232), (152, 223, 138), (31, 119, 180), (255, 187, 120), (188, 189, 34), (140, 86, 75),
    (255, 152, 150), (214, 39, 40), (197, 176, 213), (148, 103, 189), (196, 156, 148), (23, 190, 207), (178, 76, 76),
    (247, 182, 210), (66, 188, 102), (219, 219, 141), (140, 57, 197), (202, 185, 52), (51, 176, 203), (200, 54, 131),
    (92, 193, 61), (78, 71, 183), (172, 114, 82), (255, 127, 14), (91, 163, 138), (153, 98, 156), (140, 153, 101),
    (158, 218, 229), (100, 125, 154), (178, 127, 135), (120, 185, 128), (146, 111, 194), (44, 160, 44), (112, 128, 144),
    (96, 207, 209), (227, 119, 194), (213, 92, 176), (94, 106, 211), (82, 84, 163), (100, 85, 144)], np.int64)

# make_voxel_mesh (269-304): corner c takes the box max on an axis where this table has 1
CUBE_CORNERS = np.array([(1, 1, 1), (0, 1, 1), (0, 0, 1), (1, 0, 1), (1, 1, 0), (0, 1, 0), (0, 0, 0), (1, 0, 0)], bool)
CUBE_FACES = np.array([(1, 2, 3), (1, 3, 0), (0, 3, 7), (0, 7, 4), (3, 2, 6), (3, 6, 7), (1, 6, 2), (1, 5, 6), (0, 5, 1),
                       (0, 4, 5), (6, 5, 4), (6, 4, 7)], np.int64)


def ply_text(verts, colors, indices):
    """write_ply's bytes (78-101).  colors None -> zeros; indices None -> no faces."""
    verts = list(verts)
    colors = [np.zeros(3)] * len(verts) if colors is None else list(colors)
    indices = [] if indices is None else list(indices)
    out = ["ply \n", "format ascii 1.0\n", "element vertex {:d}\n".format(len(verts)), "property float x\n",
           "property float y\n", "property float z\n", "property uchar red\n", "property uchar green\n",
           "property uchar blue\n", "element face {:d}\n".format(len(indices)), "property list uchar uint vertex_indices\n",
           "end_header\n"]
    for v, c in zip(verts, colors):
        out.append("{:f} {:f} {:f} {:d} {:d} {:d}\n".format(float(v[0]), float(v[1]), float(v[2]), int(c[0] * 255),
                                                            int(c[1] * 255), int(c[2] * 255)))
    for t in indices:
        out.append("3 {:d} {:d} {:d}\n".format(int(t[0]), int(t[1]), int(t[2])))
    return "".join(out).encode("ascii")


def write_ply(verts, colors, indices, path):
    with open(path, "wb") as f:
        f.write(ply_text(verts, colors, indices))


def mask_mesh(mask):
    """-> (verts float64 [8n, 3], colors float64 [8n, 3], faces int64 [12n, 3]) of write_mask (263-324)."""
    mask = np.asarray(mask)
    zyx = np.transpose(mask, (2, 1, 0))  # visiting order: z, then y, then x
    z, y, x = np.nonzero(zyx > 0)
    vals = zyx[z, y, x]
    c = np.stack([x, y, z], 1).astype(np.int64)
    lo, hi = c - 0.05, c + 0.95
    verts = np.where(CUBE_CORNERS[None], hi[:, None], lo[:, None]).reshape(-1, 3)
    colors = np.repeat(PALETTE[(vals % 41).astype(np.int64)] / 255.0, 8, axis=0)
    faces = (CUBE_FACES[None] + 8 * np.arange(len(c))[:, None, None]).reshape(-1, 3)
    return verts, colors, faces


def write_mask(mask, path):
    write_ply(*mask_mesh(mask), path)


def paint_masks(shape, boxes, masks, classes):
    """The int64 label volume of the mask branch (444-459): box b's voxels (i, j, k) in range(int(round(lo)),
    int(round(hi))) where masks[b][i - lo, j - lo, k - lo] != 0 and the volume is still 0 get classes[b] (1 if None)."""
    vol = np.zeros(shape, np.int64)
    for b, box in enumerate(np.asarray(boxes)):
        lo = [int(round(float(v))) for v in box[:3]]
        hi = [int(round(float(v))) for v in box[3:6]]
        ext = [max(h - l, 0) for l, h in zip(lo, hi)]
        if min(ext) == 0:
            continue
        m = np.asarray(masks[b])[:ext[0], :ext[1], :ext[2]] != 0
        region = vol[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
        free = m & (region == 0)
        region[free] = 1 if classes is None else np.int64(classes[b])
    return vol
