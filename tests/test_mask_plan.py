"""CPU: the native host planner of the ragged mask stage (sis3d_mask_plan_build) -- crop packing on the canvas, brick
list coverage, region tables and offsets, checked against a direct numpy restatement of network.py:283-317's crops."""
import ctypes as C

import numpy as np
import pytest

from lib import _sis3d as S


def _plan(det, dims, ncls, use_canvas, cap=1 << 20, grow=False):
    """Run the planner; grow=True retries with the size it reports on SIS3D_EWORKSPACE (as Network._mask_branch does)."""
    while True:
        blob = np.zeros(cap, dtype=np.uint8)
        plan = S.MaskPlan()
        rc = S.lib.sis3d_mask_plan_build(C.c_void_p(det.ctypes.data), det.shape[0], *dims, ncls, use_canvas,
                                         C.c_void_p(blob.ctypes.data), C.c_size_t(cap), C.byref(plan))
        if rc == -3 and grow and plan.bytes > cap:
            cap = int(plan.bytes)
            continue
        return rc, plan, blob


def _dets(rng, n, dims):
    det = np.zeros((n, 16), dtype=np.float32)
    for i in range(n):
        lo = [int(rng.integers(0, d - 1)) for d in dims]
        hi = [int(rng.integers(l + 1, d + 1)) for l, d in zip(lo, dims)]
        det[i, 9:12], det[i, 12:15] = lo, hi
        det[i, 7] = rng.integers(0, 19)
        det[i, 8] = float(rng.random() < 0.6)  # keep flag
    return det


def _edge_dets(rng, dims):
    """Kept crops at the edges of the brick layout: extent 1 on each axis, 1x1x1, whole 4x4x8 bricks (w, h = 0 mod 4,
    l = 0 mod 8) and one voxel past them, at random positions."""
    sizes = [(1, 5, 9), (6, 1, 9), (6, 5, 1), (1, 1, 1), (4, 8, 8), (8, 4, 16), (5, 9, 17), (4, 4, 8), (1, 4, 8)]
    det = np.zeros((len(sizes), 16), dtype=np.float32)
    for i, sz in enumerate(sizes):
        lo = [int(rng.integers(0, d - s + 1)) for d, s in zip(dims, sz)]
        det[i, 9:12], det[i, 12:15] = lo, [l + s for l, s in zip(lo, sz)]
        det[i, 7], det[i, 8] = rng.integers(0, 19), 1.0
    return det


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("use_canvas", [0, 1])
def test_mask_plan_tables(seed, use_canvas):
    rng = np.random.default_rng(seed)
    dims, ncls = (45, 27, 41), 19
    det = _dets(rng, int(rng.integers(1, 40)), dims)
    edges = _edge_dets(rng, dims)
    at = int(rng.integers(0, det.shape[0] + 1))  # the edge crops sit at a random place among the others
    _check_plan(np.ascontiguousarray(np.concatenate([det[:at], edges, det[at:]])), dims, ncls, use_canvas)


def test_mask_plan_5000_kept_rows():
    """More kept rows than the planner's former fixed list of 4096: every kept row gets its crop, offsets, size and bricks."""
    rng = np.random.default_rng(11)
    dims, n = (48, 24, 40), 5000
    det = np.zeros((n + 300, 16), dtype=np.float32)
    sz = rng.integers(1, 7, (n + 300, 3))
    lo = np.stack([rng.integers(0, d - s + 1) for d, s in zip(dims, sz.T)], 1)
    det[:, 9:12], det[:, 12:15] = lo, lo + sz
    det[:, 7] = rng.integers(0, 19, n + 300)
    det[rng.permutation(n + 300)[:n], 8] = 1.0   # 5000 kept rows among 5300, the last kept one near the end
    assert int((det[:, 8] > 0.5).sum()) == n
    for use_canvas in (0, 1):
        _check_plan(det, dims, 19, use_canvas)


def _check_plan(det, dims, ncls, use_canvas):
    rc, p, blob = _plan(det, dims, ncls, use_canvas, grow=True)
    assert rc == 0
    kept = np.nonzero(det[:, 8] > 0.5)[0]
    assert p.n_kept == len(kept)
    if len(kept) == 0:
        return
    lo, hi = det[kept, 9:12].astype(np.int64), det[kept, 12:15].astype(np.int64)
    sz = hi - lo
    vox = sz.prod(1)
    assert p.total_voxels == vox.sum()
    offs = blob[p.off_offs:p.off_offs + 8 * (len(kept) + 1)].view(np.int64)
    assert np.array_equal(offs, np.concatenate([[0], np.cumsum(vox)]))
    assert np.array_equal(blob[p.off_cls:p.off_cls + 4 * len(kept)].view(np.int32), det[kept, 7].astype(np.int32))
    assert np.array_equal(blob[p.off_kept:p.off_kept + 4 * len(kept)].view(np.int32), kept.astype(np.int32))
    assert np.array_equal(blob[p.off_sizes:p.off_sizes + 12 * len(kept)].view(np.int32).reshape(-1, 3), sz.astype(np.int32))
    first = blob[p.off_first:p.off_first + S.REGION_BYTES * len(kept)].view(S.REGION_DTYPE)
    last = blob[p.off_last:p.off_last + S.REGION_BYTES * len(kept)].view(S.REGION_DTYPE)
    X, Y, Z = dims
    assert np.array_equal(first["in_off"], (lo[:, 0] * Y + lo[:, 1]) * Z + lo[:, 2])       # window into the NCDHW scene
    assert np.array_equal(first["in_dim"], sz) and np.array_equal(first["out_dim"], sz)
    assert np.array_equal(last["out_off"], offs[:-1] * ncls)                               # compact [voxels][ncls] outputs
    tiles64 = (vox + S.TILE_M - 1) // S.TILE_M
    assert np.array_equal(first["tile_begin"], np.concatenate([[0], np.cumsum(tiles64)[:-1]]))
    assert p.tiles_first == p.tiles_last == tiles64.sum()
    if not use_canvas:
        mid = blob[p.off_rest:p.off_rest + S.REGION_BYTES * len(kept)].view(S.REGION_DTYPE)
        assert np.array_equal(mid["in_off"], offs[:-1] * 64) and np.array_equal(mid["out_off"], offs[:-1] * 64)
        return
    # canvas: crops side by side along x with one zero slab between them; y/z extents = the largest crop
    Xc, Yc, Zc = p.canvas
    assert (Xc, Yc, Zc) == ((sz[:, 0] + 1).sum(), sz[:, 1].max(), sz[:, 2].max())
    xoff = np.concatenate([[0], np.cumsum(sz[:, 0] + 1)[:-1]])
    assert np.array_equal(first["out_off"], xoff * Yc * Zc * 64)
    assert np.array_equal(first["out_stride"], np.tile([Yc * Zc * 64, Zc * 64, 64], (len(kept), 1)))
    tiles = blob[p.off_rest:p.off_rest + 32 * p.n_tiles_tc].view(np.int32).reshape(-1, 8)
    cover = np.zeros((Xc, Yc, Zc), dtype=np.int32)
    for x0, y0, z0, x1, y1, z1, _, _ in tiles:  # 4x4x8 bricks clipped to their crop
        assert x0 < x1 and y0 < y1 and z0 < z1
        cover[x0:min(x0 + 4, x1), y0:min(y0 + 4, y1), z0:min(z0 + 8, z1)] += 1
    want = np.zeros_like(cover)
    for j in range(len(kept)):
        want[xoff[j]:xoff[j] + sz[j, 0], :sz[j, 1], :sz[j, 2]] = 1
    assert np.array_equal(cover, want), "every crop voxel is written by exactly one brick, the zero slabs by none"


def test_mask_plan_workspace_and_empty():
    rng = np.random.default_rng(0)
    det = _dets(rng, 12, (32, 32, 32))
    det[:, 8] = 1.0
    rc, p, _ = _plan(det, (32, 32, 32), 19, 1, cap=64)
    assert rc == -3 and p.bytes > 64          # SIS3D_EWORKSPACE reports the size needed
    rc, p2, _ = _plan(det, (32, 32, 32), 19, 1, cap=int(p.bytes))
    assert rc == 0 and p2.bytes == p.bytes
    det[:, 8] = 0.0
    rc, p3, _ = _plan(det, (32, 32, 32), 19, 1)
    assert rc == 0 and p3.n_kept == 0
