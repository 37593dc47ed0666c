// eval.cu -- voxel overlaps of predicted and ground-truth instance masks for the mask mAP of test mode.
//
// The reference expands every predicted and every GT mask into a full-scene uint8 volume and runs two full-volume passes per
// (prediction, GT) pair (lib/utils/evaluation.py:144-179, 293-307).  Only three integer counts per pair matter: the nonzero
// voxels of each mask and of their intersection (the union follows as |a| + |b| - |a & b|).  Here every mask stays packed at
// its box, and one launch counts them: one CTA per mask for its own count, one CTA per listed (prediction, GT) pair for the
// intersection, visiting only the intersection of the two boxes.  Counts are exact.
//
// The ScanNet benchmark's vertex transfer (sis3d_instance_paint, sis3d_vertex_instance_overlap) follows below the overlap
// kernel: the reference paints every kept mask into a 400x200x400 float64 canvas, looks each mesh vertex up in it, writes one
// 0/1 text line per (instance, vertex) and parses them back to count overlaps with the GT ids.  Here an int32 owner volume
// covers only the boxes' extent, and one pass over the vertices counts vertices per (box, GT id).  The GT ids themselves can
// come from ScanNet's segment annotations (sis3d_segment_gt_slots, at the end): a per-segment table replaces the reference's
// per-vertex GT text files.
#include <climits>
#include "common.cuh"

namespace sis3d {

constexpr int kOverlapThreads = 256;

// voxel (x, y, z) of a mask packed C order [w][h][l] at box lo
__device__ __forceinline__ int64_t packed_index(const int32_t *box, int x, int y, int z) {
    const int h = box[4] - box[1], l = box[5] - box[2];
    return ((int64_t)(x - box[0]) * h + (y - box[1])) * l + (z - box[2]);
}

__global__ void __launch_bounds__(kOverlapThreads)
mask_overlap_kernel(const uint8_t *pred_bits, const int64_t *pred_offs, const int32_t *pred_box, int n_pred,
                    const uint8_t *gt_bits, const int64_t *gt_offs, const int32_t *gt_box, int n_gt,
                    const int32_t *pairs, int64_t *pred_count, int64_t *gt_count, int64_t *pair_count) {
    __shared__ int warp_part[kOverlapThreads / 32];
    const int b = blockIdx.x;
    const uint8_t *a, *c = nullptr;
    const int32_t *abox, *cbox = nullptr;
    int64_t *dst;
    if (b < n_pred) {
        a = pred_bits + pred_offs[b], abox = pred_box + 6 * b, dst = pred_count + b;
    } else if (b < n_pred + n_gt) {
        const int j = b - n_pred;
        a = gt_bits + gt_offs[j], abox = gt_box + 6 * j, dst = gt_count + j;
    } else {
        const int p = b - n_pred - n_gt, i = pairs[2 * p], j = pairs[2 * p + 1];
        dst = pair_count + p;
        if (i < 0 || i >= n_pred || j < 0 || j >= n_gt) {  // a malformed pair list reads nothing and is reported as -1
            if (threadIdx.x == 0) *dst = -1;
            return;
        }
        a = pred_bits + pred_offs[i], abox = pred_box + 6 * i;
        c = gt_bits + gt_offs[j], cbox = gt_box + 6 * j;
    }
    int lo[3], ext[3];
    for (int k = 0; k < 3; ++k) {
        lo[k] = c ? max(abox[k], cbox[k]) : abox[k];
        ext[k] = max((c ? min(abox[k + 3], cbox[k + 3]) : abox[k + 3]) - lo[k], 0);
    }
    const int64_t n = (int64_t)ext[0] * ext[1] * ext[2];
    int cnt = 0;
    for (int64_t v = threadIdx.x; v < n; v += kOverlapThreads) {  // z fastest: consecutive threads read consecutive bytes
        const int64_t r = v / ext[2];
        const int z = lo[2] + (int)(v - r * ext[2]);
        const int xr = (int)(r / ext[1]);
        const int x = lo[0] + xr, y = lo[1] + (int)(r - (int64_t)xr * ext[1]);
        cnt += a[packed_index(abox, x, y, z)] != 0 && (!c || c[packed_index(cbox, x, y, z)] != 0);
    }
    cnt = warp_sum(cnt);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t total = 0;
        for (int w = 0; w < kOverlapThreads / 32; ++w) total += warp_part[w];
        *dst = total;
    }
}

// ---------------------------------------------------------------------------------------------------------- vertex transfer
constexpr int kPaintThreads = 256;
constexpr int kPaintTile = 256;  // boxes staged in shared memory per pass
constexpr int kVertexThreads = 256;

// One thread per voxel of the owner volume: the first box (in index order) whose mask covers the voxel.  Boxes are staged
// in tiles; a CTA stops as soon as all its voxels are owned.
__global__ void __launch_bounds__(kPaintThreads)
instance_paint_kernel(const uint8_t *bits, const int64_t *offs, const int32_t *box, int n_box, int x0, int y0, int z0, int X,
                      int Y, int Z, int32_t *owner) {
    __shared__ int32_t sbox[kPaintTile * 6];
    __shared__ int64_t soff[kPaintTile];
    const int64_t n = (int64_t)X * Y * Z;
    const int64_t v = (int64_t)blockIdx.x * kPaintThreads + threadIdx.x;
    const bool live = v < n;
    int x = 0, y = 0, z = 0;
    if (live) {
        const int64_t r = v / Z;
        z = z0 + (int)(v - r * Z);
        y = y0 + (int)(r % Y);
        x = x0 + (int)(r / Y);
    }
    int found = -1;
    for (int t0 = 0; t0 < n_box; t0 += kPaintTile) {
        const int m = min(kPaintTile, n_box - t0);
        if ((int)threadIdx.x < m) {
            for (int k = 0; k < 6; ++k) sbox[threadIdx.x * 6 + k] = box[6 * (int64_t)(t0 + threadIdx.x) + k];
            soff[threadIdx.x] = offs[t0 + threadIdx.x];
        }
        __syncthreads();
        if (live && found < 0) {
            for (int i = 0; i < m; ++i) {
                const int32_t *b = sbox + 6 * i;
                if (x < b[0] || x >= b[3] || y < b[1] || y >= b[4] || z < b[2] || z >= b[5]) continue;
                const int64_t at = ((int64_t)(x - b[0]) * (b[4] - b[1]) + (y - b[1])) * (b[5] - b[2]) + (z - b[2]);
                if (bits[soff[i] + at] != 0) {
                    found = t0 + i;
                    break;
                }
            }
        }
        // also the barrier before the next tile overwrites the staged boxes
        if (__syncthreads_count(live && found < 0) == 0) break;
    }
    if (live) owner[v] = found;
}

__global__ void vertex_overlap_init_kernel(int64_t *hist, int64_t n_hist, int32_t *first_vertex, int n_box) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_hist || i < n_box; i += stride) {
        if (i < n_hist) hist[i] = 0;
        if (i < n_box) first_vertex[i] = INT_MAX;
    }
}

// row r of world2grid . [x, y, z, 1] in a fixed order, each product and sum rounded on its own (no FMA contraction)
__device__ __forceinline__ double grid_row(const double *w, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(w[0], x), __dmul_rn(w[1], y)), __dmul_rn(w[2], z)), w[3]);
}

__global__ void __launch_bounds__(kVertexThreads)
vertex_overlap_kernel(const float *verts, int n_vert, const double *w2g, const int32_t *owner, int x0, int y0, int z0, int X,
                      int Y, int Z, int cx, int cy, int cz, const int32_t *gt_slot, int n_slot, int n_box, int64_t *hist,
                      int32_t *first_vertex, int32_t *vertex_box) {
    const int v = blockIdx.x * kVertexThreads + threadIdx.x;
    if (v >= n_vert) return;
    const double px = verts[3 * (int64_t)v], py = verts[3 * (int64_t)v + 1], pz = verts[3 * (int64_t)v + 2];
    const double gx = rint(grid_row(w2g, px, py, pz)), gy = rint(grid_row(w2g + 4, px, py, pz)),
                 gz = rint(grid_row(w2g + 8, px, py, pz));
    int b = -1;
    // the whole 3x3x3 neighbourhood lies on the canvas (nan fails every comparison)
    if (gx >= 1 && gx <= cx - 2 && gy >= 1 && gy <= cy - 2 && gz >= 1 && gz <= cz - 2) {
        const int ix = (int)gx - x0, iy = (int)gy - y0, iz = (int)gz - z0;
        auto at = [&](int dx, int dy, int dz) -> int {
            const int x = ix + dx, y = iy + dy, z = iz + dz;
            if (x < 0 || x >= X || y < 0 || y >= Y || z < 0 || z >= Z) return -1;
            return owner[((int64_t)x * Y + y) * Z + z];
        };
        b = at(0, 0, 0);
        for (int d = 0; b < 0 && d < 27; ++d) b = at(d / 9 - 1, (d / 3) % 3 - 1, d % 3 - 1);
        if (b >= n_box) b = -1;
    }
    if (vertex_box) vertex_box[v] = b;
    if (b < 0) return;
    const int s = gt_slot[v];
    if (s >= 0 && s < n_slot) atomicAdd((unsigned long long *)(hist + (int64_t)b * n_slot + s), 1ull);
    atomicMin(first_vertex + b, v);
}

// ------------------------------------------------------------------------------------------------------- GT from segments
// ScanNet's annotations label segments, not vertices: the host resolves export_train_mesh_for_evaluation.py's rules once per
// segment into a table sorted by segment id, and each vertex finds its segment's row by binary search.  Slot counts go
// through a per-CTA shared histogram (most vertices fall into a few slots, 0 above all), flushed once per CTA.
constexpr int kSlotThreads = 256;
constexpr int kSlotShared = 1024;  // slots counted in shared memory; higher slots go straight to global atomics

__global__ void segment_slot_init_kernel(int64_t *slot_count, int n_slot) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slot; i += stride) slot_count[i] = 0;
}

__global__ void __launch_bounds__(kSlotThreads)
segment_gt_slot_kernel(const int32_t *seg_index, int n_vert, const int32_t *seg_ids, const int32_t *seg_slot, int n_seg,
                       int n_slot, int32_t *gt_slot, int64_t *slot_count) {
    __shared__ int s_count[kSlotShared];
    const int n_shared = min(n_slot, kSlotShared);
    for (int i = threadIdx.x; i < n_shared; i += kSlotThreads) s_count[i] = 0;
    __syncthreads();
    for (int v = blockIdx.x * kSlotThreads + threadIdx.x; v < n_vert; v += gridDim.x * kSlotThreads) {
        const int32_t seg = seg_index[v];
        int slot = 0;
        if (seg >= 0) {
            int lo = 0, hi = n_seg;  // first row with seg_ids[row] >= seg
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (seg_ids[mid] < seg) lo = mid + 1;
                else hi = mid;
            }
            if (lo < n_seg && seg_ids[lo] == seg) slot = seg_slot[lo];
        }
        gt_slot[v] = slot;
        if (slot >= 0 && slot < n_shared) atomicAdd(s_count + slot, 1);
        else if (slot >= 0 && slot < n_slot) atomicAdd((unsigned long long *)(slot_count + slot), 1ull);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_shared; i += kSlotThreads)
        if (s_count[i]) atomicAdd((unsigned long long *)(slot_count + i), (unsigned long long)s_count[i]);
}

}  // namespace sis3d
using namespace sis3d;

extern "C" int sis3d_mask_overlap(const uint8_t *pred_bits, const int64_t *pred_offs, const int32_t *pred_box, int n_pred,
                                  const uint8_t *gt_bits, const int64_t *gt_offs, const int32_t *gt_box, int n_gt,
                                  const int32_t *pairs, int n_pairs, int64_t *pred_count, int64_t *gt_count,
                                  int64_t *pair_count, void *stream) {
    if (n_pred < 0 || n_gt < 0 || n_pairs < 0) return SIS3D_EINVAL;
    if (n_pred > 0 && (!pred_bits || !pred_offs || !pred_box || !pred_count)) return SIS3D_EINVAL;
    if (n_gt > 0 && (!gt_bits || !gt_offs || !gt_box || !gt_count)) return SIS3D_EINVAL;
    if (n_pairs > 0 && (!pairs || !pair_count || n_pred == 0 || n_gt == 0)) return SIS3D_EINVAL;
    const int64_t blocks = (int64_t)n_pred + n_gt + n_pairs;
    if (blocks == 0) return SIS3D_OK;
    if (blocks > 0x7fffffff) return SIS3D_EUNSUPPORTED;
    mask_overlap_kernel<<<(unsigned)blocks, kOverlapThreads, 0, (cudaStream_t)stream>>>(
        pred_bits, pred_offs, pred_box, n_pred, gt_bits, gt_offs, gt_box, n_gt, pairs, pred_count, gt_count, pair_count);
    return finish_launch();
}

extern "C" int sis3d_instance_paint(const uint8_t *bits, const int64_t *offs, const int32_t *box, int n_box, int x0, int y0,
                                    int z0, int X, int Y, int Z, int32_t *owner, void *stream) {
    if (n_box < 0 || X < 0 || Y < 0 || Z < 0) return SIS3D_EINVAL;
    if (n_box > 0 && (!bits || !offs || !box)) return SIS3D_EINVAL;
    const int64_t n = (int64_t)X * Y * Z;
    if (n == 0) return SIS3D_OK;
    if (!owner) return SIS3D_EINVAL;
    const int64_t blocks = cdiv64(n, kPaintThreads);
    if (blocks > 0x7fffffff) return SIS3D_EUNSUPPORTED;
    instance_paint_kernel<<<(unsigned)blocks, kPaintThreads, 0, (cudaStream_t)stream>>>(bits, offs, box, n_box, x0, y0, z0, X,
                                                                                         Y, Z, owner);
    return finish_launch();
}

extern "C" int sis3d_vertex_instance_overlap(const float *verts, int n_vert, const double *world2grid, const int32_t *owner,
                                             int x0, int y0, int z0, int X, int Y, int Z, int canvas_x, int canvas_y,
                                             int canvas_z, const int32_t *gt_slot, int n_slot, int n_box, int64_t *hist,
                                             int32_t *first_vertex, int32_t *vertex_box, void *stream) {
    if (n_vert < 0 || n_slot < 0 || n_box < 0 || X < 0 || Y < 0 || Z < 0 || canvas_x < 0 || canvas_y < 0 || canvas_z < 0)
        return SIS3D_EINVAL;
    if (n_vert > 0 && (!verts || !world2grid || !gt_slot)) return SIS3D_EINVAL;
    if ((int64_t)X * Y * Z > 0 && !owner) return SIS3D_EINVAL;
    if (n_box > 0 && (!first_vertex || (n_slot > 0 && !hist))) return SIS3D_EINVAL;
    const int64_t n_hist = (int64_t)n_box * n_slot;
    cudaStream_t s = (cudaStream_t)stream;
    int launches = 0;
    if (n_box > 0) {
        const int64_t work = n_hist > n_box ? n_hist : n_box;
        const int blocks = (int)imin64(cdiv64(work, 256), 4 * kNumSMs);
        vertex_overlap_init_kernel<<<blocks, 256, 0, s>>>(hist, n_hist, first_vertex, n_box);
        ++launches;
    }
    if (n_vert > 0) {
        vertex_overlap_kernel<<<cdiv(n_vert, kVertexThreads), kVertexThreads, 0, s>>>(
            verts, n_vert, world2grid, owner, x0, y0, z0, X, Y, Z, canvas_x, canvas_y, canvas_z, gt_slot, n_slot, n_box, hist,
            first_vertex, vertex_box);
        ++launches;
    }
    return launches ? finish_launch(launches) : SIS3D_OK;
}

extern "C" int sis3d_segment_gt_slots(const int32_t *seg_index, int n_vert, const int32_t *seg_ids, const int32_t *seg_slot,
                                      int n_seg, int n_slot, int32_t *gt_slot, int64_t *slot_count, void *stream) {
    if (n_vert < 0 || n_seg < 0 || n_slot < 0) return SIS3D_EINVAL;
    if (n_vert > 0 && (!seg_index || !gt_slot)) return SIS3D_EINVAL;
    if (n_seg > 0 && (!seg_ids || !seg_slot)) return SIS3D_EINVAL;
    if (n_slot > 0 && !slot_count) return SIS3D_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    int launches = 0;
    if (n_slot > 0) {
        segment_slot_init_kernel<<<(int)imin64(cdiv64(n_slot, 256), 4 * kNumSMs), 256, 0, s>>>(slot_count, n_slot);
        ++launches;
    }
    if (n_vert > 0) {
        segment_gt_slot_kernel<<<(int)imin64(cdiv64(n_vert, kSlotThreads), 4 * kNumSMs), kSlotThreads, 0, s>>>(
            seg_index, n_vert, seg_ids, seg_slot, n_seg, n_slot, gt_slot, slot_count);
        ++launches;
    }
    return launches ? finish_launch(launches) : SIS3D_OK;
}
