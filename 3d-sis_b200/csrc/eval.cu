// eval.cu -- voxel overlaps of predicted and ground-truth instance masks for the mask mAP of test mode.
//
// The reference expands every predicted and every GT mask into a full-scene uint8 volume and runs two full-volume passes per
// (prediction, GT) pair (lib/utils/evaluation.py:144-179, 293-307).  Only three integer counts per pair matter: the nonzero
// voxels of each mask and of their intersection (the union follows as |a| + |b| - |a & b|).  Here every mask stays packed at
// its box, and one launch counts them: one CTA per mask for its own count, one CTA per listed (prediction, GT) pair for the
// intersection, visiting only the intersection of the two boxes.  Counts are exact.
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
