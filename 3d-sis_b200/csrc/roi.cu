// roi.cu -- 3D RoI max pooling (forward) and the detection decode feeding the mask branch.
//
//   roi_pool_ncdhw_kernel  drop-in for ROIPoolForward (lib/layer_utils/roi_pooling/src/cuda/
//                          roi_pooling_kernel.cu:15-109) on the reference's NCDHW features
//   roi_pool_vc_kernel     same arithmetic on VC features, one CTA per RoI, channel-coalesced reads,
//                          picks the pyramid level per RoI (lib/nets/network.py:503-534)
//   detect_decode_kernel   lib/nets/network.py:285-301 / lib/model/trainval.py:825-858
#include <float.h>
#include "common.cuh"

namespace sis3d {

struct RoiBins {
    int sw, sh, sl;
    float bw, bh, bl;
};
__device__ __forceinline__ RoiBins roi_bins(const float *roi, float scale, int pw, int ph, int pl) {
    RoiBins b;
    b.sw = (int)floorf(__fmul_rn(roi[0], scale));
    b.sh = (int)floorf(__fmul_rn(roi[1], scale));
    b.sl = (int)floorf(__fmul_rn(roi[2], scale));
    const int ew = (int)ceilf(__fmul_rn(roi[3], scale)), eh = (int)ceilf(__fmul_rn(roi[4], scale));
    const int el = (int)ceilf(__fmul_rn(roi[5], scale));
    const int rw = max(ew - b.sw, 1), rh = max(eh - b.sh, 1), rl = max(el - b.sl, 1);  // malformed RoIs -> 1x1x1
    b.bw = __fdiv_rn((float)rw, (float)pw);
    b.bh = __fdiv_rn((float)rh, (float)ph);
    b.bl = __fdiv_rn((float)rl, (float)pl);
    return b;
}
__device__ __forceinline__ void bin_range(int p, float bin, int start, int dim, int &lo, int &hi) {
    lo = (int)floorf(__fmul_rn((float)p, bin));
    hi = (int)ceilf(__fmul_rn((float)(p + 1), bin));
    lo = min(max(lo + start, 0), dim);
    hi = min(max(hi + start, 0), dim);
}

__global__ void __launch_bounds__(256) roi_pool_ncdhw_kernel(int nthreads, const float *feat, float scale, int W, int H, int L,
                                                             int C, int pw_, int ph_, int pl_, const float *rois, float *top,
                                                             int *argmax) {
    for (int index = blockIdx.x * blockDim.x + threadIdx.x; index < nthreads; index += blockDim.x * gridDim.x) {
        int n = index;
        const int pl = n % pl_; n /= pl_;
        const int ph = n % ph_; n /= ph_;
        const int pw = n % pw_; n /= pw_;
        const int c = n % C; n /= C;
        const RoiBins b = roi_bins(rois + n * 6, scale, pw_, ph_, pl_);
        int ws, we, hs, he, ls, le;
        bin_range(pw, b.bw, b.sw, W, ws, we);
        bin_range(ph, b.bh, b.sh, H, hs, he);
        bin_range(pl, b.bl, b.sl, L, ls, le);
        const bool empty = (he <= hs) || (we <= ws) || (le <= ls);
        float best = empty ? 0.f : -FLT_MAX;
        int besti = -1;
        for (int w = ws; w < we; ++w)
            for (int h = hs; h < he; ++h)
                for (int l = ls; l < le; ++l) {
                    const int idx = (c * W + w) * H * L + h * L + l;
                    const float v = __ldg(feat + idx);
                    if (v > best) { best = v; besti = idx; }
                }
        top[index] = best;
        if (argmax) argmax[index] = besti;
    }
}

// grid = (RoIs, pw*ph); block = 128 threads (channels).  Each CTA pools the pl bins of one (pw, ph) column, so a
// large RoI is spread over pw*ph CTAs instead of serialising 64 bins in one.
__global__ void __launch_bounds__(128) roi_pool_vc_kernel(const float *feat1, const float *feat2, const float *feat3,
                                                          const int32_t *level_ids, float scale, int W, int H, int L, int C,
                                                          int pw_, int ph_, int pl_, const float *rois, float *top, int *argmax) {
    const int r = blockIdx.x;
    const int pw = blockIdx.y / ph_, ph = blockIdx.y % ph_;
    const int nb = pw_ * ph_ * pl_;
    const int lvl = level_ids ? level_ids[r] : 1;
    const float *feat = lvl == 1 ? feat1 : (lvl == 2 ? feat2 : (lvl == 3 ? feat3 : nullptr));
    const RoiBins b = roi_bins(rois + r * 6, scale, pw_, ph_, pl_);
    int ws, we, hs, he;
    bin_range(pw, b.bw, b.sw, W, ws, we);
    bin_range(ph, b.bh, b.sh, H, hs, he);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        for (int pl = 0; pl < pl_; ++pl) {
            int ls, le;
            bin_range(pl, b.bl, b.sl, L, ls, le);
            const bool empty = (he <= hs) || (we <= ws) || (le <= ls) || !feat;
            float best = empty ? 0.f : -FLT_MAX;
            int besti = -1;
            if (!empty)
                for (int w = ws; w < we; ++w)
                    for (int h = hs; h < he; ++h) {
                        const float *row = feat + ((int64_t)(w * H + h) * L) * C + c;
                        for (int l = ls; l < le; ++l) {
                            const float v = __ldg(row + (int64_t)l * C);
                            if (v > best) { best = v; besti = (c * W + w) * H * L + h * L + l; }
                        }
                    }
            const int64_t o = ((int64_t)r * C + c) * nb + (pw * ph_ + ph) * pl_ + pl;
            top[o] = best;
            if (argmax) argmax[o] = besti;
        }
    }
}

// Tail of the RoI classifier (lib/nets/backbones.py:225-231 layers 2,4 + lib/nets/network.py:55-57 heads) in one
// launch: 4 RoI rows per CTA, activations stay in shared memory.  Each layer streams its packed weights ([K][ldw]) through
// shared memory in 32-row slabs loaded cooperatively (8 independent float4 loads per thread in flight, next slab
// prefetched into registers while the current one is multiplied) -- a thread-per-output loop over global memory is
// latency-bound (measured 55 us).
constexpr int kMlpRows = 4;
constexpr int kMlpSlab = 32;
__device__ __forceinline__ void mlp_layer(const float (*xin)[256], int K, const float *w, int N, float *slab /*[32][256]*/,
                                          float *acc /*[kMlpRows]*/) {
    const int t = threadIdx.x;
    const int ld = (N + 3) & ~3, ld4 = ld >> 2;
    const int per_slab = kMlpSlab * ld4;            // float4 per slab
    float4 pre[8];
#pragma unroll
    for (int r = 0; r < kMlpRows; ++r) acc[r] = 0.f;
    auto fetch = [&](int k0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = t + j * 256;
            pre[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < per_slab && k0 + i / ld4 < K) pre[j] = __ldg(reinterpret_cast<const float4 *>(w + (int64_t)k0 * ld) + i);
        }
    };
    fetch(0);
    for (int k0 = 0; k0 < K; k0 += kMlpSlab) {
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int i = t + j * 256;
            if (i < per_slab) reinterpret_cast<float4 *>(slab)[i] = pre[j];
        }
        __syncthreads();
        if (k0 + kMlpSlab < K) fetch(k0 + kMlpSlab);
        if (t < N) {
            const int kn = min(kMlpSlab, K - k0);
            for (int k = 0; k < kn; ++k) {
                const float wv = slab[k * ld + t];
#pragma unroll
                for (int r = 0; r < kMlpRows; ++r) acc[r] = fmaf(xin[r][k0 + k], wv, acc[r]);
            }
        }
    }
}

__global__ void __launch_bounds__(256) mlp_tail_kernel(const float *x1, int R, int d1, const float *w2, const float *b2, int d2,
                                                       const float *w3, const float *b3, int d3, const float *wc,
                                                       const float *bc, int nc, const float *wb, const float *bb, int nb,
                                                       float *cls_score, float *bbox_pred) {
    __shared__ float sa[kMlpRows][256];
    __shared__ float sb[kMlpRows][256];
    __shared__ __align__(16) float slab[kMlpSlab * 256];
    const int r0 = blockIdx.x * kMlpRows, t = threadIdx.x;
    for (int i = t; i < kMlpRows * d1; i += 256) {
        const int r = i / d1, k = i - r * d1;
        sa[r][k] = (r0 + r < R) ? x1[(int64_t)(r0 + r) * d1 + k] : 0.f;
    }
    float acc[kMlpRows];
    mlp_layer(sa, d1, w2, d2, slab, acc);  // starts with a __syncthreads(): sa is complete
    if (t < d2)
#pragma unroll
        for (int r = 0; r < kMlpRows; ++r) sb[r][t] = fmaxf(acc[r] + b2[t], 0.f);
    mlp_layer(sb, d2, w3, d3, slab, acc);
    if (t < d3)
#pragma unroll
        for (int r = 0; r < kMlpRows; ++r) sa[r][t] = fmaxf(acc[r] + b3[t], 0.f);
    mlp_layer(sa, d3, wc, nc, slab, acc);
    if (t < nc)
#pragma unroll
        for (int r = 0; r < kMlpRows; ++r)
            if (r0 + r < R) cls_score[(int64_t)(r0 + r) * nc + t] = acc[r] + bc[t];
    mlp_layer(sa, d3, wb, nb, slab, acc);
    if (t < nb)
#pragma unroll
        for (int r = 0; r < kMlpRows; ++r)
            if (r0 + r < R) bbox_pred[(int64_t)(r0 + r) * nb + t] = acc[r] + bb[t];
}

// Predicted-class channel of every kept RoI's mask, packed back to back (what the driver saves:
// lib/model/trainval.py:900-908).  masks [total][ncls] (crop j occupies rows offs[j]..offs[j+1]); out float [total],
// bits uint8 [total] = (value >= thresh).
__global__ void mask_select_kernel(const float *masks, const int64_t *offs, const int32_t *cls, int n_crops, int ncls,
                                   float thresh, float *out, uint8_t *bits) {
    const int64_t total = offs[n_crops];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = n_crops - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (offs[mid] <= i) lo = mid; else hi = mid - 1;
        }
        const float v = masks[i * ncls + cls[lo]];
        if (out) out[i] = v;
        if (bits) bits[i] = v >= thresh ? 1 : 0;
    }
}

// one thread per RoI row
__global__ void detect_decode_kernel(const float *rois, const int32_t *num_rois, int max_rois, const float *cls_score,
                                     const float *bbox_pred, int nc, int sx, int sy, int sz, float thresh, float *cls_prob,
                                     int64_t *cls_pred, float *det) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= max_rois) return;
    const int n = min(*num_rois, max_rois);
    float *d = det + i * 16;
    const float tag = i == 0 ? (float)n : 0.f;  // row 0, column 15 carries the RoI count (one D2H for count + table)
    if (i >= n) {
        for (int k = 0; k < 15; ++k) d[k] = 0.f;
        d[15] = tag;
        cls_pred[i] = 0;
        for (int k = 0; k < nc; ++k) cls_prob[i * nc + k] = 0.f;
        return;
    }
    const float *s = cls_score + i * nc;
    int best = 0;
    float m = s[0];
    for (int k = 1; k < nc; ++k)
        if (s[k] > m) { m = s[k]; best = k; }  // first maximum (torch.max on CPU)
    float sum = 0.f;
    for (int k = 0; k < nc; ++k) sum += expf(s[k] - m);
    for (int k = 0; k < nc; ++k) cls_prob[i * nc + k] = __fdiv_rn(expf(s[k] - m), sum);
    const float conf = cls_prob[i * nc + best];
    cls_pred[i] = best;
    const float *dl = bbox_pred + (int64_t)i * nc * 6 + best * 6;
    const float dims[3] = {(float)sx, (float)sy, (float)sz};
    float box[6];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float lo = rois[i * 6 + k], hi = rois[i * 6 + 3 + k];
        const float w = __fsub_rn(hi, lo);
        const float ctr = __fadd_rn(lo, __fmul_rn(0.5f, w));
        const float pc = __fadd_rn(__fmul_rn(dl[k], w), ctr);
        const float pw = __fmul_rn(expf(dl[3 + k]), w);
        const float hw = __fmul_rn(0.5f, pw);
        box[k] = fminf(fmaxf(__fsub_rn(pc, hw), 0.f), dims[k]);
        box[3 + k] = fminf(fmaxf(__fadd_rn(pc, hw), 0.f), dims[k]);
    }
    bool keep = conf > thresh;
    float crop[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) crop[k] = rintf(box[k]);  // Python-3 round(): half to even
    if (crop[0] >= crop[3] || crop[1] >= crop[4] || crop[2] >= crop[5]) keep = false;
    for (int k = 0; k < 6; ++k) d[k] = box[k];
    d[6] = conf; d[7] = (float)best; d[8] = keep ? 1.f : 0.f;
    for (int k = 0; k < 6; ++k) d[9 + k] = crop[k];
    d[15] = tag;
}

}  // namespace sis3d
using namespace sis3d;

extern "C" int sis3d_roi_pool_fwd(const float *feat, int feat_layout, float spatial_scale, int num_rois, int width,
                                  int height, int length, int channels, int pw, int ph, int pl, const float *rois,
                                  float *top, int32_t *argmax, void *stream) {
    if (!feat || !rois || !top || num_rois < 0 || pw <= 0 || ph <= 0 || pl <= 0 || channels <= 0) return SIS3D_EINVAL;
    if (feat_layout != 0 && (int64_t)pw * ph > 65535) return SIS3D_EUNSUPPORTED;  // gridDim.y of the VC kernel
    if (num_rois == 0) return SIS3D_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (feat_layout == 0) {
        const int total = num_rois * channels * pw * ph * pl;
        roi_pool_ncdhw_kernel<<<min(cdiv(total, 256), kNumSMs * 8), 256, 0, s>>>(total, feat, spatial_scale, width, height,
                                                                                length, channels, pw, ph, pl, rois, top,
                                                                                argmax);
    } else {
        roi_pool_vc_kernel<<<dim3(num_rois, pw * ph), 128, 0, s>>>(feat, nullptr, nullptr, nullptr, spatial_scale, width, height,
                                                                  length, channels, pw, ph, pl, rois, top, argmax);
    }
    return finish_launch();
}

extern "C" int sis3d_roi_pool_levels(const float *feat1, const float *feat2, const float *feat3, const int32_t *level_ids,
                                     float spatial_scale, int num_rois, int width, int height, int length, int channels,
                                     int pw, int ph, int pl, const float *rois, float *top, int32_t *argmax, void *stream) {
    if (!feat1 || !level_ids || !rois || !top || num_rois <= 0 || channels <= 0 || pw <= 0 || ph <= 0 || pl <= 0)
        return SIS3D_EINVAL;
    if ((int64_t)pw * ph > 65535) return SIS3D_EUNSUPPORTED;  // gridDim.y
    roi_pool_vc_kernel<<<dim3(num_rois, pw * ph), 128, 0, (cudaStream_t)stream>>>(feat1, feat2, feat3, level_ids, spatial_scale,
                                                                                 width, height, length, channels, pw, ph, pl,
                                                                                 rois, top, argmax);
    return finish_launch();
}

extern "C" int sis3d_detect_decode(const float *rois, const int32_t *num_rois, int max_rois, const float *cls_score,
                                   const float *bbox_pred, int num_classes, int scene_x, int scene_y, int scene_z,
                                   float class_thresh, float *cls_prob, int64_t *cls_pred, float *det, void *stream) {
    if (!rois || !num_rois || !cls_score || !bbox_pred || !cls_prob || !cls_pred || !det || max_rois <= 0 || num_classes <= 0)
        return SIS3D_EINVAL;
    detect_decode_kernel<<<cdiv(max_rois, 128), 128, 0, (cudaStream_t)stream>>>(rois, num_rois, max_rois, cls_score, bbox_pred,
                                                                              num_classes, scene_x, scene_y, scene_z,
                                                                              class_thresh, cls_prob, cls_pred, det);
    return finish_launch();
}

extern "C" int sis3d_mlp_tail(const float *x1, int R, int d1, const float *w2, const float *b2, int d2, const float *w3,
                              const float *b3, int d3, const float *wc, const float *bc, int nc, const float *wb,
                              const float *bb, int nb, float *cls_score, float *bbox_pred, void *stream) {
    if (!x1 || !w2 || !b2 || !w3 || !b3 || !wc || !bc || !wb || !bb || !cls_score || !bbox_pred || R <= 0) return SIS3D_EINVAL;
    if (d1 > 256 || d2 > 256 || d3 > 256 || d1 <= 0 || d2 <= 0 || d3 <= 0 || nc <= 0 || nb <= 0 || nc > 256 || nb > 256)
        return SIS3D_EUNSUPPORTED;
    mlp_tail_kernel<<<cdiv(R, kMlpRows), 256, 0, (cudaStream_t)stream>>>(x1, R, d1, w2, b2, d2, w3, b3, d3, wc, bc, nc, wb, bb, nb,
                                                                        cls_score, bbox_pred);
    return finish_launch();
}

extern "C" int sis3d_mask_select(const float *masks, const int64_t *offs, const int32_t *cls, int n_crops, int ncls,
                                 int64_t total_hint, float thresh, float *out, uint8_t *bits, void *stream) {
    if (!masks || !offs || !cls || n_crops <= 0 || ncls <= 0 || (!out && !bits)) return SIS3D_EINVAL;
    const int blocks = (int)imin64(cdiv64(total_hint > 0 ? total_hint : 1, 256), kNumSMs * 8);
    mask_select_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(masks, offs, cls, n_crops, ncls, thresh, out, bits);
    return finish_launch();
}
