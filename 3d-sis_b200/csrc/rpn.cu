// rpn.cu -- 3D NMS and the fused RPN proposal stage ("rpn3d").
//
//   sis3d_nms            == gpu_nms/_nms  (lib/layer_utils/nms/src/nms_cuda.c:10-67, cuda/nms_kernel.cu:11-94)
//                           but with the greedy reduce on the device (no D2H of the bitmask).
//   sis3d_rpn_proposals  == proposal_layer (lib/layer_utils/proposal_layer.py:11-204) incl. softmax
//                           (lib/nets/network.py:546), anchors (generate_anchors.py:58-119), decode/clip
//                           (lib/utils/bbox_transform.py:59-99,4-21), stable descending top-N and NMS.
//
// IoU arithmetic is pinned with explicit intrinsics to the SASS nvcc emits for the reference's
// devIoU (Sa = FMUL,FMUL; t = FFMA(wb*hb, lb, Sa); u = t - inter; IEEE div) -- see DESIGN.md.
#include <stdlib.h>
#include "common.cuh"

namespace sis3d {

__device__ __forceinline__ float box_volume_p1(const float *b) {
    const float w = __fadd_rn(__fsub_rn(b[3], b[0]), 1.f), h = __fadd_rn(__fsub_rn(b[4], b[1]), 1.f);
    const float l = __fadd_rn(__fsub_rn(b[5], b[2]), 1.f);
    return __fmul_rn(__fmul_rn(w, h), l);
}
// a = earlier (higher score, "row") box with precomputed volume Sa; b = candidate ("column") box.
__device__ __forceinline__ float iou3d_ref(const float *a, float Sa, const float *b) {
    const float left = fmaxf(a[0], b[0]), top = fmaxf(a[1], b[1]), front = fmaxf(a[2], b[2]);
    const float right = fminf(a[3], b[3]), bottom = fminf(a[4], b[4]), back = fminf(a[5], b[5]);
    const float w = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.f), 0.f);
    const float h = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.f), 0.f);
    const float l = fmaxf(__fadd_rn(__fsub_rn(back, front), 1.f), 0.f);
    const float inter = __fmul_rn(__fmul_rn(w, h), l);
    const float wb = __fadd_rn(__fsub_rn(b[3], b[0]), 1.f), hb = __fadd_rn(__fsub_rn(b[4], b[1]), 1.f);
    const float lb = __fadd_rn(__fsub_rn(b[5], b[2]), 1.f);
    const float t = __fmaf_rn(__fmul_rn(wb, hb), lb, Sa);
    return __fdiv_rn(inter, __fsub_rn(t, inter));
}

// ---- NMS: suppression bitmask (upper triangle only) ----------------------------------------------
// mask[i][cb] bit j  <=>  IoU(box i, box 64*cb+j) > thresh, for 64*cb+j > i.
__global__ void __launch_bounds__(64) nms_mask_kernel(const float *boxes, int n, float thresh, unsigned long long *mask, int cb_total) {
    const int row_b = blockIdx.y, col_b = blockIdx.x;
    if (col_b < row_b) return;  // never read by the reduce (nms_cuda.c:52 starts at j = nblock)
    __shared__ float cbox[64 * 6];
    const int col_n = min(n - col_b * 64, 64), row_n = min(n - row_b * 64, 64);
    if (threadIdx.x < col_n)
        for (int k = 0; k < 6; ++k) cbox[threadIdx.x * 6 + k] = boxes[(col_b * 64 + threadIdx.x) * 6 + k];
    __syncthreads();
    if (threadIdx.x < row_n) {
        const int i = row_b * 64 + threadIdx.x;
        float a[6];
        for (int k = 0; k < 6; ++k) a[k] = boxes[i * 6 + k];
        const float Sa = box_volume_p1(a);
        unsigned long long bits = 0;
        const int start = (row_b == col_b) ? threadIdx.x + 1 : 0;
        for (int j = start; j < col_n; ++j)
            if (iou3d_ref(a, Sa, cbox + j * 6) > thresh) bits |= 1ULL << j;
        mask[(size_t)i * cb_total + col_b] = bits;
    }
}

// ---- NMS: greedy reduce on the device ------------------------------------------------------------
// One CTA.  For each block of 64 boxes: resolve the in-block chain serially from the diagonal words
// (warp 0), then OR the kept rows' words of all later column blocks in parallel.
// Optional gather epilogue (proposal stage): writes rois/scores/level ids of the first post_top_n kept.
struct NmsGather {
    const float *sorted_boxes;
    const float *sorted_scores;
    const int32_t *sorted_levels;
    float *rois, *scores;
    int32_t *level_ids;
    int post_top_n;
};

__global__ void __launch_bounds__(256) nms_reduce_kernel(const unsigned long long *mask, int n_rows, const int *n_limit,
                                                         int cb_total, int64_t *keep, int32_t *num_out, NmsGather g) {
    const int n = n_limit ? min(n_rows, *n_limit) : n_rows;  // rows >= n are padding and never emitted
    extern __shared__ unsigned long long s_remv[];  // [cb_total]
    __shared__ unsigned long long s_diag[64];
    __shared__ unsigned long long s_kept;
    __shared__ int s_nkept;
    for (int j = threadIdx.x; j < cb_total; j += blockDim.x) s_remv[j] = 0;
    if (threadIdx.x == 0) s_nkept = 0;
    __syncthreads();
    for (int rb = 0; rb < cb_total; ++rb) {
        const int rows = max(0, min(n - rb * 64, 64));
        if (threadIdx.x < rows) s_diag[threadIdx.x] = mask[(size_t)(rb * 64 + threadIdx.x) * cb_total + rb];
        __syncthreads();
        if (threadIdx.x == 0) {
            // greedy chain over the 64 boxes of this block, visiting only the SURVIVORS (next clear bit of the suppression word):
            // a single thread's dependent chain, so its length matters -- ~60 kept boxes instead of 400 iterations
            const unsigned long long rmask = rows >= 64 ? ~0ULL : ((1ULL << rows) - 1ULL);
            unsigned long long cur = s_remv[rb], kept = 0, avail = ~cur & rmask;
            while (avail) {
                const int i = __ffsll((long long)avail) - 1;
                kept |= 1ULL << i;
                cur |= s_diag[i];
                avail = ~cur & rmask & ~((2ULL << i) - 1ULL);  // clear bits above i (i == 63: 2 << 63 == 0 -> nothing left)
            }
            s_kept = kept;
        }
        __syncthreads();
        const unsigned long long kept = s_kept;
        // ordered output of this block's kept boxes
        if (threadIdx.x < rows && ((kept >> threadIdx.x) & 1ULL)) {
            const int pos = s_nkept + __popcll(kept & ((1ULL << threadIdx.x) - 1ULL));
            const int i = rb * 64 + threadIdx.x;
            if (keep) keep[pos] = i;
            if (g.rois && pos < g.post_top_n) {
                for (int k = 0; k < 6; ++k) g.rois[pos * 6 + k] = g.sorted_boxes[i * 6 + k];
                g.scores[pos] = g.sorted_scores[i];
                g.level_ids[pos] = g.sorted_levels[i];
            }
        }
        // propagate suppression to later column blocks
        const int ncols = cb_total - rb - 1;
        for (int w = threadIdx.x; w < ncols * 64; w += blockDim.x) {
            const int i = w & 63, j = rb + 1 + (w >> 6);
            if (i < rows && ((kept >> i) & 1ULL)) {
                const unsigned long long m = mask[(size_t)(rb * 64 + i) * cb_total + j];
                if (m) atomicOr(&s_remv[j], m);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) s_nkept += __popcll(kept);
        __syncthreads();
    }
    if (threadIdx.x == 0) *num_out = g.rois ? min(s_nkept, g.post_top_n) : s_nkept;
}

// ---- RPN stage 1: objectness, inside filter, sort keys, coarse histogram -------------------------
constexpr int kMaxLevels = 3;
constexpr int kHistBins = 2048;
struct RpnLevels {
    const float *cls[kMaxLevels], *deltas[kMaxLevels], *sizes[kMaxLevels];
    int grid[kMaxLevels][3], A[kMaxLevels], cls_mode[kMaxLevels], cls_ld[kMaxLevels], deltas_ld[kMaxLevels];
    int offset[kMaxLevels + 1];  // flat anchor index offsets
    int n_levels, feat_stride, scene[3], border;
};

__device__ __forceinline__ void decode_flat(const RpnLevels &L, int f, int &lvl, int &vox, int &a, int &x, int &y, int &z) {
    lvl = 0;
    while (lvl + 1 < L.n_levels && f >= L.offset[lvl + 1]) ++lvl;
    const int r = f - L.offset[lvl];
    vox = r / L.A[lvl];
    a = r - vox * L.A[lvl];
    z = vox % L.grid[lvl][2];
    const int t = vox / L.grid[lvl][2];
    y = t % L.grid[lvl][1];
    x = t / L.grid[lvl][1];
}

__device__ __forceinline__ int score_bin(float p) { return min(kHistBins - 1, max(0, (int)(p * (float)kHistBins))); }

__global__ void __launch_bounds__(256) rpn_score_kernel(const RpnLevels L, unsigned long long *keys, int *hist) {
    __shared__ int s_hist[kHistBins];
    for (int i = threadIdx.x; i < kHistBins; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const int total = L.offset[L.n_levels];
    for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < total; f += gridDim.x * blockDim.x) {
        int lvl, vox, a, x, y, z;
        decode_flat(L, f, lvl, vox, a, x, y, z);
        const float *sz = L.sizes[lvl] + a * 3;
        const float st = (float)L.feat_stride;
        const float cx = st * x, cy = st * y, cz = st * z;  // exact small integers
        const float hx = 0.5f * sz[0], hy = 0.5f * sz[1], hz = 0.5f * sz[2];
        const float b = (float)L.border;
        const bool inside = (cx - hx >= -b) && (cy - hy >= -b) && (cz - hz >= -b) && (cx + hx < (float)L.scene[0] + b) &&
                            (cy + hy < (float)L.scene[1] + b) && (cz + hz < (float)L.scene[2] + b);
        unsigned long long key = 0;
        if (inside) {
            const int A = L.A[lvl];
            float p;
            if (L.cls_mode[lvl] == 1) {  // caller already holds foreground probabilities [N][A]
                p = __ldg(L.cls[lvl] + (int64_t)vox * L.cls_ld[lvl] + a);
            } else {  // 2-way softmax over {bg, fg} logits (lib/nets/network.py:546)
                const float s0 = __ldg(L.cls[lvl] + (int64_t)vox * L.cls_ld[lvl] + a), s1 = __ldg(L.cls[lvl] + (int64_t)vox * L.cls_ld[lvl] + A + a);
                const float m = fmaxf(s0, s1);
                const float e0 = expf(s0 - m), e1 = expf(s1 - m);
                p = __fdiv_rn(e1, __fadd_rn(e0, e1));
            }
            key = ((unsigned long long)__float_as_uint(p) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)f);
            atomicAdd(&s_hist[score_bin(p)], 1);
        }
        keys[f] = key;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kHistBins; i += blockDim.x)
        if (s_hist[i]) atomicAdd(hist + i, s_hist[i]);
}

// ---- RPN stage 2: candidates = every key whose bin >= the bin containing the K-th best ------------
__global__ void __launch_bounds__(256) rpn_candidates_kernel(const unsigned long long *keys, int total, const int *hist, int K,
                                                             unsigned long long *cand, int *cand_count) {
    __shared__ int s_thr;
    if (threadIdx.x == 0) {
        int cum = 0, b = kHistBins - 1;
        for (; b > 0; --b) { cum += hist[b]; if (cum >= K) break; }
        s_thr = b;  // b == 0 when fewer than K candidates exist in total
    }
    __syncthreads();
    const int thr = s_thr;
    for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < total; f += gridDim.x * blockDim.x) {
        const unsigned long long key = keys[f];
        if (key && score_bin(__uint_as_float((unsigned)(key >> 32))) >= thr) cand[atomicAdd(cand_count, 1)] = key;
    }
}

// ---- RPN stage 3: exact top-K (radix select + bitonic sort), decode, clip -------------------------
__global__ void __launch_bounds__(1024) rpn_topk_decode_kernel(const RpnLevels L, const unsigned long long *cand, const int *cand_count,
                                                               int K, int Kpow2, float *sorted_boxes, float *sorted_scores,
                                                               int32_t *sorted_levels, int32_t *order_out, int *n_sorted) {
    extern __shared__ unsigned long long s_keys[];  // [Kpow2]
    __shared__ int s_hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_need, s_fill;
    const int M = *cand_count;
    const int Keff = min(K, M);
    for (int i = threadIdx.x; i < Kpow2; i += blockDim.x) s_keys[i] = 0;
    if (threadIdx.x == 0) { s_prefix = 0; s_need = Keff; s_fill = 0; }
    __syncthreads();
    unsigned long long T = 0;  // K-th largest key (0 -> take everything)
    if (M > K) {
        for (int r = 0; r < 8; ++r) {
            for (int i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
            __syncthreads();
            const unsigned long long prefix = s_prefix;
            const int shift = 56 - 8 * r;
            for (int i = threadIdx.x; i < M; i += blockDim.x) {
                const unsigned long long k = cand[i];
                if (r == 0 || (k >> (shift + 8)) == prefix) atomicAdd(&s_hist[(int)((k >> shift) & 255ULL)], 1);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                int need = s_need, d = 255;
                for (; d > 0; --d) { if (s_hist[d] >= need) break; need -= s_hist[d]; }
                s_need = need;
                s_prefix = (prefix << 8) | (unsigned long long)d;
            }
            __syncthreads();
        }
        T = s_prefix;
    }
    for (int i = threadIdx.x; i < M; i += blockDim.x) {
        const unsigned long long k = cand[i];
        if (k >= T) { const int p = atomicAdd(&s_fill, 1); if (p < Kpow2) s_keys[p] = k; }
    }
    __syncthreads();
    // bitonic sort, descending
    for (int size = 2; size <= Kpow2; size <<= 1) {
        for (int strd = size >> 1; strd > 0; strd >>= 1) {
            for (int i = threadIdx.x; i < Kpow2; i += blockDim.x) {
                const int j = i ^ strd;
                if (j > i) {
                    const unsigned long long a = s_keys[i], b = s_keys[j];
                    const bool desc = ((i & size) == 0);
                    if (desc ? (a < b) : (a > b)) { s_keys[i] = b; s_keys[j] = a; }
                }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) *n_sorted = Keff;
    for (int i = threadIdx.x; i < K; i += blockDim.x) {
        float box[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float score = 0.f;
        int lvl_id = 0, f = -1;
        if (i < Keff) {
            const unsigned long long key = s_keys[i];
            f = (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFULL));
            score = __uint_as_float((unsigned)(key >> 32));
            int lvl, vox, a, x, y, z;
            decode_flat(L, f, lvl, vox, a, x, y, z);
            lvl_id = lvl + 1;
            const float *sz = L.sizes[lvl] + a * 3;
            const float *d = L.deltas[lvl] + (int64_t)vox * L.deltas_ld[lvl] + a * 6;
            const float st = (float)L.feat_stride;
            const float pos[3] = {st * x, st * y, st * z};
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                // anchor (lo, hi) = pos -/+ size/2 are exact in fp32; bbox_transform_inv with one rounding per op
                const float lo = pos[k] - 0.5f * sz[k], hi = pos[k] + 0.5f * sz[k];
                const float w = __fsub_rn(hi, lo);
                const float ctr = __fadd_rn(lo, __fmul_rn(0.5f, w));
                const float pc = __fadd_rn(__fmul_rn(__ldg(d + k), w), ctr);
                const float pw = __fmul_rn(expf(__ldg(d + 3 + k)), w);
                const float hw = __fmul_rn(0.5f, pw);
                const float dim = (float)L.scene[k];
                box[k] = fminf(fmaxf(__fsub_rn(pc, hw), 0.f), dim);
                box[3 + k] = fminf(fmaxf(__fadd_rn(pc, hw), 0.f), dim);
            }
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) sorted_boxes[i * 6 + k] = box[k];
        sorted_scores[i] = score;
        sorted_levels[i] = lvl_id;
        if (order_out) order_out[i] = f;
    }
}

// zero-fill the padded tail of the proposal outputs (rows >= num_out) so downstream kernels that
// always process post_top_n rows are deterministic
__global__ void rpn_pad_kernel(float *rois, float *scores, int32_t *level_ids, const int32_t *num_out, int post_top_n) {
    const int n = *num_out;
    for (int i = n + threadIdx.x; i < post_top_n; i += blockDim.x) {
        for (int k = 0; k < 6; ++k) rois[i * 6 + k] = 0.f;
        scores[i] = 0.f;
        level_ids[i] = 0;
    }
}


// ---- RPN stage 3 (single CTA): exact top-K by sorting the candidates in shared memory, decode + clip -------------------
// The coarse histogram cut of stage 2 leaves K plus the population of one 1/2048-wide score bin -- a few hundred to a few
// thousand keys -- so they are bitonic-sorted directly (no 8-pass radix select, which cost ~16 us of serial latency); only
// when more than kSortCap candidates share the cut bin is the exact K-th key radix-selected over the global list first.
// Same keys (score bits | ~flat index: unique, stable descending order) and the same decode arithmetic as
// rpn_topk_decode_kernel: identical outputs.
constexpr int kSortCap = 4096;  // candidates sorted in shared memory (32 KB)
constexpr size_t kReduceSmemCap = 200 * 1024;  // largest bitmask + remv words nms_reduce_smem_kernel stages (pre_top_n <= 1279)

__device__ __forceinline__ void decode_box(const RpnLevels &L, int f, float *box, int &lvl_id) {
    int lvl, vox, a, x, y, z;
    decode_flat(L, f, lvl, vox, a, x, y, z);
    lvl_id = lvl + 1;
    const float *sz = L.sizes[lvl] + a * 3;
    const float *d = L.deltas[lvl] + (int64_t)vox * L.deltas_ld[lvl] + a * 6;
    const float st = (float)L.feat_stride;
    const float pos[3] = {st * x, st * y, st * z};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        // anchor (lo, hi) = pos -/+ size/2 are exact in fp32; bbox_transform_inv with one rounding per op
        const float lo = pos[k] - 0.5f * sz[k], hi = pos[k] + 0.5f * sz[k];
        const float w = __fsub_rn(hi, lo);
        const float ctr = __fadd_rn(lo, __fmul_rn(0.5f, w));
        const float pc = __fadd_rn(__fmul_rn(__ldg(d + k), w), ctr);
        const float pw = __fmul_rn(expf(__ldg(d + 3 + k)), w);
        const float hw = __fmul_rn(0.5f, pw);
        const float dim = (float)L.scene[k];
        box[k] = fminf(fmaxf(__fsub_rn(pc, hw), 0.f), dim);
        box[3 + k] = fminf(fmaxf(__fadd_rn(pc, hw), 0.f), dim);
    }
}

__global__ void __launch_bounds__(1024) rpn_sort_decode_kernel(const RpnLevels L, const unsigned long long *cand, const int *cand_count,
                                                               int K, float *sorted_boxes, float *sorted_scores,
                                                               int32_t *sorted_levels, int32_t *order_out, int *n_sorted) {
    __shared__ unsigned long long s_keys[kSortCap];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_hist[256], s_need, s_fill;
    const int t = threadIdx.x, nt = blockDim.x;
    const int Mtot = *cand_count;
    int M = Mtot;
    const int Keff = min(K, Mtot);
    if (t == 0) { s_prefix = 0; s_need = Keff; s_fill = 0; }
    __syncthreads();
    if (Mtot > kSortCap) {
        // thousands of scores share the histogram bin of the K-th best: radix-select the exact K-th key over the global list
        // first (8 passes), then only the K keys at or above it enter shared memory
        for (int r = 0; r < 8; ++r) {
            for (int i = t; i < 256; i += nt) s_hist[i] = 0;
            __syncthreads();
            const unsigned long long prefix = s_prefix;
            const int shift = 56 - 8 * r;
            for (int i = t; i < Mtot; i += nt) {
                const unsigned long long k = cand[i];
                if (r == 0 || (k >> (shift + 8)) == prefix) atomicAdd(&s_hist[(int)((k >> shift) & 255ULL)], 1);
            }
            __syncthreads();
            if (t == 0) {
                int need = s_need, d = 255;
                for (; d > 0; --d) { if (s_hist[d] >= need) break; need -= s_hist[d]; }
                s_need = need;
                s_prefix = (prefix << 8) | (unsigned long long)d;
            }
            __syncthreads();
        }
        const unsigned long long T = s_prefix;
        for (int i = t; i < Mtot; i += nt) {
            const unsigned long long k = cand[i];
            if (k >= T) { const int p = atomicAdd(&s_fill, 1); if (p < kSortCap) s_keys[p] = k; }
        }
        __syncthreads();
        M = min(s_fill, kSortCap);  // == K (keys are unique)
    }
    int P = 2;
    while (P < M) P <<= 1;  // sort size: every candidate, padded with zero keys (zero sorts last; real keys are non-zero)
    for (int i = t; i < P; i += nt)
        if (Mtot <= kSortCap) s_keys[i] = i < M ? cand[i] : 0ULL;
        else if (i >= M) s_keys[i] = 0ULL;
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1)  // bitonic sort, descending
        for (int strd = size >> 1; strd > 0; strd >>= 1) {
            for (int i = t; i < P; i += nt) {
                const int j = i ^ strd;
                if (j > i) {
                    const unsigned long long a = s_keys[i], b = s_keys[j];
                    const bool desc = ((i & size) == 0);
                    if (desc ? (a < b) : (a > b)) { s_keys[i] = b; s_keys[j] = a; }
                }
            }
            __syncthreads();
        }
    if (t == 0) *n_sorted = Keff;
    for (int i = t; i < K; i += nt) {  // decode + clip the K best (rows >= Keff: zero boxes that are never emitted)
        float box[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        float score = 0.f;
        int lvl_id = 0, f = -1;
        if (i < Keff) {
            const unsigned long long key = s_keys[i];
            f = (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFULL));
            score = __uint_as_float((unsigned)(key >> 32));
            decode_box(L, f, box, lvl_id);
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) sorted_boxes[i * 6 + k] = box[k];
        sorted_scores[i] = score;
        sorted_levels[i] = lvl_id;
        if (order_out) order_out[i] = f;
    }
}

// ---- NMS greedy reduce with the bitmask staged in shared memory (one coalesced pass over the 22 KB the reduce needs, instead
// of a global round trip per 64-box block), gather of the first post_top_n survivors and zero padding of the tail ----------
__global__ void __launch_bounds__(256) nms_reduce_smem_kernel(const unsigned long long *mask, int n_rows, const int *n_limit,
                                                              int cb_total, NmsGather g, int32_t *num_out) {
    extern __shared__ unsigned long long s_m[];  // [n_rows][cb_total] then remv[cb_total]
    unsigned long long *s_remv = s_m + (size_t)n_rows * cb_total;
    __shared__ unsigned long long s_kept;
    __shared__ int s_nkept;
    const int n = n_limit ? min(n_rows, *n_limit) : n_rows;  // rows >= n are padding and never emitted
    const int t = threadIdx.x, nt = blockDim.x;
    for (int w = t; w < n * cb_total; w += nt) {
        const int i = w / cb_total, c = w - i * cb_total;
        s_m[w] = c >= (i >> 6) ? mask[w] : 0ULL;  // only the upper triangle was written by nms_mask_kernel
    }
    for (int j = t; j < cb_total; j += nt) s_remv[j] = 0;
    if (t == 0) s_nkept = 0;
    __syncthreads();
    for (int rb = 0; rb * 64 < n; ++rb) {
        const int rows = min(n - rb * 64, 64);
        if (t == 0) {
            // greedy chain visiting only the survivors (see nms_reduce_kernel)
            const unsigned long long rmask = rows >= 64 ? ~0ULL : ((1ULL << rows) - 1ULL);
            unsigned long long cur = s_remv[rb], kept = 0, avail = ~cur & rmask;
            while (avail) {
                const int i = __ffsll((long long)avail) - 1;
                kept |= 1ULL << i;
                cur |= s_m[(size_t)(rb * 64 + i) * cb_total + rb];
                avail = ~cur & rmask & ~((2ULL << i) - 1ULL);
            }
            s_kept = kept;
        }
        __syncthreads();
        const unsigned long long kept = s_kept;
        if (t < rows && ((kept >> t) & 1ULL)) {
            const int pos = s_nkept + __popcll(kept & ((1ULL << t) - 1ULL));
            const int i = rb * 64 + t;
            if (pos < g.post_top_n) {
#pragma unroll
                for (int k = 0; k < 6; ++k) g.rois[pos * 6 + k] = g.sorted_boxes[i * 6 + k];
                g.scores[pos] = g.sorted_scores[i];
                g.level_ids[pos] = g.sorted_levels[i];
            }
        }
        // suppression words of the kept rows -> later column blocks: one WARP per column block ORs its 64 rows with a shuffle
        // tree and writes the word once (64 threads hammering one shared atomic per block serialised: ~2k cycles per pass)
        const int ncols = cb_total - rb - 1, lane = t & 31;
        for (int jj = t >> 5; jj < ncols; jj += nt >> 5) {
            const int j = rb + 1 + jj;
            unsigned long long m = 0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = lane + 32 * h;
                if (i < rows && ((kept >> i) & 1ULL)) m |= s_m[(size_t)(rb * 64 + i) * cb_total + j];
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
            if (lane == 0 && m) s_remv[j] |= m;
        }
        __syncthreads();
        if (t == 0) s_nkept += __popcll(kept);
        __syncthreads();
    }
    const int nk = min(s_nkept, g.post_top_n);
    if (t == 0) *num_out = nk;
    for (int i = nk + t; i < g.post_top_n; i += nt) {  // zero the padded tail (downstream kernels always process post_top_n rows)
#pragma unroll
        for (int k = 0; k < 6; ++k) g.rois[i * 6 + k] = 0.f;
        g.scores[i] = 0.f;
        g.level_ids[i] = 0;
    }
}

static inline int next_pow2(int v) { int p = 1; while (p < v) p <<= 1; return p; }

struct RpnWs {  // workspace carve-up (all 8-byte aligned)
    unsigned long long *keys, *cand, *mask;
    int *hist, *cand_count, *n_sorted;
    float *sorted_boxes, *sorted_scores;
    int32_t *sorted_levels;
    size_t bytes;
};
static RpnWs carve(void *base, int total, int K) {
    RpnWs w;
    char *p = (char *)base;
    auto take = [&](size_t n) { char *r = p; p += (n + 15) & ~(size_t)15; return r; };
    w.keys = (unsigned long long *)take(sizeof(unsigned long long) * total);
    w.cand = (unsigned long long *)take(sizeof(unsigned long long) * total);
    w.mask = (unsigned long long *)take(sizeof(unsigned long long) * (size_t)K * cdiv(K, 64));
    w.hist = (int *)take(sizeof(int) * (kHistBins + 2));
    w.cand_count = w.hist + kHistBins;
    w.n_sorted = w.hist + kHistBins + 1;
    w.sorted_boxes = (float *)take(sizeof(float) * 6 * K);
    w.sorted_scores = (float *)take(sizeof(float) * K);
    w.sorted_levels = (int32_t *)take(sizeof(int32_t) * K);
    w.bytes = (size_t)(p - (char *)base);
    return w;
}

}  // namespace sis3d
using namespace sis3d;

extern "C" size_t sis3d_nms_workspace_bytes(int n) { return sizeof(unsigned long long) * (size_t)max(n, 1) * cdiv(max(n, 1), 64); }

extern "C" int sis3d_nms(const float *boxes, int n, float thresh, int64_t *keep, int32_t *num_out, void *workspace, void *stream) {
    if (!keep || !num_out || n < 0 || (n > 0 && (!boxes || !workspace))) return SIS3D_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return cudaMemsetAsync(num_out, 0, sizeof(int32_t), s) == cudaSuccess ? SIS3D_OK : SIS3D_ELAUNCH;
    const int cb = cdiv(n, 64);
    if ((size_t)cb * 8 > 200 * 1024) return SIS3D_EUNSUPPORTED;
    if ((size_t)cb * 8 > 48 * 1024 &&
        cudaFuncSetAttribute(nms_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cb * 8) != cudaSuccess)
        return SIS3D_ELAUNCH;
    nms_mask_kernel<<<dim3(cb, cb), 64, 0, s>>>(boxes, n, thresh, (unsigned long long *)workspace, cb);
    NmsGather g = {};
    nms_reduce_kernel<<<1, 256, cb * 8, s>>>((const unsigned long long *)workspace, n, nullptr, cb, keep, num_out, g);
    return finish_launch(2);
}

extern "C" size_t sis3d_rpn_workspace_bytes(const sis3d_rpn_level *lv, int n_levels, int pre_top_n) {
    if (!lv || n_levels <= 0 || n_levels > kMaxLevels) return 0;
    int total = 0;
    for (int i = 0; i < n_levels; ++i) total += lv[i].grid[0] * lv[i].grid[1] * lv[i].grid[2] * lv[i].num_anchors;
    return carve(nullptr, total, pre_top_n).bytes + 64;
}

extern "C" int sis3d_rpn_proposals(const sis3d_rpn_level *lv, int n_levels, int feat_stride, int scene_x, int scene_y,
                                   int scene_z, int allow_border, int pre_top_n, int post_top_n, float nms_thresh,
                                   float *rois, float *scores, int32_t *level_ids, int32_t *num_out,
                                   int32_t *debug_order, void *workspace, size_t workspace_bytes, void *stream) {
    if (!lv || n_levels <= 0 || n_levels > kMaxLevels || !rois || !scores || !level_ids || !num_out || !workspace)
        return SIS3D_EINVAL;
    if (pre_top_n <= 0 || pre_top_n > 8192 || post_top_n <= 0) return SIS3D_EUNSUPPORTED;
    RpnLevels L = {};
    L.n_levels = n_levels; L.feat_stride = feat_stride; L.border = allow_border;
    L.scene[0] = scene_x; L.scene[1] = scene_y; L.scene[2] = scene_z;
    int total = 0;
    for (int i = 0; i < n_levels; ++i) {
        if (!lv[i].cls || !lv[i].deltas || !lv[i].anchor_sizes || lv[i].num_anchors <= 0) return SIS3D_EINVAL;
        L.cls[i] = lv[i].cls; L.deltas[i] = lv[i].deltas; L.sizes[i] = lv[i].anchor_sizes; L.A[i] = lv[i].num_anchors; L.cls_mode[i] = lv[i].cls_mode;
        L.cls_ld[i] = lv[i].cls_ld ? lv[i].cls_ld : (lv[i].cls_mode == 1 ? lv[i].num_anchors : 2 * lv[i].num_anchors);
        L.deltas_ld[i] = lv[i].deltas_ld ? lv[i].deltas_ld : 6 * lv[i].num_anchors;
        for (int k = 0; k < 3; ++k) L.grid[i][k] = lv[i].grid[k];
        L.offset[i] = total;
        total += lv[i].grid[0] * lv[i].grid[1] * lv[i].grid[2] * lv[i].num_anchors;
    }
    for (int i = n_levels; i <= kMaxLevels; ++i) L.offset[i] = total;
    void *base = (void *)(((uintptr_t)workspace + 15) & ~(uintptr_t)15);
    RpnWs w = carve(base, total, pre_top_n);
    if (w.bytes + 16 > workspace_bytes) return SIS3D_EWORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    if (total == 0) {  // every level grid is empty: no anchor, no proposal (a zero-block launch would fail)
        const bool ok = cudaMemsetAsync(num_out, 0, sizeof(int32_t), s) == cudaSuccess &&
                        cudaMemsetAsync(rois, 0, sizeof(float) * 6 * post_top_n, s) == cudaSuccess &&
                        cudaMemsetAsync(scores, 0, sizeof(float) * post_top_n, s) == cudaSuccess &&
                        cudaMemsetAsync(level_ids, 0, sizeof(int32_t) * post_top_n, s) == cudaSuccess &&
                        (!debug_order || cudaMemsetAsync(debug_order, 0xFF, sizeof(int32_t) * pre_top_n, s) == cudaSuccess);
        return ok ? SIS3D_OK : SIS3D_ELAUNCH;
    }
    const int cb = cdiv(pre_top_n, 64);
    const size_t reduce_smem = sizeof(unsigned long long) * ((size_t)pre_top_n * cb + cb);
    const bool fused = reduce_smem <= kReduceSmemCap && !getenv("SIS3D_RPN_UNFUSED");
    const int Kp2 = next_pow2(pre_top_n);
    // shared-memory opt-ins are checked before the first launch, so a refused call leaves every buffer untouched
    if (fused) {
        static bool attr = false;
        if (!attr) {
            if (cudaFuncSetAttribute(nms_reduce_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kReduceSmemCap) != cudaSuccess)
                return SIS3D_ELAUNCH;
            attr = true;
        }
    } else if ((size_t)Kp2 * 8 > 48 * 1024 &&
               cudaFuncSetAttribute(rpn_topk_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Kp2 * 8) != cudaSuccess) {
        return SIS3D_ELAUNCH;
    }
    if (cudaMemsetAsync(w.hist, 0, sizeof(int) * (kHistBins + 2), s) != cudaSuccess) return SIS3D_ELAUNCH;
    const int blocks = min(cdiv(total, 256), kNumSMs * 4);
    rpn_score_kernel<<<blocks, 256, 0, s>>>(L, w.keys, w.hist);
    rpn_candidates_kernel<<<blocks, 256, 0, s>>>(w.keys, total, w.hist, pre_top_n, w.cand, w.cand_count);
    if (fused) {
        // low-latency chain: sort + decode in one CTA (candidates sorted in shared memory), the K x K/64 IoU bitmask on
        // cb x cb CTAs (the parallel part), greedy reduce + gather + padding in one CTA with the bitmask staged in shared memory
        rpn_sort_decode_kernel<<<1, 1024, 0, s>>>(L, w.cand, w.cand_count, pre_top_n, w.sorted_boxes, w.sorted_scores, w.sorted_levels,
                                                debug_order, w.n_sorted);
        nms_mask_kernel<<<dim3(cb, cb), 64, 0, s>>>(w.sorted_boxes, pre_top_n, nms_thresh, w.mask, cb);
        NmsGather g = {w.sorted_boxes, w.sorted_scores, w.sorted_levels, rois, scores, level_ids, post_top_n};
        nms_reduce_smem_kernel<<<1, 256, reduce_smem, s>>>(w.mask, pre_top_n, w.n_sorted, cb, g, num_out);
        return finish_launch(5);
    }
    rpn_topk_decode_kernel<<<1, 1024, Kp2 * 8, s>>>(L, w.cand, w.cand_count, pre_top_n, Kp2, w.sorted_boxes, w.sorted_scores,
                                                  w.sorted_levels, debug_order, w.n_sorted);
    // NMS over the (zero padded) pre_top_n rows is wrong when fewer than pre_top_n candidates exist:
    // padded all-zero boxes would suppress each other only, but must not be emitted -> the reduce is
    // bounded by n_sorted on the device.
    nms_mask_kernel<<<dim3(cb, cb), 64, 0, s>>>(w.sorted_boxes, pre_top_n, nms_thresh, w.mask, cb);
    NmsGather g = {w.sorted_boxes, w.sorted_scores, w.sorted_levels, rois, scores, level_ids, post_top_n};
    nms_reduce_kernel<<<1, 256, cb * 8, s>>>(w.mask, pre_top_n, w.n_sorted, cb, nullptr, num_out, g);
    rpn_pad_kernel<<<1, 256, 0, s>>>(rois, scores, level_ids, num_out, post_top_n);
    return finish_launch(6);
}
