// mask_color.cu -- the colour-aware mask head (MASK_USE_IMAGES / MASK_ONLY_IMAGES; reference lib/nets/backbones.py:236-287,
// lib/nets/network.py:302-317) on the ragged mask stage.
//
// The reference crops the dense back-projected feature volume (128 channels, the max over the paired views) at every kept
// RoI and runs a second 3x3x3 stack on it.  Here that volume never exists: mask_color_gather_kernel writes each kept crop's
// 128-channel input straight onto the stage's input (packed canvas or compact per-crop buffers), reading the per-view
// voxel->pixel maps and the channels-last view features the static stage already made.  The max is the one of
// backproject_max_kernel (csrc/project.cu), in the same order, so every crop voxel equals the dense volume bit for bit.
// Every convolution of the stage runs on kernel instances the mask stage and the backbone already use.
#include <cuda_fp16.h>
#include "common.cuh"

namespace sis3d {

// One warp per crop voxel, one float4 of channels per lane.  crops int32[n_crops][8] = x0, y0, z0, w, h, l, canvas x, 0;
// offs int64[n_crops + 1] = the crops' first voxels in compact order.  layout 0: compact fp32 [total][C]; 1: canvas fp32
// [Xc][cy][cz][C]; 2: the same canvas in fp16.
__global__ void __launch_bounds__(256) mask_color_gather_kernel(const float *feats_t, const int16_t *pix, const int32_t *pairs,
                                                                const int32_t *n_pairs, int n_views, int C, int hw, int X, int Y,
                                                                int Z, const int32_t *crops, const int64_t *offs, int n_crops,
                                                                int cy, int cz, int layout, void *out) {
    extern __shared__ int s_pairs[];  // [2*n_views] (feat index, map index)
    __shared__ int s_npairs;
    if (threadIdx.x == 0) s_npairs = min(*n_pairs, n_views);
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * s_npairs; i += blockDim.x) s_pairs[i] = pairs[i];
    __syncthreads();
    const int npairs = s_npairs;
    const int lane = threadIdx.x & 31;
    const int warps_per_block = blockDim.x >> 5;
    const int64_t n0 = (int64_t)X * Y * Z, total = offs[n_crops];
    const int C4 = C >> 2;
    for (int64_t v = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5); v < total; v += (int64_t)gridDim.x * warps_per_block) {
        int lo = 0, hi = n_crops - 1;  // the crop holding compact voxel v
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (offs[mid] <= v) lo = mid; else hi = mid - 1;
        }
        const int32_t *cr = crops + 8 * lo;
        const int64_t m = v - offs[lo];
        const int hl = cr[4] * cr[5];
        const int x = (int)(m / hl), r = (int)(m - (int64_t)x * hl), y = r / cr[5], z = r - y * cr[5];
        const int64_t lin = ((int64_t)(cr[2] + z) * Y + (cr[1] + y)) * X + (cr[0] + x);  // the maps' index: z slowest, x fastest
        const int64_t row = layout == 0 ? v : (((int64_t)cr[6] + x) * cy + y) * cz + z;
        for (int c4 = lane; c4 < C4; c4 += 32) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            bool first = true;
            for (int p = 0; p < npairs; ++p) {
                const int fi = s_pairs[2 * p], mi = s_pairs[2 * p + 1];
                const int px = pix[(int64_t)mi * n0 + lin];
                float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
                if (px >= 0) val = __ldg(reinterpret_cast<const float4 *>(feats_t + ((int64_t)fi * hw + px) * C) + c4);
                if (first) { acc = val; first = false; }
                else { acc.x = fmaxf(acc.x, val.x); acc.y = fmaxf(acc.y, val.y); acc.z = fmaxf(acc.z, val.z); acc.w = fmaxf(acc.w, val.w); }
            }
            if (layout == 2) {
                __half *o = reinterpret_cast<__half *>(out) + row * C + 4 * c4;
                o[0] = __float2half_rn(acc.x); o[1] = __float2half_rn(acc.y); o[2] = __float2half_rn(acc.z); o[3] = __float2half_rn(acc.w);
            } else {
                reinterpret_cast<float4 *>(reinterpret_cast<float *>(out) + row * C)[c4] = acc;
            }
        }
    }
}

// [n][C][hw] -> [n][hw][C]: the channels-last view features the gather reads, for scenes whose static stage made none
// (ground-truth RoIs run no back-projection)
__global__ void mask_color_feats_t_kernel(const float *in, float *out, int C, int hw) {
    __shared__ float tile[32][33];
    const float *src = in + (int64_t)blockIdx.z * C * hw;
    float *dst = out + (int64_t)blockIdx.z * C * hw;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int c = c0 + r, p = p0 + threadIdx.x;
        tile[r][threadIdx.x] = (c < C && p < hw) ? src[(int64_t)c * hw + p] : 0.f;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int p = p0 + r, c = c0 + threadIdx.x;
        if (c < C && p < hw) dst[(int64_t)p * C + c] = tile[threadIdx.x][r];
    }
}

}  // namespace sis3d
using namespace sis3d;

extern "C" int sis3d_mask_color_feats_t(const float *feats, int n_views, int C, int hw, float *feats_t, void *stream) {
    if (!feats || !feats_t || n_views <= 0 || C <= 0 || hw <= 0) return SIS3D_EINVAL;
    dim3 tg(cdiv(hw, 32), cdiv(C, 32), n_views);
    mask_color_feats_t_kernel<<<tg, dim3(32, 8), 0, (cudaStream_t)stream>>>(feats, feats_t, C, hw);
    return finish_launch();
}

extern "C" int sis3d_mask_color_gather(const float *feats_t, const int16_t *pix, const int32_t *pairs, const int32_t *n_pairs,
                                       int n_views, int C, int hw, int X, int Y, int Z, const int32_t *crops, const int64_t *offs,
                                       int n_crops, int64_t total, int cy, int cz, int layout, void *out, void *stream) {
    if (!feats_t || !pix || !pairs || !n_pairs || !crops || !offs || !out || n_views <= 0 || C <= 0 || C % 4 || hw <= 0 ||
        n_crops < 0 || total < 0 || layout < 0 || layout > 2 || (layout && (cy <= 0 || cz <= 0)))
        return SIS3D_EINVAL;
    if ((size_t)n_views * 2 * sizeof(int) > 40000) return SIS3D_EUNSUPPORTED;
    if (n_crops == 0 || total == 0) return SIS3D_OK;
    const int blocks = (int)imin64(cdiv64(total, 8), kNumSMs * 16);
    mask_color_gather_kernel<<<blocks, 256, (size_t)n_views * 2 * sizeof(int), (cudaStream_t)stream>>>(
        feats_t, pix, pairs, n_pairs, n_views, C, hw, X, Y, Z, crops, offs, n_crops, cy, cz, layout, out);
    return finish_launch();
}

// ---- host planner: the colour stage's tables, appended to the blob of sis3d_mask_plan_build -------------------------------
static sis3d_region crop_region(int w, int h, int l, int tile_begin, int64_t in_off, int64_t in_vox_stride[3], int64_t out_off,
                                const int64_t *out_stride) {
    sis3d_region r = {};
    r.in_off = in_off;
    r.out_off = out_off;
    r.in_dim[0] = r.out_dim[0] = w; r.in_dim[1] = r.out_dim[1] = h; r.in_dim[2] = r.out_dim[2] = l;
    for (int k = 0; k < 3; ++k) {
        r.in_stride[k] = in_vox_stride[k];
        r.out_stride[k] = out_stride ? out_stride[k] : 0;
    }
    r.tile_begin = tile_begin;
    return r;
}

extern "C" int sis3d_mask_color_plan_build(const float *h_det, int n, const sis3d_mask_plan *plan, void *h_blob, size_t capacity,
                                           sis3d_mask_color_plan *cplan) {
    if (!h_det || !plan || !cplan || n < 0) return SIS3D_EINVAL;
    sis3d_mask_color_plan c = {};
    const int nk = plan->n_kept;
    const bool canvas = plan->n_tiles_tc > 0;  // the plan's mode: canvas plans list their bricks, compact plans none
    const size_t rb = sizeof(sis3d_region) * (size_t)nk;
    c.off_crops = (plan->bytes + 15) & ~(int64_t)15;
    c.off_g2c = c.off_crops + 32 * (int64_t)nk;
    c.off_last128 = c.off_g2c + (int64_t)rb;
    c.off_c0 = c.off_last128 + (int64_t)rb;
    c.off_c128 = c.off_c0 + (canvas ? 0 : (int64_t)rb);
    c.bytes = c.off_c128 + (canvas ? 0 : (int64_t)rb);
    if (nk == 0) { c.bytes = plan->bytes; *cplan = c; return SIS3D_OK; }
    if (!h_blob || capacity < (size_t)c.bytes) { *cplan = c; return SIS3D_EWORKSPACE; }
    char *blob = (char *)h_blob;
    const int64_t *offs = (const int64_t *)(blob + plan->off_offs);
    const sis3d_region *last = (const sis3d_region *)(blob + plan->off_last);
    int32_t *crops = (int32_t *)(blob + c.off_crops);
    sis3d_region *g2c = (sis3d_region *)(blob + c.off_g2c), *last128 = (sis3d_region *)(blob + c.off_last128);
    sis3d_region *c0 = (sis3d_region *)(blob + c.off_c0), *c128 = (sis3d_region *)(blob + c.off_c128);
    const int64_t ymax = plan->canvas[1], zmax = plan->canvas[2];
    int64_t xoff = 0;
    int tb = 0;
    for (int i = 0, j = 0; i < n && j < nk; ++i) {
        const float *d = h_det + i * 16;
        if (!(d[8] > 0.5f)) continue;
        const int x0 = (int)d[9], y0 = (int)d[10], z0 = (int)d[11];
        const int w = (int)d[12] - x0, h = (int)d[13] - y0, l = (int)d[14] - z0;
        const int64_t voff = offs[j];
        int32_t *cr = crops + 8 * j;
        cr[0] = x0; cr[1] = y0; cr[2] = z0; cr[3] = w; cr[4] = h; cr[5] = l; cr[6] = (int32_t)xoff; cr[7] = 0;
        if (canvas) {  // canvas voxel strides of a 64- and a 128-channel canvas
            int64_t s64[3] = {ymax * zmax * 64, zmax * 64, 64}, s128[3] = {ymax * zmax * 128, zmax * 128, 128};
            g2c[j] = crop_region(w, h, l, tb, xoff * s64[0], s64, xoff * s128[0], s128);
            last128[j] = last[j];  // the planner's last-layer region with the 128-channel input
            last128[j].in_off = xoff * s128[0];
            for (int k = 0; k < 3; ++k) last128[j].in_stride[k] = s128[k];
        } else {       // compact per-crop buffers: dense [w][h][l] rows of 64 or 128 channels
            int64_t s64[3] = {(int64_t)h * l * 64, (int64_t)l * 64, 64}, s128[3] = {(int64_t)h * l * 128, (int64_t)l * 128, 128};
            g2c[j] = crop_region(w, h, l, tb, voff * 64, s64, voff * 128, nullptr);
            last128[j] = last[j];
            last128[j].in_off = voff * 128;
            for (int k = 0; k < 3; ++k) last128[j].in_stride[k] = s128[k];
            c0[j] = crop_region(w, h, l, tb, voff * 128, s128, voff * 64, nullptr);
            c128[j] = crop_region(w, h, l, tb, voff * 128, s128, voff * 128, nullptr);
        }
        xoff += w + 1;
        tb += (int)(((int64_t)w * h * l + SIS3D_CONV_TILE_M - 1) / SIS3D_CONV_TILE_M);
        ++j;
    }
    *cplan = c;
    return SIS3D_OK;
}
