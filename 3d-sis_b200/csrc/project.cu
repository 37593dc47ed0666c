// project.cu -- back-projection of 2D feature maps into the voxel grid.
//
//   project_map_kernel      voxel -> pixel map per view (frustum cull + depth test)
//                           == ProjectionHelper.compute_projection, lib/layer_utils/projection.py:52-121
//   compact kernels         ordered compaction into the reference's (lin3d, lin2d) index lists
//   backproject_max_kernel  gather + cross-view max, writes the VC volume once
//                           == Projection.forward (projection.py:129-136) + network.py:220-239
//
// Arithmetic notes (bit parity with the torch-CPU reference, verified in tests):
//   * torch.mm on a [4,4]x[4,N] product accumulates k = 0..3 as mul, fma, fma, fma -> same chain here;
//   * (p*fx)/pz + cx is three separately rounded ops -> __fmul_rn/__fdiv_rn/__fadd_rn (no contraction);
//   * torch.round is half-to-even -> rintf; NaN/inf never pass the range tests.
#include "common.cuh"

namespace sis3d {

struct ViewParams {  // 40 floats, see sis3d.h
    float w2c[16];
    float g2w[16];
    float bmin[3];
    float bmax[3];
    float pad[2];
};

__device__ __forceinline__ float dot4(const float *m, float x, float y, float z) {
    float acc = __fmul_rn(m[0], x);
    acc = __fmaf_rn(m[1], y, acc);
    acc = __fmaf_rn(m[2], z, acc);
    acc = __fmaf_rn(m[3], 1.0f, acc);
    return acc;
}
__device__ __forceinline__ float dot4w(const float *m, float x, float y, float z, float w) {
    float acc = __fmul_rn(m[0], x);
    acc = __fmaf_rn(m[1], y, acc);
    acc = __fmaf_rn(m[2], z, acc);
    acc = __fmaf_rn(m[3], w, acc);
    return acc;
}

__global__ void __launch_bounds__(256) project_map_kernel(const ViewParams *views, const float *depth, int img_w,
                                                          int img_h, float fx, float fy, float cx, float cy,
                                                          float dmin, float dmax, float vsize, int X, int Y, int Z,
                                                          int16_t *pix, int32_t *counts) {
    const int view = blockIdx.y;
    __shared__ ViewParams vp;
    if (threadIdx.x < 40) reinterpret_cast<float *>(&vp)[threadIdx.x] = reinterpret_cast<const float *>(views + view)[threadIdx.x];
    __syncthreads();
    const int64_t n0 = (int64_t)X * Y * Z;
    const float *dimg = depth + (int64_t)view * img_w * img_h;
    int16_t *out = pix + (int64_t)view * n0;
    int local = 0;
    for (int64_t lin = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; lin < n0; lin += (int64_t)gridDim.x * blockDim.x) {
        const int z = (int)(lin / ((int64_t)X * Y));
        const int rem = (int)(lin - (int64_t)z * X * Y);
        const int y = rem / X, x = rem - y * X;
        const float fxv = (float)x, fyv = (float)y, fzv = (float)z;
        int16_t res = -1;
        if (fxv >= vp.bmin[0] && fyv >= vp.bmin[1] && fzv >= vp.bmin[2] && fxv < vp.bmax[0] && fyv < vp.bmax[1] &&
            fzv < vp.bmax[2]) {
            // world = grid_to_world @ (x,y,z,1); cam = world_to_camera @ world   (two mm's, projection.py:86)
            const float wx = dot4(vp.g2w + 0, fxv, fyv, fzv), wy = dot4(vp.g2w + 4, fxv, fyv, fzv);
            const float wz = dot4(vp.g2w + 8, fxv, fyv, fzv), ww = dot4(vp.g2w + 12, fxv, fyv, fzv);
            const float px0 = dot4w(vp.w2c + 0, wx, wy, wz, ww), py0 = dot4w(vp.w2c + 4, wx, wy, wz, ww);
            const float pz = dot4w(vp.w2c + 8, wx, wy, wz, ww);
            const float u = rintf(__fadd_rn(__fdiv_rn(__fmul_rn(px0, fx), pz), cx));
            const float v = rintf(__fadd_rn(__fdiv_rn(__fmul_rn(py0, fy), pz), cy));
            if (u >= 0.f && v >= 0.f && u < (float)img_w && v < (float)img_h) {
                const int p = (int)v * img_w + (int)u;
                const float d = __ldg(dimg + p);
                if (d >= dmin && d <= dmax && fabsf(__fsub_rn(d, pz)) <= vsize) res = (int16_t)p;
            }
        }
        out[lin] = res;
        local += res >= 0;
    }
    local = warp_sum(local);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(counts + view, local);
}

// ---- ordered compaction of one view's map -------------------------------------------------------
constexpr int kCompactBlock = 1024;
__global__ void __launch_bounds__(kCompactBlock) compact_count_kernel(const int16_t *pix, int64_t n0, int32_t *block_counts) {
    const int64_t i = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    const int flag = (i < n0 && pix[i] >= 0) ? 1 : 0;
    const int c = __syncthreads_count(flag);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}
__global__ void __launch_bounds__(1024) compact_scan_kernel(int32_t *block_counts, int nblocks, int64_t *lin3d, int64_t *lin2d) {
    // single block exclusive scan (in place); writes the total into element 0 of both lists
    __shared__ int sh[1024];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < nblocks ? block_counts[i] : 0;
        sh[threadIdx.x] = v;
        __syncthreads();
        for (int off = 1; off < 1024; off <<= 1) {
            const int t = threadIdx.x >= off ? sh[threadIdx.x - off] : 0;
            __syncthreads();
            sh[threadIdx.x] += t;
            __syncthreads();
        }
        if (i < nblocks) block_counts[i] = carry + sh[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == 0) carry += sh[1023];
        __syncthreads();
    }
    if (threadIdx.x == 0) { lin3d[0] = carry; lin2d[0] = carry; }
}
__global__ void __launch_bounds__(kCompactBlock) compact_scatter_kernel(const int16_t *pix, int64_t n0, const int32_t *block_offsets,
                                                                       int64_t *lin3d, int64_t *lin2d) {
    __shared__ int warp_tot[32];
    const int64_t i = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
    const int p = i < n0 ? pix[i] : -1;
    const unsigned b = __ballot_sync(0xffffffffu, p >= 0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) warp_tot[warp] = __popc(b);
    __syncthreads();
    if (warp == 0) {
        int v = warp_tot[lane], s = v;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
        warp_tot[lane] = s - v;
    }
    __syncthreads();
    if (p >= 0) {
        const int pos = block_offsets[blockIdx.x] + warp_tot[warp] + __popc(b & ((1u << lane) - 1u));
        lin3d[1 + pos] = i;
        lin2d[1 + pos] = p;
    }
}

// ---- feature transpose [n][C][hw] -> [n][hw][C] --------------------------------------------------
__global__ void feats_transpose_kernel(const float *in, float *out, int C, int hw) {
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

// ---- fused gather + cross-view max ---------------------------------------------------------------
// One warp per output voxel (VC order).  Pairing of feature maps with index lists follows the
// reference exactly, including its behaviour when a view has no valid projection:
//   real = [v : counts[v] > 0];  for k < len(real): if counts[k] > 0: use (feats[k], map real[k])
// (lib/model/trainval.py:805-820 stacks only surviving lists; lib/nets/network.py:220-223 zips them
// with ALL feature maps and skips by position).
__global__ void backproject_pairs_kernel(const int32_t *counts, int n_views, int32_t *pairs, int32_t *n_pairs) {
    if (threadIdx.x || blockIdx.x) return;
    int nreal = 0;
    for (int v = 0; v < n_views; ++v)
        if (counts[v] > 0) pairs[2 * n_views + nreal++] = v;  // real[] scratch in the tail third
    int np = 0;
    for (int k = 0; k < nreal; ++k)
        if (counts[k] > 0) { pairs[2 * np] = k; pairs[2 * np + 1] = pairs[2 * n_views + k]; ++np; }
    *n_pairs = np;
}

// dense map from one reference-style index list pair (element 0 = count)
__global__ void scatter_lists_kernel(const int64_t *lin3d, const int64_t *lin2d, int64_t n0, int16_t *pix) {
    const int64_t cnt = lin3d[0];
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cnt; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t v = lin3d[1 + i];
        if (v >= 0 && v < n0) pix[v] = (int16_t)lin2d[1 + i];
    }
}

__global__ void __launch_bounds__(256) backproject_max_kernel(const float *feats_t, const int16_t *pix, const int32_t *pairs,
                                                              const int32_t *n_pairs, int n_views, int C, int hw, int X, int Y,
                                                              int Z, float *vol) {
    extern __shared__ int s_pairs[];  // [2*n_views] (feat index, map index)
    __shared__ int s_npairs;
    if (threadIdx.x == 0) s_npairs = min(*n_pairs, n_views);
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * s_npairs; i += blockDim.x) s_pairs[i] = pairs[i];
    __syncthreads();
    const int npairs = s_npairs;
    const int lane = threadIdx.x & 31;
    const int warps_per_block = blockDim.x >> 5;
    const int64_t n0 = (int64_t)X * Y * Z;
    const int C4 = C >> 2;
    for (int64_t v = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5); v < n0; v += (int64_t)gridDim.x * warps_per_block) {
        const int z = (int)(v % Z);
        const int64_t t = v / Z;
        const int y = (int)(t % Y), x = (int)(t / Y);
        const int64_t lin = ((int64_t)z * Y + y) * X + x;
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
            reinterpret_cast<float4 *>(vol + v * C)[c4] = acc;
        }
    }
}

}  // namespace sis3d
using namespace sis3d;

extern "C" int sis3d_project_map(const float *views, const float *depth, int n_views, int img_w, int img_h,
                                 float fx, float fy, float cx, float cy, float depth_min, float depth_max, float voxel_size, int X, int Y,
                                 int Z, int16_t *pix, int32_t *counts, void *stream) {
    if (!views || !depth || !pix || !counts || n_views <= 0 || img_w * img_h > 32767 || X < 0 || Y < 0 || Z < 0) return SIS3D_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(counts, 0, sizeof(int32_t) * n_views, s) != cudaSuccess) return SIS3D_ELAUNCH;
    const int64_t n0 = (int64_t)X * Y * Z;
    if (n0 == 0) return SIS3D_OK;  // empty volume: every count is 0, no map entry exists
    dim3 grid((unsigned)imin64(cdiv64(n0, 256), kNumSMs * 8), n_views);
    project_map_kernel<<<grid, 256, 0, s>>>((const ViewParams *)views, depth, img_w, img_h, fx, fy, cx,
                                            cy, depth_min, depth_max, voxel_size, X, Y, Z, pix, counts);
    return finish_launch();
}

extern "C" size_t sis3d_project_compact_workspace_bytes(int X, int Y, int Z) {
    return sizeof(int32_t) * (size_t)cdiv64((int64_t)X * Y * Z, kCompactBlock);
}

extern "C" int sis3d_project_compact(const int16_t *pix, int X, int Y, int Z, int64_t *lin3d, int64_t *lin2d,
                                     void *workspace, size_t workspace_bytes, void *stream) {
    const int64_t n0 = (int64_t)X * Y * Z;
    const int nblocks = (int)cdiv64(n0, kCompactBlock);
    if (!pix || !lin3d || !lin2d || !workspace || X < 0 || Y < 0 || Z < 0) return SIS3D_EINVAL;
    if (workspace_bytes < sizeof(int32_t) * (size_t)nblocks) return SIS3D_EWORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    if (nblocks == 0)  // empty volume: both lists hold only their count, 0
        return cudaMemsetAsync(lin3d, 0, sizeof(int64_t), s) == cudaSuccess && cudaMemsetAsync(lin2d, 0, sizeof(int64_t), s) == cudaSuccess
                   ? SIS3D_OK : SIS3D_ELAUNCH;
    int32_t *bc = (int32_t *)workspace;
    compact_count_kernel<<<nblocks, kCompactBlock, 0, s>>>(pix, n0, bc);
    compact_scan_kernel<<<1, 1024, 0, s>>>(bc, nblocks, lin3d, lin2d);
    compact_scatter_kernel<<<nblocks, kCompactBlock, 0, s>>>(pix, n0, bc, lin3d, lin2d);
    return finish_launch(3);
}

extern "C" int sis3d_backproject_pairs(const int32_t *counts, int n_views, int32_t *pairs, int32_t *n_pairs, void *stream) {
    if (!counts || !pairs || !n_pairs || n_views <= 0) return SIS3D_EINVAL;
    backproject_pairs_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(counts, n_views, pairs, n_pairs);
    return finish_launch();
}

extern "C" int sis3d_project_scatter_lists(const int64_t *lin3d, const int64_t *lin2d, int n_lists, int X, int Y, int Z,
                                           int16_t *pix, void *stream) {
    if (!lin3d || !lin2d || !pix || n_lists <= 0) return SIS3D_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t n0 = (int64_t)X * Y * Z;
    if (cudaMemsetAsync(pix, 0xFF, sizeof(int16_t) * n0 * n_lists, s) != cudaSuccess) return SIS3D_ELAUNCH;
    for (int i = 0; i < n_lists; ++i)
        scatter_lists_kernel<<<kNumSMs, 256, 0, s>>>(lin3d + (int64_t)i * (n0 + 1), lin2d + (int64_t)i * (n0 + 1), n0, pix + (int64_t)i * n0);
    return finish_launch(n_lists);
}

extern "C" int sis3d_backproject_max(const float *feats, float *feats_t, const int16_t *pix, const int32_t *pairs,
                                     const int32_t *n_pairs, int n_views, int C, int img_w, int img_h, int X, int Y, int Z,
                                     float *volume_vc, void *stream) {
    if (!feats || !feats_t || !pix || !pairs || !n_pairs || !volume_vc || n_views <= 0 || C % 4 != 0) return SIS3D_EINVAL;
    if ((size_t)n_views * 2 * sizeof(int) > 40000) return SIS3D_EUNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    const int hw = img_w * img_h;
    dim3 tg(cdiv(hw, 32), cdiv(C, 32), n_views);
    feats_transpose_kernel<<<tg, dim3(32, 8), 0, s>>>(feats, feats_t, C, hw);
    const int64_t n0 = (int64_t)X * Y * Z;
    const int blocks = (int)imin64(cdiv64(n0, 8), kNumSMs * 16);
    backproject_max_kernel<<<blocks, 256, (size_t)n_views * 2 * sizeof(int), s>>>(feats_t, pix, pairs, n_pairs, n_views, C, hw,
                                                                                 X, Y, Z, volume_vc);
    return finish_launch(2);
}
