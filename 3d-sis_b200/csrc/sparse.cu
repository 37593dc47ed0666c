// sparse.cu -- back-projection fused into the first colour convolution, exploiting sparsity.
//
// The back-projected feature volume (lib/nets/network.py:220-239) is zero except at voxels within one
// voxel of an observed depth sample: at most ~3 voxels per depth pixel and view, i.e. <= ~5 % of the
// chunk.  Its only consumer is color.0, a 2x2x2 / stride-2 convolution without bias
// (lib/nets/backbones.py:203), whose taps do not overlap.  So instead of writing the 226 MB volume and
// reading it back (453 MB of the 807 MB algorithmic traffic of the whole forward) we
//   1. sparse_cover_kernel   : list the covered input voxels per tap (t = (x&1)*4 + (y&1)*2 + (z&1)),
//   2. sparse_gemm_kernel    : for tiles of 64 covered voxels of one tap, gather their feature rows
//                              (max over paired views, 0 where a view does not cover the voxel) and
//                              multiply by that tap's [C_in x C_out] weight slice,
//   3. sparse_combine_kernel : per output voxel add its (<= 8) tap contributions in tap order, ReLU.
// The result equals relu(conv3d(imageft, W, stride 2)) up to fp32 summation order; summation order is
// fixed (no atomics on data), so results are run-to-run reproducible.
#include <cuda_fp16.h>
#include "common.cuh"

namespace sis3d {

struct SparseArgs {
    const float *feats_t;    // [n_views][hw][C]
    const int16_t *pix;      // [n_maps][N0]
    const int32_t *pairs;    // (feat, map) pairs
    const int32_t *n_pairs;
    int C, hw, X, Y, Z, OX, OY, OZ, n_views;
    int64_t n0;
    int32_t *counts;  // [8]
    int32_t *lists;   // [8][N1] : linear input index (z*X*Y + y*X + x) of covered voxels per tap
    int32_t *slot;    // [N1][8] : row of `partial` holding (o, tap), or -1
    float *partial;   // [8][N1][cout]
    int n1;
};

__global__ void __launch_bounds__(256) sparse_cover_kernel(const SparseArgs a) {
    __shared__ int s_pairs_map[64];
    __shared__ int s_np;
    if (threadIdx.x == 0) s_np = min(*a.n_pairs, a.n_views);
    __syncthreads();
    const int np = s_np;
    for (int i = threadIdx.x; i < min(np, 64); i += blockDim.x) s_pairs_map[i] = a.pairs[2 * i + 1];
    __syncthreads();
    for (int64_t lin = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; lin < a.n0; lin += (int64_t)gridDim.x * blockDim.x) {
        const int z = (int)(lin / ((int64_t)a.X * a.Y));
        const int rem = (int)(lin - (int64_t)z * a.X * a.Y);
        const int y = rem / a.X, x = rem - y * a.X;
        const int ox = x >> 1, oy = y >> 1, oz = z >> 1;
        if (ox >= a.OX || oy >= a.OY || oz >= a.OZ) continue;  // odd extents: last plane is not read by a k2s2 conv
        bool covered = false;
        for (int p = 0; p < np && !covered; ++p) {
            const int mi = p < 64 ? s_pairs_map[p] : a.pairs[2 * p + 1];
            covered = a.pix[(int64_t)mi * a.n0 + lin] >= 0;
        }
        const int tap = ((x & 1) << 2) | ((y & 1) << 1) | (z & 1);
        const int o = (ox * a.OY + oy) * a.OZ + oz;
        int s = -1;
        if (covered) {
            s = atomicAdd(a.counts + tap, 1);
            a.lists[(int64_t)tap * a.n1 + s] = (int)lin;
        }
        a.slot[(int64_t)o * 8 + tap] = s;
    }
}

constexpr int SP_BM = 64;
// one tile = 64 covered voxels of one tap; A [64][C] gathered into smem, W_tap [C][cout] staged in smem
template <int COUT>
__global__ void __launch_bounds__(256) sparse_gemm_kernel(const SparseArgs a, const float *w /*[8*C][COUT]*/) {
    extern __shared__ __align__(16) float sm[];
    float *As = sm;                        // [C][SP_BM + 4]  (k-major, padded)
    float *Ws = sm + a.C * (SP_BM + 4);    // [C][COUT]
    __shared__ int s_cnt[8];
    __shared__ int s_np;
    if (threadIdx.x < 8) s_cnt[threadIdx.x] = a.counts[threadIdx.x];
    if (threadIdx.x == 0) s_np = min(*a.n_pairs, a.n_views);
    __syncthreads();
    const int np = s_np;
    int tile_base[9];
    tile_base[0] = 0;
    for (int t = 0; t < 8; ++t) tile_base[t + 1] = tile_base[t] + (s_cnt[t] + SP_BM - 1) / SP_BM;
    const int t_ = threadIdx.x;
    constexpr int NTX = COUT / 4;          // threads along N, 4 columns each
    constexpr int TM = SP_BM * NTX / 256;  // rows per thread
    const int tx = t_ % NTX, ty = t_ / NTX;
    int cur_tap = -1;
    for (int tile = blockIdx.x; tile < tile_base[8]; tile += gridDim.x) {
        int tap = 0;
        while (tile >= tile_base[tap + 1]) ++tap;
        const int row0 = (tile - tile_base[tap]) * SP_BM;
        const int rows = min(SP_BM, s_cnt[tap] - row0);
        __syncthreads();  // previous tile's smem fully consumed
        if (tap != cur_tap) {
            const float4 *src = reinterpret_cast<const float4 *>(w + (int64_t)tap * a.C * COUT);
            for (int i = t_; i < a.C * COUT / 4; i += 256) reinterpret_cast<float4 *>(Ws)[i] = __ldg(src + i);
            cur_tap = tap;
        }
        // gather: 4 threads per row, each covers channels q*4 + 16*j
        {
            const int r = t_ >> 2, q = t_ & 3;
            int lin = -1;
            if (r < rows) lin = a.lists[(int64_t)tap * a.n1 + row0 + r];
            for (int c = q * 4; c < a.C; c += 16) {
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (lin >= 0) {
                    bool first = true;
                    for (int p = 0; p < np; ++p) {
                        const int fi = a.pairs[2 * p], mi = a.pairs[2 * p + 1];
                        const int px = a.pix[(int64_t)mi * a.n0 + lin];
                        float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (px >= 0) f = __ldg(reinterpret_cast<const float4 *>(a.feats_t + ((int64_t)fi * a.hw + px) * a.C + c));
                        if (first) { v = f; first = false; }
                        else { v.x = fmaxf(v.x, f.x); v.y = fmaxf(v.y, f.y); v.z = fmaxf(v.z, f.z); v.w = fmaxf(v.w, f.w); }
                    }
                }
                As[(c + 0) * (SP_BM + 4) + r] = v.x;
                As[(c + 1) * (SP_BM + 4) + r] = v.y;
                As[(c + 2) * (SP_BM + 4) + r] = v.z;
                As[(c + 3) * (SP_BM + 4) + r] = v.w;
            }
        }
        __syncthreads();
        float acc[TM][4];
#pragma unroll
        for (int i = 0; i < TM; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
        for (int k = 0; k < a.C; ++k) {
            const float4 b = *reinterpret_cast<const float4 *>(Ws + k * COUT + tx * 4);
            float ar[TM];
#pragma unroll
            for (int i = 0; i < TM; ++i) ar[i] = As[k * (SP_BM + 4) + ty * TM + i];
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                acc[i][0] = fmaf(ar[i], b.x, acc[i][0]);
                acc[i][1] = fmaf(ar[i], b.y, acc[i][1]);
                acc[i][2] = fmaf(ar[i], b.z, acc[i][2]);
                acc[i][3] = fmaf(ar[i], b.w, acc[i][3]);
            }
        }
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            const int r = ty * TM + i;
            if (r < rows)
                *reinterpret_cast<float4 *>(a.partial + ((int64_t)tap * a.n1 + row0 + r) * COUT + tx * 4) =
                    make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        }
    }
}

__global__ void __launch_bounds__(256) sparse_combine_kernel(const SparseArgs a, int cout, float *out, int out_ld, int out_coff,
                                                             __half *out16) {
    const int c4n = cout / 4;
    const int64_t total = (int64_t)a.n1 * c4n;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % c4n);
        const int64_t o = i / c4n;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            const int sl = a.slot[o * 8 + t];
            if (sl >= 0) {
                const float4 p = *reinterpret_cast<const float4 *>(a.partial + ((int64_t)t * a.n1 + sl) * cout + c4 * 4);
                s.x += p.x; s.y += p.y; s.z += p.z; s.w += p.w;
            }
        }
        s.x = fmaxf(s.x, 0.f); s.y = fmaxf(s.y, 0.f); s.z = fmaxf(s.z, 0.f); s.w = fmaxf(s.w, 0.f);
        *reinterpret_cast<float4 *>(out + o * out_ld + out_coff + c4 * 4) = s;
        if (out16) {
            const __half2 h0 = __floats2half2_rn(s.x, s.y), h1 = __floats2half2_rn(s.z, s.w);
            uint2 pk;
            pk.x = *reinterpret_cast<const uint32_t *>(&h0);
            pk.y = *reinterpret_cast<const uint32_t *>(&h1);
            *reinterpret_cast<uint2 *>(out16 + o * out_ld + out_coff + c4 * 4) = pk;
        }
    }
}

__global__ void feats_transpose_kernel2(const float *in, float *out, int C, int hw, int32_t *zero8) {
    __shared__ float tile[32][33];
    if (zero8 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.y == 0 && threadIdx.x < 8)
        zero8[threadIdx.x] = 0;  // per-tap counters of the cover pass (saves a memset node)
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

static size_t sparse_ws_layout(int n1, int cout, size_t *o_lists, size_t *o_slot, size_t *o_partial) {
    size_t p = 64;  // counts[8] + pad
    *o_lists = p; p += sizeof(int32_t) * 8 * (size_t)n1; p = (p + 15) & ~(size_t)15;
    *o_slot = p; p += sizeof(int32_t) * 8 * (size_t)n1; p = (p + 15) & ~(size_t)15;
    *o_partial = p; p += sizeof(float) * 8 * (size_t)n1 * cout;
    return p + 16;
}

}  // namespace sis3d
using namespace sis3d;

extern "C" size_t sis3d_backproject_conv_k2s2_workspace_bytes(int X, int Y, int Z, int cout) {
    size_t a, b, c;
    return sparse_ws_layout((X / 2) * (Y / 2) * (Z / 2), cout, &a, &b, &c);
}

extern "C" int sis3d_backproject_conv_k2s2(const float *feats, float *feats_t, const int16_t *pix, const int32_t *pairs,
                                           const int32_t *n_pairs, int n_views, int C, int img_w, int img_h, int X, int Y,
                                           int Z, const float *w_packed, int cout, float *out, int out_ld, int out_coff,
                                           void *workspace, size_t workspace_bytes, void *stream) {
    return sis3d_backproject_conv_k2s2_ex(feats, feats_t, pix, pairs, n_pairs, n_views, C, img_w, img_h, X, Y, Z, w_packed, cout, out,
                                          nullptr, out_ld, out_coff, workspace, workspace_bytes, stream);
}

extern "C" int sis3d_backproject_conv_k2s2_ex(const float *feats, float *feats_t, const int16_t *pix, const int32_t *pairs,
                                              const int32_t *n_pairs, int n_views, int C, int img_w, int img_h, int X, int Y,
                                              int Z, const float *w_packed, int cout, float *out, uint16_t *out16, int out_ld,
                                              int out_coff, void *workspace, size_t workspace_bytes, void *stream) {
    if (!feats || !feats_t || !pix || !pairs || !n_pairs || !w_packed || !out || !workspace) return SIS3D_EINVAL;
    if (C % 16 != 0 || (cout != 32 && cout != 64) || (out_ld | out_coff) & 3 || n_views <= 0) return SIS3D_EUNSUPPORTED;
    SparseArgs a;
    a.OX = X / 2; a.OY = Y / 2; a.OZ = Z / 2;
    a.n1 = a.OX * a.OY * a.OZ;
    if (a.n1 <= 0) return SIS3D_OK;
    size_t o_lists, o_slot, o_partial;
    if (sparse_ws_layout(a.n1, cout, &o_lists, &o_slot, &o_partial) > workspace_bytes) return SIS3D_EWORKSPACE;
    char *ws = (char *)workspace;
    a.counts = (int32_t *)ws; a.lists = (int32_t *)(ws + o_lists); a.slot = (int32_t *)(ws + o_slot);
    a.partial = (float *)(ws + o_partial);
    a.feats_t = feats_t; a.pix = pix; a.pairs = pairs; a.n_pairs = n_pairs;
    a.C = C; a.hw = img_w * img_h; a.X = X; a.Y = Y; a.Z = Z; a.n_views = n_views; a.n0 = (int64_t)X * Y * Z;
    // everything that can refuse the call is checked before the first launch, so a refused call writes nothing
    const size_t smem = sizeof(float) * ((size_t)C * (SP_BM + 4) + (size_t)C * cout);
    if (smem > 200 * 1024) return SIS3D_EUNSUPPORTED;
    if (cudaFuncSetAttribute(cout == 64 ? (const void *)sparse_gemm_kernel<64> : (const void *)sparse_gemm_kernel<32>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return SIS3D_ELAUNCH;
    cudaStream_t s = (cudaStream_t)stream;
    dim3 tg(cdiv(a.hw, 32), cdiv(C, 32), n_views);
    feats_transpose_kernel2<<<tg, dim3(32, 8), 0, s>>>(feats, feats_t, C, a.hw, a.counts);
    sparse_cover_kernel<<<(int)imin64(cdiv64(a.n0, 256), kNumSMs * 8), 256, 0, s>>>(a);
    if (cout == 64) sparse_gemm_kernel<64><<<kNumSMs * 2, 256, smem, s>>>(a, w_packed);
    else sparse_gemm_kernel<32><<<kNumSMs * 2, 256, smem, s>>>(a, w_packed);
    sparse_combine_kernel<<<(int)imin64(cdiv64((int64_t)a.n1 * (cout / 4), 256), kNumSMs * 8), 256, 0, s>>>(a, cout, out, out_ld,
                                                                                                             out_coff, (__half *)out16);
    return finish_launch(4);
}
