// conv_simt.cu -- fp32 implicit-GEMM 3D convolution on CUDA cores + MaxPool3d(3,1,1) + layout helpers.
//
// Role in the design (DESIGN.md "kernels"): exact-fp32 path for every conv call site of
// lib/nets/backbones.py / lib/nets/network.py.  The 3x3x3 / wide-channel layers are served by the
// wgmma kernel (conv_tc.cu); this kernel keeps the narrow layers (C_in = 2, tiny C_out heads) and
// is the fp32 parity reference for the tensor-core path.
//
// GEMM view: M = output voxels of all regions (tiles of 64), N = C_out, K = ks^3 * C_in with
// k = tap*C_in + c.  A is gathered on the fly from the VC (or strided NCDHW) input with zero fill
// outside the region (== PyTorch zero padding of the *crop*, lib/nets/network.py:303-311); B is the
// pre-packed weight [K][ldw].
#include <cuda_fp16.h>
#include "common.cuh"

namespace sis3d {

constexpr int BM = SIS3D_CONV_TILE_M;  // 64
constexpr int BK = 16;
constexpr int kConvThreads = 256;
constexpr int AS_LD = BM + 4;
constexpr int kKtab = 128;  // tap-table entries of the gather path (K = ks^3 * C_in of the narrow layers: 16, 54, ...)

struct ConvArgs {
    const float *in, *w, *bias, *res;
    float *out;
    const sis3d_region *regions;
    int n_regions, cin, cout, ldw, ks, stride, pad, act, K;
    int out_ld, out_coff, res_ld, res_coff;
    int64_t in_sc;
    int fast;  // in_sc == 1 && cin % 16 == 0
    int dense_m;          // > 0: no region table, input is a dense [dense_m][cin] matrix (linear layer)
    int k_per_split;      // > 0: split-K, blockIdx.z owns K range [z*k_per_split, ...), raw partials to out + z*split_stride
    int64_t split_stride;
    __half *out16;        // optional fp16 twin of the output, same element offsets as `out` (`out` may then be null)
};

template <int BN, int TM>
__global__ void __launch_bounds__(kConvThreads) conv3d_igemm_f32(const ConvArgs a) {
    constexpr int TN = 4;
    constexpr int NTX = BN / TN;  // threads along N
    __shared__ __align__(16) float As[BK][AS_LD];
    __shared__ __align__(16) float Bs[BK][BN];
    __shared__ int s_region;
    __shared__ int s_ktab[kKtab];  // gather path: k -> (kx | ky << 4 | kz << 8 | c << 12), replaces four integer divisions per element

    const int t = threadIdx.x;
    if (!a.fast && !a.dense_m) {
        const int ks2_ = a.ks * a.ks;
        for (int k = t; k < min(a.K, kKtab); k += kConvThreads) {
            const int tap = k / a.cin, c = k - tap * a.cin;
            const int kx = tap / ks2_, kr = tap - kx * ks2_, ky = kr / a.ks, kz = kr - ky * a.ks;
            s_ktab[k] = kx | (ky << 4) | (kz << 8) | (c << 12);
        }
    }
    const int tile = blockIdx.x;
    const int n0 = blockIdx.y * BN;
    if (t == 0 && !a.dense_m) {
        int lo = 0, hi = a.n_regions - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (a.regions[mid].tile_begin <= tile) lo = mid; else hi = mid - 1;
        }
        s_region = lo;
    }
    __syncthreads();
    sis3d_region R;
    if (a.dense_m) {
        R.in_off = R.out_off = R.res_off = 0;
        R.in_dim[0] = R.out_dim[0] = a.dense_m; R.in_dim[1] = R.in_dim[2] = R.out_dim[1] = R.out_dim[2] = 1;
        R.in_stride[0] = R.in_stride[1] = R.in_stride[2] = a.cin;
        R.out_stride[0] = R.out_stride[1] = R.out_stride[2] = 0;
        R.tile_begin = 0;
    } else {
        R = a.regions[s_region];
    }
    const int oyz = R.out_dim[1] * R.out_dim[2];
    const int m_total = R.out_dim[0] * oyz;
    const int m_base = (tile - R.tile_begin) * BM;

    // ---- A loader role: row lr, 4 consecutive k at lq*4
    const int lr = t >> 2, lq = t & 3;
    const int lm = m_base + lr;
    const bool lvalid = lm < m_total;
    int lx = 0, ly = 0, lz = 0;
    if (lvalid) {
        lx = lm / oyz;
        int rem = lm - lx * oyz;
        ly = rem / R.out_dim[2];
        lz = rem - ly * R.out_dim[2];
    }
    const int bx = lx * a.stride - a.pad, by = ly * a.stride - a.pad, bz = lz * a.stride - a.pad;
    const float *in_base = a.in + R.in_off;
    // ---- B loader role
    const int bk = t / (BN / 4), bc = (t % (BN / 4)) * 4;
    const bool b_thread = t < BK * (BN / 4);

    const int tx = t % NTX, ty = t / NTX;
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    const int ks2 = a.ks * a.ks;
    const int k_begin = a.k_per_split ? blockIdx.z * a.k_per_split : 0;
    const int k_end = a.k_per_split ? min(a.K, k_begin + a.k_per_split) : a.K;
    // global -> register fetch of one K chunk (A gathered from the voxel tensor, B from the packed weights)
    auto fetch = [&](int k0, float4 &av, float4 &bv) {
        av = make_float4(0.f, 0.f, 0.f, 0.f);
        if (a.fast) {
            const int tap = k0 / a.cin, c0 = k0 - tap * a.cin + lq * 4;
            const int kx = tap / ks2, kr = tap - kx * ks2, ky = kr / a.ks, kz = kr - ky * a.ks;
            const int ix = bx + kx, iy = by + ky, iz = bz + kz;
            if (lvalid && (unsigned)ix < (unsigned)R.in_dim[0] && (unsigned)iy < (unsigned)R.in_dim[1] &&
                (unsigned)iz < (unsigned)R.in_dim[2]) {
                const float *p = in_base + ix * R.in_stride[0] + iy * R.in_stride[1] + iz * R.in_stride[2] + c0;
                av = __ldg(reinterpret_cast<const float4 *>(p));
            }
        } else {
            float tmp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int k = k0 + lq * 4 + i;
                if (lvalid && k < k_end) {
                    int kx, ky, kz, c;
                    if (k < kKtab) {
                        const int e = s_ktab[k];
                        kx = e & 15; ky = (e >> 4) & 15; kz = (e >> 8) & 15; c = e >> 12;
                    } else {
                        const int tap = k / a.cin;
                        c = k - tap * a.cin;
                        kx = tap / ks2;
                        const int kr = tap - kx * ks2;
                        ky = kr / a.ks; kz = kr - ky * a.ks;
                    }
                    const int ix = bx + kx, iy = by + ky, iz = bz + kz;
                    if ((unsigned)ix < (unsigned)R.in_dim[0] && (unsigned)iy < (unsigned)R.in_dim[1] &&
                        (unsigned)iz < (unsigned)R.in_dim[2])
                        tmp[i] = __ldg(in_base + ix * R.in_stride[0] + iy * R.in_stride[1] +
                                       iz * R.in_stride[2] + c * a.in_sc);
                }
            }
            av = make_float4(tmp[0], tmp[1], tmp[2], tmp[3]);
        }
        bv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b_thread) {
            const int k = k0 + bk, n = n0 + bc;
            if (k < k_end && n < a.ldw) bv = __ldg(reinterpret_cast<const float4 *>(a.w + (int64_t)k * a.ldw + n));
        }
    };
    float4 av, bv;
    if (k_begin < k_end) fetch(k_begin, av, bv);
    for (int k0 = k_begin; k0 < k_end; k0 += BK) {
        __syncthreads();  // previous chunk fully consumed
        As[lq * 4 + 0][lr] = av.x;
        As[lq * 4 + 1][lr] = av.y;
        As[lq * 4 + 2][lr] = av.z;
        As[lq * 4 + 3][lr] = av.w;
        if (b_thread) *reinterpret_cast<float4 *>(&Bs[bk][bc]) = bv;
        __syncthreads();
        if (k0 + BK < k_end) fetch(k0 + BK, av, bv);  // next chunk's global loads fly while this one is multiplied
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float ar[TM];
            if constexpr (TM == 4) {
                const float4 v = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
                ar[0] = v.x; ar[1] = v.y; ar[2] = v.z; ar[3] = v.w;
            } else {
                const float2 v = *reinterpret_cast<const float2 *>(&As[k][ty * 2]);
                ar[0] = v.x; ar[1] = v.y;
            }
            const float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                acc[i][0] = fmaf(ar[i], b.x, acc[i][0]);
                acc[i][1] = fmaf(ar[i], b.y, acc[i][1]);
                acc[i][2] = fmaf(ar[i], b.z, acc[i][2]);
                acc[i][3] = fmaf(ar[i], b.w, acc[i][3]);
            }
        }
    }
    // ---------------- epilogue
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m_base + ty * TM + i;
        if (m >= m_total) continue;
        int64_t ooff = (int64_t)m * a.out_ld;
        if (R.out_stride[0] | R.out_stride[1] | R.out_stride[2]) {
            const int ox = m / oyz, orem = m - ox * oyz, oy = orem / R.out_dim[2], oz = orem - oy * R.out_dim[2];
            ooff = ox * R.out_stride[0] + oy * R.out_stride[1] + oz * R.out_stride[2];
        }
        const int64_t eoff = R.out_off + ooff + a.out_coff;
        float *orow = a.out ? a.out + eoff : nullptr;
        if (a.k_per_split) {  // raw partial sums; bias/activation applied by splitk_reduce_kernel
            orow = a.out + (int64_t)blockIdx.z * a.split_stride + (int64_t)m * a.out_ld;
#pragma unroll
            for (int j = 0; j < TN; ++j) {
                const int n = n0 + tx * TN + j;
                if (n < a.cout) orow[n] = acc[i][j];
            }
            continue;
        }
        const float *rrow = a.res ? a.res + R.res_off + (int64_t)m * a.res_ld + a.res_coff : nullptr;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + tx * TN + j;
            if (n >= a.cout) continue;
            float v = acc[i][j];
            if (a.bias) v += a.bias[n];
            if (rrow) v += rrow[n];
            if (a.act == 1) v = fmaxf(v, 0.f);
            else if (a.act == 2) v = 1.f / (1.f + expf(-v));
            if (orow) orow[n] = v;
            if (a.out16) a.out16[eoff + n] = __float2half_rn(v);
        }
    }
}

__global__ void splitk_reduce_kernel(const float *part, int splits, int64_t split_stride, const float *bias, float *y, int M,
                                     int N, int act) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * N) return;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += part[(int64_t)s * split_stride + i];  // fixed order -> deterministic
    if (bias) v += bias[i % N];
    if (act == 1) v = fmaxf(v, 0.f);
    y[i] = v;
}

// weights [cout][cin][ks][ks][ks] -> [K = tap*cin + c][ldw], zero padded columns
__global__ void pack_conv_weight_kernel(const float *w, int cout, int cin, int ks3, int ldw, float *out) {
    const int64_t total = (int64_t)ks3 * cin * ldw;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int n = (int)(i % ldw);
        const int64_t k = i / ldw;
        const int c = (int)(k % cin), tap = (int)(k / cin);
        out[i] = n < cout ? w[((int64_t)n * cin + c) * ks3 + tap] : 0.f;
    }
}

// MaxPool3d(kernel 3, stride 1, pad 1) on VC; out-of-range taps ignored (PyTorch pads with -inf).
// One thread per (voxel, channel quad); the 27 neighbours are L1/L2 hits (a z-sliding-window variant with 9 loads per
// output was measured slower: too little parallelism at 24x12x24).
__global__ void __launch_bounds__(256) maxpool3_vc_kernel(const float4 *in, float4 *out, int X, int Y, int Z, int C4, int out_ld4,
                                                          int out_coff4) {
    const int64_t total = (int64_t)X * Y * Z * C4;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        int64_t v = i / C4;
        const int z = (int)(v % Z);
        v /= Z;
        const int y = (int)(v % Y), x = (int)(v / Y);
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int dx = -1; dx <= 1; ++dx) {
            const int xx = x + dx;
            if ((unsigned)xx >= (unsigned)X) continue;
            for (int dy = -1; dy <= 1; ++dy) {
                const int yy = y + dy;
                if ((unsigned)yy >= (unsigned)Y) continue;
#pragma unroll
                for (int dz = -1; dz <= 1; ++dz) {
                    const int zz = z + dz;
                    if ((unsigned)zz >= (unsigned)Z) continue;
                    const float4 q = __ldg(in + (((int64_t)xx * Y + yy) * Z + zz) * C4 + c);
                    m.x = fmaxf(m.x, q.x); m.y = fmaxf(m.y, q.y); m.z = fmaxf(m.z, q.z); m.w = fmaxf(m.w, q.w);
                }
            }
        }
        out[(i / C4) * out_ld4 + out_coff4 + c] = m;
    }
}

// Tiled MaxPool3d(3,1,1): one CTA = an 8x8x8 brick of voxels x 16 channels.  Phase 1 reduces along z in registers while the
// halo'd brick streams in from global memory (1.95 loads per output instead of 27), phase 2 takes the 3x3 (x,y) maximum
// from shared memory (9 conflict-free 16-byte reads).  Out-of-volume neighbours count as -inf (== PyTorch's padding).
constexpr int kPoolT = 8, kPoolH = kPoolT + 2, kPoolCG4 = 4, kPoolPS = (kPoolT + 1) * kPoolCG4;  // PS: padded per-column stride
constexpr int kPoolSmem = kPoolH * kPoolH * kPoolPS * 16;
__device__ __forceinline__ float4 max4(float4 a, float4 b) {
    return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__global__ void __launch_bounds__(256) maxpool3_tiled_kernel(const float4 *in, float4 *out, int X, int Y, int Z, int C4, int out_ld4,
                                                             int out_coff4, int gy, int gz) {
    constexpr int T = kPoolT, H = kPoolH, CG4 = kPoolCG4, PS = kPoolPS;
    extern __shared__ float4 pool_sm[];
    int b = blockIdx.x;
    const int ncg = C4 / CG4;
    const int cg = b % ncg; b /= ncg;
    const int tz = b % gz; b /= gz;
    const int ty = b % gy, tx = b / gy;
    const int x0 = tx * T, y0 = ty * T, z0 = tz * T, c0 = cg * CG4;
    const float4 ninf = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int i = threadIdx.x; i < H * H * CG4; i += 256) {
        const int c = i % CG4, p = i / CG4;
        const int x = x0 + p / H - 1, y = y0 + p % H - 1;
        const bool in_xy = (unsigned)x < (unsigned)X && (unsigned)y < (unsigned)Y;
        const float4 *col = in + (((int64_t)x * Y + y) * Z) * C4 + c0 + c;
        float4 v[T + 2];
#pragma unroll
        for (int k = 0; k < T + 2; ++k) {
            const int z = z0 + k - 1;
            v[k] = (in_xy && (unsigned)z < (unsigned)Z) ? __ldg(col + (int64_t)z * C4) : ninf;
        }
#pragma unroll
        for (int k = 0; k < T; ++k) pool_sm[p * PS + k * CG4 + c] = max4(max4(v[k], v[k + 1]), v[k + 2]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < T * T * T * CG4; i += 256) {
        const int c = i % CG4;
        int q = i / CG4;
        const int z = q % T; q /= T;
        const int y = q % T, x = q / T;
        if (x0 + x >= X || y0 + y >= Y || z0 + z >= Z) continue;
        float4 m = ninf;
#pragma unroll
        for (int dx = 0; dx < 3; ++dx)
#pragma unroll
            for (int dy = 0; dy < 3; ++dy) m = max4(m, pool_sm[((x + dx) * H + (y + dy)) * PS + z * CG4 + c]);
        out[(((int64_t)(x0 + x) * Y + (y0 + y)) * Z + (z0 + z)) * out_ld4 + out_coff4 + c0 + c] = m;
    }
}

// VC [nvox][C] -> [C][nvox] through a 32x32 smem transpose
__global__ void vc_to_ncdhw_kernel(const float *in, float *out, int64_t nvox, int C) {
    __shared__ float tile[32][33];
    const int64_t v0 = (int64_t)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int64_t v = v0 + r;
        const int c = c0 + threadIdx.x;
        tile[r][threadIdx.x] = (v < nvox && c < C) ? in[v * C + c] : 0.f;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int c = c0 + r;
        const int64_t v = v0 + threadIdx.x;
        if (v < nvox && c < C) out[(int64_t)c * nvox + v] = tile[threadIdx.x][r];
    }
}

}  // namespace sis3d

using namespace sis3d;

extern "C" int sis3d_pack_conv_weight(const float *w, int cout, int cin, int ks, float *w_packed, void *stream) {
    if (!w || !w_packed || cout <= 0 || cin <= 0 || ks <= 0) return SIS3D_EINVAL;
    const int ldw = (cout + 3) & ~3;
    const int64_t total = (int64_t)ks * ks * ks * cin * ldw;
    const int blocks = (int)imin64(cdiv64(total, 256), kNumSMs * 8);
    pack_conv_weight_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, cout, cin, ks * ks * ks, ldw, w_packed);
    return finish_launch();
}

extern "C" int sis3d_conv3d(const float *in, int64_t in_chan_stride, const float *w_packed, const float *bias,
                            const float *residual, int res_ld, int res_coff, float *out, int out_ld, int out_coff,
                            const sis3d_region *regions, int n_regions, int n_tiles, int cin, int cout, int ks,
                            int stride, int pad, int act, void *stream) {
    return sis3d_conv3d_ex(in, in_chan_stride, w_packed, bias, residual, res_ld, res_coff, out, nullptr, out_ld, out_coff, regions,
                           n_regions, n_tiles, cin, cout, ks, stride, pad, act, stream);
}

extern "C" int sis3d_conv3d_ex(const float *in, int64_t in_chan_stride, const float *w_packed, const float *bias,
                               const float *residual, int res_ld, int res_coff, float *out, uint16_t *out16, int out_ld,
                               int out_coff, const sis3d_region *regions, int n_regions, int n_tiles, int cin, int cout, int ks,
                               int stride, int pad, int act, void *stream) {
    if (!in || !w_packed || (!out && !out16) || !regions || n_regions <= 0 || cin <= 0 || cout <= 0) return SIS3D_EINVAL;
    if (n_tiles <= 0) return SIS3D_OK;
    ConvArgs a;
    a.in = in; a.w = w_packed; a.bias = bias; a.res = residual; a.out = out; a.regions = regions;
    a.n_regions = n_regions; a.cin = cin; a.cout = cout; a.ldw = (cout + 3) & ~3; a.ks = ks; a.stride = stride;
    a.pad = pad; a.act = act; a.K = ks * ks * ks * cin; a.out_ld = out_ld; a.out_coff = out_coff;
    a.res_ld = res_ld; a.res_coff = res_coff; a.in_sc = in_chan_stride;
    a.fast = (in_chan_stride == 1 && cin % 16 == 0 && ((uintptr_t)in % 16 == 0)) ? 1 : 0;
    a.dense_m = 0; a.k_per_split = 0; a.split_stride = 0; a.out16 = (__half *)out16;
    cudaStream_t s = (cudaStream_t)stream;
    if (cout <= 32) {
        dim3 grid(n_tiles, cdiv(cout, 32));
        conv3d_igemm_f32<32, 2><<<grid, kConvThreads, 0, s>>>(a);
    } else {
        dim3 grid(n_tiles, cdiv(cout, 64));
        conv3d_igemm_f32<64, 4><<<grid, kConvThreads, 0, s>>>(a);
    }
    return finish_launch();
}

static int linear_splits(int M, int N, int K) {
    const int tiles = cdiv(M, BM) * cdiv(N, 64);
    int splits = max(1, min(K / 64, (2 * kNumSMs + tiles - 1) / tiles));
    return splits;
}
extern "C" size_t sis3d_linear_workspace_bytes(int M, int N, int K) {
    if (M <= 0 || N <= 0 || K <= 0) return 0;  // linear_splits divides by the tile count
    return sizeof(float) * (size_t)linear_splits(M, N, K) * M * N + 16;
}
extern "C" int sis3d_linear(const float *x, const float *w_packed, const float *bias, float *y, int M, int K, int N, int act,
                            void *workspace, size_t workspace_bytes, void *stream) {
    if (!x || !w_packed || !y || M <= 0 || K <= 0 || N <= 0 || K % 16 != 0 || ((uintptr_t)x & 15)) return SIS3D_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    int splits = linear_splits(M, N, K);
    ConvArgs a;
    a.in = x; a.w = w_packed; a.bias = bias; a.res = nullptr; a.out = y; a.regions = nullptr; a.n_regions = 0;
    a.cin = K; a.cout = N; a.ldw = (N + 3) & ~3; a.ks = 1; a.stride = 1; a.pad = 0; a.act = act; a.K = K;
    a.out_ld = N; a.out_coff = 0; a.res_ld = 0; a.res_coff = 0; a.in_sc = 1; a.fast = 1; a.dense_m = M;
    a.k_per_split = 0; a.split_stride = 0; a.out16 = nullptr;
    if (splits > 1) {
        if (!workspace || workspace_bytes < sizeof(float) * (size_t)splits * M * N) return SIS3D_EWORKSPACE;
        a.k_per_split = cdiv(cdiv(K, splits), BK) * BK;
        splits = cdiv(K, a.k_per_split);
        a.split_stride = (int64_t)M * N;
        a.out = (float *)workspace;
        a.bias = nullptr; a.act = 0;
    }
    dim3 grid(cdiv(M, BM), cdiv(N, N <= 32 ? 32 : 64), splits > 1 ? splits : 1);
    if (N <= 32) conv3d_igemm_f32<32, 2><<<grid, kConvThreads, 0, s>>>(a);
    else conv3d_igemm_f32<64, 4><<<grid, kConvThreads, 0, s>>>(a);
    if (splits > 1) {
        splitk_reduce_kernel<<<cdiv(M * N, 256), 256, 0, s>>>((const float *)workspace, splits, a.split_stride, bias, y, M, N, act);
        return finish_launch(2);
    }
    return finish_launch();
}

extern "C" int sis3d_maxpool3(const float *in, float *out, int out_ld, int out_coff, int X, int Y, int Z, int C, void *stream) {
    if (!in || !out || C % 4 != 0 || out_ld % 4 != 0 || out_coff % 4 != 0 || X <= 0 || Y <= 0 || Z <= 0) return SIS3D_EINVAL;
    if (C % (4 * kPoolCG4) == 0) {
        static bool attr_done = false;
        if (!attr_done) {
            if (cudaFuncSetAttribute(maxpool3_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPoolSmem) != cudaSuccess)
                return SIS3D_ELAUNCH;
            attr_done = true;
        }
        const int gx = cdiv(X, kPoolT), gy = cdiv(Y, kPoolT), gz = cdiv(Z, kPoolT);
        const int64_t nblk = (int64_t)gx * gy * gz * (C / (4 * kPoolCG4));
        if (nblk > 0x7fffffff) return SIS3D_EINVAL;
        maxpool3_tiled_kernel<<<(int)nblk, 256, kPoolSmem, (cudaStream_t)stream>>>((const float4 *)in, (float4 *)out, X, Y, Z, C / 4,
                                                                                 out_ld / 4, out_coff / 4, gy, gz);
        return finish_launch();
    }
    const int64_t total = (int64_t)X * Y * Z * (C / 4);
    const int blocks = (int)imin64(cdiv64(total, 256), kNumSMs * 16);
    maxpool3_vc_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4 *)in, (float4 *)out, X, Y, Z, C / 4, out_ld / 4, out_coff / 4);
    return finish_launch();
}

extern "C" int sis3d_vc_to_ncdhw(const float *in, float *out, int64_t nvox, int C, void *stream) {
    if (!in || !out || nvox <= 0 || C <= 0) return SIS3D_EINVAL;
    dim3 grid((unsigned)cdiv64(nvox, 32), cdiv(C, 32));
    vc_to_ncdhw_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(in, out, nvox, C);
    return finish_launch();
}
