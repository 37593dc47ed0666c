// enet2d.cu -- SURVEY row f2: fp32 implicit-GEMM 2-D convolution with a fused bias / residual / PReLU epilogue for the
// ENet encoder (reference: lib/nets/enet.py:130-590, called at lib/nets/network.py:204-205), NHWC activations.
// Part of libsis3d.so (C ABI in include/sis3d_enet.h); validated on the GPU against features of the unmodified reference
// ENet (tests/test_gpu_enet.py, max abs error 2e-6).
//
// GEMM view: M = N*Ho*Wo output pixels (tiles of 64), N = C_out, K = kh*kw*C_in with k = (ky*kw + kx)*C_in + c.
// A is gathered on the fly (zero outside the image == PyTorch zero padding), dilation and stride in the tap offsets;
// B is the packed weight [K][ldw].  Register tile 4 x 4 per thread (256 threads: 16 x 16), BK = 16, next chunk's global
// loads in flight while the current one is multiplied -- the structure of conv3d_igemm_f32 (conv_simt.cu).
#ifdef SIS3D_HOST_EMU  // host emulation build (tests/test_enet_executor.py): same source, blocks run as std::threads
#include "../emu_shims/host_emu.h"
#define SIS3D_LAUNCH(kernel, grid, block, stream, ...) emu_launch(kernel, grid, block, __VA_ARGS__)
#else
#include <cuda_runtime.h>
#define SIS3D_LAUNCH(kernel, grid, block, stream, ...) kernel<<<grid, block, 0, (cudaStream_t)(stream)>>>(__VA_ARGS__)
#endif
#include <math.h>
#include <stdint.h>
#include "sis3d_enet.h"

namespace {

constexpr int BK = 16, THREADS = 256, TN = 4, KTAB = 512;
constexpr int NUM_SMS = 132;  // H100 SXM

// N tile BN_ in {16, 32, 64} (ENet's bottleneck convs produce 16 / 32 channels: a fixed 64-wide tile wasted 50-75 % of the FMAs);
// 256 threads = (BN_/4) x (1024/BN_) register tiles of TM x 4, so the M tile is BM_ = TM * 1024 / BN_ rows (TM = 4: 256 / 128 /
// 64 rows; TM = 2 halves it for the launches whose grid would otherwise leave most SMs idle: 5 views of 32 x 41 pixels are
// only 6560 rows).
// VEC: NHWC input with C_in % 4 == 0 (every layer but the first): four consecutive k = four channels of one tap = ONE float4 load
// instead of four scalar gathers with their index arithmetic.  Per output the products are still accumulated k = 0 .. K-1 in
// order with fmaf, so every variant produces the same bits.
template <int BN_, bool VEC, int TM = 4>
__global__ void __launch_bounds__(THREADS) enet_conv2d_kernel(const sis3d_enet_conv a) {
    constexpr int NTX = BN_ / TN, NTY = THREADS / NTX, BM_ = NTY * TM, AS_LD = BM_ + 4;
    static_assert(BM_ % 64 == 0, "the A loader fills 64 rows per pass");
    constexpr int ROWS_PER_T = BM_ / 64;  // A loader: 64 rows x 4 k-quads per pass
    __shared__ __align__(16) float As[BK][AS_LD];
    __shared__ __align__(16) float Bs[BK][BN_];
    __shared__ int s_ktab[KTAB];  // k -> ky | kx << 4 | c << 8

    const int t = threadIdx.x;
    const int K = a.kh * a.kw * a.cin;
    for (int k = t; k < min(K, KTAB); k += THREADS) {
        const int tap = k / a.cin, c = k - tap * a.cin;
        const int ky = tap / a.kw, kx = tap - ky * a.kw;
        s_ktab[k] = ky | (kx << 4) | (c << 8);
    }
    __syncthreads();

    const int64_t m_total = (int64_t)a.N * a.Ho * a.Wo;
    const int64_t m_base = (int64_t)blockIdx.x * BM_;
    const int n0 = blockIdx.y * BN_;

    // A loader: rows lr + 64 p (p < ROWS_PER_T) of the tile, 4 consecutive k at lq*4
    const int lr = t >> 2, lq = t & 3;
    bool lvalid[ROWS_PER_T];
    int by[ROWS_PER_T], bx[ROWS_PER_T];
    const float *in_base[ROWS_PER_T];
#pragma unroll
    for (int p = 0; p < ROWS_PER_T; ++p) {
        const int64_t lm = m_base + lr + 64 * p;
        lvalid[p] = lm < m_total;
        int ln = 0, loy = 0, lox = 0;
        if (lvalid[p]) {
            ln = (int)(lm / ((int64_t)a.Ho * a.Wo));
            const int rem = (int)(lm - (int64_t)ln * a.Ho * a.Wo);
            loy = rem / a.Wo;
            lox = rem - loy * a.Wo;
        }
        by[p] = loy * a.stride - a.pad_y;
        bx[p] = lox * a.stride - a.pad_x;
        in_base[p] = a.in + (int64_t)ln * a.in_sn;
    }
    // B loader: row bk, 4 consecutive columns at bc
    const int bk = t / (BN_ / 4), bc = (t % (BN_ / 4)) * 4;
    const bool b_thread = t < BK * (BN_ / 4);

    const int tx = t % NTX, ty = t / NTX;
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    auto fetch = [&](int k0, float4 *av, float4 &bv) {
        const int kq = k0 + lq * 4;
        if constexpr (VEC) {
            int ky = 0, kx = 0, c = 0;
            const bool kin = kq < K;  // K % 4 == 0: the quad is either entirely inside or entirely outside
            if (kin) {
                if (kq < KTAB) {
                    const int e = s_ktab[kq];
                    ky = e & 15; kx = (e >> 4) & 15; c = e >> 8;
                } else {
                    const int tap = kq / a.cin;
                    c = kq - tap * a.cin;
                    ky = tap / a.kw;
                    kx = tap - ky * a.kw;
                }
            }
#pragma unroll
            for (int p = 0; p < ROWS_PER_T; ++p) {
                av[p] = make_float4(0.f, 0.f, 0.f, 0.f);
                const int iy = by[p] + ky * a.dil, ix = bx[p] + kx * a.dil;
                if (kin && lvalid[p] && (unsigned)iy < (unsigned)a.H && (unsigned)ix < (unsigned)a.W)
                    av[p] = __ldg(reinterpret_cast<const float4 *>(in_base[p] + (int64_t)iy * a.in_sy + (int64_t)ix * a.in_sx + c));
            }
        } else {
#pragma unroll
            for (int p = 0; p < ROWS_PER_T; ++p) {
                float tmp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int k = kq + i;
                    if (lvalid[p] && k < K) {
                        int ky, kx, c;
                        if (k < KTAB) {
                            const int e = s_ktab[k];
                            ky = e & 15; kx = (e >> 4) & 15; c = e >> 8;
                        } else {
                            const int tap = k / a.cin;
                            c = k - tap * a.cin;
                            ky = tap / a.kw;
                            kx = tap - ky * a.kw;
                        }
                        const int iy = by[p] + ky * a.dil, ix = bx[p] + kx * a.dil;
                        if ((unsigned)iy < (unsigned)a.H && (unsigned)ix < (unsigned)a.W)
                            tmp[i] = __ldg(in_base[p] + (int64_t)iy * a.in_sy + (int64_t)ix * a.in_sx + (int64_t)c * a.in_sc);
                    }
                }
                av[p] = make_float4(tmp[0], tmp[1], tmp[2], tmp[3]);
            }
        }
        bv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b_thread) {
            const int k = k0 + bk, n = n0 + bc;
            if (k < K && n < a.ldw) bv = __ldg(reinterpret_cast<const float4 *>(a.w + (int64_t)k * a.ldw + n));
        }
    };

    float4 av[ROWS_PER_T], bv;
    if (K > 0) fetch(0, av, bv);
    for (int k0 = 0; k0 < K; k0 += BK) {
        __syncthreads();
#pragma unroll
        for (int p = 0; p < ROWS_PER_T; ++p) {
            As[lq * 4 + 0][lr + 64 * p] = av[p].x;
            As[lq * 4 + 1][lr + 64 * p] = av[p].y;
            As[lq * 4 + 2][lr + 64 * p] = av[p].z;
            As[lq * 4 + 3][lr + 64 * p] = av[p].w;
        }
        if (b_thread) *reinterpret_cast<float4 *>(&Bs[bk][bc]) = bv;
        __syncthreads();
        if (k0 + BK < K) fetch(k0 + BK, av, bv);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float ar[TM];
            if constexpr (TM == 4) {
                const float4 v = *reinterpret_cast<const float4 *>(&As[k][ty * TM]);
                ar[0] = v.x; ar[1] = v.y; ar[2] = v.z; ar[3] = v.w;
            } else {
                const float2 v = *reinterpret_cast<const float2 *>(&As[k][ty * TM]);
                ar[0] = v.x; ar[1] = v.y;
            }
            const float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tx * TN]);
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                acc[i][0] = fmaf(ar[i], b.x, acc[i][0]);
                acc[i][1] = fmaf(ar[i], b.y, acc[i][1]);
                acc[i][2] = fmaf(ar[i], b.z, acc[i][2]);
                acc[i][3] = fmaf(ar[i], b.w, acc[i][3]);
            }
        }
    }

    // epilogue: + bias, + residual (optionally the floor-mode 2x2 max-pool of a res_h x res_w tensor, zero beyond res_c), PReLU
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t m = m_base + ty * TM + i;
        if (m >= m_total) continue;
        const int n_img = (int)(m / ((int64_t)a.Ho * a.Wo));
        const int rem = (int)(m - (int64_t)n_img * a.Ho * a.Wo);
        const int oy = rem / a.Wo, ox = rem - oy * a.Wo;
        float *orow = a.out + m * a.out_ld + a.out_coff;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int n = n0 + tx * TN + j;
            if (n >= a.cout) continue;
            float v = acc[i][j];
            if (a.bias) v += a.bias[n];
            if (a.res && n < a.res_c) {
                if (a.res_pool) {  // floor-mode pool: an odd res_h / res_w leaves the last row / column out
                    const int rw = a.res_w;
                    const float *r = a.res + (((int64_t)n_img * a.res_h + 2 * oy) * rw + 2 * ox) * a.res_ld + n;
                    v += fmaxf(fmaxf(r[0], r[a.res_ld]), fmaxf(r[(int64_t)rw * a.res_ld], r[((int64_t)rw + 1) * a.res_ld]));
                } else {
                    v += a.res[m * a.res_ld + n];
                }
            }
            if (a.slope) v = v >= 0.f ? v : v * a.slope[n];
            orow[n] = v;
        }
    }
}

__global__ void enet_pack_weight_kernel(const float *w, int cout, int cin, int kh, int kw, int ldw, float *out) {
    const int64_t total = (int64_t)kh * kw * cin * ldw;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int n = (int)(i % ldw);
        const int64_t k = i / ldw;
        const int c = (int)(k % cin), tap = (int)(k / cin);
        out[i] = n < cout ? w[((int64_t)n * cin + c) * (kh * kw) + tap] : 0.f;
    }
}

__global__ void enet_pool_affine_kernel(const float *in, int64_t sn, int64_t sy, int64_t sx, int64_t sc, int N, int H, int W, int C,
                                        const float *scale, const float *shift, const float *slope, float *out, int out_ld,
                                        int out_coff) {
    const int Ho = H / 2, Wo = W / 2;
    const int64_t total = (int64_t)N * Ho * Wo * C;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        int64_t p = i / C;
        const int ox = (int)(p % Wo);
        p /= Wo;
        const int oy = (int)(p % Ho), n = (int)(p / Ho);
        const float *q = in + n * sn + (int64_t)(2 * oy) * sy + (int64_t)(2 * ox) * sx + c * sc;
        float v = fmaxf(fmaxf(q[0], q[sx]), fmaxf(q[sy], q[sy + sx]));
        v = v * scale[c] + shift[c];
        v = v >= 0.f ? v : v * slope[c];
        out[(i / C) * out_ld + out_coff + c] = v;
    }
}

__global__ void enet_to_nchw_kernel(const float *in, int ld, int coff, int64_t P, int C, float *out) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int64_t p0 = (int64_t)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int64_t p = p0 + r;
        const int c = c0 + threadIdx.x;
        tile[r][threadIdx.x] = (p < P && c < C) ? in[((int64_t)n * P + p) * ld + coff + c] : 0.f;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int c = c0 + r;
        const int64_t p = p0 + threadIdx.x;
        if (p < P && c < C) out[((int64_t)n * C + c) * P + p] = tile[threadIdx.x][r];
    }
}

#ifdef SIS3D_HOST_EMU
inline int done() { return cudaGetLastError() == cudaSuccess ? 0 : -2; }
#else
}  // namespace
namespace sis3d { extern unsigned long long g_launch_count; }  // api.cu: host-side launch counter of libsis3d.so
namespace {
inline int done() {
    ++sis3d::g_launch_count;
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}
#endif

}  // namespace

extern "C" int sis3d_enet_pack_weight(const float *w, int cout, int cin, int kh, int kw, float *packed, void *stream) {
    if (!w || !packed || cout <= 0 || cin <= 0 || kh <= 0 || kw <= 0 || kh > 15 || kw > 15) return -1;
    const int ldw = (cout + 3) / 4 * 4;
    const int64_t total = (int64_t)kh * kw * cin * ldw;
    const int blocks = (int)((total + 255) / 256 < NUM_SMS * 8 ? (total + 255) / 256 : NUM_SMS * 8);
    SIS3D_LAUNCH(enet_pack_weight_kernel, dim3(blocks), dim3(256), stream, w, cout, cin, kh, kw, ldw, packed);
    return done();
}

extern "C" int sis3d_enet_conv2d(const sis3d_enet_conv *p, void *stream) {
    if (!p || !p->in || !p->w || !p->out) return -1;
    sis3d_enet_conv a = *p;
    if (a.N <= 0 || a.H <= 0 || a.W <= 0 || a.cin <= 0 || a.cout <= 0 || a.Ho <= 0 || a.Wo <= 0 || a.kh <= 0 || a.kw <= 0 ||
        a.kh > 15 || a.kw > 15 || a.stride <= 0 || a.dil <= 0 || a.ldw < a.cout || (a.ldw & 3) || a.out_ld < a.out_coff + a.cout)
        return -1;
    if (a.res && (a.res_c <= 0 || a.res_c > a.cout || a.res_ld < a.res_c)) return -1;
    // residual extent: [Ho][Wo], or for the pooled skip [2Ho or 2Ho + 1][2Wo or 2Wo + 1] (floor-mode 2x2/2 max-pool)
    if (a.res_h == 0 && a.res_w == 0) {  // extent not given: the output's, or twice it for the pooled skip
        a.res_h = (int16_t)(a.res_pool ? 2 * a.Ho : a.Ho);
        a.res_w = (int16_t)(a.res_pool ? 2 * a.Wo : a.Wo);
    }
    const bool res_fits = a.res_pool ? (a.res_h == 2 * a.Ho || a.res_h == 2 * a.Ho + 1) && (a.res_w == 2 * a.Wo || a.res_w == 2 * a.Wo + 1)
                                     : a.res_h == a.Ho && a.res_w == a.Wo;
    if (a.res && !res_fits) return -1;
    if (((uintptr_t)a.w) & 15) return -1;
    const int64_t m_total = (int64_t)a.N * a.Ho * a.Wo;
    // narrowest N tile that covers cout (16 / 32 / 64 per grid column), vectorised gather for NHWC inputs with C_in % 4 == 0
    const bool vec = a.in_sc == 1 && a.cin % 4 == 0 && ((uintptr_t)a.in & 15) == 0 && a.in_sx % 4 == 0 && a.in_sy % 4 == 0 && a.in_sn % 4 == 0;
    const int bn = a.cout <= 16 ? 16 : (a.cout <= 32 ? 32 : 64);
    const int ntiles = (a.cout + bn - 1) / bn;
    // TM = 2 (half-height M tiles) when the 4-row tiling would launch fewer than two CTAs per SM and the narrow N tile allows it
    const bool half = bn < 64 && ((m_total + 4096 / bn - 1) / (4096 / bn)) * ntiles < 2 * NUM_SMS;
    const int bm = (half ? 2048 : 4096) / bn;
    dim3 grid((unsigned)((m_total + bm - 1) / bm), (unsigned)ntiles);
#define SIS3D_ENET_GO(BNV, VECV, TMV) SIS3D_LAUNCH((enet_conv2d_kernel<BNV, VECV, TMV>), grid, dim3(THREADS), stream, a)
    if (bn == 16) {
        if (vec) { if (half) SIS3D_ENET_GO(16, true, 2); else SIS3D_ENET_GO(16, true, 4); }
        else { if (half) SIS3D_ENET_GO(16, false, 2); else SIS3D_ENET_GO(16, false, 4); }
    } else if (bn == 32) {
        if (vec) { if (half) SIS3D_ENET_GO(32, true, 2); else SIS3D_ENET_GO(32, true, 4); }
        else { if (half) SIS3D_ENET_GO(32, false, 2); else SIS3D_ENET_GO(32, false, 4); }
    } else {
        if (vec) SIS3D_ENET_GO(64, true, 4); else SIS3D_ENET_GO(64, false, 4);
    }
#undef SIS3D_ENET_GO
    return done();
}

extern "C" int sis3d_enet_pool_affine(const float *in, int64_t sn, int64_t sy, int64_t sx, int64_t sc, int N, int H, int W, int C,
                                      const float *scale, const float *shift, const float *slope, float *out, int out_ld,
                                      int out_coff, void *stream) {
    if (!in || !scale || !shift || !slope || !out || N <= 0 || H < 2 || W < 2 || C <= 0 || out_ld < out_coff + C) return -1;
    const int64_t total = (int64_t)N * (H / 2) * (W / 2) * C;
    const int blocks = (int)((total + 255) / 256 < NUM_SMS * 16 ? (total + 255) / 256 : NUM_SMS * 16);
    SIS3D_LAUNCH(enet_pool_affine_kernel, dim3(blocks), dim3(256), stream, in, sn, sy, sx, sc, N, H, W, C, scale, shift, slope, out, out_ld,
                 out_coff);
    return done();
}

extern "C" int sis3d_enet_to_nchw(const float *in, int ld, int coff, int N, int64_t P, int C, float *out, void *stream) {
    if (!in || !out || N <= 0 || P <= 0 || C <= 0 || ld < coff + C) return -1;
    dim3 grid((unsigned)((P + 31) / 32), (unsigned)((C + 31) / 32), (unsigned)N);
    SIS3D_LAUNCH(enet_to_nchw_kernel, grid, dim3(32, 8), stream, in, ld, coff, P, C, out);
    return done();
}
