// conv_tc.cu -- 3x3x3 (pad 1), 2x2x2 / stride 2 and 1x1x1 convolutions and fully connected layers as an implicit GEMM on the
// Hopper tensor cores (wgmma).
//
//   D[128 voxels x BN] (registers, fp32)  +=  A[128 x 32] (smem, TF32 / FP16)  x  B[BN x 32]^T (smem)
//
// * M tile = an 8x2x8 (x,y,z) brick of output voxels, rows ordered z (8 rows = one swizzle atom), y, x.  For every
//   (dy, dz) tap pair (9) and every 32-channel slice of C_in, ONE 4-D TMA box {32 ch, 8 z, 2 y, 10 x} fetches the
//   shifted input slab -- with a one-plane halo in x -- straight from the VC activation tensor; the three x-taps then
//   read rows [16 dx, 16 dx + 128) of that slab, an offset of two whole swizzle atoms, so the descriptor just moves by
//   2 KB: A traffic is 9 x 1.25 instead of 27 bricks per K slice (2.4x less).  Voxels outside the volume are zero-filled
//   by the TMA unit, which *is* the convolution's zero padding -- no halo logic, no im2col buffer.  Rows land 128 B
//   apart in the canonical K-major SWIZZLE_128B layout wgmma reads through its shared-memory descriptors.
// * B tiles = BN rows of the weight matrix W[C_out][27*C_in] (k = tap*C_in + c) for the three x-taps, 2-D TMA, same swizzle.
// * Warp roles (384 threads = three warpgroups): warpgroup 0: thread 0 = TMA producer, warps 1-3 = operand splitters (X3);
//   warpgroups 1 and 2 = consumers: each issues wgmma.mma_async m64nBNk8 (tf32) / m64nBNk16 (f16) for its 64 rows of the
//   brick, keeps the fp32 accumulator in registers and runs the epilogue (bias / residual / ReLU -> global) from them.
//   Full/empty mbarrier ring; a consumer warpgroup releases a stage once its wgmma group has retired.
// * Tiles may be listed explicitly (ragged RoI crops packed on one zero-separated canvas, mask head)
//   or implied by the volume.
//
// Reference call sites: Bottleneck.conv2 (lib/nets/backbones.py:21), geometry2.0 (:216),
// rpn_net_level{1,2} (lib/nets/network.py:40,45), MaskBackbone.geometry.{2,4,6,8} (backbones.py:243-249).
#include <cuda.h>
#include <stdlib.h>
#include <string.h>
#include <cuda_fp16.h>
#include "common.cuh"

namespace sis3d {

constexpr int TC_BZ = 8;  // brick = (16/BY) x BY x 8 voxels (x,y,z), BY in {2,4}; rows ordered z (8 = one swizzle atom), y, x
constexpr int TC_BM = 128;
constexpr int TC_KC = 32;  // channels per stage: 32 * 4 B = 128 B = one swizzle row
constexpr int TC_THREADS = 384;

struct TcArgs {
    const float *bias, *res;
    float *out;
    const int32_t *tiles;  // [n_tiles][8] = x0,y0,z0,x1,y1,z1,-,- (origin, exclusive valid end) or null
    int X, Y, Z, cin, cout, act, out_ld, out_coff, res_ld, res_coff;
    int tiles_y, tiles_z;
    int gemm_m, gemm_chunks_per_split;  // KS == 0 (plain GEMM y = x W^T, split-K over blockIdx.z)
    __half *out16;                      // optional fp16 twin of the output (same geometry as `out`); `out` may be null
    const float *bias_mid;              // N2 > 0: bias of the 3x3x3 conv (added before the inner ReLU), or null
    int n_tiles;                        // bricks of this launch (the grid may be padded to a multiple of the cluster size)
    __half *out_split;                  // X3 = 2, KS = 1: optional split-pair output ([32 hi | 32 lo] halves per voxel and
                                        // 32-channel slice, row stride 2 cout); `out` may then be null
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done, spins = 0;
    do {
        if (++spins > (1u << 28)) __trap();  // a broken pipeline becomes a CUDA error, never a hung GPU
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}
// arrive on the barrier at the same shared-memory offset in CTA `rank` of the cluster (rank = own rank for CL = 1)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t *bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// cluster variants (CL = 2: two CTAs = two bricks of the same N tile share every weight tile: each CTA fetches half of them and
// multicasts to both -> half the weight bytes per SM over the L2->SM crossbar, which bounds the wide / weight-heavy layers)
__device__ __forceinline__ void tma_load_2d_mc(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%4, %5}], [%2], %3;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

// K-major shared-memory matrix descriptor of wgmma (cute::GMMA::DescriptorIterator bit layout):
// start>>4 [0,14) | LBO=1 [16,30) (unused by the swizzled K-major layouts) | SBO = 8 rows >>4 [32,46) | layout [62,64)
// ROWB = 128: SWIZZLE_128B (layout 1, 8-row atom = 1024 B);  ROWB = 64: SWIZZLE_64B (layout 2, 8-row atom = 512 B)
template <int ROWB>
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr) {
    constexpr uint64_t sbo = (8 * ROWB) >> 4, layout = ROWB == 128 ? 1 : 2;
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (sbo << 32) | (layout << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (+)= A[64 x K] . B[N x K]^T, both operands K-major in shared memory; d = this thread's N/2 accumulator registers
// (d[4j + 2h + e] = row 16 (warp % 4) + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e); scale_d = 0 overwrites d
__device__ __forceinline__ void wgmma_tf32_n32(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n64(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n128(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n32(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n64(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n128(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d));
}
template <int N, bool F16>
__device__ __forceinline__ void wgmma(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
    static_assert(N == 32 || N == 64 || N == 128, "wgmma tile widths of this file");
    if constexpr (F16) {
        if constexpr (N == 32) wgmma_f16_n32(d, a, b, scale_d);
        else if constexpr (N == 64) wgmma_f16_n64(d, a, b, scale_d);
        else wgmma_f16_n128(d, a, b, scale_d);
    } else {
        if constexpr (N == 32) wgmma_tf32_n32(d, a, b, scale_d);
        else if constexpr (N == 64) wgmma_tf32_n64(d, a, b, scale_d);
        else wgmma_tf32_n128(d, a, b, scale_d);
    }
}

// v = hi + lo with hi = tf32(v) (round to nearest, low 13 bits zero) and lo = tf32(v - hi) (v - hi is exact in fp32)
__device__ __forceinline__ float tf32_rna_bits(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ void split_tf32(float v, float &hi, float &lo) {
    hi = tf32_rna_bits(v);
    lo = tf32_rna_bits(v - hi);
}

// fp16 split (X3 = 2): v = hi + lo / 2048 with hi = fp16(v) (round to nearest) and lo = fp16((v - hi) * 2048): the same
// 11 + 11 significand bits as the TF32 split, but the MMAs run at the fp16 rate (twice the TF32 rate of the H100 tensor core).
// Scaling the low part keeps it out of fp16's subnormal range; |v| is clamped to the fp16 range first.
__device__ __forceinline__ void split_f16(float v, __half &hi, __half &lo) {
    v = fminf(fmaxf(v, -65504.f), 65504.f);
    hi = __float2half_rn(v);
    lo = __float2half_rn((v - __half2float(hi)) * 2048.0f);
}
// activations, two at a time with packed conversions (4 ALU ops per element); precondition |v| < 65504 (not clamped here: the
// fp16-operand mask stage of the default math mode has the same range requirement)
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t &hi, uint32_t &lo) {
    const __half2 h = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn((a - hf.x) * 2048.0f, (b - hf.y) * 2048.0f);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}
__device__ __forceinline__ void split_f16x8(const float4 a, const float4 b, uint4 &hi, uint4 &lo) {
    split_f16x2(a.x, a.y, hi.x, lo.x);
    split_f16x2(a.z, a.w, hi.y, lo.y);
    split_f16x2(b.x, b.y, hi.z, lo.z);
    split_f16x2(b.z, b.w, hi.w, lo.w);
}

// stages: 4 for BN = 128 (128 KB), 3 for BN <= 64
template <int BN>
struct TcStages { static constexpr int value = BN >= 128 ? 4 : 3; };
// stage count per kernel flavour: the 3x3x3 stages are 3x bigger (slab + three weight tiles)
// X3 = 1 (error-compensated 3xTF32, 64-byte K rows): every stage also holds the low parts of A and B; BN = 32 keeps three
// stages (96 KB), BN = 64 two (88 KB), BN = 128 three (204 KB)
// X3 = 2 (fp16 split, 128-byte fp32 source rows): a stage = the slab (fp32 as it lands, split IN PLACE into fp16 hi / lo tiles of
// half the size each) + fp16 hi/lo weight tiles.  3x3x3: BN = 32: three stages of 32 KB, BN = 64: four of 44 KB, BN = 128:
// three of 68 KB; 1x1 / 2x2x2 / GEMM: four.  A fused tail fed split-pair activations (PS) uses the same stages: its slab lands
// as [hi | lo] fp16 rows of the same 128 bytes and is read where it landed.
// Every configuration stays within the 227 KB of shared memory an H100 block may use.  How many CTAs share an SM is set by
// registers (tc_min_blocks below), not by shared memory.
template <int BN, int KS, int ROWB, int X3 = 0, int N2 = 0>
struct TcStagesOf {
    static constexpr int value =
        X3 == 2 ? (KS == 3 ? (BN == 64 ? 4 : 3) : 4)
                : (KS == 3 ? (X3 ? (BN == 64 ? 2 : 3) : (BN >= 128 ? 3 : 2)) : TcStages<BN>::value);
};
// CTAs per SM the kernel is compiled for (384 threads each): two for BN = 32, whose 16-register accumulators fit the 80
// registers that leaves (one CTA's prologue / epilogue runs under the other's main loop), except the fp16-split 1x1, 2x2x2
// and fused-tail kernels that split their A operand in shared memory: the splitter warps' staging registers would spill or
// have the wgmmas serialized at 80 registers.  The fused tail fed a pre-split A operand (PS) has no splitter and runs two
// CTAs per SM (2 x 104-108 KB of shared memory).  Every BN >= 64 kernel needs more than 80 registers and runs one CTA per SM.
template <int BN, int KS, int N2, int X3, bool PS = false>
constexpr int tc_min_blocks() {
    return (BN == 32 && (PS || !(X3 == 2 && (KS == 1 || KS == 2 || N2 > 0)))) ? 2 : 1;
}
template <int BN, int KS, int ROWB, int BY, int N2 = 0, int X3 = 0>
constexpr size_t tc_smem_bytes() {
    // bytes of one weight row in shared memory: ROWB, or 64 (32 fp16 channels) in the fp16-split mode
    return (size_t)TcStagesOf<BN, KS, ROWB, X3, N2>::value *
               ((X3 == 1 ? 2 : 1) * (KS == 3 ? (16 / BY + 2) * BY * TC_BZ : TC_BM) * ROWB +
                (X3 == 1 ? 2 : 1) * (KS == 3 ? 3 : 1) * BN * (X3 == 2 ? 128 : ROWB)) +
           (size_t)(X3 == 1 ? 2 : 1) * N2 * 128 * (BN / 32) + 1024 + 256;
}

// EB = operand element bytes: 4 -> fp32 storage, TF32 wgmma;  2 -> fp16 storage, f16 wgmma (same 11-bit significand,
// half the operand bytes through L2).  ROWB = bytes of one K slice row in shared memory (128, or 64 for C_in = 32 in fp16).
//
// N2 > 0 (KS = 3, EB = 4) fuses the bottleneck's trailing 1x1 convolution (lib/nets/backbones.py:28-40: conv2 -> relu ->
// conv3 -> +x -> relu): the ReLU'd 128 x BN accumulator is written back to shared memory as a K-major swizzled operand
// (aliasing the drained pipeline stages), multiplied by W3[N2][BN] (its own TMA tile, fetched at kernel start) into a second
// register accumulator, and only that N2-wide result -- plus residual and ReLU -- goes to global memory.  The BN-wide
// intermediate never leaves the SM; operand values and summation order equal the two-kernel path bit for bit.
//
// X3 = 1 (EB = 4 only): error-compensated 3xTF32.  Every fp32 operand is split as v = hi + lo with hi = tf32(v) (round to
// nearest) and lo = tf32(v - hi); the product is accumulated as A_lo.B_hi + A_hi.B_lo + A_hi.B_hi (the dropped A_lo.B_lo term
// is ~2^-22 relative).  Weights are split once at pack time ([2][cout][K]: hi rows, then lo rows); the activation slab is split
// IN SHARED MEMORY by the splitter warps after the TMA lands (hi overwrites the slab, lo goes to a second buffer of the same
// swizzled layout -- the split is elementwise, so the layout is untouched), published to wgmma's async proxy with
// fence.proxy.async + the conv_done mbarrier.  No extra L2->SM traffic for activations.  The tensor core adds into its fp32
// accumulator with truncation, a bias that grows with the length of the accumulation chain -- invisible next to TF32 operand
// rounding, but the dominant error of the compensated product.  So each stage's products go to a fresh register
// accumulator (a chain of at most 18 MMAs), which is then added to the running sum with round-to-nearest FADDs.  Result:
// fp32-class accuracy (the integer outputs of the detector -- top-N order, NMS keep lists, class argmax, crop bounds -- match
// the fp32 path) on the tensor cores.
//
// X3 = 2 (EB = 4, ROWB = 128): the same compensation with an fp16 split (split_f16 above): the fp32 slab lands in a staging
// buffer, the splitter warps write its hi and (scaled) lo parts as two fp16 K-major SWIZZLE_64B tiles, the weights are
// pre-split fp16 tiles, and the three products are f16 wgmmas -- same 22 significand bits, twice the MMA rate.  The scaled
// cross terms are a wgmma group of their own, folded into the running sum as fmaf(cross, 2^-11, sum).
//
// Split-pair activations (X3 = 2): [32 fp16 hi | 32 fp16 lo] per voxel and 32-channel slice, one 128-byte row, hi and lo
// exactly as split_f16x2 makes them (the layout of the fp16-split weights).  The 1x1 kernel writes this format from its
// post-bias / ReLU fp32 value when a.out_split is set; the fused tail with PS = true reads it as its A operand: the TMA box
// {64 halves, 8 z, 2 y, 10 x} lands as SWIZZLE_128B rows, hi at +0 and lo at +64 -- the same descriptors as the weights --
// so there are no splitter warps, no conv_done handoff and no proxy fence per stage.  The operand bits and the MMA order are
// those of the fp32-input tail, so its result is bit-identical.
template <int BN, int KS, int EB = 4, int ROWB = 128, int BY = 2, int N2 = 0, int X3 = 0, int CL = 1, bool PS = false>
__global__ void __launch_bounds__(TC_THREADS, tc_min_blocks<BN, KS, N2, X3, PS>()) conv3d_k3_tc_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                                  const __grid_constant__ CUtensorMap tmB,
                                                                                  const __grid_constant__ CUtensorMap tmB2,
                                                                                  const TcArgs a) {
    static_assert(N2 == 0 || (KS == 3 && EB == 4), "conv3 fusion: fp32-stored 3x3x3 kernels only");
    static_assert(X3 == 0 || EB == 4, "3xTF32 splits fp32-stored operands");
    static_assert(X3 != 2 || ROWB == 128, "the fp16 split reads 128-byte fp32 rows and writes 64-byte fp16 rows");
    static_assert(CL == 1 || (CL == 2 && KS == 3), "weight-tile multicast: pairs of 3x3x3 bricks");
    static_assert(!PS || (X3 == 2 && KS == 3 && N2 > 0 && CL == 1), "pre-split A operand: fp16-split fused tails");
    constexpr bool XH = X3 == 2;             // fp16 split
    constexpr bool SPLITTER = X3 && !PS;     // warps 1-3 split the A slab in shared memory
    constexpr int AOPB = PS ? 128 : (XH ? 64 : ROWB);  // bytes of one A operand row in shared memory (PS: [hi | lo] per row)
    constexpr bool F16 = EB == 2 || XH;      // f16 (else TF32) wgmma
    constexpr int NSPLIT = 96;               // splitter threads: warps 1-3
    constexpr int OPB = XH ? 64 : ROWB;      // bytes of one K-slice row of the MMA operands in shared memory
    constexpr int KC = ROWB / EB;            // channels per pipeline stage
    constexpr int TC_BY = BY, TC_BX = 16 / BY;  // brick: BY = 2 -> 8x2x8 (whole volumes), BY = 4 -> 4x4x8 (small RoI crops)
    // 3x3x3: one stage = one (dy, dz) pair: an x-halo slab of (8+2) x-planes (160 rows) serves the three x-taps --
    // tap dx reads rows [dx*16, dx*16+128), a whole-swizzle-atom offset -- plus the three taps' weight tiles.
    constexpr int XT = KS == 3 ? 3 : 1;      // x-taps per stage
    constexpr int A_ROWS = KS == 3 ? (TC_BX + 2) * TC_BY * TC_BZ : TC_BM;
    constexpr int A_BYTES = A_ROWS * ROWB;
    // weight tiles: X3 = 2 keeps the hi and lo halves of a 32-channel K slice side by side in ONE 128-byte row (one TMA row
    // request instead of two 64-byte ones), SWIZZLE_128B; hi = first 64 bytes, lo = last 64
    constexpr int BROW = XH ? 128 : OPB;
    constexpr int NBT = XT * (X3 == 1 ? 2 : 1);  // weight tiles per stage
    constexpr int B_BYTES = BN * BROW;
    // stage layout: X3 = 0: [A | B x XT];  X3 = 1: [A_hi (in place) | A_lo | B_hi x XT | B_lo x XT];
    //               X3 = 2: [A: fp32 as landed -> split in place into A_hi fp16 | A_lo fp16 (half of A_BYTES each) | B x XT]
    constexpr int B_OFF = (X3 == 1 ? 2 : 1) * A_BYTES;
    constexpr int STAGE_BYTES = B_OFF + NBT * B_BYTES;
    constexpr int TC_STAGES = TcStagesOf<BN, KS, ROWB, X3, N2>::value;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // SWIZZLE_128B needs 1024 B alignment
    // W3 as BN/32 K slices of [N2 rows][32 ch] (X3 = 1: hi slices, then lo slices; fp16 split: [32 hi | 32 lo] halves per row)
    constexpr int B2_SLICE = N2 * 128;
    constexpr int B2_BYTES = (X3 == 1 ? 2 : 1) * B2_SLICE * (BN / 32);
    uint8_t *smem_b2 = smem + TC_STAGES * STAGE_BYTES;
    uint64_t *full = reinterpret_cast<uint64_t *>(smem_b2 + B2_BYTES);
    uint64_t *empty = full + TC_STAGES;
    uint64_t *b2_full = empty + TC_STAGES;
    uint64_t *conv_done = b2_full + 1;  // X3: the splitter warps finished splitting stage s

    const int warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        // empty: one arrival per consumer warpgroup of every CTA of the cluster (the peer's producer multicasts into this slot too)
        for (int i = 0; i < TC_STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 2 * CL); mbar_init(conv_done + i, NSPLIT); }
        mbar_init(b2_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    uint32_t crank = 0;
    if constexpr (CL > 1) {
        // both CTAs' barriers are initialised before either multicasts into the other's shared memory / arrives on its barriers
        cluster_sync_all();
        crank = cluster_ctarank();
    }

    // ---- which brick
    int x0 = 0, y0 = 0, z0 = 0, x1 = 0, y1 = 0, z1 = 0;
    if constexpr (KS == 0) {
        // GEMM mode: rows instead of bricks (x0 = first row, set below)
    } else if (a.tiles) {
        const int32_t *t = a.tiles + (size_t)min((int)blockIdx.x, a.n_tiles - 1) * 8;
        x0 = t[0]; y0 = t[1]; z0 = t[2]; x1 = t[3]; y1 = t[4]; z1 = t[5];
        if ((int)blockIdx.x >= a.n_tiles) x1 = y1 = z1 = 0;  // cluster padding: runs the pipeline (its peer needs it), stores nothing
    } else {
        const int tz = blockIdx.x % a.tiles_z, ty = (blockIdx.x / a.tiles_z) % a.tiles_y, tx = blockIdx.x / (a.tiles_z * a.tiles_y);
        x0 = tx * TC_BX; y0 = ty * TC_BY; z0 = tz * TC_BZ;
        x1 = min(x0 + TC_BX, a.X); y1 = min(y0 + TC_BY, a.Y); z1 = min(z0 + TC_BZ, a.Z);
    }
    const int n0 = blockIdx.y * BN;
    const int kchunks = a.cin / KC;
    constexpr int TAPS = KS == 3 ? 9 : KS == 2 ? 8 : 1;  // pipeline steps per K slice: 9 (dy,dz) pairs (3x3x3), 8 taps (2x2x2/s2), else 1
    int total = TAPS * kchunks, chunk0 = 0;
    if constexpr (KS == 0) {  // split-K GEMM: this CTA owns K chunks [chunk0, chunk0 + total)
        chunk0 = blockIdx.z * a.gemm_chunks_per_split;
        total = max(0, min(a.gemm_chunks_per_split, kchunks - chunk0));
        x0 = blockIdx.x * TC_BM;  // row offset m0
    }

    if (threadIdx.x == 0) {
        // ===== TMA producer =====
        if constexpr (N2 > 0) {
            mbar_expect_tx(b2_full, B2_BYTES);
#pragma unroll
            for (int h = 0; h < (X3 == 1 ? 2 : 1); ++h)  // X3 = 1: rows [N2, 2 N2) of the split W3 are the low parts
#pragma unroll
                for (int kc = 0; kc < BN / 32; ++kc)  // X3 = 2: one 64-half row per K slice = [32 hi | 32 lo]
                    tma_load_2d(smem_b2 + (h * (BN / 32) + kc) * B2_SLICE, &tmB2, b2_full, kc * (XH ? 64 : 32), h * N2);
        }
        for (int it = 0; it < total; ++it) {
            const int s = it % TC_STAGES;
            const uint32_t ph = (it / TC_STAGES) & 1;
            mbar_wait(empty + s, ph ^ 1);
            mbar_expect_tx(full + s, STAGE_BYTES - (X3 == 1 ? A_BYTES : 0));  // X3 = 1: A_lo is written by the splitter warps, not by TMA
            const int tap = it / kchunks, kc = it - tap * kchunks;
            uint8_t *sa = smem + s * STAGE_BYTES;
            if constexpr (KS == 0) {
                tma_load_2d(sa, &tmA, full + s, (chunk0 + it) * KC, x0);
                tma_load_2d(sa + B_OFF, &tmB, full + s, (chunk0 + it) * KC * (XH ? 2 : 1), n0);
                if constexpr (X3 == 1) tma_load_2d(sa + B_OFF + B_BYTES, &tmB, full + s, (chunk0 + it) * KC, a.cout + n0);
            } else if constexpr (KS == 1) {
                tma_load_4d(sa, &tmA, full + s, kc * KC, z0, y0, x0);
                tma_load_2d(sa + B_OFF, &tmB, full + s, kc * KC * (XH ? 2 : 1), n0);
                if constexpr (X3 == 1) tma_load_2d(sa + B_OFF + B_BYTES, &tmB, full + s, kc * KC, a.cout + n0);
            } else if constexpr (KS == 2) {
                // 2x2x2 / stride 2: the tensor map traverses the input with element strides {1,2,2,2}, so the box that starts
                // at input voxel (2 x0 + dx, 2 y0 + dy, 2 z0 + dz) lands as the 128 output rows of this brick for tap (dx,dy,dz)
                const int dx = tap >> 2, dy = (tap >> 1) & 1, dz = tap & 1;
                tma_load_4d(sa, &tmA, full + s, kc * KC, 2 * z0 + dz, 2 * y0 + dy, 2 * x0 + dx);
                tma_load_2d(sa + B_OFF, &tmB, full + s, (tap * a.cin + kc * KC) * (XH ? 2 : 1), n0);
                if constexpr (X3 == 1) tma_load_2d(sa + B_OFF + B_BYTES, &tmB, full + s, tap * a.cin + kc * KC, a.cout + n0);
            } else {
                const int dy = tap / 3, dz = tap % 3;  // tap = (dy, dz) pair; the slab covers x0-1 .. x0+8
                // (PS: the channel coordinate counts halves, two per channel)
                tma_load_4d(sa, &tmA, full + s, kc * KC * (PS ? 2 : 1), z0 + dz - 1, y0 + dy - 1, x0 - 1);
#pragma unroll
                for (int j = 0; j < NBT; ++j) {  // weight tiles: x-taps 0..2 (X3 = 1: hi tiles, then the low parts' tiles)
                    const int dx = j % 3, row0 = (j >= 3 ? a.cout : 0) + n0;
                    // weight columns k = ((dx*3+dy)*3+dz)*C_in + c  (X3 = 2: two halves per k -- [32 hi | 32 lo] per K slice)
                    const int kcol = (((dx * 3 + dy) * 3 + dz) * a.cin + kc * KC) * (XH ? 2 : 1);
                    if constexpr (CL == 1) {
                        tma_load_2d(sa + B_OFF + j * B_BYTES, &tmB, full + s, kcol, row0);
                    } else if ((uint32_t)(j % CL) == crank) {  // this CTA's share of the pair's weight tiles, delivered to both
                        tma_load_2d_mc(sa + B_OFF + j * B_BYTES, &tmB, full + s, kcol, row0, (uint16_t)((1u << CL) - 1u));
                    }
                }
            }
        }
    } else if (SPLITTER && warp >= 1 && warp <= 3) {
        // ===== operand splitter (warps 1-3) =====
        const int t = threadIdx.x - 32;
        for (int it = 0; it < total; ++it) {
            const int s = it % TC_STAGES;
            mbar_wait(full + s, (it / TC_STAGES) & 1);
            uint8_t *st = smem + s * STAGE_BYTES;
            if constexpr (XH) {
                // fp32 slab (128-byte rows, SWIZZLE_128B: 16-byte chunk j of row r at r*128 + ((j ^ (r & 7)) << 4)) ->
                // fp16 hi / lo tiles (64-byte rows, SWIZZLE_64B: chunk q of row r at r*64 + ((q ^ ((r >> 1) & 3)) << 4)), IN PLACE:
                // hi takes the first half of the slab's bytes, lo the second.  One work item = 8 channels of one row = source
                // chunks 2q, 2q+1 -> destination chunk q.  Every splitter thread converts its items into registers, the splitter
                // warps meet at a named barrier (all of the fp32 data has been read), then the fp16 tiles are stored.
                constexpr int ITEMS = (A_ROWS * 4 + NSPLIT - 1) / NSPLIT;
                uint4 h[ITEMS], l[ITEMS];
#pragma unroll
                for (int u = 0; u < ITEMS; ++u) {
                    const int i = t + u * NSPLIT;
                    if (i < A_ROWS * 4) {
                        const int r = i >> 2, q = i & 3;
                        const float4 v0 = *reinterpret_cast<const float4 *>(st + r * 128 + (((2 * q) ^ (r & 7)) << 4));
                        const float4 v1 = *reinterpret_cast<const float4 *>(st + r * 128 + (((2 * q + 1) ^ (r & 7)) << 4));
                        split_f16x8(v0, v1, h[u], l[u]);
                    }
                }
                asm volatile("bar.sync 1, %0;" ::"n"(NSPLIT) : "memory");
#pragma unroll
                for (int u = 0; u < ITEMS; ++u) {
                    const int i = t + u * NSPLIT;
                    if (i < A_ROWS * 4) {
                        const int r = i >> 2, q = i & 3;
                        const int d = r * 64 + ((q ^ ((r >> 1) & 3)) << 4);
                        *reinterpret_cast<uint4 *>(st + d) = h[u];
                        *reinterpret_cast<uint4 *>(st + A_BYTES / 2 + d) = l[u];
                    }
                }
            } else {
                // slab -> hi (in place) + lo (second buffer): the split is elementwise, so the swizzled layout is untouched
                float4 *hi = reinterpret_cast<float4 *>(st);
                float4 *lo = reinterpret_cast<float4 *>(st + A_BYTES);
#pragma unroll 2
                for (int i = t; i < A_BYTES / 16; i += NSPLIT) {
                    const float4 v = hi[i];
                    float4 h, l;
                    split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y); split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
                    hi[i] = h;
                    lo[i] = l;
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to wgmma's async proxy
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(conv_done + s)) : "memory");
        }
    } else if (warp >= 4) {
        // ===== consumer warpgroups: wgmma over rows [64 wg, 64 wg + 64) of the brick, then the epilogue =====
        const int wg = (warp >> 2) - 1, tw = threadIdx.x & 127;
        const uint32_t row_off = (uint32_t)(wg * 64);  // first A row of this warpgroup
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int it = 0; it < total; ++it) {
            const int s = it % TC_STAGES;
            const uint32_t ph = (it / TC_STAGES) & 1;
            mbar_wait(SPLITTER ? conv_done + s : full + s, ph);  // splitter: the split (which itself waited for the TMA) is done
            const uint32_t sa = smem_u32(smem + s * STAGE_BYTES), sb = sa + B_OFF;
            // operand tiles: X3 = 1: hi at sa (in place), lo at sa + A_BYTES; X3 = 2: fp16 hi at sa (in place), lo half an A_BYTES on;
            // PS: [hi | lo] halves of each 128-byte row as landed
            const uint32_t a_hi = sa + row_off * AOPB;
            const uint32_t a_lo = PS ? a_hi + 64 : sa + (XH ? A_BYTES / 2 : A_BYTES) + row_off * OPB;
            float part[X3 ? BN / 2 : 1];  // X3: this stage's products (a fresh, short accumulation chain)
            // X3 = 1: one group, A_lo.B_hi + A_hi.B_lo + A_hi.B_hi (smallest terms first).  X3 = 2: the low parts are scaled by
            // 2^11, so the cross terms are a group of their own, added scaled back (pass 0), before the A_hi.B_hi group (pass 1)
#pragma unroll
            for (int pass = 0; pass < (XH ? 2 : 1); ++pass) {
                wgmma_fence();
#pragma unroll
                for (int dx = 0; dx < XT; ++dx) {
                    // x-tap dx: A rows start 16 rows (= two 8-row swizzle atoms) further into the slab
                    const uint32_t ax = a_hi + dx * (TC_BY * TC_BZ) * AOPB, al_x = a_lo + dx * (TC_BY * TC_BZ) * AOPB, bx = sb + dx * B_BYTES;
#pragma unroll
                    for (int k = 0; k < OPB / 32; ++k) {  // one MMA consumes 32 B of K (8 tf32 / 16 f16): advance inside the swizzle atom
                        if constexpr (X3) {
                            const uint64_t ah = gmma_desc<AOPB>(ax + k * 32), al = gmma_desc<AOPB>(al_x + k * 32);
                            const uint64_t bh = gmma_desc<BROW>(bx + k * 32);
                            const uint64_t bl = XH ? gmma_desc<BROW>(bx + 64 + k * 32) : gmma_desc<BROW>(bx + XT * B_BYTES + k * 32);
                            if (pass == 0) {
                                wgmma<BN, F16>(part, al, bh, (dx | k) ? 1u : 0u);
                                wgmma<BN, F16>(part, ah, bl, 1u);
                            }
                            if (!XH || pass == 1) wgmma<BN, F16>(part, ah, bh, (XH && !(dx | k)) ? 0u : 1u);
                        } else {
                            wgmma<BN, F16>(acc, gmma_desc<ROWB>(ax + k * 32), gmma_desc<ROWB>(bx + k * 32), 1u);
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait_all();
                if constexpr (X3) {
                    const float sc = (XH && pass == 0) ? 1.0f / 2048.0f : 1.0f;
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) acc[i] = fmaf(part[i], sc, acc[i]);  // round-to-nearest
                }
            }
            // this warpgroup no longer reads stage s (cluster: release it in BOTH CTAs -- the peer's producer multicasts into it)
            if (tw == 0) {
                if constexpr (CL == 1) {
                    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(empty + s)) : "memory");
                } else {
#pragma unroll
                    for (int c = 0; c < CL; ++c) mbar_arrive_cluster(empty + s, (uint32_t)c);
                }
            }
        }

        const int g = (tw & 31) >> 2, q = tw & 3;
        const int rbase = wg * 64 + (tw >> 5) * 16 + g;  // this thread's brick rows: rbase, rbase + 8
        if constexpr (KS == 0) {
            // ===== GEMM epilogue: raw fp32 partial sums of this K split -> partial[z][m][n] (bias/ReLU in the reduce pass)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = x0 + rbase + 8 * h;
                if (m >= a.gemm_m) continue;
                float *prow = a.out + ((int64_t)blockIdx.z * a.gemm_m + m) * a.out_ld + n0;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
                    *reinterpret_cast<float2 *>(prow + 8 * j + 2 * q) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        } else {
            constexpr int NOUT = N2 > 0 ? N2 : BN;
            float acc2[N2 > 0 ? N2 / 2 : 1];
            const float *res_acc = acc;
            if constexpr (N2 > 0) {
                // conv2's tile -> ReLU -> shared memory as the A operand of the 1x1 conv: row r, 16-byte chunk j of K slice kc at
                // kc*16 KB + r*128 + ((j ^ (r & 7)) << 4)  (the canonical SWIZZLE_128B K-major layout TMA would have produced);
                // fp16 split: 64-byte rows, chunk q of 8 channels at r*64 + ((q ^ ((r >> 1) & 3)) << 4) (SWIZZLE_64B)
                uint8_t *a2 = smem;  // aliases the pipeline stages: every TMA write landed and every MMA reading them retired
                constexpr int A2_SLICE = TC_BM * (XH ? 64 : 128);
                constexpr int A2_BYTES = (BN / 32) * A2_SLICE;
                asm volatile("bar.sync 2, 256;" ::: "memory");  // both consumer warpgroups are past their last read of the stages
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = rbase + 8 * h;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j) {
                        const int c = 8 * j + 2 * q, kc = c >> 5, cc = c & 31;
                        float o0 = acc[4 * j + 2 * h], o1 = acc[4 * j + 2 * h + 1];
                        if (a.bias_mid) {
                            const float2 b = __ldg(reinterpret_cast<const float2 *>(a.bias_mid + c));
                            o0 += b.x; o1 += b.y;
                        }
                        o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f);
                        uint8_t *row = a2 + kc * A2_SLICE;
                        if constexpr (XH) {
                            uint32_t hi, lo;
                            split_f16x2(o0, o1, hi, lo);
                            const int d = r * 64 + ((((cc >> 3)) ^ ((r >> 1) & 3)) << 4) + (cc & 7) * 2;
                            *reinterpret_cast<uint32_t *>(row + d) = hi;
                            *reinterpret_cast<uint32_t *>(row + A2_BYTES + d) = lo;
                        } else {
                            const int d = r * 128 + (((cc >> 2) ^ (r & 7)) << 4) + (cc & 3) * 4;
                            if constexpr (X3 == 1) {
                                float h0, l0, h1, l1;
                                split_tf32(o0, h0, l0); split_tf32(o1, h1, l1);
                                *reinterpret_cast<float2 *>(row + d) = make_float2(h0, h1);
                                *reinterpret_cast<float2 *>(row + A2_BYTES + d) = make_float2(l0, l1);
                            } else {
                                *reinterpret_cast<float2 *>(row + d) = make_float2(o0, o1);
                            }
                        }
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to wgmma's async proxy
                // the 1x1 conv of this warpgroup reads only its own 64 rows of A2
                asm volatile("bar.sync %0, 128;" ::"r"(3 + wg) : "memory");
                mbar_wait(b2_full, 0);
                const uint32_t sa2 = smem_u32(a2) + row_off * (XH ? 64 : 128), sb2 = smem_u32(smem_b2);
                constexpr int OP2 = XH ? 64 : 128;
                // X3 = 2: the cross terms (scaled by 2^11), added scaled back after the hi.hi group.  A kernel compiled for two
                // CTAs per SM (80 registers) cannot hold two N2 = 64 accumulators, so it parks the cross terms in the drained
                // stages behind A2, one column-major block per warpgroup (thread tw's i-th value at [i][tw]: no bank conflicts).
                // Like A2 this relies on the kernel handling one brick: once the main loop is over no TMA is in flight, so the
                // stages are free (a schedule that prefetched the next brick's slabs here would need its own space)
                constexpr bool STASH = XH && N2 > 32 && tc_min_blocks<BN, KS, N2, X3, PS>() == 2;
                static_assert(!STASH || 2 * A2_BYTES + 2 * (N2 / 2) * 128 * 4 <= TC_STAGES * STAGE_BYTES, "stash fits the stages");
                float cross[XH && !STASH ? N2 / 2 : 1];
                float *stash = reinterpret_cast<float *>(smem + 2 * A2_BYTES) + wg * (N2 / 2) * 128 + tw;
#pragma unroll
                for (int pass = 0; pass < (XH ? 2 : 1); ++pass) {
                    wgmma_fence();
#pragma unroll
                    for (int kc = 0; kc < BN / 32; ++kc)
#pragma unroll
                        for (int k = 0; k < OP2 / 32; ++k) {
                            const uint64_t ah = gmma_desc<OP2>(sa2 + kc * A2_SLICE + k * 32), bh = gmma_desc<128>(sb2 + kc * B2_SLICE + k * 32);
                            const uint32_t first = (kc | k) ? 1u : 0u;
                            if constexpr (X3) {
                                const uint64_t al = gmma_desc<OP2>(sa2 + A2_BYTES + kc * A2_SLICE + k * 32);
                                const uint64_t bl = XH ? gmma_desc<128>(sb2 + kc * B2_SLICE + 64 + k * 32)
                                                       : gmma_desc<128>(sb2 + (BN / 32 + kc) * B2_SLICE + k * 32);
                                if (pass == 0) {
                                    wgmma<N2, F16>(acc2, al, bh, first);
                                    wgmma<N2, F16>(acc2, ah, bl, 1u);
                                }
                                if (!XH || pass == 1) wgmma<N2, F16>(acc2, ah, bh, XH ? first : 1u);
                            } else {
                                wgmma<N2, false>(acc2, ah, bh, first);
                            }
                        }
                    wgmma_commit();
                    wgmma_wait_all();
                    if constexpr (XH) {
                        if (pass == 0) {
#pragma unroll
                            for (int i = 0; i < N2 / 2; ++i) {
                                if constexpr (STASH) stash[i * 128] = acc2[i];
                                else cross[i] = acc2[i];
                            }
                        } else {
#pragma unroll
                            for (int i = 0; i < N2 / 2; ++i) acc2[i] = fmaf(STASH ? stash[i * 128] : cross[i], 1.0f / 2048.0f, acc2[i]);
                        }
                    }
                }
                res_acc = acc2;
            }
            // ===== epilogue: bias / residual / ReLU -> global, two columns per store =====
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rbase + 8 * h;
                const int vz = z0 + (r & (TC_BZ - 1)), vy = y0 + ((r / TC_BZ) % TC_BY), vx = x0 + r / (TC_BZ * TC_BY);
                if (!(vx < x1 && vy < y1 && vz < z1)) continue;
                const int64_t vox = ((int64_t)vx * a.Y + vy) * a.Z + vz;
                float *orow = a.out ? a.out + vox * a.out_ld + a.out_coff + n0 : nullptr;
                __half *hrow = a.out16 ? a.out16 + vox * a.out_ld + a.out_coff + n0 : nullptr;
                const float *rrow = a.res ? a.res + vox * a.res_ld + a.res_coff + n0 : nullptr;
                __half *srow = nullptr;  // split-pair row of this voxel (channel c at (c / 32) * 64 + c % 32, its lo 32 halves on)
                if constexpr (XH && KS == 1) srow = a.out_split ? a.out_split + vox * 2 * a.cout + 2 * n0 : nullptr;
#pragma unroll
                for (int j = 0; j < NOUT / 8; ++j) {
                    const int c = 8 * j + 2 * q;
                    float2 o = make_float2(res_acc[4 * j + 2 * h], res_acc[4 * j + 2 * h + 1]);
                    if (a.bias) {
                        const float2 b = __ldg(reinterpret_cast<const float2 *>(a.bias + n0 + c));
                        o.x += b.x; o.y += b.y;
                    }
                    if (rrow) {
                        const float2 v = __ldg(reinterpret_cast<const float2 *>(rrow + c));
                        o.x += v.x; o.y += v.y;
                    }
                    if (a.act == 1) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                    if (orow) *reinterpret_cast<float2 *>(orow + c) = o;
                    if (hrow) *reinterpret_cast<__half2 *>(hrow + c) = __floats2half2_rn(o.x, o.y);
                    if constexpr (XH && KS == 1) {
                        if (srow) {
                            uint32_t hi, lo;
                            split_f16x2(o.x, o.y, hi, lo);
                            __half *p = srow + (c >> 5) * 64 + (c & 31);
                            *reinterpret_cast<uint32_t *>(p) = hi;
                            *reinterpret_cast<uint32_t *>(p + 32) = lo;
                        }
                    }
                }
            }
        }
    }
    __syncwarp();
    if constexpr (CL > 1) cluster_sync_all();  // no CTA exits while its peer may still multicast into it / arrive on its barriers
}

__global__ void gemm_splitk_reduce_kernel(const float *part, int splits, int64_t split_stride, const float *bias, float *y, int M,
                                          int N, int act) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * N) return;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += part[(int64_t)s * split_stride + i];  // fixed order -> deterministic
    if (bias) v += bias[i % N];
    if (act == 1) v = fmaxf(v, 0.f);
    y[i] = v;
}

// weights [cout][cin][3][3][3] -> [cout][27*cin] with k = tap*cin + c
__global__ void pack_conv_weight_tc_kernel(const float *w, int cout, int cin, int taps, float *out) {
    const int64_t total = (int64_t)cout * taps * cin;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cin);
        const int tap = (int)((i / cin) % taps);
        const int n = (int)(i / ((int64_t)cin * taps));
        out[i] = w[((int64_t)n * cin + c) * taps + tap];
    }
}

// 3xTF32 weights: rows [0, cout) = tf32(w) (round to nearest), rows [cout, 2 cout) = tf32(w - tf32(w)); same k order
__global__ void pack_conv_weight_tc_x3_kernel(const float *w, int cout, int cin, int taps, float *out) {
    const int64_t total = (int64_t)cout * taps * cin;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cin);
        const int tap = (int)((i / cin) % taps);
        const int n = (int)(i / ((int64_t)cin * taps));
        float hi, lo;
        split_tf32(w[((int64_t)n * cin + c) * taps + tap], hi, lo);
        out[i] = hi;
        out[total + i] = lo;
    }
}

// fp16-split weights [cout][K/32][64]: per 32-channel K slice (k = tap*cin + c) 32 hi halves = fp16(w), then 32 lo halves =
// fp16((w - fp16(w)) * 2048) -- one 128-byte row per (output channel, K slice), so a TMA box row carries both parts
__global__ void pack_conv_weight_tc_h3_kernel(const float *w, int cout, int cin, int taps, __half *out) {
    const int64_t total = (int64_t)cout * taps * cin;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cin);
        const int tap = (int)((i / cin) % taps);
        const int n = (int)(i / ((int64_t)cin * taps));
        __half hi, lo;
        split_f16(w[((int64_t)n * cin + c) * taps + tap], hi, lo);
        const int64_t k = (int64_t)tap * cin + c;
        const int64_t o = ((int64_t)n * taps * cin + (k & ~(int64_t)31)) * 2 + (k & 31);
        out[o] = hi;
        out[o + 32] = lo;
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {  // resolved through the runtime so libsis3d.so has no link-time dependency on libcuda
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// template arguments of one conv3d_k3_tc_kernel instance
struct TcInst {
    int bn, ks, eb, rowb, by, n2, x3, cl, ps;
    bool operator==(const TcInst &o) const { return memcmp(this, &o, sizeof o) == 0; }
};

// Launches this instance if t holds its template arguments, and sets rc to the launch's return code; false otherwise.
template <int BN, int KS, int EB, int ROWB, int BY, int N2, int X3, int CL, bool PS>
static bool launch_tc(const TcInst &t, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmB2, const TcArgs &a,
                      cudaStream_t s, int grid_z, int &rc) {
    if (!(t == TcInst{BN, KS, EB, ROWB, BY, N2, X3, CL, PS})) return false;
    const size_t smem = tc_smem_bytes<BN, KS, ROWB, BY, N2, X3>();
    auto kern = conv3d_k3_tc_kernel<BN, KS, EB, ROWB, BY, N2, X3, CL, PS>;
    static bool attr_done = false;
    rc = SIS3D_ELAUNCH;
    if (!attr_done) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return true;
        attr_done = true;
    }
    dim3 grid((a.n_tiles + CL - 1) / CL * CL, N2 > 0 ? 1 : a.cout / BN, grid_z);
    if constexpr (CL == 1) {
        kern<<<grid, TC_THREADS, smem, s>>>(tmA, tmB, tmB2, a);
    } else {  // thread-block cluster of CL CTAs along x (pairs of bricks)
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = grid; cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmB2, a) != cudaSuccess) return true;
    }
    rc = finish_launch();
    return true;
}

// fp32 [cout][cin][taps] -> fp16 [cout][taps*cin] (k = tap*cin + c), round to nearest even
__global__ void pack_conv_weight_tc_f16_kernel(const float *w, int cout, int cin, int taps, __half *out) {
    const int64_t total = (int64_t)cout * taps * cin;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cin);
        const int tap = (int)((i / cin) % taps);
        const int n = (int)(i / ((int64_t)cin * taps));
        out[i] = __float2half_rn(w[((int64_t)n * cin + c) * taps + tap]);
    }
}
// VC fp32 (row stride in_ld, channel offset in_coff) -> dense VC fp16 [rows][C]
__global__ void cast_f16_kernel(const float *in, int in_ld, int in_coff, int64_t rows, int C4, __half *out) {
    const int64_t total = rows * C4;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / C4;
        const int c = (int)(i - r * C4) * 4;
        const float4 v = __ldg(reinterpret_cast<const float4 *>(in + r * in_ld + in_coff + c));
        const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t *>(&h0);
        pk.y = *reinterpret_cast<const uint32_t *>(&h1);
        *reinterpret_cast<uint2 *>(out + r * (int64_t)C4 * 4 + c) = pk;
    }
}

}  // namespace sis3d
using namespace sis3d;

extern "C" int sis3d_pack_conv_weight_tc(const float *w, int cout, int cin, int ks, float *w_tc, void *stream) {
    if (!w || !w_tc || cout <= 0 || cin <= 0 || (ks != 1 && ks != 2 && ks != 3)) return SIS3D_EINVAL;
    const int taps = ks * ks * ks;
    const int64_t total = (int64_t)cout * taps * cin;
    pack_conv_weight_tc_kernel<<<(int)imin64(cdiv64(total, 256), kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(w, cout, cin, taps, w_tc);
    return finish_launch();
}

extern "C" int sis3d_conv3d_k3_tc_supported(int cin, int cout) {
    return (cin > 0 && cout > 0 && cin % TC_KC == 0 && (cout == 32 || cout == 64 || cout % 128 == 0)) ? 1 : 0;
}

extern "C" int sis3d_pack_conv_weight_tc_x3(const float *w, int cout, int cin, int ks, float *w_x3, void *stream) {
    if (!w || !w_x3 || cout <= 0 || cin <= 0 || (ks != 1 && ks != 2 && ks != 3)) return SIS3D_EINVAL;
    const int taps = ks * ks * ks;
    const int64_t total = (int64_t)cout * taps * cin;
    pack_conv_weight_tc_x3_kernel<<<(int)imin64(cdiv64(total, 256), kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(w, cout, cin, taps, w_x3);
    return finish_launch();
}

extern "C" int sis3d_pack_conv_weight_tc_h3(const float *w, int cout, int cin, int ks, uint16_t *w_h3, void *stream) {
    if (!w || !w_h3 || cout <= 0 || cin <= 0 || (ks != 1 && ks != 2 && ks != 3)) return SIS3D_EINVAL;
    const int taps = ks * ks * ks;
    const int64_t total = (int64_t)cout * taps * cin;
    pack_conv_weight_tc_h3_kernel<<<(int)imin64(cdiv64(total, 256), kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(w, cout, cin, taps, (__half *)w_h3);
    return finish_launch();
}

// ---- fp16-operand variant (f16 wgmma): activations and weights stored as fp16, fp32 accumulation in registers ------
extern "C" int sis3d_pack_conv_weight_tc_f16(const float *w, int cout, int cin, int ks, uint16_t *w16, void *stream) {
    if (!w || !w16 || cout <= 0 || cin <= 0 || (ks != 1 && ks != 3)) return SIS3D_EINVAL;
    const int taps = ks * ks * ks;
    const int64_t total = (int64_t)cout * taps * cin;
    pack_conv_weight_tc_f16_kernel<<<(int)imin64(cdiv64(total, 256), kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(w, cout, cin, taps, (__half *)w16);
    return finish_launch();
}
extern "C" int sis3d_cast_f16(const float *in, int in_ld, int in_coff, int64_t rows, int C, uint16_t *out, void *stream) {
    if (!in || !out || rows <= 0 || C % 4 != 0 || (in_ld | in_coff) & 3) return SIS3D_EINVAL;
    cast_f16_kernel<<<(int)imin64(cdiv64(rows * (C / 4), 256), kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(in, in_ld, in_coff, rows, C / 4, (__half *)out);
    return finish_launch();
}

// ---- launching the tensor-core kernel -------------------------------------------------------------------------------
// Operand form of the math modes: one TF32 product, the TF32 split (x3), the fp16 split (h3) with fp32 or pre-split input,
// and fp16 operands (f16).
enum TcForm { TC_TF32, TC_TF32_SPLIT, TC_F16_SPLIT, TC_F16_PRESPLIT, TC_F16 };

// A (activations, GEMM rows) and B (weights) of every form carry eb bytes per K index (channel x tap), so one K slice of
// kc channels is one kc * eb-byte shared-memory row of either operand (ROWB), and every TMA box row is one swizzle span.
struct TcOperands {
    int kc, eb, x3;                // K slice width; EB; X3 (0: one product, 1: TF32 split, 2: fp16 split)
    bool ps;                       // PS: A holds split pairs, 32 hi then 32 lo halves per 32-channel slice
    CUtensorMapDataType adt, wdt;  // element types of A and of the packed weights in global memory
    int wrows;                     // weight rows per output channel (TF32 split: hi rows, then lo rows)
    int bn_max;                    // widest N tile
};
static TcOperands tc_operands(TcForm form, int cin) {
    const CUtensorMapDataType F32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32, F16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    switch (form) {
        case TC_TF32: return {TC_KC, 4, 0, false, F32, F32, 1, 128};
        case TC_TF32_SPLIT: return {16, 4, 1, false, F32, F32, 2, 128};  // 64-byte K rows, so hi + lo tiles fit the same smem
        case TC_F16_SPLIT: return {TC_KC, 4, 2, false, F32, F16, 1, 128};  // weight rows: [32 hi | 32 lo] halves per K slice
        case TC_F16_PRESPLIT: return {TC_KC, 4, 2, true, F16, F16, 1, 128};
        default:  // fp16 operands: cin % 64 == 0 in 128-byte rows; cin == 32 in 64-byte rows, with N tiles of at most 64
            if (cin % 64 == 0) return {64, 2, 0, false, F16, F16, 1, 128};
            return {32, 2, 0, false, F16, F16, 1, 64};
    }
}
static int tc_block_n(const TcOperands &op, int cout) { return cout < op.bn_max ? cout : op.bn_max; }
// explicit tile lists (ragged RoI crops) of 64 -> 64 3x3x3 layers use 4x4x8 bricks, everything else 8x2x8 (x, y, z)
static int tc_brick_y(bool tiles, int ks, int cin, int cout) { return tiles && ks == 3 && cout == 64 && cin % 64 == 0 ? 4 : 2; }

static CUtensorMapSwizzle tc_swizzle(uint32_t row_bytes) {
    return row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
}
static uint32_t tc_elem_bytes(CUtensorMapDataType dt) { return dt == CU_TENSOR_MAP_DATA_TYPE_FLOAT16 ? 2 : 4; }
// dense channels-last activation [X][Y][Z][vb bytes]; a box is row_bytes of channels by bz x by x bx voxels, taking every
// sd-th voxel (sd = 2: the 2x2x2 stride-2 conv)
static bool tmap_act(EncodeTiledFn enc, CUtensorMap *m, CUtensorMapDataType dt, const void *p, int X, int Y, int Z, uint64_t vb,
                     uint32_t row_bytes, uint32_t bz, uint32_t by, uint32_t bx, uint32_t sd) {
    const uint32_t e = tc_elem_bytes(dt);
    cuuint64_t dims[4] = {vb / e, (cuuint64_t)Z, (cuuint64_t)Y, (cuuint64_t)X};
    cuuint64_t strides[3] = {vb, (cuuint64_t)Z * vb, (cuuint64_t)Y * Z * vb};
    // with element strides the box is given in traversed elements: N loaded voxels = boxDim / stride
    cuuint32_t box[4] = {row_bytes / e, bz * sd, by * sd, bx * sd};
    cuuint32_t estr[4] = {1, sd, sd, sd};
    return enc(m, dt, 4, (void *)p, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, tc_swizzle(row_bytes),
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// row-major matrix [rows][rb bytes] (weights, W3, GEMM A); a box is row_bytes by box_rows rows
static bool tmap_matrix(EncodeTiledFn enc, CUtensorMap *m, CUtensorMapDataType dt, const void *p, uint64_t rb, uint64_t rows,
                        uint32_t row_bytes, uint32_t box_rows, CUtensorMapL2promotion l2) {
    const uint32_t e = tc_elem_bytes(dt);
    cuuint64_t dims[2] = {rb / e, rows}, strides[1] = {rb};
    cuuint32_t box[2] = {row_bytes / e, box_rows}, estr[2] = {1, 1};
    return enc(m, dt, 2, (void *)p, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, tc_swizzle(row_bytes), l2,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// SIS3D_CLUSTER=1 turns the 2-CTA weight-tile multicast ON (off by default: multicast halves the weight bytes each SM
// fetches, but not the rate at which an SM receives TMA rows; kept as an A/B switch)
static bool use_cluster() {
    static const bool on = getenv("SIS3D_CLUSTER") != nullptr && getenv("SIS3D_CLUSTER")[0] == '1';
    return on;
}

// Every instance of the kernel, each listed once (tests/test_tc_instance_coverage.py reads this list): runs instance t
static int tc_launch(TcInst t, const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmB2, const TcArgs &a,
                     cudaStream_t s, int grid_z) {
    int rc = SIS3D_EUNSUPPORTED;
    if (use_cluster()) {  // the layers with a 2-CTA twin run it
        t.cl = 2;
        if (launch_tc<128, 3, 4, 128, 2, 0, 2, 2, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
        if (launch_tc<64, 3, 4, 128, 4, 0, 0, 2, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
        if (launch_tc<64, 3, 2, 128, 4, 0, 0, 2, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
        if (launch_tc<64, 3, 4, 128, 2, 128, 2, 2, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
        t.cl = 1;
    }
    // convs (BN, KS): TF32, TF32 split, fp16 split; the TF32 4x4x8-brick tile-list layer
    if (launch_tc<32, 3, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 3, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 2, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 2, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 2, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 1, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 1, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 1, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 3, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 2, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 2, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 2, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 1, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 1, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 1, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 3, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 2, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 2, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 2, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 1, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 1, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 1, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 128, 4, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    // fused tails (cmid, cout): TF32, TF32 split, fp16 split, fp16 split on split-pair input
    if (launch_tc<32, 3, 4, 128, 2, 32, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 128, 2, 64, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 128, 2, 128, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 64, 2, 32, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 64, 2, 64, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 64, 2, 128, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 128, 2, 32, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 128, 2, 64, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 128, 2, 128, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 128, 2, 32, 2, 1, true>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 4, 128, 2, 64, 2, 1, true>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 4, 128, 2, 128, 2, 1, true>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    // GEMMs (BN): TF32, TF32 split, fp16 split
    if (launch_tc<32, 0, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 0, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 0, 4, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 0, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 0, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 0, 4, 64, 2, 0, 1, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 0, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 0, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 0, 4, 128, 2, 0, 2, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    // fp16-operand convs (BN, KS): 128-byte rows, the 4x4x8-brick tile-list layer, 64-byte rows
    if (launch_tc<32, 3, 2, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 2, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 3, 2, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 1, 2, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 1, 2, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<128, 1, 2, 128, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 2, 128, 4, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 3, 2, 64, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 3, 2, 64, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<32, 1, 2, 64, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    if (launch_tc<64, 1, 2, 64, 2, 0, 0, 1, false>(t, tmA, tmB, tmB2, a, s, grid_z, rc)) return rc;
    return rc;
}

extern "C" int sis3d_conv3d_k3_tc_fused_supported(int cin, int cmid, int cout) {
    return (cin > 0 && cin % TC_KC == 0 && ((cmid == 32 && (cout == 32 || cout == 64)) || (cmid == 64 && cout == 128))) ? 1 : 0;
}
extern "C" int sis3d_linear_tc_supported(int K, int N) { return sis3d_conv3d_k3_tc_supported(K, N); }
static int gemm_tc_splits(int M, int N, int K, const TcOperands &op) {
    const int tiles = cdiv(M, TC_BM) * (N / tc_block_n(op, N));
    const int chunks = K / op.kc;
    return max(1, min(chunks / (128 / op.kc), (kNumSMs + tiles - 1) / tiles));
}
extern "C" size_t sis3d_linear_tc_workspace_bytes(int M, int N, int K) {
    if (M <= 0 || !sis3d_linear_tc_supported(K, N)) return 0;  // gemm_tc_splits divides by the tile and chunk counts
    // the TF32 split's 16-channel K slices split K finest: covers every mode
    return sizeof(float) * (size_t)gemm_tc_splits(M, N, K, tc_operands(TC_TF32_SPLIT, K)) * M * N + 16;
}

// One launch as an entry point describes it.  The fields up to `stream` follow sis3d_conv3d_k3_tc's arguments.
enum TcOp { TC_CONV, TC_FUSED, TC_GEMM };
struct TcLaunch {
    TcOp op;
    TcForm form;
    const void *in, *w;
    const float *bias, *res;
    int res_ld, res_coff;
    float *out;                                    // GEMM: y
    int out_ld, out_coff, X, Y, Z, cin, cout, ks;  // GEMM: X = M, Y = Z = 1, cin = K, cout = N, ks = 1
    const int32_t *tiles;
    int n_tiles, act;
    void *stream;
    void *workspace;          // GEMM: split-K partial sums, reduced into y
    size_t workspace_bytes;
    const void *w3;           // fused tail: the 1x1 conv's weights, its input width and the 3x3x3 conv's bias
    int cmid;
    const float *bias_mid;
    __half *out16, *out_split;
};

static int tc_run(const TcLaunch &L) {
    const bool fused = L.op == TC_FUSED, gemm = L.op == TC_GEMM;
    // argument checks, in the order that decides which code a call with several faults gets
    if (!L.in || !L.w || !(L.out || L.out16 || L.out_split) || (fused && !L.w3) || (gemm && !L.workspace) || L.X <= 0 ||
        L.Y <= 0 || L.Z <= 0 || L.cin <= 0 || L.cout <= 0 || (fused && L.cmid <= 0) ||
        !(L.ks == 1 || L.ks == 3 || (L.ks == 2 && L.form != TC_F16)))
        return SIS3D_EINVAL;
    if (L.out_split && (L.cout % TC_KC || ((uintptr_t)L.out_split & 15))) return SIS3D_EINVAL;
    if (L.ks == 2 && (L.tiles || L.X < 2 || L.Y < 2 || L.Z < 2)) return SIS3D_EINVAL;
    if (!(fused ? sis3d_conv3d_k3_tc_fused_supported(L.cin, L.cmid, L.cout) : sis3d_conv3d_k3_tc_supported(L.cin, L.cout)))
        return SIS3D_EUNSUPPORTED;
    // TMA reads and the kernel's vector stores need 16-byte alignment; the GEMM's y is written by the scalar reduce
    if (((uintptr_t)L.in | (uintptr_t)L.w | (uintptr_t)L.w3 | (uintptr_t)(gemm ? L.workspace : L.out) | (uintptr_t)L.out16) & 15)
        return SIS3D_EINVAL;
    if ((L.out_ld | L.out_coff | L.res_ld | L.res_coff) & 3) return SIS3D_EINVAL;
    const TcOperands op = tc_operands(L.form, L.cin);
    if (L.form == TC_F16 && op.kc == 32 && L.cin != 32) return SIS3D_EUNSUPPORTED;  // fp16 rows: 32 or a multiple of 64 channels
    EncodeTiledFn enc = get_encode();
    if (!enc) return SIS3D_EUNSUPPORTED;

    const int rowb = op.kc * op.eb, taps = L.ks * L.ks * L.ks;
    const int by = tc_brick_y(L.tiles, L.ks, L.cin, L.cout), bx = 16 / by;
    const int width = fused ? L.cmid : L.cout;  // the weight rows of the main loop (the fused tail's 3x3x3 conv)
    const int BN = tc_block_n(op, width);
    int splits = 1, per = 0;
    if (gemm) {
        splits = gemm_tc_splits(L.X, L.cout, L.cin, op);
        const int chunks = L.cin / op.kc;
        per = cdiv(chunks, splits);
        splits = cdiv(chunks, per);
        // the documented size, not this mode's need: a buffer that is too small for the finest split is rejected in every mode
        if (L.workspace_bytes < sis3d_linear_tc_workspace_bytes(L.X, L.cout, L.cin)) return SIS3D_EWORKSPACE;
    }
    const int sd = L.ks == 2 ? 2 : 1;                       // ks == 2 is the stride-2, pad-0 conv: X, Y, Z are the INPUT extents
    const int Xo = L.X / sd, Yo = L.Y / sd, Zo = L.Z / sd;  // output extents (floor, as nn.Conv3d)
    const uint64_t kb = (uint64_t)L.cin * op.eb;            // bytes of A per voxel (GEMM row), of B per tap and output channel
    const CUtensorMapL2promotion l2w = CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
    CUtensorMap tmA, tmB, tmB2;
    if (!(gemm ? tmap_matrix(enc, &tmA, op.adt, L.in, kb, L.X, rowb, TC_BM, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)
               : tmap_act(enc, &tmA, op.adt, L.in, L.X, L.Y, L.Z, kb, rowb, TC_BZ, by, L.ks == 3 ? bx + 2 : bx, sd)) ||
        !tmap_matrix(enc, &tmB, op.wdt, L.w, taps * kb, (uint64_t)width * op.wrows, rowb, BN, l2w) ||
        (fused && !tmap_matrix(enc, &tmB2, op.wdt, L.w3, (uint64_t)L.cmid * op.eb, (uint64_t)L.cout * op.wrows, TC_KC * op.eb,
                               L.cout, l2w)))
        return SIS3D_EINVAL;

    TcArgs a = {};
    a.n_tiles = L.n_tiles;
    if (gemm) {
        a.out = (float *)L.workspace; a.out_ld = L.cout; a.cin = L.cin; a.cout = L.cout;
        a.gemm_m = L.X; a.gemm_chunks_per_split = per; a.n_tiles = cdiv(L.X, TC_BM);
    } else {
        a.bias = L.bias; a.bias_mid = L.bias_mid; a.res = L.res; a.out = L.out; a.out16 = L.out16; a.out_split = L.out_split;
        a.tiles = L.tiles;
        // the fused tail's compensated main loop indexes weight rows (and their lo halves) with cmid, the epilogue with cout
        a.X = Xo; a.Y = Yo; a.Z = Zo; a.cin = L.cin; a.cout = fused && op.x3 ? L.cmid : L.cout; a.act = L.act;
        a.out_ld = L.out_ld; a.out_coff = L.out_coff; a.res_ld = L.res_ld; a.res_coff = L.res_coff;
        a.tiles_y = cdiv(Yo, by); a.tiles_z = cdiv(Zo, TC_BZ);
        if (!L.tiles) a.n_tiles = cdiv(Xo, bx) * a.tiles_y * a.tiles_z;
    }
    if (a.n_tiles <= 0) return SIS3D_OK;
    cudaStream_t s = (cudaStream_t)L.stream;
    const TcInst t = {BN, gemm ? 0 : L.ks, op.eb, rowb, by, fused ? L.cout : 0, op.x3, 1, op.ps};
    const int rc = tc_launch(t, tmA, tmB, fused ? tmB2 : tmB, a, s, splits);
    if (rc || !gemm) return rc;
    gemm_splitk_reduce_kernel<<<cdiv(L.X * L.cout, 256), 256, 0, s>>>((const float *)L.workspace, splits, (int64_t)L.X * L.cout,
                                                                       L.bias, L.out, L.X, L.cout, L.act);
    return finish_launch();
}

extern "C" int sis3d_conv3d_k3_tc(const float *in, const float *w_tc, const float *bias, const float *residual, int res_ld,
                                  int res_coff, float *out, int out_ld, int out_coff, int X, int Y, int Z, int cin, int cout,
                                  int ks, const int32_t *tiles, int n_tiles, int act, void *stream) {
    return tc_run({TC_CONV, TC_TF32, in, w_tc, bias, residual, res_ld, res_coff, out, out_ld, out_coff, X, Y, Z, cin, cout, ks,
                   tiles, n_tiles, act, stream});
}
// error-compensated 3xTF32 (fp32-class accuracy on the tensor cores): w_x3 from sis3d_pack_conv_weight_tc_x3
extern "C" int sis3d_conv3d_k3_tc_x3(const float *in, const float *w_x3, const float *bias, const float *residual, int res_ld,
                                     int res_coff, float *out, int out_ld, int out_coff, int X, int Y, int Z, int cin, int cout,
                                     int ks, int act, void *stream) {
    return tc_run({TC_CONV, TC_TF32_SPLIT, in, w_x3, bias, residual, res_ld, res_coff, out, out_ld, out_coff, X, Y, Z, cin, cout,
                   ks, nullptr, 0, act, stream});
}
// the same compensation with an fp16 operand split (2.5x the MMA rate): w_h3 from sis3d_pack_conv_weight_tc_h3
extern "C" int sis3d_conv3d_k3_tc_h3(const float *in, const uint16_t *w_h3, const float *bias, const float *residual, int res_ld,
                                     int res_coff, float *out, int out_ld, int out_coff, int X, int Y, int Z, int cin, int cout,
                                     int ks, int act, void *stream) {
    return tc_run({TC_CONV, TC_F16_SPLIT, in, w_h3, bias, residual, res_ld, res_coff, out, out_ld, out_coff, X, Y, Z, cin, cout,
                   ks, nullptr, 0, act, stream});
}
// the fp16-split 1x1 conv writing split-pair activations (the A operand of sis3d_conv3d_k3_tc_fused_h3_split) instead of fp32
extern "C" int sis3d_conv3d_k1_tc_h3_split(const float *in, const uint16_t *w_h3, const float *bias, uint16_t *out_split, int X,
                                           int Y, int Z, int cin, int cout, int act, void *stream) {
    return tc_run({TC_CONV, TC_F16_SPLIT, in, w_h3, bias, nullptr, 0, 0, nullptr, cout, 0, X, Y, Z, cin, cout, 1, nullptr, 0, act,
                   stream, nullptr, 0, nullptr, 0, nullptr, nullptr, (__half *)out_split});
}

// ---- bottleneck tail: 3x3x3 conv (cin -> cmid) + ReLU + 1x1 conv (cmid -> cout) + residual + act, one kernel ----------------
extern "C" int sis3d_conv3d_k3_tc_fused(const float *in, const float *w2_tc, const float *bias2, const float *w3_tc,
                                        const float *bias3, const float *residual, int res_ld, int res_coff, float *out,
                                        int out_ld, int out_coff, int X, int Y, int Z, int cin, int cmid, int cout, int act,
                                        void *stream) {
    return tc_run({TC_FUSED, TC_TF32, in, w2_tc, bias3, residual, res_ld, res_coff, out, out_ld, out_coff, X, Y, Z, cin, cout, 3,
                   nullptr, 0, act, stream, nullptr, 0, w3_tc, cmid, bias2});
}
extern "C" int sis3d_conv3d_k3_tc_fused_x3(const float *in, const float *w2_x3, const float *bias2, const float *w3_x3,
                                           const float *bias3, const float *residual, int res_ld, int res_coff, float *out,
                                           int out_ld, int out_coff, int X, int Y, int Z, int cin, int cmid, int cout, int act,
                                           void *stream) {
    return tc_run({TC_FUSED, TC_TF32_SPLIT, in, w2_x3, bias3, residual, res_ld, res_coff, out, out_ld, out_coff, X, Y, Z, cin,
                   cout, 3, nullptr, 0, act, stream, nullptr, 0, w3_x3, cmid, bias2});
}
extern "C" int sis3d_conv3d_k3_tc_fused_h3(const float *in, const uint16_t *w2_h3, const float *bias2, const uint16_t *w3_h3,
                                           const float *bias3, const float *residual, int res_ld, int res_coff, float *out,
                                           int out_ld, int out_coff, int X, int Y, int Z, int cin, int cmid, int cout, int act,
                                           void *stream) {
    return tc_run({TC_FUSED, TC_F16_SPLIT, in, w2_h3, bias3, residual, res_ld, res_coff, out, out_ld, out_coff, X, Y, Z, cin,
                   cout, 3, nullptr, 0, act, stream, nullptr, 0, w3_h3, cmid, bias2});
}
// the same tail fed split-pair activations (from sis3d_conv3d_k1_tc_h3_split): no operand split on the SM, same result bits
extern "C" int sis3d_conv3d_k3_tc_fused_h3_split(const uint16_t *in_split, const uint16_t *w2_h3, const float *bias2,
                                                 const uint16_t *w3_h3, const float *bias3, const float *residual, int res_ld,
                                                 int res_coff, float *out, int out_ld, int out_coff, int X, int Y, int Z, int cin,
                                                 int cmid, int cout, int act, void *stream) {
    return tc_run({TC_FUSED, TC_F16_PRESPLIT, in_split, w2_h3, bias3, residual, res_ld, res_coff, out, out_ld, out_coff, X, Y, Z,
                   cin, cout, 3, nullptr, 0, act, stream, nullptr, 0, w3_h3, cmid, bias2});
}

// ---- y[M][N] = act(x[M][K] . w[N][K]^T + b): fully connected layer on the tensor cores, split-K ------------
extern "C" int sis3d_linear_tc(const float *x, const float *w_nk, const float *bias, float *y, int M, int K, int N, int act,
                               void *workspace, size_t workspace_bytes, void *stream) {
    return tc_run({TC_GEMM, TC_TF32, x, w_nk, bias, nullptr, 0, 0, y, 0, 0, M, 1, 1, K, N, 1, nullptr, 0, act, stream,
                   workspace, workspace_bytes});
}
// w_x3 = sis3d_pack_conv_weight_tc_x3(w[N][K] viewed as a 1x1 conv): [2][N][K]
extern "C" int sis3d_linear_tc_x3(const float *x, const float *w_x3, const float *bias, float *y, int M, int K, int N, int act,
                                  void *workspace, size_t workspace_bytes, void *stream) {
    return tc_run({TC_GEMM, TC_TF32_SPLIT, x, w_x3, bias, nullptr, 0, 0, y, 0, 0, M, 1, 1, K, N, 1, nullptr, 0, act, stream,
                   workspace, workspace_bytes});
}
extern "C" int sis3d_linear_tc_h3(const float *x, const uint16_t *w_h3, const float *bias, float *y, int M, int K, int N, int act,
                                  void *workspace, size_t workspace_bytes, void *stream) {
    return tc_run({TC_GEMM, TC_F16_SPLIT, x, w_h3, bias, nullptr, 0, 0, y, 0, 0, M, 1, 1, K, N, 1, nullptr, 0, act, stream,
                   workspace, workspace_bytes});
}

extern "C" int sis3d_conv3d_tc_f16(const uint16_t *in16, const uint16_t *w16, const float *bias, const float *residual,
                                   int res_ld, int res_coff, float *out32, uint16_t *out16, int out_ld, int out_coff, int X, int Y,
                                   int Z, int cin, int cout, int ks, const int32_t *tiles, int n_tiles, int act, void *stream) {
    return tc_run({TC_CONV, TC_F16, in16, w16, bias, residual, res_ld, res_coff, out32, out_ld, out_coff, X, Y, Z, cin, cout, ks,
                   tiles, n_tiles, act, stream, nullptr, 0, nullptr, 0, nullptr, (__half *)out16});
}

// brick shape the tensor-core kernel uses for a layer (so callers can build matching tile lists)
extern "C" void sis3d_conv3d_tc_brick(int with_tile_list, int ks, int cin, int cout, int32_t *bx, int32_t *by, int32_t *bz) {
    const int y = tc_brick_y(with_tile_list, ks, cin, cout);
    if (bx) *bx = 16 / y;
    if (by) *by = y;
    if (bz) *bz = TC_BZ;
}
