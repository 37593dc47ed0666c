// ply.cu -- the result visualisation's voxel meshes and ASCII PLY text (tools/visualization.py,
// tools/scannet_benchmark/visualize_benchmark.py).
//
// The reference builds every cube of a label volume as Python lists in a triple loop over the volume and formats one text
// line per vertex and per face with str.format (tools/visualization.py:78-101, 263-324).  Here:
// - sis3d_voxel_mesh_count / sis3d_voxel_mesh number the occupied voxels in the reference's visiting order (z outermost,
//   then y, x innermost) and emit the cubes of any range of them, so a large volume can be written in slabs;
// - sis3d_ply_ascii_lengths / sis3d_ply_ascii turn vertex and face arrays into the exact bytes Python's '{:f}' / '{:d}'
//   produce, each line at its scanned offset in one buffer.
// No CUB: the scans are three plain kernels (tile sums, one block over the tile sums, tiles), so the file also builds under
// tools/cuda_host_emu.py.
#include "common.cuh"

namespace sis3d {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;
static_assert(kScanTile == SIS3D_PLY_SCAN_TILE, "scratch size contract of include/sis3d.h");
constexpr int kMeshThreads = 256;  // one warp per (z, y) row
constexpr int kLineThreads = 256;  // one thread per text line

// ------------------------------------------------------------------------------------------------------------- scans
// exclusive prefix of v in threadIdx.x order; *total = the block's sum.  Every thread of the block calls it.
__device__ int64_t block_exclusive_scan(int64_t v, int64_t *total) {
    __shared__ int64_t warp_total[kScanThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_total[w] = inc;
    __syncthreads();
    int64_t before = 0, sum = 0;
    for (int i = 0; i < kScanThreads / 32; ++i) {
        if (i < w) before += warp_total[i];
        sum += warp_total[i];
    }
    __syncthreads();  // warp_total is reused by the next call
    *total = sum;
    return before + inc - v;
}

// v[t0, t0 + kScanTile) (clipped to n) -> exclusive prefix + carry, in place; returns the tile's sum
__device__ int64_t scan_tile(int64_t *v, int64_t n, int64_t t0, int64_t carry) {
    int64_t loc[kScanItems], s = 0;
    const int64_t i0 = t0 + (int64_t)threadIdx.x * kScanItems;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        loc[j] = i0 + j < n ? v[i0 + j] : 0;
        s += loc[j];
    }
    int64_t total;
    int64_t ex = block_exclusive_scan(s, &total) + carry;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        if (i0 + j < n) v[i0 + j] = ex;
        ex += loc[j];
    }
    return total;
}

__global__ void __launch_bounds__(kScanThreads) scan_tile_sum_kernel(const int64_t *v, int64_t n, int64_t *tile_sum) {
    const int64_t i0 = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    int64_t s = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) s += i0 + j < n ? v[i0 + j] : 0;
    int64_t total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// one block: tile sums -> their exclusive prefix; *total = the sum of everything
__global__ void __launch_bounds__(kScanThreads) scan_carry_kernel(int64_t *tile_sum, int64_t n_tiles, int64_t *total) {
    int64_t carry = 0;
    for (int64_t t0 = 0; t0 < n_tiles; t0 += kScanTile) carry += scan_tile(tile_sum, n_tiles, t0, carry);
    if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(int64_t *v, int64_t n, const int64_t *tile_sum) {
    scan_tile(v, n, (int64_t)blockIdx.x * kScanTile, tile_sum[blockIdx.x]);
}

// v[0, n) -> exclusive prefix in place, v[n] = the sum; scratch holds cdiv(n, kScanTile) int64.  Returns launches or -1.
int launch_scan(int64_t *v, int64_t n, int64_t *scratch, cudaStream_t s) {
    const int64_t tiles = cdiv64(n, kScanTile);
    if (tiles > 0x7fffffff) return -1;
    if (tiles == 0) {
        cudaMemsetAsync(v, 0, sizeof(int64_t), s);
        return 0;
    }
    scan_tile_sum_kernel<<<(unsigned)tiles, kScanThreads, 0, s>>>(v, n, scratch);
    scan_carry_kernel<<<1, kScanThreads, 0, s>>>(scratch, tiles, v + n);
    scan_apply_kernel<<<(unsigned)tiles, kScanThreads, 0, s>>>(v, n, scratch);
    return 3;
}

// ------------------------------------------------------------------------------------------------------- voxel mesh
__device__ __forceinline__ int voxel_label(const int32_t *labels, const int32_t *lut, int n_lut, int64_t i) {
    const int v = labels[i];
    return lut ? (v >= 0 && v < n_lut ? lut[v] : 0) : v;
}

// corner c of make_voxel_mesh (visualization.py:270-279) takes the high x / y / z when bit c of these masks is set
constexpr unsigned kCornerHiX = 0x99, kCornerHiY = 0x33, kCornerHiZ = 0x0F;
// its twelve faces (visualization.py:291-304), three 3-bit local vertex ids per face, six faces per word
constexpr uint64_t face_bits(int a, int b, int c, int slot) { return (uint64_t)(a | b << 3 | c << 6) << (9 * slot); }
constexpr uint64_t kFaces0 = face_bits(1, 2, 3, 0) | face_bits(1, 3, 0, 1) | face_bits(0, 3, 7, 2) | face_bits(0, 7, 4, 3) |
                             face_bits(3, 2, 6, 4) | face_bits(3, 6, 7, 5);
constexpr uint64_t kFaces1 = face_bits(1, 6, 2, 0) | face_bits(1, 5, 6, 1) | face_bits(0, 5, 1, 2) | face_bits(0, 4, 5, 3) |
                             face_bits(6, 5, 4, 4) | face_bits(6, 4, 7, 5);

// warp r: row r = z * Y + y of the visiting order; lane l reads x = l, l + 32, ...
__global__ void __launch_bounds__(kMeshThreads)
voxel_row_count_kernel(const int32_t *labels, const int32_t *lut, int n_lut, int X, int Y, int Z, int64_t *count) {
    const int64_t r = ((int64_t)blockIdx.x * kMeshThreads + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= (int64_t)Y * Z) return;  // whole warps
    const int z = (int)(r / Y), y = (int)(r - (int64_t)z * Y);
    const int64_t stride = (int64_t)Y * Z, base = (int64_t)y * Z + z;
    int64_t cnt = 0;
    for (int x0 = 0; x0 < X; x0 += 32) {
        const int x = x0 + lane;
        cnt += __popc(__ballot_sync(0xffffffffu, x < X && voxel_label(labels, lut, n_lut, base + x * stride) > 0));
    }
    if (lane == 0) count[r] = cnt;
}

__global__ void __launch_bounds__(kMeshThreads)
voxel_mesh_kernel(const int32_t *labels, const int32_t *lut, int n_lut, int X, int Y, int Z, const int64_t *row_offsets,
                  const int64_t *palette, int64_t k0, int64_t k1, double *verts, int64_t *colors, int64_t *faces) {
    const int64_t r = ((int64_t)blockIdx.x * kMeshThreads + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= (int64_t)Y * Z) return;
    int64_t k = row_offsets[r];
    if (k >= k1 || row_offsets[r + 1] <= k0) return;
    const int z = (int)(r / Y), y = (int)(r - (int64_t)z * Y);
    const int64_t stride = (int64_t)Y * Z, base = (int64_t)y * Z + z;
    for (int x0 = 0; x0 < X && k < k1; x0 += 32) {
        const int x = x0 + lane;
        const int lab = x < X ? voxel_label(labels, lut, n_lut, base + x * stride) : 0;
        const unsigned m = __ballot_sync(0xffffffffu, lab > 0);
        const int64_t kv = k + __popc(m & ((1u << lane) - 1u));
        k += __popc(m);
        if (lab <= 0 || kv < k0 || kv >= k1) continue;
        const int64_t j = kv - k0;
        if (verts) {  // fl(c - 0.05) and fl(c + 0.95): (np.array([x, y, z]) - 0.05) * 1 + 0 (visualization.py:316-317)
            const double lo[3] = {(double)x - 0.05, (double)y - 0.05, (double)z - 0.05};
            const double hi[3] = {(double)x + 0.95, (double)y + 0.95, (double)z + 0.95};
            double *o = verts + j * 24;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                o[3 * c] = (kCornerHiX >> c & 1) ? hi[0] : lo[0];
                o[3 * c + 1] = (kCornerHiY >> c & 1) ? hi[1] : lo[1];
                o[3 * c + 2] = (kCornerHiZ >> c & 1) ? hi[2] : lo[2];
            }
        }
        if (colors) {
            const int64_t *p = palette + 3 * (lab % 41);
            const int64_t p0 = p[0], p1 = p[1], p2 = p[2];
            int64_t *o = colors + j * 24;
#pragma unroll
            for (int c = 0; c < 8; ++c) o[3 * c] = p0, o[3 * c + 1] = p1, o[3 * c + 2] = p2;
        }
        if (faces) {
            int64_t *o = faces + j * 36;
#pragma unroll
            for (int f = 0; f < 12; ++f)
#pragma unroll
                for (int e = 0; e < 3; ++e) o[3 * f + e] = 8 * kv + (int64_t)(((f < 6 ? kFaces0 : kFaces1) >> (9 * (f % 6) + 3 * e)) & 7);
        }
    }
}

// ------------------------------------------------------------------------------------------------------- PLY text
// bytes of u in decimal
__device__ __forceinline__ int decimal_digits(uint64_t u) {
    int n = 1;
    while (u >= 10) u /= 10, ++n;
    return n;
}

__device__ __forceinline__ void put_decimal(char *p, uint64_t u, int n) {
    for (int i = n - 1; i >= 0; --i) p[i] = (char)('0' + u % 10), u /= 10;
}

__device__ __forceinline__ int put_text(char *p, const char *s, int n) {
    if (p)
        for (int i = 0; i < n; ++i) p[i] = s[i];
    return n;
}

// '{:f}'.format(v) for a float64: 6 fractional digits, correctly rounded from the exact binary value with ties to even, the
// sign of a negative value kept when it rounds to zero, nan / inf / -inf.  Writes the bytes at p unless p is null and
// returns their count; -1 (nothing written) when |v| >= 2^64.
//   v = m * 2^e.  e >= 0: the integer m << e.  e < 0: q = m * 10^6 >> -e, rounded half to even on the shifted-out bits, as
//   one 128-bit integer (m < 2^53, so m * 10^6 < 2^73); q = round(v * 10^6) and the integer part is floor(v) = m >> -e.
__device__ int format_fixed6(double v, char *p) {
    const uint64_t b = (uint64_t)__double_as_longlong(v);
    const int neg = (int)(b >> 63), ex = (int)(b >> 52 & 0x7ff);
    const uint64_t frac = b & ((1ull << 52) - 1);
    if (ex == 0x7ff) {
        if (frac) return put_text(p, "nan", 3);
        return neg ? put_text(p, "-inf", 4) : put_text(p, "inf", 3);
    }
    if (ex >= 1023 + 64) return -1;
    uint64_t ip = 0;
    unsigned fr = 0;
    if (ex || frac) {
        const uint64_t m = ex ? frac | 1ull << 52 : frac;
        const int e = (ex ? ex : 1) - 1075;
        if (e >= 0) {
            ip = m << e;
        } else {
            const int s = -e;
            ip = s < 64 ? m >> s : 0;
            const unsigned __int128 P = (unsigned __int128)m * 1000000u;
            unsigned __int128 q = 0;
            if (s < 128) {
                q = P >> s;
                const unsigned __int128 rem = P - (q << s), half = (unsigned __int128)1 << (s - 1);
                if (rem > half || (rem == half && (q & 1))) ++q;
            }
            fr = (unsigned)(uint64_t)(q - (unsigned __int128)ip * 1000000u);  // in [0, 10^6]
            if (fr == 1000000u) ++ip, fr = 0;
        }
    }
    const int nd = decimal_digits(ip);
    if (p) {
        if (neg) *p++ = '-';
        put_decimal(p, ip, nd);
        p[nd] = '.';
        put_decimal(p + nd + 1, fr, 6);
    }
    return neg + nd + 7;
}

// '{:d}'.format(v) for an int64
__device__ __forceinline__ int format_int(int64_t v, char *p) {
    const int neg = v < 0;
    const uint64_t u = neg ? 0ull - (uint64_t)v : (uint64_t)v;
    const int nd = decimal_digits(u);
    if (p) {
        if (neg) *p++ = '-';
        put_decimal(p, u, nd);
    }
    return neg + nd;
}

struct PlyLines {
    const double *verts;    // [n_vert][3]
    const int64_t *colors;  // [n_vert][3]
    int64_t n_vert;
    const int64_t *faces;   // [n_face][3]
    int64_t n_face;
};

// line i: vertex i, or face i - n_vert.  -> bytes (written at p unless null), -1 for a vertex with a coordinate >= 2^64
__device__ int format_line(const PlyLines &L, int64_t i, char *p) {
    int n = 0;
    if (i < L.n_vert) {
        for (int a = 0; a < 3; ++a) {
            const int m = format_fixed6(L.verts[3 * i + a], p ? p + n : nullptr);
            if (m < 0) return -1;
            n += m;
            if (p) p[n] = ' ';
            ++n;
        }
        for (int a = 0; a < 3; ++a) {
            n += format_int(L.colors[3 * i + a], p ? p + n : nullptr);
            if (p) p[n] = a < 2 ? ' ' : '\n';
            ++n;
        }
        return n;
    }
    i -= L.n_vert;
    n = put_text(p, "3 ", 2);
    for (int a = 0; a < 3; ++a) {
        n += format_int(L.faces[3 * i + a], p ? p + n : nullptr);
        if (p) p[n] = a < 2 ? ' ' : '\n';
        ++n;
    }
    return n;
}

__global__ void __launch_bounds__(kLineThreads) line_length_kernel(PlyLines L, int64_t l0, int64_t n, int64_t *offsets) {
    const int64_t i = (int64_t)blockIdx.x * kLineThreads + threadIdx.x;
    if (i >= n) return;
    int len = format_line(L, l0 + i, nullptr);
    if (len < 0) {
        atomicAdd((unsigned long long *)(offsets + n + 1), 1ull);
        len = 0;
    }
    offsets[i] = len;
}

__global__ void __launch_bounds__(kLineThreads)
line_write_kernel(PlyLines L, int64_t l0, int64_t n, const int64_t *offsets, char *out) {
    const int64_t i = (int64_t)blockIdx.x * kLineThreads + threadIdx.x;
    if (i < n) format_line(L, l0 + i, out + offsets[i]);
}

// the arguments both text entry points share
int check_lines(const PlyLines &L, int64_t l0, int64_t l1) {
    if (L.n_vert < 0 || L.n_face < 0 || l0 < 0 || l1 < l0 || l1 > L.n_vert + L.n_face) return SIS3D_EINVAL;
    if (l0 < L.n_vert && (!L.verts || !L.colors)) return SIS3D_EINVAL;
    if (l1 > L.n_vert && !L.faces) return SIS3D_EINVAL;
    if (cdiv64(l1 - l0, kLineThreads) > 0x7fffffff) return SIS3D_EUNSUPPORTED;
    return SIS3D_OK;
}

}  // namespace sis3d
using namespace sis3d;

extern "C" int sis3d_voxel_mesh_count(const int32_t *labels, const int32_t *lut, int n_lut, int X, int Y, int Z,
                                      int64_t *row_offsets, int64_t *scratch, void *stream) {
    if (X < 0 || Y < 0 || Z < 0 || n_lut < 0 || !row_offsets) return SIS3D_EINVAL;
    const int64_t n_rows = (int64_t)Y * Z;
    if ((int64_t)X * n_rows > 0 && !labels) return SIS3D_EINVAL;
    if (n_rows > 0 && !scratch) return SIS3D_EINVAL;
    const int64_t blocks = cdiv64(n_rows, kMeshThreads / 32);
    if (blocks > 0x7fffffff) return SIS3D_EUNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    int launches = 0;
    if (blocks > 0) {
        voxel_row_count_kernel<<<(unsigned)blocks, kMeshThreads, 0, s>>>(labels, lut, n_lut, X, Y, Z, row_offsets);
        ++launches;
    }
    const int scans = launch_scan(row_offsets, n_rows, scratch, s);
    if (scans < 0) return SIS3D_EUNSUPPORTED;
    return finish_launch(launches + scans);
}

extern "C" int sis3d_voxel_mesh(const int32_t *labels, const int32_t *lut, int n_lut, int X, int Y, int Z,
                                const int64_t *row_offsets, const int64_t *palette, int64_t k0, int64_t k1, double *verts,
                                int64_t *colors, int64_t *faces, void *stream) {
    if (X < 0 || Y < 0 || Z < 0 || n_lut < 0 || k0 < 0 || k1 < k0) return SIS3D_EINVAL;
    const int64_t n_rows = (int64_t)Y * Z;
    if (k1 == k0 || (int64_t)X * n_rows == 0) return SIS3D_OK;
    if (!labels || !row_offsets || (colors && !palette)) return SIS3D_EINVAL;
    const int64_t blocks = cdiv64(n_rows, kMeshThreads / 32);
    if (blocks > 0x7fffffff) return SIS3D_EUNSUPPORTED;
    voxel_mesh_kernel<<<(unsigned)blocks, kMeshThreads, 0, (cudaStream_t)stream>>>(labels, lut, n_lut, X, Y, Z, row_offsets,
                                                                                    palette, k0, k1, verts, colors, faces);
    return finish_launch();
}

extern "C" int sis3d_ply_ascii_lengths(const double *verts, const int64_t *colors, int64_t n_vert, const int64_t *faces,
                                       int64_t n_face, int64_t l0, int64_t l1, int64_t *offsets, int64_t *scratch,
                                       void *stream) {
    const PlyLines L{verts, colors, n_vert, faces, n_face};
    const int rc = check_lines(L, l0, l1);
    if (rc != SIS3D_OK) return rc;
    const int64_t n = l1 - l0;
    if (!offsets || (n > 0 && !scratch)) return SIS3D_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    cudaMemsetAsync(offsets + n + 1, 0, sizeof(int64_t), s);
    int launches = 0;
    if (n > 0) {
        line_length_kernel<<<(unsigned)cdiv64(n, kLineThreads), kLineThreads, 0, s>>>(L, l0, n, offsets);
        ++launches;
    }
    const int scans = launch_scan(offsets, n, scratch, s);
    if (scans < 0) return SIS3D_EUNSUPPORTED;
    return finish_launch(launches + scans);
}

extern "C" int sis3d_ply_ascii(const double *verts, const int64_t *colors, int64_t n_vert, const int64_t *faces,
                               int64_t n_face, int64_t l0, int64_t l1, const int64_t *offsets, char *out, void *stream) {
    const PlyLines L{verts, colors, n_vert, faces, n_face};
    const int rc = check_lines(L, l0, l1);
    if (rc != SIS3D_OK) return rc;
    const int64_t n = l1 - l0;
    if (n == 0) return SIS3D_OK;
    if (!offsets || !out) return SIS3D_EINVAL;
    line_write_kernel<<<(unsigned)cdiv64(n, kLineThreads), kLineThreads, 0, (cudaStream_t)stream>>>(L, l0, n, offsets, out);
    return finish_launch();
}
