// api.cu -- library-wide entry points of libsis3d.so.
#include <math.h>
#include "common.cuh"
namespace sis3d { unsigned long long g_launch_count = 0; }

extern "C" const char *sis3d_strerror(int code) {
    switch (code) {
        case SIS3D_OK: return "ok";
        case SIS3D_EINVAL: return "invalid argument";
        case SIS3D_ELAUNCH: return "CUDA launch/runtime error";
        case SIS3D_EWORKSPACE: return "workspace too small";
        case SIS3D_EUNSUPPORTED: return "unsupported configuration";
        default: return "unknown sis3d error";
    }
}
extern "C" int sis3d_version(void) { return 100; }
extern "C" int64_t sis3d_launch_count(void) { return (int64_t)sis3d::g_launch_count; }

// ---- host-side planner of the ragged mask stage (pure CPU code: the "runtime" part of the per-RoI mask head) ------
// From the decoded detection table it lays out, in one byte blob that the caller ships with a single pinned H2D copy:
// region tables of the first (windowed NCDHW scene -> canvas/compact) and last (-> dense per-crop output) layers, the
// brick list of the tensor-core layers (canvas mode; 4x4x8 bricks, from sis3d_conv3d_tc_brick) or the region table of the
// middle layers (compact mode), voxel offsets, predicted classes, kept row indices and crop sizes.  Mirrors
// lib/nets/network.py:296-311 (crop selection).
extern "C" int sis3d_mask_plan_build(const float *h_det, int n, int X, int Y, int Z, int ncls, int use_canvas, void *h_blob,
                                     size_t capacity, sis3d_mask_plan *plan) {
    if (!h_det || !plan || n < 0) return SIS3D_EINVAL;
    sis3d_mask_plan p = {};
    // every row with the keep flag set gets a crop (the list is as long as the detection table: no cap, no allocation)
    for (int i = 0; i < n; ++i)
        if (h_det[i * 16 + 8] > 0.5f) ++p.n_kept;
    const int nk = p.n_kept;
    if (nk == 0) { *plan = p; return SIS3D_OK; }
    // pass 1: sizes
    int64_t total = 0, xsum = 0;
    int ymax = 0, zmax = 0;
    int64_t ntiles = 0, t_mid = 0;
    int32_t brick[3];  // the bricks of the tensor-core layers' tile lists
    sis3d_conv3d_tc_brick(1, 3, 64, 64, &brick[0], &brick[1], &brick[2]);
    for (int i = 0; i < n; ++i) {
        const float *d = h_det + i * 16;
        if (!(d[8] > 0.5f)) continue;
        const int w = (int)d[12] - (int)d[9], h = (int)d[13] - (int)d[10], l = (int)d[14] - (int)d[11];
        total += (int64_t)w * h * l;
        xsum += w + 1;
        ymax = h > ymax ? h : ymax;
        zmax = l > zmax ? l : zmax;
        ntiles += (int64_t)((w + brick[0] - 1) / brick[0]) * ((h + brick[1] - 1) / brick[1]) * ((l + brick[2] - 1) / brick[2]);
        t_mid += ((int64_t)w * h * l + SIS3D_CONV_TILE_M - 1) / SIS3D_CONV_TILE_M;
    }
    p.total_voxels = total;
    p.canvas[0] = (int)xsum; p.canvas[1] = ymax; p.canvas[2] = zmax;
    p.n_tiles_tc = use_canvas ? (int)ntiles : 0;
    const size_t rb = sizeof(sis3d_region) * (size_t)nk;
    p.off_first = 0;
    p.off_last = rb;
    p.off_rest = 2 * rb;
    const size_t rest = use_canvas ? (size_t)ntiles * 32 : rb;
    p.off_offs = (p.off_rest + rest + 7) & ~(size_t)7;
    p.off_cls = p.off_offs + 8 * (size_t)(nk + 1);
    p.off_kept = p.off_cls + 4 * (size_t)nk;
    p.off_sizes = p.off_kept + 4 * (size_t)nk;
    p.bytes = p.off_sizes + 12 * (size_t)nk;
    if (!h_blob || capacity < (size_t)p.bytes) { *plan = p; return SIS3D_EWORKSPACE; }
    char *blob = (char *)h_blob;
    sis3d_region *first = (sis3d_region *)(blob + p.off_first), *last = (sis3d_region *)(blob + p.off_last);
    sis3d_region *mid = (sis3d_region *)(blob + p.off_rest);
    int32_t *tiles = (int32_t *)(blob + p.off_rest);
    int64_t *offs = (int64_t *)(blob + p.off_offs);
    int32_t *cls = (int32_t *)(blob + p.off_cls), *kidx = (int32_t *)(blob + p.off_kept), *sizes = (int32_t *)(blob + p.off_sizes);
    const int64_t cs0 = (int64_t)ymax * zmax * 64, cs1 = (int64_t)zmax * 64, cs2 = 64;
    int64_t voff = 0, xoff = 0, tile_no = 0;
    int tb = 0;
    for (int i = 0, j = 0; i < n; ++i) {
        const float *d = h_det + i * 16;
        if (!(d[8] > 0.5f)) continue;
        const int x0 = (int)d[9], y0 = (int)d[10], z0 = (int)d[11];
        const int w = (int)d[12] - x0, h = (int)d[13] - y0, l = (int)d[14] - z0;
        const int64_t vox = (int64_t)w * h * l;
        const int tl = (int)((vox + SIS3D_CONV_TILE_M - 1) / SIS3D_CONV_TILE_M);
        sis3d_region f = {}, q = {};
        f.in_off = ((int64_t)x0 * Y + y0) * Z + z0;
        f.in_dim[0] = f.out_dim[0] = w; f.in_dim[1] = f.out_dim[1] = h; f.in_dim[2] = f.out_dim[2] = l;
        f.in_stride[0] = (int64_t)Y * Z; f.in_stride[1] = Z; f.in_stride[2] = 1;
        f.tile_begin = tb;
        q.in_dim[0] = q.out_dim[0] = w; q.in_dim[1] = q.out_dim[1] = h; q.in_dim[2] = q.out_dim[2] = l;
        q.out_off = voff * ncls;
        q.tile_begin = tb;
        if (use_canvas) {
            f.out_off = xoff * cs0;
            f.out_stride[0] = cs0; f.out_stride[1] = cs1; f.out_stride[2] = cs2;
            q.in_off = xoff * cs0;
            q.in_stride[0] = cs0; q.in_stride[1] = cs1; q.in_stride[2] = cs2;
            for (int bx = 0; bx < w; bx += brick[0])
                for (int by = 0; by < h; by += brick[1])
                    for (int bz = 0; bz < l; bz += brick[2]) {
                        int32_t *t = tiles + tile_no * 8;
                        t[0] = (int32_t)xoff + bx; t[1] = by; t[2] = bz;
                        t[3] = (int32_t)xoff + w; t[4] = h; t[5] = l; t[6] = t[7] = 0;
                        ++tile_no;
                    }
        } else {
            f.out_off = voff * 64;
            q.in_off = voff * 64;
            q.in_stride[0] = (int64_t)h * l * 64; q.in_stride[1] = (int64_t)l * 64; q.in_stride[2] = 64;
            sis3d_region m = q;
            m.out_off = voff * 64;
            mid[j] = m;
        }
        first[j] = f;
        last[j] = q;
        offs[j] = voff;
        cls[j] = (int32_t)d[7];
        kidx[j] = i;
        sizes[3 * j] = w; sizes[3 * j + 1] = h; sizes[3 * j + 2] = l;
        voff += vox;
        xoff += w + 1;
        tb += tl;
        ++j;
    }
    offs[nk] = voff;
    p.tiles_first = p.tiles_last = p.tiles_mid = tb;
    *plan = p;
    return SIS3D_OK;
}

// ---- ragged mask stage: every launch of one scene's mask head behind ONE host call ---------------------------------------
// (reference: lib/nets/network.py:283-317 loops over the kept RoIs and runs mask_backbone on each crop).  The tables come
// from sis3d_mask_plan_build (pinned host blob); this call queues their H2D copy, zeroes the canvases, launches the six
// layers + the predicted-class select and, when bits_host is given, the D2H copy of the thresholded masks.
extern "C" int sis3d_mask_stage_launch(const sis3d_mask_plan *p, const void *h_blob, const sis3d_mask_stage *a, void *stream) {
    if (!p || !h_blob || !a || !a->scene || !a->w_first || !a->w_last || !a->tables || !a->canvas || !a->masks) return SIS3D_EINVAL;
    const int nk = p->n_kept, ncls = a->ncls;
    if (nk <= 0) return SIS3D_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t total = p->total_voxels;
    const int Xc = p->canvas[0], Yc = p->canvas[1], Zc = p->canvas[2];
    const int64_t cvox = (int64_t)Xc * Yc * Zc;
    const size_t need = a->math == 0 ? (size_t)total * 64 * 4 * 2 : (size_t)cvox * 64 * (a->math == 2 ? 2 : 4) * 2;
    if (a->canvas_bytes < need) return SIS3D_EWORKSPACE;
    if (a->math == 2 && (!a->canvas32 || a->canvas32_bytes < (size_t)cvox * 64 * 4)) return SIS3D_EWORKSPACE;
    for (int i = 0; i < 4; ++i)
        if (!a->w_mid[i]) return SIS3D_EINVAL;
    if (cudaMemcpyAsync(a->tables, h_blob, (size_t)p->bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return SIS3D_ELAUNCH;
    char *tb = (char *)a->tables;
    const sis3d_region *r_first = (const sis3d_region *)(tb + p->off_first), *r_last = (const sis3d_region *)(tb + p->off_last);
    const int64_t scene_vox = (int64_t)a->X * a->Y * a->Z;
    int rc;
    const float *x32 = nullptr;
    if (a->math == 0) {  // compact per-crop buffers, fp32 CUDA-core kernel throughout
        float *b0 = (float *)a->canvas, *b1 = b0 + total * 64;
        const sis3d_region *r_mid = (const sis3d_region *)(tb + p->off_rest);
        if ((rc = sis3d_conv3d_ex(a->scene, scene_vox, a->w_first, nullptr, nullptr, 0, 0, b0, nullptr, 64, 0, r_first, nk,
                                  p->tiles_first, 2, 64, 3, 1, 1, 1, stream))) return rc;
        float *cur = b0, *nxt = b1;
        for (int i = 0; i < 4; ++i) {
            if ((rc = sis3d_conv3d_ex(cur, 1, (const float *)a->w_mid[i], nullptr, nullptr, 0, 0, nxt, nullptr, 64, 0, r_mid, nk,
                                      p->tiles_mid, 64, 64, 3, 1, 1, 1, stream))) return rc;
            float *t = cur; cur = nxt; nxt = t;
        }
        x32 = cur;
    } else {
        const int32_t *tiles = (const int32_t *)(tb + p->off_rest);
        if (cudaMemsetAsync(a->canvas, 0, need, st) != cudaSuccess) return SIS3D_ELAUNCH;
        if (a->math == 2) {
            uint16_t *h0 = (uint16_t *)a->canvas, *h1 = h0 + cvox * 64;
            if ((rc = sis3d_conv3d_ex(a->scene, scene_vox, a->w_first, nullptr, nullptr, 0, 0, nullptr, h0, 64, 0, r_first, nk,
                                      p->tiles_first, 2, 64, 3, 1, 1, 1, stream))) return rc;
            uint16_t *cur = h0, *nxt = h1;
            for (int i = 0; i < 4; ++i) {
                const bool last3 = i == 3;
                if ((rc = sis3d_conv3d_tc_f16(cur, (const uint16_t *)a->w_mid[i], nullptr, nullptr, 0, 0, last3 ? a->canvas32 : nullptr,
                                              last3 ? nullptr : nxt, 64, 0, Xc, Yc, Zc, 64, 64, 3, tiles, p->n_tiles_tc, 1, stream)))
                    return rc;
                uint16_t *t = cur; cur = nxt; nxt = t;
            }
            x32 = a->canvas32;
        } else {
            float *b0 = (float *)a->canvas, *b1 = b0 + cvox * 64;
            if ((rc = sis3d_conv3d_ex(a->scene, scene_vox, a->w_first, nullptr, nullptr, 0, 0, b0, nullptr, 64, 0, r_first, nk,
                                      p->tiles_first, 2, 64, 3, 1, 1, 1, stream))) return rc;
            float *cur = b0, *nxt = b1;
            for (int i = 0; i < 4; ++i) {
                if ((rc = sis3d_conv3d_k3_tc(cur, (const float *)a->w_mid[i], nullptr, nullptr, 0, 0, nxt, 64, 0, Xc, Yc, Zc, 64, 64,
                                             3, tiles, p->n_tiles_tc, 1, stream))) return rc;
                float *t = cur; cur = nxt; nxt = t;
            }
            x32 = cur;
        }
    }
    if ((rc = sis3d_conv3d_ex(x32, 1, a->w_last, nullptr, nullptr, 0, 0, a->masks, nullptr, ncls, 0, r_last, nk, p->tiles_last, 64,
                              ncls, 1, 1, 0, 2, stream))) return rc;
    if (a->bits) {
        if ((rc = sis3d_mask_select(a->masks, (const int64_t *)(tb + p->off_offs), (const int32_t *)(tb + p->off_cls), nk, ncls,
                                    total, a->thresh, nullptr, a->bits, stream))) return rc;
        if (a->bits_host && cudaMemcpyAsync(a->bits_host, a->bits, (size_t)total, cudaMemcpyDeviceToHost, st) != cudaSuccess)
            return SIS3D_ELAUNCH;
    }
    return SIS3D_OK;
}

// ---- colour-aware ragged mask stage (MASK_USE_IMAGES / MASK_ONLY_IMAGES) -----------------------------------------------------
// Buffers, in the route's operand type: A and B (64 channels) ping-pong through each stack; I (128 channels) holds the
// gathered colour input until colour.0 has read it, then the concatenation [geometry | colour] that the two 1x1s write; A and B
// together (128 channels) then hold combine.0's output (math 2: canvas32).  The canvas routes keep every voxel outside the
// crops zero (the crops' padding): nothing writes there.  The 128 -> 128 combine.0 runs as two 128 -> 64 halves on the
// 4x4x8-brick instances, the ones colour.0 and the 64 -> 64 layers use.
extern "C" int sis3d_mask_stage_color_launch(const sis3d_mask_plan *p, const sis3d_mask_color_plan *cp, const void *h_blob,
                                             const sis3d_mask_stage_color *a, void *stream) {
    if (!p || !cp || !h_blob || !a || !a->scene || !a->w_color_first || !a->w_color_last || !a->tables || !a->canvas || !a->masks)
        return SIS3D_EINVAL;
    const bool full = !a->only_images;
    if (full && (!a->w_geom_first || !a->w_geom_last || !a->w_combine || !a->w_combine_last)) return SIS3D_EINVAL;
    for (int i = 0; i < 4; ++i)
        if (!a->w_color_mid[i] || (full && !a->w_geom_mid[i])) return SIS3D_EINVAL;
    if (a->math < 0 || a->math > 2) return SIS3D_EINVAL;
    const int nk = p->n_kept, ncls = a->ncls;
    if (nk <= 0) return SIS3D_OK;
    if (a->crop_in ? nk != 1 : (!a->feats_t || !a->pix || !a->pairs || !a->n_pairs || a->n_views <= 0 || a->hw <= 0))
        return SIS3D_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t total = p->total_voxels;
    const int Xc = p->canvas[0], Yc = p->canvas[1], Zc = p->canvas[2];
    const int64_t cvox = (int64_t)Xc * Yc * Zc, vox = a->math == 0 ? total : cvox;
    const size_t eb = a->math == 2 ? 2 : 4, need = (size_t)vox * 64 * eb * 4;
    if (a->canvas_bytes < need) return SIS3D_EWORKSPACE;
    if (a->math == 2 && (!a->canvas32 || a->canvas32_bytes < (size_t)cvox * (full ? 128 : 64) * 4)) return SIS3D_EWORKSPACE;
    if (cudaMemcpyAsync(a->tables, h_blob, (size_t)cp->bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return SIS3D_ELAUNCH;
    if (a->math && cudaMemsetAsync(a->canvas, 0, need, st) != cudaSuccess) return SIS3D_ELAUNCH;
    char *tb = (char *)a->tables;
    const sis3d_region *r_first = (const sis3d_region *)(tb + p->off_first), *r_last = (const sis3d_region *)(tb + p->off_last);
    const sis3d_region *r_mid = (const sis3d_region *)(tb + p->off_rest), *r_g2c = (const sis3d_region *)(tb + cp->off_g2c);
    const sis3d_region *r_last128 = (const sis3d_region *)(tb + cp->off_last128);
    const int32_t *tiles = (const int32_t *)(tb + p->off_rest);
    const int nt = p->n_tiles_tc;
    const int64_t scene_vox = (int64_t)a->X * a->Y * a->Z;
    char *A = (char *)a->canvas, *B = A + (size_t)vox * 64 * eb, *I = B + (size_t)vox * 64 * eb;
    int rc;
    // colour input
    if (a->crop_in) {  // one crop at canvas x 0 (canvas y, z = the crop's h, l): its voxels are the first w*h*l rows, as compact
        if (a->math == 2) {
            if ((rc = sis3d_cast_f16(a->crop_in, 128, 0, total, 128, (uint16_t *)I, stream))) return rc;
        } else if (cudaMemcpyAsync(I, a->crop_in, (size_t)total * 128 * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
            return SIS3D_ELAUNCH;
        }
    } else if ((rc = sis3d_mask_color_gather(a->feats_t, a->pix, a->pairs, a->n_pairs, a->n_views, 128, a->hw, a->X, a->Y, a->Z,
                                             (const int32_t *)(tb + cp->off_crops), (const int64_t *)(tb + p->off_offs), nk, total,
                                             Yc, Zc, a->math, I, stream))) {
        return rc;
    }
    // one 3x3x3 stack: first layer (scene or colour input) -> A, four 64 -> 64 layers; returns the fp32 input of its 1x1
    auto stack = [&](bool colour, const float **x32) -> int {
        const void *const *mid = colour ? a->w_color_mid : a->w_geom_mid;
        if (a->math == 0) {
            float *cur = (float *)A, *nxt = (float *)B;
            if (colour) rc = sis3d_conv3d_ex((const float *)I, 1, (const float *)a->w_color_first, nullptr, nullptr, 0, 0, cur, nullptr,
                                             64, 0, (const sis3d_region *)(tb + cp->off_c0), nk, p->tiles_mid, 128, 64, 3, 1, 1, 1, stream);
            else rc = sis3d_conv3d_ex(a->scene, scene_vox, a->w_geom_first, nullptr, nullptr, 0, 0, cur, nullptr, 64, 0, r_first, nk,
                                      p->tiles_first, 2, 64, 3, 1, 1, 1, stream);
            if (rc) return rc;
            for (int i = 0; i < 4; ++i) {
                if ((rc = sis3d_conv3d_ex(cur, 1, (const float *)mid[i], nullptr, nullptr, 0, 0, nxt, nullptr, 64, 0, r_mid, nk,
                                          p->tiles_mid, 64, 64, 3, 1, 1, 1, stream))) return rc;
                float *t = cur; cur = nxt; nxt = t;
            }
            *x32 = cur;
        } else if (a->math == 2) {
            uint16_t *cur = (uint16_t *)A, *nxt = (uint16_t *)B;
            if (colour) rc = sis3d_conv3d_tc_f16((const uint16_t *)I, (const uint16_t *)a->w_color_first, nullptr, nullptr, 0, 0, nullptr,
                                                 cur, 64, 0, Xc, Yc, Zc, 128, 64, 3, tiles, nt, 1, stream);
            else rc = sis3d_conv3d_ex(a->scene, scene_vox, a->w_geom_first, nullptr, nullptr, 0, 0, nullptr, cur, 64, 0, r_first, nk,
                                      p->tiles_first, 2, 64, 3, 1, 1, 1, stream);
            if (rc) return rc;
            for (int i = 0; i < 4; ++i) {
                const bool last3 = i == 3;
                if ((rc = sis3d_conv3d_tc_f16(cur, (const uint16_t *)mid[i], nullptr, nullptr, 0, 0, last3 ? a->canvas32 : nullptr,
                                              last3 ? nullptr : nxt, 64, 0, Xc, Yc, Zc, 64, 64, 3, tiles, nt, 1, stream))) return rc;
                uint16_t *t = cur; cur = nxt; nxt = t;
            }
            *x32 = a->canvas32;
        } else {
            float *cur = (float *)A, *nxt = (float *)B;
            if (colour) rc = sis3d_conv3d_k3_tc((const float *)I, (const float *)a->w_color_first, nullptr, nullptr, 0, 0, cur, 64, 0,
                                                Xc, Yc, Zc, 128, 64, 3, tiles, nt, 1, stream);
            else rc = sis3d_conv3d_ex(a->scene, scene_vox, a->w_geom_first, nullptr, nullptr, 0, 0, cur, nullptr, 64, 0, r_first, nk,
                                      p->tiles_first, 2, 64, 3, 1, 1, 1, stream);
            if (rc) return rc;
            for (int i = 0; i < 4; ++i) {
                if ((rc = sis3d_conv3d_k3_tc(cur, (const float *)mid[i], nullptr, nullptr, 0, 0, nxt, 64, 0, Xc, Yc, Zc, 64, 64, 3, tiles,
                                             nt, 1, stream))) return rc;
                float *t = cur; cur = nxt; nxt = t;
            }
            *x32 = cur;
        }
        return SIS3D_OK;
    };
    // a stack's 1x1 (64 -> 64, no ReLU) writing channels [coff, coff + 64) of the concatenation in I
    auto to_cat = [&](const float *x32, const float *w, int coff) -> int {
        return sis3d_conv3d_ex(x32, 1, w, nullptr, nullptr, 0, 0, a->math == 2 ? nullptr : (float *)I,
                               a->math == 2 ? (uint16_t *)I : nullptr, 128, coff, r_g2c, nk, p->tiles_last, 64, 64, 1, 1, 0, 0, stream);
    };
    const float *x32 = nullptr, *head_in = nullptr;
    if ((rc = stack(true, &x32))) return rc;
    if (!full) {
        if ((rc = sis3d_conv3d_ex(x32, 1, a->w_color_last, nullptr, nullptr, 0, 0, a->masks, nullptr, ncls, 0, r_last, nk, p->tiles_last,
                                  64, ncls, 1, 1, 0, 2, stream))) return rc;
    } else {
        if ((rc = to_cat(x32, a->w_color_last, 64))) return rc;
        if ((rc = stack(false, &x32))) return rc;
        if ((rc = to_cat(x32, a->w_geom_last, 0))) return rc;
        // combine.0: 128 -> 128 + ReLU
        if (a->math == 0) {
            rc = sis3d_conv3d_ex((const float *)I, 1, (const float *)a->w_combine, nullptr, nullptr, 0, 0, (float *)A, nullptr, 128, 0,
                                 (const sis3d_region *)(tb + cp->off_c128), nk, p->tiles_mid, 128, 128, 3, 1, 1, 1, stream);
            head_in = (const float *)A;
        } else {
            const size_t half = (size_t)64 * 27 * 128;  // weight rows of 64 output channels
            for (int hh = 0; hh < 2 && !rc; ++hh) {
                if (a->math == 2)
                    rc = sis3d_conv3d_tc_f16((const uint16_t *)I, (const uint16_t *)a->w_combine + hh * half, nullptr, nullptr, 0, 0,
                                             a->canvas32, nullptr, 128, 64 * hh, Xc, Yc, Zc, 128, 64, 3, tiles, nt, 1, stream);
                else
                    rc = sis3d_conv3d_k3_tc((const float *)I, (const float *)a->w_combine + hh * half, nullptr, nullptr, 0, 0,
                                            (float *)A, 128, 64 * hh, Xc, Yc, Zc, 128, 64, 3, tiles, nt, 1, stream);
            }
            head_in = a->math == 2 ? a->canvas32 : (const float *)A;
        }
        if (rc) return rc;
        if ((rc = sis3d_conv3d_ex(head_in, 1, a->w_combine_last, nullptr, nullptr, 0, 0, a->masks, nullptr, ncls, 0, r_last128, nk,
                                  p->tiles_last, 128, ncls, 1, 1, 0, 2, stream))) return rc;
    }
    if (a->bits) {
        if ((rc = sis3d_mask_select(a->masks, (const int64_t *)(tb + p->off_offs), (const int32_t *)(tb + p->off_cls), nk, ncls,
                                    total, a->thresh, nullptr, a->bits, stream))) return rc;
        if (a->bits_host && cudaMemcpyAsync(a->bits_host, a->bits, (size_t)total, cudaMemcpyDeviceToHost, st) != cudaSuccess)
            return SIS3D_ELAUNCH;
    }
    return SIS3D_OK;
}

// thin async-copy entry point for hosts that stage their own pinned buffers (kind: 1 H2D, 2 D2H, 3 D2D)
extern "C" int sis3d_memcpy_async(void *dst, const void *src, size_t bytes, int kind, void *stream) {
    if (!dst || !src) return SIS3D_EINVAL;
    if (bytes == 0) return SIS3D_OK;
    const cudaMemcpyKind k = kind == 1 ? cudaMemcpyHostToDevice : kind == 2 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    return cudaMemcpyAsync(dst, src, bytes, k, (cudaStream_t)stream) == cudaSuccess ? SIS3D_OK : SIS3D_ELAUNCH;
}

// ---- per-view constants of the back-projection, host code (lib/layer_utils/projection.py:27-60) ---------------------------
// Packs world_to_camera | grid_to_world | clamped frustum AABB for every view into out[n][40] (layout of sis3d_project_map).
// The two 4x4 inverses are supplied by the caller (torch.inverse, as in the reference); the 8-corner frustum bounds are
// computed here with the arithmetic of the reference's tiny torch.bmm calls (fp32, separate multiply and add, k = 0..3)
// so the cull bounds are bit-identical (checked on random poses in tests/test_view_params.py).
static inline void matvec4(const float *m, const float *v, float *o) {
    for (int r = 0; r < 4; ++r) {
        volatile float acc = 0.f;  // volatile: one rounding per multiply and per add, never an FMA
        for (int k = 0; k < 4; ++k) {
            volatile float p = m[r * 4 + k] * v[k];
            acc = acc + p;
        }
        o[r] = acc;
    }
}
extern "C" int sis3d_view_params_host(const float *poses, const float *w2g, const float *inv_poses, const float *inv_w2g, int n,
                                      int n_w2g, double fx, double fy, double cx, double cy, int img_w, int img_h,
                                      double depth_min, double depth_max, int X, int Y, int Z, float *out) {
    if (!poses || !w2g || !inv_poses || !inv_w2g || !out || n <= 0 || (n_w2g != 1 && n_w2g != n)) return SIS3D_EINVAL;
    float corners[8][4];
    int c = 0;
    const double ds[2] = {depth_min, depth_max};
    for (int di = 0; di < 2; ++di) {
        const int ux[4] = {0, img_w - 1, img_w - 1, 0}, uy[4] = {0, 0, img_h - 1, img_h - 1};
        for (int j = 0; j < 4; ++j, ++c) {  // depth_to_skeleton in Python doubles, stored as fp32 (projection.py:16-19)
            const double x = (ux[j] - cx) / fx, y = (uy[j] - cy) / fy;
            corners[c][0] = (float)(ds[di] * x); corners[c][1] = (float)(ds[di] * y); corners[c][2] = (float)ds[di]; corners[c][3] = 1.f;
        }
    }
    const float dims[3] = {(float)X, (float)Y, (float)Z};
    for (int i = 0; i < n; ++i) {
        const float *c2w = poses + 16 * i, *g = w2g + 16 * (n_w2g == 1 ? 0 : i);
        float *o = out + 40 * i;
        for (int k = 0; k < 16; ++k) { o[k] = inv_poses[16 * i + k]; o[16 + k] = inv_w2g[16 * (n_w2g == 1 ? 0 : i) + k]; }
        float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int k = 0; k < 8; ++k) {
            float p[4], pf[4], pc[4], l[4], u[4];
            matvec4(c2w, corners[k], p);
            for (int r = 0; r < 4; ++r) { pf[r] = floorf(p[r]); pc[r] = ceilf(p[r]); }
            matvec4(g, pf, l);
            matvec4(g, pc, u);
            for (int r = 0; r < 3; ++r) {
                const float a = nearbyintf(l[r]), b = nearbyintf(u[r]);  // torch.round: half to even
                lo[r] = fminf(lo[r], fminf(a, b));
                hi[r] = fmaxf(hi[r], fmaxf(a, b));
            }
        }
        for (int r = 0; r < 3; ++r) { o[32 + r] = fmaxf(lo[r], 0.f); o[35 + r] = fminf(hi[r], dims[r]); }
        o[38] = o[39] = 0.f;
    }
    return SIS3D_OK;
}
