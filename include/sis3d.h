/*
 * sis3d.h -- C ABI of libsis3d.so: the H100 (sm_90a) dense-voxel inference hot path of 3D-SIS.
 *
 * Conventions (all entry points):
 *   - plain pointers + sizes, no torch types; every pointer is a DEVICE pointer unless named h_*;
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on that stream, allocate
 *     nothing and never call exit(); caller owns all memory (workspace sizes via *_workspace_bytes);
 *   - return 0 on success, a negative SIS3D_E* code otherwise (see sis3d_strerror);
 *   - "VC layout" = channels-last voxel tensor [X][Y][Z][C] fp32 (C contiguous); "NCDHW" = the
 *     reference's [1][C][X][Y][Z] layout.
 *
 * Each entry cites the reference interface it replaces (paths relative to the reference root).
 */
#ifndef SIS3D_H
#define SIS3D_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define SIS3D_OK 0
#define SIS3D_EINVAL (-1)   /* bad argument (shape, alignment, null pointer) */
#define SIS3D_ELAUNCH (-2)  /* CUDA launch / runtime error (cudaGetLastError) */
#define SIS3D_EWORKSPACE (-3)
#define SIS3D_EUNSUPPORTED (-4)

const char *sis3d_strerror(int code);
int sis3d_version(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
int64_t sis3d_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * 3D greedy NMS.  Replaces  int gpu_nms(THLongTensor* keep, THLongTensor* num_out, THCudaTensor*
 * boxes, float thresh)  (lib/layer_utils/nms/src/nms_cuda.h:1, src/nms_cuda.c:10-67) and the kernel
 * ABI  void _nms(int, float*, unsigned long long*, float)  (src/cuda/nms_kernel.h:14).
 * boxes [n,6] fp32 sorted by descending score; keep int64[n] (device), num_out int32[1] (device).
 * IoU arithmetic is bit-identical to the reference CUDA build (inclusive +1 extents, one FFMA).
 * workspace: sis3d_nms_workspace_bytes(n) bytes, 8-byte aligned.
 * ---------------------------------------------------------------------------------------------- */
size_t sis3d_nms_workspace_bytes(int n);
int sis3d_nms(const float *boxes, int n, float thresh, int64_t *keep, int32_t *num_out,
              void *workspace, void *stream);

/* ------------------------------------------------------------------------------------------------
 * 3D RoI max pooling forward.  Replaces  int ROIPoolForwardLaucher(const float* bottom, float
 * scale, int num_rois, int width, int height, int length, int channels, int pw, int ph, int pl,
 * const float* rois, float* top, int* argmax, cudaStream_t)
 * (lib/layer_utils/roi_pooling/src/cuda/roi_pooling_kernel.h:8-12) and roi_pooling_forward_cuda
 * (src/roi_pooling_cuda.h:1-2).  feat_layout: 0 = NCDHW (reference), 1 = VC.
 * rois [n,6]; top [n,C,pw,ph,pl]; argmax int32 same shape or NULL (indices in the NCDHW convention).
 * sis3d_roi_pool_levels is the pyramid form used by the forward (lib/nets/network.py:503-534): VC
 * features of up to three levels, level_ids int32[n] (1-based, 0 = padded row -> zeros) pick the map.
 * channels, pw, ph and pl must be positive (SIS3D_EINVAL); the VC kernels need pw*ph <= 65535
 * (SIS3D_EUNSUPPORTED).
 * ---------------------------------------------------------------------------------------------- */
int sis3d_roi_pool_fwd(const float *feat, int feat_layout, float spatial_scale, int num_rois,
                       int width, int height, int length, int channels, int pw, int ph, int pl,
                       const float *rois, float *top, int32_t *argmax, void *stream);
int sis3d_roi_pool_levels(const float *feat1, const float *feat2, const float *feat3,
                          const int32_t *level_ids, float spatial_scale, int num_rois, int width,
                          int height, int length, int channels, int pw, int ph, int pl,
                          const float *rois, float *top, int32_t *argmax, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Back-projection.  Replaces ProjectionHelper.compute_projection (lib/layer_utils/projection.py:
 * 52-121) and Projection.forward + the running max of lib/nets/network.py:220-239.
 *
 * views: float[n_views][40] per view = world_to_camera(16) | grid_to_world(16) | bounds_min(3) |
 *        bounds_max(3) | pad(2)   (row-major 4x4; bounds already clamped to the volume)
 * depth: float[n_views][img_h][img_w];   fx, fy, cx, cy = pinhole intrinsics of the depth image
 * sis3d_project_map     : pix int16[n_views][Z*Y*X] = v*img_w+u of the pixel a voxel projects to or
 *                         -1; index = z*X*Y + y*X + x (the reference's linear index); counts
 *                         int32[n_views] = number of valid voxels per view (zeroed by the call).
 * sis3d_project_compact : ordered compaction of one view's map into the reference's (lin3d, lin2d)
 *                         int64 lists of length 1+Z*Y*X with element 0 = count.
 * An empty volume (X*Y*Z == 0) is a defined empty result: the map call zeroes counts, the compaction
 * writes count 0, and neither launches a kernel.  Negative extents are SIS3D_EINVAL.
 * sis3d_backproject_max : fused gather + cross-view max into a VC volume [X][Y][Z][C]; reproduces
 *                         the reference's pairing of feature maps with surviving index lists when
 *                         views are dropped (pairs from sis3d_backproject_pairs), see DESIGN.md.  feats [n_views][C][h][w]
 *                         (reference layout) are first transposed to [n_views][h*w][C] into
 *                         `feats_t` (workspace of the same size).
 * ---------------------------------------------------------------------------------------------- */
/* Host helper (CPU code): packs the per-view constants views[n][40] from the poses, world2grid and their inverses
 * (the caller inverts the 4x4s, e.g. torch.inverse as the reference does); frustum bounds per projection.py:27-60. */
int sis3d_view_params_host(const float *h_poses, const float *h_w2g, const float *h_inv_poses, const float *h_inv_w2g,
                           int n, int n_w2g, double fx, double fy, double cx, double cy, int img_w, int img_h,
                           double depth_min, double depth_max, int X, int Y, int Z, float *h_out);
int sis3d_project_map(const float *views, const float *depth, int n_views, int img_w, int img_h,
                      float fx, float fy, float cx, float cy, float depth_min, float depth_max, float voxel_size,
                      int X, int Y, int Z, int16_t *pix, int32_t *counts, void *stream);
int sis3d_project_compact(const int16_t *pix, int X, int Y, int Z, int64_t *lin3d, int64_t *lin2d,
                          void *workspace, size_t workspace_bytes, void *stream);
size_t sis3d_project_compact_workspace_bytes(int X, int Y, int Z);
/* pairs int32[3*n_views] (2*n_pairs used), n_pairs int32[1]: (feature map, index map) pairing derived
 * on the device from counts -- no host round trip. */
int sis3d_backproject_pairs(const int32_t *counts, int n_views, int32_t *pairs, int32_t *n_pairs, void *stream);
/* reference-style index lists [n_lists][1+Z*Y*X] (lib/layer_utils/projection.py:110-121) -> dense maps */
int sis3d_project_scatter_lists(const int64_t *lin3d, const int64_t *lin2d, int n_lists, int X, int Y, int Z,
                                int16_t *pix, void *stream);
int sis3d_backproject_max(const float *feats, float *feats_t, const int16_t *pix,
                          const int32_t *pairs, const int32_t *n_pairs, int n_views, int C,
                          int img_w, int img_h, int X, int Y, int Z, float *volume_vc, void *stream);

/* Back-projection fused with the first colour convolution (2x2x2, stride 2, no bias, ReLU;
 * lib/nets/backbones.py:203 / :137): out = relu(conv3d(max-over-views back-projection, W, stride 2))
 * WITHOUT materialising the (>= 95 % zero) feature volume: covered voxels are listed per tap, multiplied by
 * that tap's weight slice and combined per output voxel in tap order (csrc/sparse.cu).  Arguments as for
 * sis3d_backproject_max; w_packed from sis3d_pack_conv_weight(ks=2) ([8*C][cout]); out is VC
 * [X/2][Y/2][Z/2][cout] with row stride out_ld / channel offset out_coff.  C % 16 == 0, cout in {32,64}. */
size_t sis3d_backproject_conv_k2s2_workspace_bytes(int X, int Y, int Z, int cout);
int sis3d_backproject_conv_k2s2(const float *feats, float *feats_t, const int16_t *pix, const int32_t *pairs,
                                const int32_t *n_pairs, int n_views, int C, int img_w, int img_h, int X,
                                int Y, int Z, const float *w_packed, int cout, float *out, int out_ld,
                                int out_coff, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * 3D convolution (implicit GEMM) over a table of regions.  Replaces the nn.Conv3d call sites of
 * lib/nets/backbones.py:20-22,126-169,188-231,241-272 and lib/nets/network.py:40-52 (cuDNN in the
 * reference).  One launch processes `n_regions` independent volumes (1 for the backbone, one per
 * RoI crop for the mask head, lib/nets/network.py:303-317).
 * Weights are pre-packed by sis3d_pack_conv_weight into [ks^3*cin][cout] (k = tap*cin + c,
 * tap = (kx*ks+ky)*ks+kz).  Output is VC with row stride out_ld and channel offset out_coff (lets a
 * producer write straight into a concatenated tensor); optional bias[cout], residual (VC, res_ld /
 * res_coff), act: 0 none, 1 relu, 2 sigmoid.
 * ---------------------------------------------------------------------------------------------- */
typedef struct sis3d_region {
    int64_t in_off;   /* element offset of the region's input voxel (0,0,0) */
    int64_t out_off;  /* element offset of the region's output voxel (0,0,0), before out_coff */
    int64_t res_off;
    int32_t in_dim[3];     /* input extent (x,y,z): taps outside read as zero */
    int32_t out_dim[3];    /* output extent */
    int64_t in_stride[3];  /* input voxel strides in elements (x,y,z) */
    int64_t out_stride[3]; /* output voxel strides in elements; all zero = dense rows (m * out_ld) */
    int32_t tile_begin;    /* first M-tile of this region (exclusive prefix sum of tile counts) */
    int32_t pad_;
} sis3d_region;

#define SIS3D_CONV_TILE_M 64
int sis3d_pack_conv_weight(const float *w_oidhw, int cout, int cin, int ks, float *w_packed, void *stream);
int sis3d_conv3d(const float *in, int64_t in_chan_stride, const float *w_packed, const float *bias,
                 const float *residual, int res_ld, int res_coff, float *out, int out_ld, int out_coff,
                 const sis3d_region *regions, int n_regions, int n_tiles, int cin, int cout, int ks,
                 int stride, int pad, int act, void *stream);
/* Fully connected layer y[M][N] = act(x[M][K] . W + b) for the RoI classifier MLP (lib/nets/backbones.py:
 * 92-96,225-231): split-K over `splits` CTAs-per-tile with a deterministic second-pass reduction.
 * w_packed from sis3d_pack_conv_weight(ks=1).  workspace >= sis3d_linear_workspace_bytes(M,N,K). */
size_t sis3d_linear_workspace_bytes(int M, int N, int K);
int sis3d_linear(const float *x, const float *w_packed, const float *bias, float *y, int M, int K, int N,
                 int act, void *workspace, size_t workspace_bytes, void *stream);

/* Same layer on the tensor cores (TF32 wgmma, fp32 accumulate, split-K + deterministic reduce): w_nk is the
 * nn.Linear weight as stored, [N][K].  K % 32 == 0, N in {32, 64, 128k}, all sizes positive (the predicate is 0 and the
 * workspace size 0 otherwise; the call returns SIS3D_EINVAL).  workspace >= sis3d_linear_tc_workspace_bytes(M, N, K) bytes in
 * every mode (_tc, _tc_x3, _tc_h3), SIS3D_EWORKSPACE otherwise. */
int sis3d_linear_tc_supported(int K, int N);
size_t sis3d_linear_tc_workspace_bytes(int M, int N, int K);
int sis3d_linear_tc(const float *x, const float *w_nk, const float *bias, float *y, int M, int K, int N, int act,
                    void *workspace, size_t workspace_bytes, void *stream);

/* Layers 2-3 of the classifier MLP and both heads in one launch (activations stay in shared memory):
 * x1 [R][d1] -> relu(W2) [d2] -> relu(W3) [d3] -> cls_score [R][nc] and bbox_pred [R][nb].  All weights packed by
 * sis3d_pack_conv_weight(ks=1); d1,d2,d3 <= 256.  (lib/nets/backbones.py:225-231, lib/nets/network.py:55-57) */
int sis3d_mlp_tail(const float *x1, int R, int d1, const float *w2, const float *b2, int d2, const float *w3,
                   const float *b3, int d3, const float *wc, const float *bc, int nc, const float *wb,
                   const float *bb, int nb, float *cls_score, float *bbox_pred, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Tensor-core path: ks = 3 (stride 1, pad 1), ks = 1, or ks = 2 (the 2x2x2 / stride-2 / pad-0 downsampling convs,
 * lib/nets/backbones.py:182-205; X,Y,Z are then the INPUT extents, the output is [X/2][Y/2][Z/2][cout], tiles must be NULL;
 * the A operand is fetched by TMA boxes with element strides {1,2,2,2}) -- same call sites as sis3d_conv3d:
 * wgmma.mma_async (TF32) with fp32 accumulation in registers, operands staged by 4-D/2-D TMA boxes
 * (csrc/conv_tc.cu).  `in` is a dense VC tensor [X][Y][Z][cin]; w_tc comes from
 * sis3d_pack_conv_weight_tc ([cout][ks^3*cin]).  tiles == NULL covers the whole volume with 8x2x8 (x,y,z)
 * bricks; otherwise (brick shape from sis3d_conv3d_tc_brick) tiles int32[n_tiles][8] = {x0,y0,z0,x1,y1,z1,0,0} lists brick origins and the
 * exclusive end of the voxels to be written (ragged RoI crops packed on one canvas).
 * Requires cin % 32 == 0 and cout in {32, 64, 128k}; returns SIS3D_EUNSUPPORTED otherwise (SIS3D_EINVAL for cin or cout <= 0).
 * ---------------------------------------------------------------------------------------------- */
int sis3d_pack_conv_weight_tc(const float *w_oidhw, int cout, int cin, int ks, float *w_tc, void *stream);
int sis3d_conv3d_k3_tc_supported(int cin, int cout);
/* brick shape (x,y,z) the kernel uses for a layer: 8x2x8 for whole volumes, 4x4x8 for explicit tile lists of 64->64 layers */
void sis3d_conv3d_tc_brick(int with_tile_list, int ks, int cin, int cout, int32_t *bx, int32_t *by, int32_t *bz);
int sis3d_conv3d_k3_tc(const float *in, const float *w_tc, const float *bias, const float *residual,
                       int res_ld, int res_coff, float *out, int out_ld, int out_coff, int X, int Y,
                       int Z, int cin, int cout, int ks, const int32_t *tiles, int n_tiles, int act, void *stream);

/* Bottleneck tail in ONE kernel (lib/nets/backbones.py:28-40: conv2 3x3x3 (+bias2) -> ReLU -> conv3 1x1 (+bias3) -> + residual -> act;
 * biases may be NULL):
 * the cmid-wide intermediate stays in shared memory / registers.  w2_tc / w3_tc from sis3d_pack_conv_weight_tc (ks 3 / ks 1).
 * Supported: cin % 32 == 0 and (cmid, cout) in {(32,32), (32,64), (64,128)}; results equal the two-kernel TF32 path
 * bit for bit (same operand values, same accumulation order). */
int sis3d_conv3d_k3_tc_fused_supported(int cin, int cmid, int cout);
int sis3d_conv3d_k3_tc_fused(const float *in, const float *w2_tc, const float *bias2, const float *w3_tc, const float *bias3,
                             const float *residual, int res_ld, int res_coff, float *out, int out_ld, int out_coff, int X,
                             int Y, int Z, int cin, int cmid, int cout, int act, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Voxel block of a `.scene` / `.chunk` file -> network input, on the device (replaces the host numpy passes of
 * lib/datasets/dataset.py:50-68 + the height crop :192-205).  sdf_xfast: the raw float32 block as stored in the file
 * (index = x + X*(y + Y*z)); data: [2][X][min(Y, y_keep)][Z] (z fastest): channel 0 = |clip(sdf, -truncation, truncation)|,
 * channel 1 = (sdf > -1) as 0/1.  Exact (no rounding involved).
 * ---------------------------------------------------------------------------------------------- */
int sis3d_chunk_decode(const float *sdf_xfast, int X, int Y, int Z, int y_keep, float truncation, float *data, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Error-compensated 3xTF32 on the tensor cores ("x3"): same call sites and arguments as sis3d_conv3d_k3_tc /
 * _fused / sis3d_linear_tc, fp32-class accuracy.  Every fp32 operand is split v = hi + lo (hi = tf32(v), round to
 * nearest; lo = tf32(v - hi)) and the product accumulated as A_lo.B_hi + A_hi.B_lo + A_hi.B_hi in an fp32
 * register accumulator per pipeline stage, added to the running sum with round-to-nearest adds.  Weights are split once (sis3d_pack_conv_weight_tc_x3 -> [2][cout][ks^3*cin]: hi rows, then lo rows; a
 * [N][K] nn.Linear weight is packed as a ks = 1 conv); activations are split in shared memory after the TMA load, so
 * they cross L2->SM once.  This is the mode in which the detector's integer outputs (top-N order, NMS keep lists, class
 * argmax, crop bounds) match the fp32 reference (lib/layer_utils/proposal_layer.py:181-197, lib/nets/network.py:296-301)
 * while the convolutions still run on the tensor cores (wgmma).  Whole volumes only (tiles = NULL).
 * ---------------------------------------------------------------------------------------------- */
int sis3d_pack_conv_weight_tc_x3(const float *w_oidhw, int cout, int cin, int ks, float *w_x3, void *stream);
int sis3d_conv3d_k3_tc_x3(const float *in, const float *w_x3, const float *bias, const float *residual,
                          int res_ld, int res_coff, float *out, int out_ld, int out_coff, int X, int Y,
                          int Z, int cin, int cout, int ks, int act, void *stream);
int sis3d_conv3d_k3_tc_fused_x3(const float *in, const float *w2_x3, const float *bias2, const float *w3_x3,
                                const float *bias3, const float *residual, int res_ld, int res_coff, float *out,
                                int out_ld, int out_coff, int X, int Y, int Z, int cin, int cmid, int cout, int act,
                                void *stream);
int sis3d_linear_tc_x3(const float *x, const float *w_x3, const float *bias, float *y, int M, int K, int N, int act,
                       void *workspace, size_t workspace_bytes, void *stream);
/* The same compensation with an fp16 operand split ("h3"): v = hi + lo / 2048, hi = fp16(v), lo = fp16((v - hi) * 2048) -- the
 * same 11 + 11 significand bits as the TF32 split -- so the three products are f16 wgmmas (twice the TF32 rate
 * of the H100 tensor core) over 32-channel stages.  Activations stay fp32 in HBM (split in shared memory after the TMA load, |v|
 * range-limited to fp16: |v| < 65504); weights from sis3d_pack_conv_weight_tc_h3: fp16 [cout][ks^3*cin/32][64], each 128-byte
 * row = the 32 hi halves of a 32-channel K slice followed by its 32 lo halves (2*cout*ks^3*cin halves in total), so one TMA
 * row request carries both parts.  Same arguments as _x3.
 * Accuracy: per output element |err| <= 2^-15 sqrt(sum_k (x_k w_k)^2) + 2^-22 (|bias| + |residual| + |result|), plus, where an
 * operand lies below fp16's normal range (|v| < 2^-14: its hi part is subnormal and the split keeps its value to 2^-35 absolute),
 * an absolute floor of 2^-34 sum_k |x_k| for weights that small (2^-34 sum_k |w_k| for activations that small).  Checked per
 * element against fp64 by tests/test_gpu_tc_accuracy.py. */
int sis3d_pack_conv_weight_tc_h3(const float *w_oidhw, int cout, int cin, int ks, uint16_t *w_h3, void *stream);
int sis3d_conv3d_k3_tc_h3(const float *in, const uint16_t *w_h3, const float *bias, const float *residual,
                          int res_ld, int res_coff, float *out, int out_ld, int out_coff, int X, int Y,
                          int Z, int cin, int cout, int ks, int act, void *stream);
int sis3d_conv3d_k3_tc_fused_h3(const float *in, const uint16_t *w2_h3, const float *bias2, const uint16_t *w3_h3,
                                const float *bias3, const float *residual, int res_ld, int res_coff, float *out,
                                int out_ld, int out_coff, int X, int Y, int Z, int cin, int cmid, int cout, int act,
                                void *stream);
int sis3d_linear_tc_h3(const float *x, const uint16_t *w_h3, const float *bias, float *y, int M, int K, int N, int act,
                       void *workspace, size_t workspace_bytes, void *stream);
/* Split-pair activations: the fp16 split done once, by the layer that produces the activation.  Per voxel and 32-channel
 * slice one 128-byte row of 32 hi halves = fp16(v) followed by 32 lo halves = fp16((v - hi) * 2048) (the layout of the _h3
 * weights): a dense VC tensor of 2 * C halves per voxel, 4 bytes per channel like fp32.
 * sis3d_conv3d_k1_tc_h3_split: the 1x1 conv of sis3d_conv3d_k3_tc_h3 (ks = 1, no residual, cout % 32 == 0) writing out_split
 * in this format from the same post-bias / activation fp32 value.
 * sis3d_conv3d_k3_tc_fused_h3_split: sis3d_conv3d_k3_tc_fused_h3 reading its input in this format; the result is
 * bit-identical to the fp32-input entry point on the fp32 tensor the split was made from. */
int sis3d_conv3d_k1_tc_h3_split(const float *in, const uint16_t *w_h3, const float *bias, uint16_t *out_split, int X, int Y,
                                int Z, int cin, int cout, int act, void *stream);
int sis3d_conv3d_k3_tc_fused_h3_split(const uint16_t *in_split, const uint16_t *w2_h3, const float *bias2,
                                      const uint16_t *w3_h3, const float *bias3, const float *residual, int res_ld,
                                      int res_coff, float *out, int out_ld, int out_coff, int X, int Y, int Z, int cin,
                                      int cmid, int cout, int act, void *stream);

/* ------------------------------------------------------------------------------------------------
 * fp16-operand tensor-core path (f16 wgmma, fp32 accumulate): activations and weights are STORED as fp16 (same
 * 11-bit significand TF32 keeps, half the bytes through L2 -- the kernel is bound by operand feed).  in16 is a dense VC
 * fp16 tensor; w16 from sis3d_pack_conv_weight_tc_f16; outputs: out32 (fp32, may be NULL) and/or out16 (fp16 twin with
 * the same row stride / channel offset, may be NULL).  cin % 64 == 0 uses 128-B rows, cin == 32 64-B rows.
 * sis3d_cast_f16 makes the fp16 copy of an fp32 VC tensor; sis3d_conv3d_ex / sis3d_backproject_conv_k2s2_ex are the
 * fp32 kernels with an optional fp16 twin output.
 * ---------------------------------------------------------------------------------------------- */
int sis3d_pack_conv_weight_tc_f16(const float *w_oidhw, int cout, int cin, int ks, uint16_t *w16, void *stream);
int sis3d_cast_f16(const float *in, int in_ld, int in_coff, int64_t rows, int C, uint16_t *out, void *stream);
int sis3d_conv3d_tc_f16(const uint16_t *in16, const uint16_t *w16, const float *bias, const float *residual,
                        int res_ld, int res_coff, float *out32, uint16_t *out16, int out_ld, int out_coff, int X,
                        int Y, int Z, int cin, int cout, int ks, const int32_t *tiles, int n_tiles, int act, void *stream);
int sis3d_conv3d_ex(const float *in, int64_t in_chan_stride, const float *w_packed, const float *bias,
                    const float *residual, int res_ld, int res_coff, float *out, uint16_t *out16, int out_ld,
                    int out_coff, const sis3d_region *regions, int n_regions, int n_tiles, int cin, int cout, int ks,
                    int stride, int pad, int act, void *stream);
int sis3d_backproject_conv_k2s2_ex(const float *feats, float *feats_t, const int16_t *pix, const int32_t *pairs,
                                   const int32_t *n_pairs, int n_views, int C, int img_w, int img_h, int X, int Y,
                                   int Z, const float *w_packed, int cout, float *out, uint16_t *out16, int out_ld,
                                   int out_coff, void *workspace, size_t workspace_bytes, void *stream);

/* MaxPool3d(3,1,1) on a VC tensor (lib/nets/backbones.py:207,212,220); output row stride out_ld and
 * channel offset out_coff as for the convolution. */
int sis3d_maxpool3(const float *in, float *out, int out_ld, int out_coff, int X, int Y, int Z, int C, void *stream);
/* VC [X][Y][Z][C] -> NCDHW [C][X][Y][Z] (to hand tensors back in the reference layout). */
int sis3d_vc_to_ncdhw(const float *in, float *out, int64_t nvox, int C, void *stream);

/* ------------------------------------------------------------------------------------------------
 * RPN proposals ("rpn3d").  Replaces proposal_layer (lib/layer_utils/proposal_layer.py:11-204),
 * the softmax of lib/nets/network.py:546, generate_anchors (lib/layer_utils/generate_anchors.py:
 * 58-119), bbox_transform_inv / clip_boxes (lib/utils/bbox_transform.py:59-99,4-21) and the nms call
 * (proposal_layer.py:190) in three launches with no host round trip.
 * Per level l: cls [N_l][2*A_l] VC logits (channel = cls*A+a), deltas [N_l][6*A_l] VC,
 * anchor_sizes float[A_l][3], grid (gx,gy,gz), N_l = gx*gy*gz.
 * Outputs: rois [post_top_n][6], scores [post_top_n], level_ids int32[post_top_n] (1-based),
 * num_out int32[1]; debug_order int32[pre_top_n] (flat anchor index of each pre-NMS box, or NULL).
 * Tie rule: equal scores are ordered by ascending flat index (level, x, y, z, a).
 * Rows from num_out to post_top_n are zero; debug_order rows past the candidate count are -1.  When every level
 * grid is empty the call launches nothing and returns that empty result (num_out = 0).
 * pre_top_n in 1..8192 and post_top_n >= 1, SIS3D_EUNSUPPORTED otherwise.
 * ---------------------------------------------------------------------------------------------- */
typedef struct sis3d_rpn_level {
    const float *cls;
    const float *deltas;
    const float *anchor_sizes;
    int32_t grid[3];
    int32_t num_anchors;
    int32_t cls_mode; /* 0: cls = logits [N][2A]; 1: cls = foreground probability [N][A] */
    int32_t cls_ld;    /* row stride of cls in elements (0 = dense) -- lets both heads share one conv output */
    int32_t deltas_ld; /* row stride of deltas in elements (0 = dense 6A) */
    int32_t pad_;
} sis3d_rpn_level;
size_t sis3d_rpn_workspace_bytes(const sis3d_rpn_level *h_levels, int n_levels, int pre_top_n);
int sis3d_rpn_proposals(const sis3d_rpn_level *h_levels, int n_levels, int feat_stride,
                        int scene_x, int scene_y, int scene_z, int allow_border, int pre_top_n,
                        int post_top_n, float nms_thresh, float *rois, float *scores,
                        int32_t *level_ids, int32_t *num_out, int32_t *debug_order,
                        void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Detection decode for the mask branch.  Replaces lib/nets/network.py:285-301 (== lib/model/
 * trainval.py:825-858): argmax class, softmax confidence, class-specific bbox_transform_inv,
 * clip, conf > class_thresh and round()-degenerate filter (Python-3 half-to-even).
 * det float[n][16] = pred_box(6) | conf | cls | keep | crop lo(3) hi(3) | pad   (all as float)
 * n is read from device num_rois (int32[1]) and clamped to max_rois.  Rows n..max_rois-1 are zero,
 * except det[0][15], which holds n.  max_rois and num_classes must be positive (SIS3D_EINVAL).
 * ---------------------------------------------------------------------------------------------- */
int sis3d_detect_decode(const float *rois, const int32_t *num_rois, int max_rois,
                        const float *cls_score, const float *bbox_pred, int num_classes,
                        int scene_x, int scene_y, int scene_z, float class_thresh,
                        float *cls_prob, int64_t *cls_pred, float *det, void *stream);

/* Host-side planner of the ragged mask stage (CPU code, no CUDA calls): from the decoded detection table
 * h_det [n][16] (sis3d_detect_decode layout) builds every table the six mask-head launches need into one host blob
 * (ship it with a single pinned H2D copy).  use_canvas = 1: crops packed along x on a zero canvas of size plan.canvas
 * (tensor-core path, brick list at off_rest); 0: compact per-crop buffers (region table of the middle layers at
 * off_rest).  Returns SIS3D_EWORKSPACE with plan->bytes set when `capacity` is too small. */
typedef struct sis3d_mask_plan {
    int32_t n_kept, canvas[3], n_tiles_tc, tiles_first, tiles_last, tiles_mid;
    int64_t total_voxels;
    int64_t off_first, off_last, off_rest, off_offs, off_cls, off_kept, off_sizes, bytes;
} sis3d_mask_plan;
int sis3d_mask_plan_build(const float *h_det, int n, int X, int Y, int Z, int ncls, int use_canvas, void *h_blob,
                          size_t capacity, sis3d_mask_plan *plan);

/* One host call for every launch of a scene's ragged mask stage: H2D of the planner's tables, canvas zeroing, the six
 * layers (math 0: fp32 CUDA-core kernel on compact crops; 1: TF32 wgmma on the canvas; 2: fp16-operand wgmma), the
 * predicted-class select and (bits_host != NULL) the D2H of the thresholded masks.  w_first / w_last: sis3d_pack_conv_weight
 * of geometry.0 / geometry.10; w_mid[i]: geometry.{2,4,6,8} packed for `math` (pack_conv_weight / _tc / _tc_f16).
 * canvas_bytes >= 2 layers x voxels x 64 channels in the operand type; SIS3D_EWORKSPACE otherwise. */
typedef struct sis3d_mask_stage {
    const float *scene;            /* NCDHW [2][X][Y][Z] */
    int32_t X, Y, Z, ncls, math, reserved;
    const float *w_first, *w_last;
    const void *w_mid[4];
    void *tables;                  /* device, >= plan->bytes */
    void *canvas;
    size_t canvas_bytes;
    float *canvas32;               /* math 2 only: fp32 output of the last 3x3x3 layer */
    size_t canvas32_bytes;
    float *masks;                  /* [total_voxels][ncls] sigmoid outputs */
    uint8_t *bits;                 /* [total_voxels] thresholded predicted-class masks, or NULL */
    uint8_t *bits_host;            /* pinned host destination for `bits`, or NULL */
    float thresh;
    int32_t reserved2;
} sis3d_mask_stage;
int sis3d_mask_stage_launch(const sis3d_mask_plan *plan, const void *h_blob, const sis3d_mask_stage *args, void *stream);

/* Colour-aware mask head (MASK_USE_IMAGES / MASK_ONLY_IMAGES; lib/nets/backbones.py:236-287, lib/nets/network.py:302-317):
 * mask = sigmoid(combine(cat[geometry(scene crop), color(imageft crop)])), or sigmoid(color(imageft crop)) with only_images.
 * imageft is the 128-channel back-projected volume (max over the paired views, 0 where a view sees nothing); it is never
 * built: every kept crop's channels are gathered onto the stage input from the per-view maps (csrc/mask_color.cu).
 *
 * sis3d_mask_color_plan_build appends the colour stage's tables to a blob that sis3d_mask_plan_build has just filled for the
 * same h_det (plan = its result; canvas mode when plan->n_tiles_tc > 0): crops int32[n_kept][8] = x0, y0, z0, w, h, l, canvas
 * x, 0; region tables of the 1x1 convs that write a half of the 128-channel concatenation (g2c), of combine's 1x1 (last128),
 * and, on compact buffers only, of colour.0 (128 -> 64) and combine.0 (128 -> 128).  cplan->bytes = the blob's whole size
 * (ship it with one H2D copy); SIS3D_EWORKSPACE when capacity is smaller. */
typedef struct sis3d_mask_color_plan {
    int64_t off_crops, off_g2c, off_last128, off_c0, off_c128, bytes;
} sis3d_mask_color_plan;
int sis3d_mask_color_plan_build(const float *h_det, int n, const sis3d_mask_plan *plan, void *h_blob, size_t capacity,
                                sis3d_mask_color_plan *cplan);
/* The gather: for every voxel of every crop, out[row][c] = max over the (feature map, index map) pairs of
 * (pix[map][voxel] >= 0 ? feats_t[feat][pix][c] : 0), the first pair's value taken as it is -- sis3d_backproject_max's value
 * at that voxel, bit for bit.  feats_t [n_views][hw][C] channels-last features, pix int16[n_views][Z*Y*X], pairs / n_pairs
 * from sis3d_backproject_pairs (or the caller's pairing); crops / offs as in the plans above.  layout 0: compact fp32
 * rows (row = offs[j] + voxel); 1: fp32 canvas [.][cy][cz][C] at x = crops[j][6] + x; 2: the same canvas in fp16 (round to
 * nearest).  Voxels outside the crops are not written.  C % 4 == 0. */
int sis3d_mask_color_gather(const float *feats_t, const int16_t *pix, const int32_t *pairs, const int32_t *n_pairs, int n_views,
                            int C, int hw, int X, int Y, int Z, const int32_t *crops, const int64_t *offs, int n_crops,
                            int64_t total, int cy, int cz, int layout, void *out, void *stream);
/* [n_views][C][hw] -> [n_views][hw][C] (the gather's feats_t when no back-projection made one) */
int sis3d_mask_color_feats_t(const float *feats, int n_views, int C, int hw, float *feats_t, void *stream);
/* Every launch of a colour-aware scene's mask stage behind one call, on the routes of sis3d_mask_stage_launch (math 0 compact
 * fp32 CUDA-core, 1 TF32 canvas, 2 fp16-operand canvas).  Layers: colour input (gather, or crop_in: a dense fp32 VC crop
 * [w][h][l][128] of the single kept RoI, copied), color.0 .. color.8, color.10 -> channels [64, 128) of the concatenation
 * (only_images: -> sigmoid masks), geometry.0 .. geometry.8, geometry.10 -> channels [0, 64), combine.0, combine.2 ->
 * sigmoid masks, the predicted-class select, bits and their D2H.  Weights: *_first / *_last / *_combine_last fp32
 * (sis3d_pack_conv_weight); *_mid and w_color_first / w_combine packed for `math` as w_mid of sis3d_mask_stage.  geometry
 * and combine weights are not read with only_images.  canvas_bytes >= 4 x voxels (compact total or canvas) x 64 channels in
 * the operand type; math 2: canvas32_bytes >= canvas voxels x 128 (only_images: 64) x 4. */
typedef struct sis3d_mask_stage_color {
    const float *scene;            /* NCDHW [2][X][Y][Z] */
    int32_t X, Y, Z, ncls, math, only_images;
    const float *w_geom_first, *w_geom_last;
    const void *w_geom_mid[4];
    const void *w_color_first;
    const void *w_color_mid[4];
    const float *w_color_last;
    const void *w_combine;
    const float *w_combine_last;
    const float *feats_t;          /* gather inputs (see sis3d_mask_color_gather) */
    const int16_t *pix;
    const int32_t *pairs, *n_pairs;
    int32_t n_views, hw;
    const float *crop_in;          /* instead of the gather (n_kept must be 1), or NULL */
    void *tables;                  /* device, >= cplan->bytes */
    void *canvas;
    size_t canvas_bytes;
    float *canvas32;
    size_t canvas32_bytes;
    float *masks;
    uint8_t *bits;
    uint8_t *bits_host;
    float thresh;
    int32_t reserved;
} sis3d_mask_stage_color;
int sis3d_mask_stage_color_launch(const sis3d_mask_plan *plan, const sis3d_mask_color_plan *cplan, const void *h_blob,
                                  const sis3d_mask_stage_color *args, void *stream);
/* cudaMemcpyAsync behind the C ABI (kind 1 H2D, 2 D2H, 3 D2D) for hosts that stage their own pinned buffers. */
int sis3d_memcpy_async(void *dst, const void *src, size_t bytes, int kind, void *stream);

/* Predicted-class mask channel of every kept RoI, packed back to back, optionally thresholded to bits
 * (lib/model/trainval.py:900-908).  masks [total][ncls]; offs int64[n_crops+1] voxel offsets; cls int32[n_crops]. */
int sis3d_mask_select(const float *masks, const int64_t *offs, const int32_t *cls, int n_crops, int ncls,
                      int64_t total_hint, float thresh, float *out, uint8_t *bits, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Voxel overlaps of predicted and GT instance masks for the mask mAP of test mode.  Replaces the
 * full-scene unmold_mask + jaccard_mask of lib/utils/evaluation.py:144-179, 293-307.
 * Each mask is packed uint8, C order [w][h][l], at its box: *_bits + *_offs[i] (int64 offsets, one per
 * mask), *_box int32[n][6] = lo xyz | hi xyz (hi exclusive, extent = the mask's shape).  The predicted
 * side is the mask stage's `bits` with the crop bounds of sis3d_detect_decode (columns 9-14).
 * pairs int32[n_pairs][2] = (prediction, GT) indices; only the intersection of the two boxes is visited,
 * so list the pairs whose boxes intersect (the others have no common voxel).
 * Outputs (exact int64 counts of nonzero voxels): pred_count[n_pred], gt_count[n_gt],
 * pair_count[n_pairs] (voxels nonzero in both masks; -1 for a pair index out of range).
 * One launch, no workspace, capturable in a CUDA graph.
 * ---------------------------------------------------------------------------------------------- */
int sis3d_mask_overlap(const uint8_t *pred_bits, const int64_t *pred_offs, const int32_t *pred_box, int n_pred,
                       const uint8_t *gt_bits, const int64_t *gt_offs, const int32_t *gt_box, int n_gt,
                       const int32_t *pairs, int n_pairs, int64_t *pred_count, int64_t *gt_count,
                       int64_t *pair_count, void *stream);

/* ------------------------------------------------------------------------------------------------
 * ScanNet benchmark: voxel instances -> mesh vertices -> per-(box, GT id) vertex counts, without the
 * painted float64 canvas or per-vertex text files (tools/scannet_benchmark/vox2mesh.py:40-108 of the
 * reference, tools/scannet_benchmark/evaluate_predictions.py here).
 *
 * sis3d_instance_paint: owner volume int32 [X][Y][Z] (C order) over the canvas voxels [x0, x0+X) x
 * [y0, y0+Y) x [z0, z0+Z).  owner = the smallest box index b whose mask covers the voxel, -1 if none
 * ("first box wins"; vox2mesh's painting order).  Masks in the sis3d_mask_overlap layout: bits +
 * offs[b], box int32[n_box][6] = lo | hi in canvas voxels (hi exclusive, extent = the mask's shape); a
 * box with hi <= lo on any axis paints nothing.  One launch.
 *
 * sis3d_vertex_instance_overlap: per vertex v (float32 xyz), g = rint(world2grid . [v, 1]) in fp64
 * (row r: ((w[r][0]*x + w[r][1]*y) + w[r][2]*z) + w[r][3], each operation rounded, no FMA).  If
 * 1 <= g <= canvas - 2 on every axis, the vertex takes the owner at g, else the first owned voxel of
 * g's 3x3x3 neighbourhood in (dx, dy, dz) order, dx slowest, each in -1, 0, 1 (vox2mesh nn_search).
 * Voxels outside the owner volume are unowned.  Outputs, for vertices that take a box b < n_box:
 * hist int64[n_box][n_slot] += 1 at [b][gt_slot[v]] (slots outside [0, n_slot) are not counted),
 * first_vertex int32[n_box] = the smallest such v (INT32_MAX for a box no vertex takes), and, when
 * vertex_box is not NULL, vertex_box int32[n_vert] = b or -1.  hist and first_vertex are initialised
 * by the call.  world2grid: 16 doubles, row major, on the device.  Two launches.
 *
 * Both: no workspace, no host synchronisation, capturable in a CUDA graph.
 * ---------------------------------------------------------------------------------------------- */
int sis3d_instance_paint(const uint8_t *bits, const int64_t *offs, const int32_t *box, int n_box, int x0, int y0, int z0,
                         int X, int Y, int Z, int32_t *owner, void *stream);
int sis3d_vertex_instance_overlap(const float *verts, int n_vert, const double *world2grid, const int32_t *owner, int x0,
                                  int y0, int z0, int X, int Y, int Z, int canvas_x, int canvas_y, int canvas_z,
                                  const int32_t *gt_slot, int n_slot, int n_box, int64_t *hist, int32_t *first_vertex,
                                  int32_t *vertex_box, void *stream);

/* sis3d_segment_gt_slots: per-vertex GT slots from ScanNet's segment annotations (the reference's
 * tools/scannet_benchmark/export_train_mesh_for_evaluation.py, resolved per segment on the host).
 * Table: seg_ids int32[n_seg] sorted ascending and unique, seg_slot int32[n_seg] the slot of each
 * segment's GT id (slot s = index of the id in the sorted distinct ids of the table with 0 added).
 * Per vertex v: gt_slot[v] = seg_slot[row] for the row whose seg_ids equals seg_index[v]; 0 (id 0,
 * unannotated) for a segment id not in the table or negative.  slot_count int64[n_slot] = the number
 * of vertices per slot (slots outside [0, n_slot) are not counted); initialised by the call.  gt_slot
 * feeds sis3d_vertex_instance_overlap directly.  SIS3D_EINVAL on a negative size or a missing
 * pointer; n_vert = 0 only initialises slot_count.  No workspace, no host synchronisation,
 * capturable in a CUDA graph.  Two launches.
 * ---------------------------------------------------------------------------------------------- */
int sis3d_segment_gt_slots(const int32_t *seg_index, int n_vert, const int32_t *seg_ids, const int32_t *seg_slot, int n_seg,
                           int n_slot, int32_t *gt_slot, int64_t *slot_count, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Result visualisation: cube meshes of label volumes and ASCII PLY text (tools/visualization.py and
 * tools/scannet_benchmark/visualize_benchmark.py; the reference's write_mask / write_ply,
 * tools/visualization.py:78-101, 263-324).  No allocation, no host synchronisation; every pointer is
 * on the device.  Scans use scratch of ceil(n / SIS3D_PLY_SCAN_TILE) int64.
 *
 * sis3d_voxel_mesh_count: labels int32 [X][Y][Z] (C order, numpy's mask[x, y, z]).  A voxel's label is
 * labels[i], or, when lut is not NULL, lut[labels[i]] (0 for an index outside [0, n_lut)).  A voxel is
 * occupied when its label is > 0.  Occupied voxels are numbered in the reference's visiting order: z
 * outermost, then y, x innermost (row r = z * Y + y).  Writes row_offsets int64 [Y*Z + 1]: the
 * exclusive prefix of the per-row counts, row_offsets[Y*Z] = the number of occupied voxels (the one
 * value the host reads back).  Scratch: ceil(Y*Z / SIS3D_PLY_SCAN_TILE) int64.  Four launches.
 *
 * sis3d_voxel_mesh: the cubes of occupied voxels k in [k0, k1) (row_offsets from the count call on the
 * same labels; k beyond the total emits nothing), output row j = k - k0:
 *   verts  float64 [8j .. 8j+8)[3]: make_voxel_mesh's corners from fl(c - 0.05) and fl(c + 0.95);
 *   colors int64   [8j .. 8j+8)[3]: palette[label % 41] (palette int64 [41][3], the host's
 *                                   int(p / 255.0 * 255), as write_ply truncates it);
 *   faces  int64   [12j .. 12j+12)[3]: the reference's twelve triangles, vertex ids 8k + local.
 * Any of verts / colors / faces may be NULL to skip it.  One launch.
 *
 * sis3d_ply_ascii_lengths / sis3d_ply_ascii: the text lines [l0, l1) of vertices then faces, line i
 * being vertex i ("{:f} {:f} {:f} {:d} {:d} {:d}\n" of verts[i], colors[i]) for i < n_vert, else face
 * i - n_vert ("3 {:d} {:d} {:d}\n").  '{:f}' is Python's on float64: six fractional digits correctly
 * rounded (ties to even), "-0.000000" for negative values that round to zero, nan / inf / -inf.
 * lengths writes offsets int64 [n + 2] (n = l1 - l0): offsets[0..n] = the exclusive prefix of the
 * line lengths (offsets[n] = the bytes of the range) and offsets[n + 1] = the number of lines with a
 * coordinate |v| >= 2^64, which the formatter does not handle: when it is nonzero the caller formats
 * that range itself and does not call sis3d_ply_ascii.  The host reads offsets[n .. n+2) back.
 * sis3d_ply_ascii writes line l0 + i at out + offsets[i].  lengths: a memset and four launches;
 * ascii: one launch.
 * ---------------------------------------------------------------------------------------------- */
#define SIS3D_PLY_SCAN_TILE 2048
int sis3d_voxel_mesh_count(const int32_t *labels, const int32_t *lut, int n_lut, int X, int Y, int Z,
                           int64_t *row_offsets, int64_t *scratch, void *stream);
int sis3d_voxel_mesh(const int32_t *labels, const int32_t *lut, int n_lut, int X, int Y, int Z,
                     const int64_t *row_offsets, const int64_t *palette, int64_t k0, int64_t k1, double *verts,
                     int64_t *colors, int64_t *faces, void *stream);
int sis3d_ply_ascii_lengths(const double *verts, const int64_t *colors, int64_t n_vert, const int64_t *faces,
                            int64_t n_face, int64_t l0, int64_t l1, int64_t *offsets, int64_t *scratch, void *stream);
int sis3d_ply_ascii(const double *verts, const int64_t *colors, int64_t n_vert, const int64_t *faces, int64_t n_face,
                    int64_t l0, int64_t l1, const int64_t *offsets, char *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SIS3D_H */
