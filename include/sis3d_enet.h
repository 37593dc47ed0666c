/* sis3d_enet.h -- C ABI of the 2-D ENet encoder kernels of libsis3d.so (SURVEY row f2; replaces the cuDNN nn.Sequential of
 * lib/nets/enet.py:130-590 that lib/nets/network.py:204-205 runs in front of the back-projection when USE_IMAGES_GT=False).
 *
 * Layout: NHWC fp32 activations (channel stride 1, row stride `ld` >= C so that producers can write channel slices of a wider
 * tensor); the very first layer reads the NCHW image through explicit element strides.  BatchNorm is folded on the host
 * (lib/nets/enet_program.py), so every layer is conv + bias (+ residual) + PReLU.  fp32 CUDA-core math (exact parity path).
 * Return codes: 0 ok, -1 invalid argument, -2 CUDA launch error.  Nothing is allocated; re-entrant per stream. */
#ifndef SIS3D_ENET_H
#define SIS3D_ENET_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sis3d_enet_conv {
    const float *in;                       /* input activations */
    int64_t in_sn, in_sy, in_sx, in_sc;    /* element strides of (image, row, column, channel) */
    const float *w;                        /* packed weights [kh*kw*cin][ldw], k = (ky*kw + kx)*cin + c */
    const float *bias;                     /* [cout] or NULL */
    const float *slope;                    /* PReLU slope per output channel, or NULL (no activation) */
    const float *res;                      /* residual, NHWC [N][res_h][res_w][res_ld], or NULL; added for c < res_c */
    float *out;                            /* NHWC [N][Ho][Wo][out_ld], channels [out_coff, out_coff + cout) are written */
    int32_t N, H, W, cin, Ho, Wo, cout, ldw;
    int32_t kh, kw, stride, pad_y, pad_x, dil;
    int32_t out_ld, out_coff;
    int32_t res_ld, res_c, res_pool;       /* res_pool = 1: the residual is the floor-mode 2x2/2 max-pool of the tensor */
    int16_t res_h, res_w;                  /* residual extent: Ho x Wo, or with res_pool (2Ho | 2Ho + 1) x (2Wo | 2Wo + 1);
                                              0 (both): Ho x Wo, with res_pool 2Ho x 2Wo (the layout before these fields) */
} sis3d_enet_conv;

/* weights [cout][cin][kh][kw] -> [kh*kw*cin][ldw] (ldw = cout rounded up to 4, zero padded) */
int sis3d_enet_pack_weight(const float *w_oihw, int cout, int cin, int kh, int kw, float *packed, void *stream);
/* out = prelu(conv(in) + bias + residual, slope) */
int sis3d_enet_conv2d(const sis3d_enet_conv *args, void *stream);
/* initial block's second branch: out[..., coff + c] = prelu(scale[c] * maxpool2x2(in)[c] + shift[c], slope[c]); `in` is read
 * through element strides (NCHW image), out is NHWC with row stride out_ld */
int sis3d_enet_pool_affine(const float *in, int64_t in_sn, int64_t in_sy, int64_t in_sx, int64_t in_sc, int N, int H, int W, int C,
                           const float *scale, const float *shift, const float *slope, float *out, int out_ld, int out_coff,
                           void *stream);
/* NHWC [N][P][ld] (channels [coff, coff + C)) -> NCHW [N][C][P] */
int sis3d_enet_to_nchw(const float *in, int ld, int coff, int N, int64_t P, int C, float *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif
