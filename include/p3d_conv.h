/*
 * p3d_conv.h - C ABI of the fp32 training convolutions on the tensor cores (conv2d_gradfix's conv2d / conv_transpose2d
 * at the shapes the generator's synthesis layers and the discriminator's fp32 blocks produce, and their weight gradients).
 *
 * Arithmetic: 3xTF32.  Each fp32 operand v is split into big = tf32(v) and small = tf32(v - big) (cvt.rna: nearest, ties
 * away); a product is big*big + big*small + small*big, accumulated in fp32 by m64n128k8.f32.tf32.tf32 wgmma.
 * No atomics: two calls with the same inputs give bit-identical outputs.
 *
 * Envelope (kernel / stride / padding), for both conv2d and conv_transpose2d:  3 / 1 / 1,  1 / 1 / 0,  3 / 2 / 0.
 * groups 1, dilation 1, no bias; output_padding 0 (conv2d) or 0 .. stride - 1 per axis (conv_transpose2d).
 * Tensors are fp32 and contiguous: x (N, Cin, H, W), y (N, Cout, outH, outW); the weight is (Cout, Cin, k, k) for conv2d
 * and (Cin, Cout, k, k) for conv_transpose2d, as torch lays them out.
 * Return codes / p3d_last_error() as in p3d_render.h.
 */
#ifndef P3D_CONV_H_
#define P3D_CONV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct p3d_conv_params {
    int32_t batch;           /* N */
    int32_t in_channels;     /* Cin: channels of x */
    int32_t out_channels;    /* Cout: channels of y */
    int32_t in_h, in_w;      /* resolution of x */
    int32_t kernel_size;     /* 1 or 3 */
    int32_t stride;          /* 1 or 2 */
    int32_t padding;         /* 1 (kernel 3, stride 1) or 0 */
    int32_t transpose;       /* 0: conv2d, 1: conv_transpose2d */
    int32_t output_padding_h, output_padding_w;   /* conv_transpose2d only, each in [0, stride) */
} p3d_conv_params;

/* 1 when the kernels cover this call: (kernel, stride, padding) in the envelope above, transpose 0 or 1, output_padding
   as above, 1 <= N <= 16384 (conv_transpose2d stride 2: N <= 16383, four phases per sample), 1 <= Cin, Cout <= 8192, H, W in [1, 4096] and a non-empty output (conv2d stride 2: H, W >= 3),
   every tensor below 2^31 elements per sample and the weight below 2^31 elements. */
int p3d_conv_supported(const p3d_conv_params* p);

/* output resolution: conv2d (H + 2 padding - k) / stride + 1, conv_transpose2d (H - 1) stride - 2 padding + k + output_padding_h (W: _w) */
int p3d_conv_out_size(const p3d_conv_params* p, int32_t* out_h, int32_t* out_w);

/* bytes of the workspace p3d_conv_forward needs: the weight reordered K-major, Cout * Cin * k * k fp32 (0 when unsupported) */
size_t p3d_conv_forward_workspace_bytes(const p3d_conv_params* p);

/* y = conv2d(x, w) or conv_transpose2d(x, w) (p->transpose); ws: p3d_conv_forward_workspace_bytes(p) bytes, 16-byte aligned */
int p3d_conv_forward(const p3d_conv_params* p, const float* x, const float* w, void* ws, size_t ws_bytes, float* y, void* stream);

/* bytes of the split-K partials p3d_conv_weight_grad needs (0 when it needs none or the call is unsupported) */
size_t p3d_conv_weight_grad_workspace_bytes(const p3d_conv_params* p);

/* dw = the gradient of sum(y * dy) with respect to the weight of the call p describes, for its input x (N, Cin, H, W) and an
   output gradient dy (N, Cout, outH, outW); dw has the weight's shape.  The split-K partials are summed in a fixed order.
   ws: p3d_conv_weight_grad_workspace_bytes(p) bytes, 16-byte aligned (may be NULL when that is 0). */
int p3d_conv_weight_grad(const p3d_conv_params* p, const float* x, const float* dy, void* ws, size_t ws_bytes, float* dw, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* P3D_CONV_H_ */
