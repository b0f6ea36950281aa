/*
 * p3d_ops.h - C ABI of the H100-native StyleGAN custom ops (bias_act, upfirdn2d, filtered_lrelu).
 *
 * Each entry point replaces one pybind11 function of the reference's JIT plugins
 * (/root/reference/_train/eg3dc/src/torch_utils/ops/): same argument meaning, but plain device
 * pointers + sizes + strides instead of torch::Tensor, and the caller allocates the output.
 * Return codes / p3d_last_error() as in p3d_render.h.
 */
#ifndef P3D_OPS_H_
#define P3D_OPS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* element types */
#define P3D_F32  0
#define P3D_F16  1
#define P3D_BF16 2   /* not offered by the reference plugins (fp16/fp32/fp64 only) */
#define P3D_F64  3

/* activation ids = `cuda_idx` of bias_act.activation_funcs (ops/bias_act.py:23-33) */
#define P3D_ACT_LINEAR   1
#define P3D_ACT_RELU     2
#define P3D_ACT_LRELU    3
#define P3D_ACT_TANH     4
#define P3D_ACT_SIGMOID  5
#define P3D_ACT_ELU      6
#define P3D_ACT_SELU     7
#define P3D_ACT_SOFTPLUS 8
#define P3D_ACT_SWISH    9

/* bias_act_plugin.bias_act(x, b, xref, yref, dy, grad, dim, act, alpha, gain, clamp) -> y
   (ops/bias_act.cpp:36-101, kernel ops/bias_act.cu:27-151).
     x, xref, yref, dy, y : `numel` elements of `dtype`, all with the SAME dense layout (any memory format);
                            xref / yref / dy may be NULL exactly where the reference passes empty tensors
     b                    : `size_b` elements of `dtype` or NULL; element i of memory uses b[(i / step_b) % size_b]
                            (step_b = x.stride(dim), bias_act.cpp:78)
     grad                 : 0 forward, 1 first derivative (x = incoming gradient), 2 second derivative
     clamp < 0 disables clamping. */
int p3d_bias_act(const void* x, const void* b, const void* xref, const void* yref, const void* dy, void* y,
                 int64_t numel, int32_t dtype, int32_t grad, int64_t step_b, int32_t size_b,
                 int32_t act, float alpha, float gain, float clamp, void* stream);

/* upfirdn2d_plugin.upfirdn2d(x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip, gain) -> y
   (ops/upfirdn2d.cpp:20-103, kernels ops/upfirdn2d.cu:33-204).
     x : (N,C,inH,inW) of `dtype` with element strides x_stride[4] = {sN, sC, sH, sW} (any layout)
     f : (fH,fW) fp32 taps, element strides {f_stride_h, f_stride_w}
     y : (N,C,outH,outW) of `dtype`, element strides y_stride[4]; outW = (inW*upx + padx0 + padx1 - fW + downx)/downx,
         outH likewise (the caller allocates it with exactly that size). */
int p3d_upfirdn2d(const void* x, const float* f, void* y, int32_t dtype,
                  int32_t n, int32_t c, int32_t in_h, int32_t in_w, const int64_t* x_stride,
                  int32_t f_h, int32_t f_w, int64_t f_stride_h, int64_t f_stride_w,
                  int32_t out_h, int32_t out_w, const int64_t* y_stride,
                  int32_t upx, int32_t upy, int32_t downx, int32_t downy,
                  int32_t padx0, int32_t padx1, int32_t pady0, int32_t pady1,
                  int32_t flip, float gain, void* stream);

/* filtered_lrelu_plugin.filtered_lrelu(x, fu, fd, b, si, up, down, px0, px1, py0, py1, sx, sy, gain, slope,
                                        clamp, flip_filter, writeSigns) -> (y, so, return_code)
   (ops/filtered_lrelu.cpp:20-214, kernel ops/filtered_lrelu.cu:143-1103).  One generic tiled kernel covers every
   (up, down, filter size, separable or not) combination, so there is no "-1: no kernel" return path.
     x  : (N,C,inH,inW) `dtype` (f32/f16/bf16), element strides x_stride[4]
     fu : up-sampling FIR, fp32, (fu_h, fu_w) row-major; fu_h == 1 with fu_sep != 0 means separable taps (fu_w)
     fd : down-sampling FIR, same convention
     b  : C biases of `dtype` (never NULL; the Python host passes zeros like the reference does)
     s  : sign/clamp tensor, 2 bits per element, 4 per byte: (N,C,sH,sW4) uint8 contiguous with
          sW4 = ceil16(sW)/4 bytes per row (filtered_lrelu.cpp:91-98).  Written when sign_mode == 1,
          read when sign_mode == 2 (then no bias/lrelu/clamp maths is done, the gradient is gated by s),
          ignored when sign_mode == 0.  sx, sy: offset of the up-sampled image inside the sign tensor.
     y  : (N,C,outH,outW) `dtype`, element strides y_stride[4]. */
int p3d_filtered_lrelu(const void* x, const float* fu, const float* fd, const void* b, uint8_t* s, void* y,
                       int32_t dtype, int32_t n, int32_t c, int32_t in_h, int32_t in_w, const int64_t* x_stride,
                       int32_t out_h, int32_t out_w, const int64_t* y_stride,
                       int32_t fu_h, int32_t fu_w, int32_t fu_sep, int32_t fd_h, int32_t fd_w, int32_t fd_sep,
                       int32_t up, int32_t down, int32_t px0, int32_t px1, int32_t py0, int32_t py1,
                       int32_t s_h, int32_t s_w, int32_t sx, int32_t sy,
                       float gain, float slope, float clamp, int32_t flip, int32_t sign_mode, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* P3D_OPS_H_ */
