/*
 * p3d_modconv.h - C ABI of the fused modulated convolution at inference (StyleGAN2 SynthesisLayer / ToRGBLayer with
 * fused_modconv=True: reference _train/eg3dc/src/training/networks_stylegan2.py:40-98, 334-354, 376-380).
 *
 * Two steps per layer call:
 *   p3d_modconv_prep     per-sample weights W[o,i,ky,kx] * styles[n,i] (fp16 layers: after the inf-norm pre-normalisation
 *                        of :60-63), demodulated by rsqrt(sum w^2 + 1e-8) when `demodulate`, rounded to the compute type and
 *                        written in the shared-memory operand layout the conv kernel loads (a workspace the caller allocates:
 *                        p3d_modconv_workspace_bytes).
 *   p3d_modconv_forward  implicit-GEMM convolution on Hopper wgmma with a fused epilogue
 *                        (+ noise, + bias, lrelu 0.2 or linear, x gain, clamp, one rounding to the layer dtype).
 *
 * Tap sets: kernel 3 / up 1 (correlation, padding 1), kernel 1 / up 1 (ToRGB), kernel 3 / up 2 (the stride-2 transposed
 * conv of conv2d_resample's up > 1 branch, padding 0: output (2H+1) x (2W+1), the tensor conv_transpose2d writes before
 * the FIR; the caller runs upfirdn2d, the noise and bias_act after it).
 * Compute types: fp16 layers  m64nNk16.f32.f16.f16 (fp16 operands, fp32 accumulation);
 *                fp32 layers  m64nNk8.f32.tf32.tf32, both operands rounded to tf32 with cvt.rna (nearest, ties away).
 * No atomics: two calls with the same inputs give bit-identical outputs.
 * Return codes / p3d_last_error() as in p3d_render.h.
 */
#ifndef P3D_MODCONV_H_
#define P3D_MODCONV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct p3d_modconv_params {
    int32_t batch;          /* N (one group of the reference's grouped conv per sample) */
    int32_t in_channels;    /* Cin */
    int32_t out_channels;   /* Cout */
    int32_t in_h, in_w;     /* input resolution */
    int32_t kernel_size;    /* 1 or 3 */
    int32_t up, down;       /* up 1 or 2 (up 2 needs kernel 3); down 1 */
    int32_t dtype;          /* P3D_F32 or P3D_F16 (p3d_ops.h): dtype of x, y and bias */
    int32_t demodulate;     /* 1: SynthesisLayer, 0: ToRGBLayer */
    int32_t allow_tf32;     /* fp32 layers run on TF32 tensor cores only when the caller allows it */
    int32_t reserved0;
} p3d_modconv_params;

/* 1 when the kernel covers this layer call: kernel 1 or 3, up 1 or 2 (up 2 only with kernel 3), down 1, fp16 or fp32 with
   allow_tf32, Cin a positive multiple of 16, 1 <= Cout <= 4096, N <= 65535 / (phases), H, W in [1, 4096]. */
int p3d_modconv_supported(const p3d_modconv_params* p);

/* output resolution of p3d_modconv_forward: H (up 1) or 2H + 1 (up 2) */
int p3d_modconv_out_size(const p3d_modconv_params* p, int32_t* out_h, int32_t* out_w);

/* bytes of the per-sample operand buffer p3d_modconv_prep writes (0 when unsupported) */
size_t p3d_modconv_workspace_bytes(const p3d_modconv_params* p);

/* weight  (Cout, Cin, k, k) fp32, contiguous
   styles  (N, Cin) fp32, contiguous (ToRGB: already multiplied by weight_gain, as the reference passes them)
   ws      p3d_modconv_workspace_bytes(p) bytes, 16-byte aligned */
int p3d_modconv_prep(const p3d_modconv_params* p, const float* weight, const float* styles, void* ws, void* stream);

/* x      (N, Cin, H, W) of dtype, element strides x_stride[4] (NCHW-contiguous, channels_last or any other)
   ws     written by p3d_modconv_prep for the same params
   bias   Cout elements of dtype, or NULL
   noise  fp32, element (n, oy, ox) at noise[n * noise_stride[0] + oy * noise_stride[1] + ox * noise_stride[2]], or NULL
          (noise_stride[0] = 0 broadcasts one [H, W] image over the batch)
   y      (N, Cout, outH, outW) of dtype, element strides y_stride[4]
   act    P3D_ACT_LINEAR or P3D_ACT_LRELU (slope 0.2);  clamp < 0 disables clamping
   y = clamp((act(acc + noise + bias)) * gain), rounded once to dtype. */
int p3d_modconv_forward(const p3d_modconv_params* p, const void* x, const int64_t* x_stride, const void* ws,
                        const void* bias, const float* noise, const int64_t* noise_stride,
                        void* y, const int64_t* y_stride, int32_t act, float gain, float clamp, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* P3D_MODCONV_H_ */
