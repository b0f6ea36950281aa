// filtered_lrelu for sm_90a: bias -> up-FIR -> gain*lrelu/clamp (with the 2-bit sign tensor) -> down-FIR,
// one CTA per 32x16 output tile of one (n,c) image, everything between the input read and the output write
// lives in shared memory.  Semantics follow the reference plugin (ops/filtered_lrelu.cu:143-1103, host side
// ops/filtered_lrelu.cpp:20-214) and its Python composition (ops/filtered_lrelu.py:123-155):
//     u = upfirdn2d(x + b, fu, up, padding, gain = up^2)        (px0,px1,py0,py1 in up-sampled pixels)
//     v = clamp(lrelu(u * gain, slope), +-clamp)                 sign tensor: 0 plain, 1 negative, 2 clamped
//     y = upfirdn2d(v, fd, down)
// The reference ships 31 hand-specialised tile/filter configurations and returns -1 ("no kernel") for the rest;
// here ONE runtime-generic kernel covers every (up, down, filter shape, separable or full) combination:
// shared memory on H100 (227 KB/CTA) holds the up-sampled tile for every practical filter, and the op is
// far from compute bound, so per-shape template specialisation buys nothing.
//   A) input footprint -> smem (bias added on real pixels, zeros outside);
//   B) each thread produces a 4-wide strip of the up-sampled tile (polyphase taps only), applies the
//      activation, and - in write mode - emits one byte of four 2-bit codes; byte ownership follows the
//      tile's non-overlapping region, so no two CTAs ever touch the same byte;
//   C) down-FIR from smem, coalesced store.
#include "p3d_common.cuh"
#include "../../include/p3d_ops.h"

namespace p3d {
namespace {

template <typename T> struct Fx;
template <> struct Fx<float> { static __device__ float ld(float v) { return v; } static __device__ float st(float v) { return v; } };
template <> struct Fx<__half> { static __device__ float ld(__half v) { return __half2float(v); } static __device__ __half st(float v) { return __float2half_rn(v); } };
template <> struct Fx<__nv_bfloat16> { static __device__ float ld(__nv_bfloat16 v) { return __bfloat162float(v); } static __device__ __nv_bfloat16 st(float v) { return __float2bfloat16_rn(v); } };

constexpr int kOutW = 32, kOutH = 16, kThr = 256;

struct FlParams {
    const void* x;
    const float *fu, *fd;
    const void* b;
    unsigned char* s;
    void* y;
    int N, C, inH, inW, outH, outW;
    long long xs[4], ys[4];
    int fuH, fuW, fuSep, fdH, fdW, fdSep;
    int up, down, px0, py0;
    int sH, sW, sx, sy;              // sign tensor: rows, width in ELEMENTS (multiple of 16), offsets
    int upH, upW;                    // size of the up-sampled (post up-FIR) image
    float gain, slope, clamp;
    int flip, sign_mode;
    int tilesX, tilesY, inTW, inTH, upTW, upTH;
};

__device__ __forceinline__ int fdiv(int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
__device__ __forceinline__ int pmod(int a, int b) { int m = a % b; return m < 0 ? m + b : m; }

// tap (ky,kx) of a filter given as full (h,w) row-major taps or as separable 1-D taps (w entries, h == w logically)
__device__ __forceinline__ float tap(const float* f, int fh, int fw, int sep, int ky, int kx, int flip) {
    const int yy = flip ? ky : fh - 1 - ky, xx = flip ? kx : fw - 1 - kx;
    return sep ? f[yy] * f[xx] : f[yy * fw + xx];
}

// SEP: both filters were given as 1-D taps (the way StyleGAN3 layers and setup_filter(>= 8 taps) pass them).  The two FIRs then run as
// four 1-D passes through shared memory - up-x, up-y (+ activation / signs), down-x, down-y - e.g. 6+6 and 12+12 instead of 36 and 144
// multiply-adds per up-sampled / output pixel for the 12-tap up 2 / down 2 layer; the rounding differs from the 2-D sum in the last bit.
template <typename T, bool SEP>
__global__ void __launch_bounds__(kThr) k_filtered_lrelu(const FlParams p) {
    extern __shared__ float smem[];
    float* s_wu = smem;                                   // fuH*fuW (gain up^2*gain folded)   SEP: 2 x fuW (x taps with the gain, y taps)
    float* s_wd = s_wu + (SEP ? 2 * p.fuW : p.fuH * p.fuW);   // fdH*fdW                        SEP: fdW
    float* s_in = s_wd + (SEP ? p.fdW : p.fdH * p.fdW);   // inTH*inTW
    float* s_up = s_in + p.inTH * p.inTW;                 // upTH*upTW
    float* s_t1 = s_up + p.upTH * p.upTW;                 // SEP: inTH*upTW  rows of the input footprint after the horizontal up-pass
    float* s_t2 = s_t1 + p.inTH * p.upTW;                 // SEP: upTH*kOutW rows of the activated tile after the horizontal down-pass
    const int tid = threadIdx.x;
    const float ugain = (float)p.up * (float)p.up * p.gain;
    if (SEP) {
        for (int i = tid; i < p.fuW; i += kThr) {
            const float t = p.fu[p.flip ? i : p.fuW - 1 - i];
            s_wu[i] = t * ugain; s_wu[p.fuW + i] = t;
        }
        for (int i = tid; i < p.fdW; i += kThr) s_wd[i] = p.fd[p.flip ? i : p.fdW - 1 - i];
    } else {
        for (int i = tid; i < p.fuH * p.fuW; i += kThr) s_wu[i] = tap(p.fu, p.fuH, p.fuW, p.fuSep, i / p.fuW, i % p.fuW, p.flip) * ugain;
        for (int i = tid; i < p.fdH * p.fdW; i += kThr) s_wd[i] = tap(p.fd, p.fdH, p.fdW, p.fdSep, i / p.fdW, i % p.fdW, p.flip);
    }

    const int tile = blockIdx.x, tyi = tile / p.tilesX, txi = tile - tyi * p.tilesX;
    const int ox0 = txi * kOutW, oy0 = tyi * kOutH;
    const int ux0 = ox0 * p.down, uy0 = oy0 * p.down;     // origin of this tile in the up-sampled image
    // first input column/row that can contribute to up-sampled pixel ux0:  P index = ux0 + k - px0, k >= 0
    const int ix0 = fdiv(ux0 - p.px0, p.up), iy0 = fdiv(uy0 - p.py0, p.up);
    const T* xp = reinterpret_cast<const T*>(p.x);
    const T* bp = reinterpret_cast<const T*>(p.b);
    T* yp = reinterpret_cast<T*>(p.y);
    // rows/cols of the up-sampled tile this CTA owns for sign writing (non-overlapping partition)
    const int own_x1 = (txi == p.tilesX - 1) ? p.sW : ux0 + kOutW * p.down;
    const int own_y1 = (tyi == p.tilesY - 1) ? p.sH : uy0 + kOutH * p.down;

    for (long long img = blockIdx.y; img < (long long)p.N * p.C; img += gridDim.y) {
        const int n = (int)(img / p.C), c = (int)(img - (long long)n * p.C);
        const T* xi = xp + n * p.xs[0] + c * p.xs[1];
        const float bias = bp ? Fx<T>::ld(bp[c]) : 0.f;
        __syncthreads();
        // ---- A) input footprint
        for (int i = tid; i < p.inTH * p.inTW; i += kThr) {
            const int r = i / p.inTW, q = i - r * p.inTW;
            const int iy = iy0 + r, ix = ix0 + q;
            s_in[i] = (iy >= 0 && iy < p.inH && ix >= 0 && ix < p.inW) ? Fx<T>::ld(xi[iy * p.xs[2] + ix * p.xs[3]]) + bias : 0.f;
        }
        __syncthreads();
        if (SEP) {
            // ---- B1) horizontal up-pass over every footprint row
            for (int i = tid; i < p.inTH * p.upTW; i += kThr) {
                const int r = i / p.upTW, q = i - r * p.upTW;
                const int tx0 = ux0 + q - p.px0;
                const int kx0 = pmod(-tx0, p.up);
                const float* row = s_in + r * p.inTW + ((tx0 + kx0) / p.up - ix0);
                float acc = 0.f;
                for (int kx = kx0, j = 0; kx < p.fuW; kx += p.up, ++j) acc = fmaf(row[j], s_wu[kx], acc);
                s_t1[i] = acc;
            }
            __syncthreads();
        }
        // ---- B) up-FIR + activation, 4-wide strips
        const int strips = (p.upTW + 3) >> 2;
        unsigned char* srow_base = p.s ? p.s + (size_t)img * p.sH * (p.sW >> 2) : nullptr;
        for (int i = tid; i < p.upTH * strips; i += kThr) {
            const int r = i / strips, q4 = (i - r * strips) * 4;
            const int uy = uy0 + r;
            const int ty0 = uy - p.py0;                    // P row of tap ky = 0 is ty0 + ky ... (in up-sampled input coords)
            const int ky0 = pmod(-ty0, p.up);
            const int sy0 = (ty0 + ky0) / p.up - iy0;
            float v[4];
            unsigned int code = 0;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int ux = ux0 + q4 + e;
                float acc = 0.f;
                if (q4 + e < p.upTW && uy < p.upH && ux < p.upW) {
                    if (SEP) {                             // vertical up-pass over the horizontally filtered rows
                        const float* col = s_t1 + sy0 * p.upTW + q4 + e;
                        for (int ky = ky0, j = 0; ky < p.fuW; ky += p.up, ++j) acc = fmaf(col[j * p.upTW], s_wu[p.fuW + ky], acc);
                    } else {
                    const int tx0 = ux - p.px0;
                    const int kx0 = pmod(-tx0, p.up);
                    const int sx0 = (tx0 + kx0) / p.up - ix0;
                    for (int ky = ky0, sy = sy0; ky < p.fuH; ky += p.up, ++sy) {
                        const float* row = s_in + sy * p.inTW + sx0;
                        const float* wr = s_wu + ky * p.fuW;
                        for (int kx = kx0, j = 0; kx < p.fuW; kx += p.up, ++j) acc = fmaf(row[j], wr[kx], acc);
                    }
                    }
                    if (p.sign_mode == 2) {                // gradient pass: gate by the stored signs
                        const int qx = ux + p.sx, qy = uy + p.sy;
                        if (qx >= 0 && qx < p.sW && qy >= 0 && qy < p.sH) {
                            const unsigned int sc = (srow_base[(size_t)qy * (p.sW >> 2) + (qx >> 2)] >> ((qx & 3) << 1)) & 3u;
                            if (sc & 1u) acc *= p.slope;
                            if (sc & 2u) acc = 0.f;
                        }
                    } else {
                        unsigned int sc = 0;
                        if (acc < 0.f) { acc *= p.slope; sc = 1; }
                        if (fabsf(acc) > p.clamp) { acc = acc < 0.f ? -p.clamp : p.clamp; sc = 2; }
                        code |= sc << (2 * e);
                    }
                }
                v[e] = acc;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (q4 + e < p.upTW) s_up[r * p.upTW + q4 + e] = v[e];
            if (p.sign_mode == 1) {
                const int ux = ux0 + q4;
                if (ux < own_x1 && uy < own_y1 && ux < p.sW && uy < p.sH) srow_base[(size_t)uy * (p.sW >> 2) + (ux >> 2)] = (unsigned char)code;
            }
        }
        __syncthreads();
        if (SEP) {
            // ---- C1) horizontal down-pass over every row of the activated tile
            for (int i = tid; i < p.upTH * kOutW; i += kThr) {
                const int r = i / kOutW, tx = i - r * kOutW;
                const float* base = s_up + r * p.upTW + tx * p.down;
                float acc = 0.f;
                for (int kx = 0; kx < p.fdW; ++kx) acc = fmaf(base[kx], s_wd[kx], acc);
                s_t2[i] = acc;
            }
            __syncthreads();
        }
        // ---- C) down-FIR
        for (int i = tid; i < kOutW * kOutH; i += kThr) {
            const int ty = i / kOutW, tx = i - ty * kOutW;
            const int ox = ox0 + tx, oy = oy0 + ty;
            if (ox >= p.outW || oy >= p.outH) continue;
            const float* base = s_up + (ty * p.down) * p.upTW + tx * p.down;
            float acc = 0.f;
            if (SEP) {
                const float* col = s_t2 + (ty * p.down) * kOutW + tx;
                for (int ky = 0; ky < p.fdW; ++ky) acc = fmaf(col[ky * kOutW], s_wd[ky], acc);
            } else
            for (int ky = 0; ky < p.fdH; ++ky)
                for (int kx = 0; kx < p.fdW; ++kx) acc = fmaf(base[ky * p.upTW + kx], s_wd[ky * p.fdW + kx], acc);
            yp[n * p.ys[0] + c * p.ys[1] + oy * p.ys[2] + ox * p.ys[3]] = Fx<T>::st(acc);
        }
    }
}

template <typename T>
int launch_fl(FlParams p, cudaStream_t stream) {
    p.tilesX = (p.outW + kOutW - 1) / kOutW;
    p.tilesY = (p.outH + kOutH - 1) / kOutH;
    p.upTW = kOutW * p.down + p.fdW - 1 - (p.down - 1);
    p.upTH = kOutH * p.down + p.fdH - 1 - (p.down - 1);
    p.inTW = (p.upTW + p.fuW - 1 + p.up - 1) / p.up + 1;
    p.inTH = (p.upTH + p.fuH - 1 + p.up - 1) / p.up + 1;
    const bool sep = p.fuSep && p.fdSep;
    const size_t smem = sep ? ((size_t)2 * p.fuW + p.fdW + (size_t)p.inTW * p.inTH + (size_t)p.upTW * p.upTH + (size_t)p.inTH * p.upTW + (size_t)p.upTH * kOutW) * sizeof(float)
                            : ((size_t)p.fuH * p.fuW + (size_t)p.fdH * p.fdW + (size_t)p.inTW * p.inTH + (size_t)p.upTW * p.upTH) * sizeof(float);
    if (smem > 200 * 1024) {
        set_error("filtered_lrelu: tile needs %zu bytes of shared memory (filters %dx%d / %dx%d, up %d, down %d)", smem, p.fuH, p.fuW, p.fdH, p.fdW, p.up, p.down);
        return P3D_EUNSUPPORTED;
    }
    auto kern = sep ? k_filtered_lrelu<T, true> : k_filtered_lrelu<T, false>;
    if (smem > 48 * 1024) P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long nc = (long long)p.N * p.C;
    dim3 grid((unsigned)(p.tilesX * p.tilesY), (unsigned)(nc < 32768 ? nc : 32768));
    kern<<<grid, kThr, smem, stream>>>(p);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_filtered_lrelu(const void* x, const float* fu, const float* fd, const void* b, uint8_t* s, void* y,
                                  int32_t dtype, int32_t n, int32_t c, int32_t in_h, int32_t in_w, const int64_t* x_stride,
                                  int32_t out_h, int32_t out_w, const int64_t* y_stride, int32_t fu_h, int32_t fu_w,
                                  int32_t fu_sep, int32_t fd_h, int32_t fd_w, int32_t fd_sep, int32_t up, int32_t down,
                                  int32_t px0, int32_t px1, int32_t py0, int32_t py1, int32_t s_h, int32_t s_w, int32_t sx,
                                  int32_t sy, float gain, float slope, float clamp, int32_t flip, int32_t sign_mode,
                                  void* stream) {
    P3D_REQUIRE(x && fu && fd && y && x_stride && y_stride, "null pointer");
    P3D_REQUIRE(n > 0 && c > 0 && in_h > 0 && in_w > 0, "x has zero size");
    P3D_REQUIRE(up >= 1 && down >= 1, "up/down must be >= 1");
    P3D_REQUIRE(fu_h >= 1 && fu_w >= 1 && fd_h >= 1 && fd_w >= 1, "filters must be at least 1x1");
    P3D_REQUIRE(sign_mode >= 0 && sign_mode <= 2, "bad sign_mode");
    P3D_REQUIRE(sign_mode == 0 || (s != nullptr && s_w % 16 == 0 && s_h > 0 && s_w > 0), "sign tensor needs s != NULL and a width that is a multiple of 16");
    if (fu_sep) fu_h = fu_w;                       // separable taps: logical filter is the outer product (fu_w x fu_w)
    if (fd_sep) fd_h = fd_w;
    const int cw = in_w * up + px0 + px1 - (fu_w - 1), ch = in_h * up + py0 + py1 - (fu_h - 1);
    P3D_REQUIRE(cw > fd_w - 1 && ch > fd_h - 1, "upsampled buffer must be at least the size of downsampling filter");
    const int yw = (cw - (fd_w - 1) + (down - 1)) / down, yh = (ch - (fd_h - 1) + (down - 1)) / down;
    P3D_REQUIRE(yw == out_w && yh == out_h, "output size mismatch: expected %dx%d, got %dx%d", yh, yw, out_h, out_w);
    FlParams p{};
    p.x = x; p.fu = fu; p.fd = fd; p.b = b; p.s = s; p.y = y; p.N = n; p.C = c; p.inH = in_h; p.inW = in_w; p.outH = out_h; p.outW = out_w;
    for (int i = 0; i < 4; ++i) { p.xs[i] = x_stride[i]; p.ys[i] = y_stride[i]; }
    p.fuH = fu_h; p.fuW = fu_w; p.fuSep = fu_sep; p.fdH = fd_h; p.fdW = fd_w; p.fdSep = fd_sep;
    p.up = up; p.down = down; p.px0 = px0; p.py0 = py0; p.sH = s_h; p.sW = s_w; p.sx = sx; p.sy = sy;
    p.upH = ch; p.upW = cw; p.gain = gain; p.slope = slope; p.clamp = clamp; p.flip = flip ? 1 : 0; p.sign_mode = sign_mode;
    if (sign_mode == 0) { p.s = nullptr; p.sH = 0; p.sW = 0; }
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case P3D_F32: return launch_fl<float>(p, st);
        case P3D_F16: return launch_fl<__half>(p, st);
        case P3D_BF16: return launch_fl<__nv_bfloat16>(p, st);
    }
    set_error("filtered_lrelu supports fp32 / fp16 / bf16 (dtype %d)", dtype);
    return P3D_EINVAL;
}
