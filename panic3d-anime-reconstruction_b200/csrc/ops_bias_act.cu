// bias_act for sm_90a: y = clamp(gain * act(x + b)), and its first / second derivatives.
//
// Semantics follow the reference plugin kernel (ops/bias_act.cu:27-151) exactly - same activation
// table, same G=0/1/2 formulas expressed through the saved xref / yref, same clamp rule - but the
// kernel is rebuilt for H100's memory system: it is a pure HBM-streaming op (1 read + 1 write per
// element forward, up to 4 reads in the gradient modes), so
//   * every tensor moves as 128-bit vectors (4 fp32 / 8 fp16|bf16 per access);
//   * the bias index costs one 64-bit div+mod per VECTOR (NCHW: all lanes of a vector share one
//     bias; channels-last / (N,C): the vector reads a contiguous bias run), not one per element;
//   * the grid is persistent: #SMs x 8 CTAs of 256 threads, grid-stride over vectors;
//   * bf16 is supported next to fp16/fp32/fp64 (maths in fp32, fp64 for double).
#include "p3d_common.cuh"
#include "../../include/p3d_ops.h"

namespace p3d {
namespace {

template <typename T> struct Elem;
template <> struct Elem<float> { using acc = float; static __device__ float ld(float v) { return v; } static __device__ float st(float v) { return v; } };
template <> struct Elem<double> { using acc = double; static __device__ double ld(double v) { return v; } static __device__ double st(double v) { return v; } };
template <> struct Elem<__half> { using acc = float; static __device__ float ld(__half v) { return __half2float(v); } static __device__ __half st(float v) { return __float2half_rn(v); } };
template <> struct Elem<__nv_bfloat16> { using acc = float; static __device__ float ld(__nv_bfloat16 v) { return __bfloat162float(v); } static __device__ __nv_bfloat16 st(float v) { return __float2bfloat16_rn(v); } };

__device__ __forceinline__ float xexp(float v) { return expf(v); }
__device__ __forceinline__ double xexp(double v) { return exp(v); }
__device__ __forceinline__ float xlog(float v) { return logf(v); }
__device__ __forceinline__ double xlog(double v) { return log(v); }

struct BiasActParams {
    const void *x, *b, *xref, *yref, *dy;
    void* y;
    long long numel, step_b, base;      // base: element index of x[0] in the full tensor (tail launches)
    int size_b, grad;
    float alpha, gain, clamp;
};

// one element; A = activation id, G = derivative order.  Mirrors ops/bias_act.cu:58-146.
template <typename S, int A>
__device__ __forceinline__ S bias_act_elem(int G, S x, S b, S xref, S yref, S dy, S alpha, S gain, S clamp) {
    const S one = (S)1, two = (S)2, expRange = (S)80, halfExpRange = (S)40;
    const S seluScale = (S)1.0507009873554804934193349852946, seluAlpha = (S)1.6732632423543772848170429916717;
    S yy = (gain != (S)0) ? yref / gain : (S)0;
    S y = (S)0;
    if (G == 0) x += b; else xref += b;
    if (A == P3D_ACT_LINEAR) { y = x; }
    if (A == P3D_ACT_RELU) { y = (G == 0) ? ((x > 0) ? x : (S)0) : ((yy > 0) ? x : (S)0); }
    if (A == P3D_ACT_LRELU) { y = (G == 0) ? ((x > 0) ? x : x * alpha) : ((yy > 0) ? x : x * alpha); }
    if (A == P3D_ACT_TANH) {
        if (G == 0) { S c = xexp(x), d = one / c; y = (x < -expRange) ? -one : (x > expRange) ? one : (c - d) / (c + d); }
        if (G == 1) y = x * (one - yy * yy);
        if (G == 2) y = x * (one - yy * yy) * (-two * yy);
    }
    if (A == P3D_ACT_SIGMOID) {
        if (G == 0) y = (x < -expRange) ? (S)0 : one / (xexp(-x) + one);
        if (G == 1) y = x * yy * (one - yy);
        if (G == 2) y = x * yy * (one - yy) * (one - two * yy);
    }
    if (A == P3D_ACT_ELU) {
        if (G == 0) y = (x >= 0) ? x : xexp(x) - one;
        if (G == 1) y = (yy >= 0) ? x : x * (yy + one);
        if (G == 2) y = (yy >= 0) ? (S)0 : x * (yy + one);
    }
    if (A == P3D_ACT_SELU) {
        if (G == 0) y = (x >= 0) ? seluScale * x : (seluScale * seluAlpha) * (xexp(x) - one);
        if (G == 1) y = (yy >= 0) ? x * seluScale : x * (yy + seluScale * seluAlpha);
        if (G == 2) y = (yy >= 0) ? (S)0 : x * (yy + seluScale * seluAlpha);
    }
    if (A == P3D_ACT_SOFTPLUS) {
        if (G == 0) y = (x > expRange) ? x : xlog(xexp(x) + one);
        if (G == 1) y = x * (one - xexp(-yy));
        if (G == 2) { S c = xexp(-yy); y = x * c * (one - c); }
    }
    if (A == P3D_ACT_SWISH) {
        if (G == 0) y = (x < -expRange) ? (S)0 : x / (xexp(-x) + one);
        else {
            S c = xexp(xref), d = c + one;
            if (G == 1) y = (xref > halfExpRange) ? x : x * c * (xref + d) / (d * d);
            else y = (xref > halfExpRange) ? (S)0 : x * c * (xref * (two - d) + two * d) / (d * d * d);
            yref = (xref < -expRange) ? (S)0 : xref / (xexp(-xref) + one) * gain;
        }
    }
    y *= gain * dy;
    if (clamp >= 0) {
        if (G == 0) y = (y > -clamp && y < clamp) ? y : (y >= 0) ? clamp : -clamp;
        else y = (yref > -clamp && yref < clamp) ? y : (S)0;
    }
    return y;
}

template <typename T, int VEC> struct alignas(sizeof(T) * VEC) Vec { T v[VEC]; };

// BIAS: 0 = no bias, 1 = one bias per vector (NCHW-like: step_b % VEC == 0), 2 = contiguous bias run per vector
// (channels-last / (N,C): step_b == 1, size_b % VEC == 0, bias 16-byte aligned), 3 = generic per-element index,
// 4 = row mode (NCHW with >= 128 vectors per (n,c) image: the bias is CTA-uniform).
// numel <= 2^31-1 is enforced at the ABI, so all index arithmetic is 32-bit unsigned (a 64-bit div/mod per vector was
// the dominant cost of the first version on channels-last inputs).
template <typename T, int A, int VEC, int BIAS, bool FWD>
__global__ void __launch_bounds__(256) k_bias_act(const BiasActParams p) {
    using S = typename Elem<T>::acc;
    using V = Vec<T, VEC>;
    constexpr bool REFS = !FWD;                                   // FWD: plain forward (G = 0, no xref/yref/dy) - the hot case
    const int G = FWD ? 0 : p.grad;
    constexpr int UNROLL = FWD ? 4 : 2;                            // independent 16-byte vectors in flight per thread
    constexpr unsigned kItem = 256 * UNROLL;                       // vectors per CTA iteration (contiguous)
    const S alpha = (S)p.alpha, gain = (S)p.gain, clamp = (S)p.clamp;
    const T* bp = reinterpret_cast<const T*>(p.b);
    const unsigned nvec = (unsigned)(p.numel / VEC);
    const unsigned step_b = (unsigned)p.step_b, size_b = (unsigned)p.size_b, base = (unsigned)p.base;
    // BIAS == 4 walks the tensor row by row (a row = step_b elements sharing one bias), so the bias index is one
    // uniform div/mod per CTA iteration; the other modes see a single row of nvec vectors.
    const unsigned row_vecs = (BIAS == 4) ? step_b / VEC : nvec;
    const unsigned items_per_row = (row_vecs + kItem - 1) / kItem;
    const unsigned n_items = (nvec / row_vecs) * items_per_row;
    for (unsigned item = blockIdx.x; item < n_items; item += gridDim.x) {
        const unsigned r = item / items_per_row, kk = (item - r * items_per_row) * kItem + threadIdx.x;
        const unsigned vrow = r * row_vecs;
        V xv[UNROLL], xr[UNROLL], yr[UNROLL], dv[UNROLL];
        bool live[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const unsigned vi = vrow + kk + u * 256;
            live[u] = kk + u * 256 < row_vecs;
            if (live[u]) {
                xv[u] = reinterpret_cast<const V*>(p.x)[vi];
                if (REFS) {
                    if (p.xref) xr[u] = reinterpret_cast<const V*>(p.xref)[vi];
                    if (p.yref) yr[u] = reinterpret_cast<const V*>(p.yref)[vi];
                    if (p.dy) dv[u] = reinterpret_cast<const V*>(p.dy)[vi];
                }
            }
        }
        S brow = (S)0;
        if (BIAS == 4) brow = Elem<T>::ld(bp[r % size_b]);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            if (!live[u]) continue;
            const unsigned vi = vrow + kk + u * 256;
            const unsigned ge = vi * VEC + base;
            S bshared = brow;
            V bv;
            unsigned bi0 = 0;
            if (BIAS == 1) bshared = Elem<T>::ld(bp[(ge / step_b) % size_b]);
            if (BIAS == 2) bv = *reinterpret_cast<const V*>(bp + ge % size_b);
            if (BIAS == 3) bi0 = (step_b == 1) ? ge % size_b : 0;
            V out;
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                S b = bshared;
                if (BIAS == 2) b = Elem<T>::ld(bv.v[k]);
                if (BIAS == 3) b = Elem<T>::ld(bp[step_b == 1 ? (bi0 + k) % size_b : ((ge + k) / step_b) % size_b]);
                out.v[k] = Elem<T>::st(bias_act_elem<S, A>(G, Elem<T>::ld(xv[u].v[k]), b,
                                                           (REFS && p.xref) ? Elem<T>::ld(xr[u].v[k]) : (S)0,
                                                           (REFS && p.yref) ? Elem<T>::ld(yr[u].v[k]) : (S)0,
                                                           (REFS && p.dy) ? Elem<T>::ld(dv[u].v[k]) : (S)1, alpha, gain, clamp));
            }
            reinterpret_cast<V*>(p.y)[vi] = out;
        }
    }
}

template <typename T, int A, int VEC, int BIAS>
void launch_bias_act_g(const BiasActParams& q, int grid, cudaStream_t stream) {
    if (q.grad == 0 && !q.xref && !q.yref && !q.dy) k_bias_act<T, A, VEC, BIAS, true><<<grid, 256, 0, stream>>>(q);
    else k_bias_act<T, A, VEC, BIAS, false><<<grid, 256, 0, stream>>>(q);
}

template <typename T, int A, int VEC>
void launch_bias_act_v(const BiasActParams& q, int grid, cudaStream_t stream) {
    auto aligned = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
    if (!q.b) launch_bias_act_g<T, A, VEC, 0>(q, grid, stream);
    else if (q.step_b % VEC == 0 && q.step_b / VEC >= 128 && q.base == 0 && (q.numel / VEC) % (q.step_b / VEC) == 0)
        launch_bias_act_g<T, A, VEC, 4>(q, grid, stream);
    else if (q.step_b % VEC == 0) launch_bias_act_g<T, A, VEC, 1>(q, grid, stream);
    else if (VEC > 1 && q.step_b == 1 && q.size_b % VEC == 0 && q.base % VEC == 0 && aligned(q.b)) launch_bias_act_g<T, A, VEC, 2>(q, grid, stream);
    else launch_bias_act_g<T, A, VEC, 3>(q, grid, stream);
}

template <typename T, int A>
int launch_bias_act_t(const BiasActParams& p, cudaStream_t stream) {
    constexpr int VEC = 16 / sizeof(T);
    static int n_sm = 0;
    if (!n_sm) {
        int dev = 0;
        P3D_CUDA_TRY(cudaGetDevice(&dev));
        P3D_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    auto aligned = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    const bool vec_ok = aligned(p.x) && aligned(p.y) && aligned(p.xref) && aligned(p.yref) && aligned(p.dy);
    const long long main_n = vec_ok ? (p.numel / VEC) * VEC : 0;
    if (main_n > 0) {
        BiasActParams q = p;
        q.numel = main_n;
        const long long nvec = main_n / VEC;
        const int grid = (int)((nvec + 255) / 256 < (long long)n_sm * 8 ? (nvec + 255) / 256 : (long long)n_sm * 8);
        launch_bias_act_v<T, A, VEC>(q, grid, stream);
        P3D_LAUNCH_CHECK();
    }
    if (main_n < p.numel) {                                       // scalar tail (numel % VEC) or unaligned caller
        BiasActParams q = p;
        q.x = reinterpret_cast<const T*>(p.x) + main_n;
        q.y = reinterpret_cast<T*>(p.y) + main_n;
        if (p.xref) q.xref = reinterpret_cast<const T*>(p.xref) + main_n;
        if (p.yref) q.yref = reinterpret_cast<const T*>(p.yref) + main_n;
        if (p.dy) q.dy = reinterpret_cast<const T*>(p.dy) + main_n;
        q.numel = p.numel - main_n;
        q.base = main_n;
        const long long n = q.numel;
        const int grid = (int)((n + 255) / 256 < (long long)n_sm * 8 ? (n + 255) / 256 : (long long)n_sm * 8);
        launch_bias_act_v<T, A, 1>(q, grid, stream);
        P3D_LAUNCH_CHECK();
    }
    return P3D_OK;
}

template <typename T>
int launch_bias_act(const BiasActParams& p, int act, cudaStream_t stream) {
    switch (act) {
        case P3D_ACT_LINEAR: return launch_bias_act_t<T, P3D_ACT_LINEAR>(p, stream);
        case P3D_ACT_RELU: return launch_bias_act_t<T, P3D_ACT_RELU>(p, stream);
        case P3D_ACT_LRELU: return launch_bias_act_t<T, P3D_ACT_LRELU>(p, stream);
        case P3D_ACT_TANH: return launch_bias_act_t<T, P3D_ACT_TANH>(p, stream);
        case P3D_ACT_SIGMOID: return launch_bias_act_t<T, P3D_ACT_SIGMOID>(p, stream);
        case P3D_ACT_ELU: return launch_bias_act_t<T, P3D_ACT_ELU>(p, stream);
        case P3D_ACT_SELU: return launch_bias_act_t<T, P3D_ACT_SELU>(p, stream);
        case P3D_ACT_SOFTPLUS: return launch_bias_act_t<T, P3D_ACT_SOFTPLUS>(p, stream);
        case P3D_ACT_SWISH: return launch_bias_act_t<T, P3D_ACT_SWISH>(p, stream);
    }
    set_error("no CUDA kernel found for the specified activation func (act=%d)", act);
    return P3D_EINVAL;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_bias_act(const void* x, const void* b, const void* xref, const void* yref, const void* dy, void* y,
                            int64_t numel, int32_t dtype, int32_t grad, int64_t step_b, int32_t size_b, int32_t act,
                            float alpha, float gain, float clamp, void* stream) {
    P3D_REQUIRE(x && y, "x / y must not be NULL");
    P3D_REQUIRE(numel >= 0 && numel <= 0x7fffffffll, "x is too large");
    P3D_REQUIRE(grad >= 0 && grad <= 2, "grad must be 0, 1 or 2");
    P3D_REQUIRE(b == nullptr || (size_b > 0 && step_b > 0), "bias needs size_b > 0 and step_b > 0");
    if (numel == 0) return P3D_OK;
    BiasActParams p{x, b, xref, yref, dy, y, (long long)numel, b ? (long long)step_b : 1, 0ll, b ? size_b : 1, grad, alpha, gain, clamp};
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case P3D_F32: return launch_bias_act<float>(p, act, st);
        case P3D_F16: return launch_bias_act<__half>(p, act, st);
        case P3D_BF16: return launch_bias_act<__nv_bfloat16>(p, act, st);
        case P3D_F64: return launch_bias_act<double>(p, act, st);
    }
    set_error("unsupported dtype %d", dtype);
    return P3D_EINVAL;
}
