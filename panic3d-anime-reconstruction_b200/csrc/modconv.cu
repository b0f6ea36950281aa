// Modulated convolution at inference (StyleGAN2 modulated_conv2d with fused_modconv=True, reference
// _train/eg3dc/src/training/networks_stylegan2.py:40-98) as an implicit GEMM on Hopper wgmma.
//
//   p3d_modconv_prep     one CTA per (output channel, sample): modulate, demodulate, round to the compute type, write
//                        the B operand tiles (K-major, no swizzle, fused::tile_off geometry) the conv kernel copies as is.
//   p3d_modconv_forward  GEMM per sample and sub-pixel phase: M = output pixels of the phase, N = output channels,
//                        K = taps x input channels.  A CTA owns 128 output pixels x BN channels; two warpgroups each own
//                        64 rows.  K is streamed in chunks of 128 bytes per row (64 fp16 / 32 fp32 channels) of one tap
//                        through a 3-stage shared-memory ring: all 256 threads fill a stage (the im2col gather of A, a
//                        cp.async copy of the prepared B tile) while the tensor cores run on the previous one.
//
// Tap sets (one table per call, TapTable): kernel 3 / up 1 = 9 taps of a correlation with padding 1; kernel 1 = 1 tap;
// kernel 3 / up 2 = conv_transpose2d(stride 2, padding 0) split into the four sub-pixel phases (oy, ox parity):
// output row oy = 2 a + py takes kernel rows ky = py (mod 2) at input row a + (py - ky) / 2, i.e. 2 x 2 / 2 x 1 / 1 x 2 /
// 1 x 1 taps, and writes the (2H+1) x (2W+1) tensor conv_transpose2d writes (conv2d_resample.py up > 1 branch:
// w transposed per group, flip_weight=False -> no flip, padding [0, 0]).
#include "p3d_common.cuh"
#include "fused_common.cuh"
#include "../../include/p3d_ops.h"
#include "../../include/p3d_modconv.h"

namespace p3d {
namespace {

constexpr int kBM = 128, kThreads = 256, kKB = 128, kStages = 3;
constexpr int kLboA = kBM * 16;                  // bytes between 16-byte K columns of the A tile
constexpr int kTileA = kBM * kKB;
enum Mode { MODE_K3 = 0, MODE_K1 = 1, MODE_UP2 = 2 };

// Sub-pixel phases and their taps.  Slots [base[ph], base[ph] + cnt[ph]) of the operand are phase ph's taps, row-major
// over (jy, jx); tap slot s reads input (a + dy[s], b + dx[s]) for output (a, b) of the phase grid, with kernel tap w[s].
struct TapTable {
    int nphase, stride, ntaps;
    int base[4], cnt[4], oh[4], ow[4], oy0[4], ox0[4];
    int w[9], dy[9], dx[9];
};

// one axis: taps of phase ph (kernel index k, input offset d)
inline int ntaps_1d(int mode, int ph) { return mode == MODE_K3 ? 3 : mode == MODE_K1 ? 1 : (ph == 0 ? 2 : 1); }
inline void tap_1d(int mode, int ph, int j, int& k, int& d) {
    if (mode == MODE_K3) { k = j; d = j - 1; }
    else if (mode == MODE_K1) { k = 0; d = 0; }
    else { k = ph == 0 ? 2 * j : 1; d = -j; }
}

inline int mode_of(const p3d_modconv_params* p) { return p->up == 2 ? MODE_UP2 : p->kernel_size == 1 ? MODE_K1 : MODE_K3; }

TapTable make_taps(const p3d_modconv_params* p) {
    TapTable t{};
    const int mode = mode_of(p), nph = mode == MODE_UP2 ? 2 : 1, ks = p->kernel_size;
    t.nphase = nph * nph;
    t.stride = nph;
    int s = 0;
    for (int py = 0; py < nph; ++py)
        for (int px = 0; px < nph; ++px) {
            const int ph = py * nph + px, nty = ntaps_1d(mode, py), ntx = ntaps_1d(mode, px);
            t.base[ph] = s;
            t.cnt[ph] = nty * ntx;
            t.oh[ph] = mode == MODE_UP2 ? (py == 0 ? p->in_h + 1 : p->in_h) : p->in_h;
            t.ow[ph] = mode == MODE_UP2 ? (px == 0 ? p->in_w + 1 : p->in_w) : p->in_w;
            t.oy0[ph] = py;
            t.ox0[ph] = px;
            for (int jy = 0; jy < nty; ++jy)
                for (int jx = 0; jx < ntx; ++jx, ++s) {
                    int ky, kx, dy, dx;
                    tap_1d(mode, py, jy, ky, dy);
                    tap_1d(mode, px, jx, kx, dx);
                    t.w[s] = ky * ks + kx;
                    t.dy[s] = dy;
                    t.dx[s] = dx;
                }
        }
    t.ntaps = s;
    return t;
}

struct Geometry {
    int es, kce, nchunks, bn, nnb;       // element bytes, channels per chunk, chunks, N tile, N tiles
    size_t btile;                        // bytes of one B tile (bn x kKB)
};
Geometry geometry(const p3d_modconv_params* p) {
    Geometry g;
    g.es = p->dtype == P3D_F16 ? 2 : 4;
    g.kce = kKB / g.es;
    g.nchunks = (p->in_channels + g.kce - 1) / g.kce;
    g.bn = p->out_channels <= 8 ? 8 : 128;
    g.nnb = (p->out_channels + g.bn - 1) / g.bn;
    g.btile = (size_t)g.bn * kKB;
    return g;
}

__device__ __forceinline__ uint32_t to_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}
// byte offset of (row r, K byte b) in a K-major tile with `lbo` bytes between 16-byte K columns
__device__ __forceinline__ int tile_byte(int r, int b, int lbo) { return (r >> 3) * fused::kSBO + (b >> 4) * lbo + (r & 7) * 16 + (b & 15); }

// ------------------------------------------------------------------------------------------ prep
struct PrepArgs {
    const float *weight, *styles;
    unsigned char* ws;
    int Cin, Cout, kk, nnb, nchunks, bn, ntaps, f16, demod, prenorm;
    int cin_pad;
    float prenorm_c;                     // (float)(1 / sqrt(Cin k k)), networks_stylegan2.py:61
    size_t btile;
    TapTable tt;
};

__device__ float block_reduce(float v, bool is_max, float* red) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float u = __shfl_xor_sync(0xffffffffu, v, o);
        v = is_max ? fmaxf(v, u) : v + u;
    }
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    if (wid == 0) {
        v = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.f;   // |.| maxima and sums are >= 0
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float u = __shfl_xor_sync(0xffffffffu, v, o);
            v = is_max ? fmaxf(v, u) : v + u;
        }
        if (lane == 0) red[0] = v;
    }
    __syncthreads();
    return red[0];
}

__global__ void __launch_bounds__(256) k_modconv_prep(PrepArgs a) {
    __shared__ float red[32];
    const int co = blockIdx.x, n = blockIdx.y, tid = threadIdx.x;
    const bool live = co < a.Cout;
    const int K = a.Cin * a.kk;
    const float* wrow = a.weight + (size_t)(live ? co : 0) * K;
    const float* srow = a.styles + (size_t)n * a.Cin;
    // fp16 layers: weight * (1/sqrt(Cin k k) / max|W[co]|), styles / max|styles[n]| (networks_stylegan2.py:60-63)
    float rw = 1.f, smax = 1.f;
    if (a.prenorm) {
        float m = 0.f;
        for (int i = tid; i < K; i += blockDim.x) m = fmaxf(m, fabsf(wrow[i]));
        const float wmax = block_reduce(m, true, red);
        m = 0.f;
        for (int i = tid; i < a.Cin; i += blockDim.x) m = fmaxf(m, fabsf(srow[i]));
        smax = block_reduce(m, true, red);
        rw = __fdiv_rn(a.prenorm_c, wmax);
    }
    auto value = [&](int ci, int t) {
        float w = wrow[ci * a.kk + t], s = srow[ci];
        if (a.prenorm) { w = __fmul_rn(w, rw); s = __fdiv_rn(s, smax); }
        return __fmul_rn(w, s);
    };
    // dcoefs = rsqrt(sum w^2 + 1e-8) in fp32 (:69)
    float dcoef = 1.f;
    if (a.demod) {
        float ss = 0.f;
        for (int i = tid; i < K; i += blockDim.x) { const float v = value(i / a.kk, i % a.kk); ss = fmaf(v, v, ss); }
        dcoef = __frsqrt_rn(block_reduce(ss, false, red) + 1e-8f);
    }
    const int nb = co / a.bn, r = co % a.bn, es = a.f16 ? 2 : 4, kce = kKB / es, lbo = a.bn * 16;
    unsigned char* base = a.ws + ((size_t)n * a.nnb + nb) * a.ntaps * a.nchunks * a.btile;
    for (int i = tid; i < a.ntaps * a.cin_pad; i += blockDim.x) {
        const int s = i / a.cin_pad, ci = i % a.cin_pad;
        const float v = (live && ci < a.Cin) ? __fmul_rn(value(ci, a.tt.w[s]), dcoef) : 0.f;
        unsigned char* dst = base + ((size_t)s * a.nchunks + ci / kce) * a.btile + tile_byte(r, (ci % kce) * es, lbo);
        if (a.f16) *reinterpret_cast<__half*>(dst) = __float2half_rn(v);
        else *reinterpret_cast<uint32_t*>(dst) = to_tf32(v);
    }
}

// ------------------------------------------------------------------------------------------ conv
struct ConvArgs {
    const unsigned char* x;
    long long sxn, sxc, sxh, sxw;        // element strides
    const unsigned char* ws;
    const void* bias;
    const float* noise;
    long long snn, snh, snw;
    unsigned char* y;
    long long syn, syc, syh, syw;
    int Cin, Cout, H, W, nnb, nchunks, vec, act;
    float gain, clamp;
    size_t btile;
    TapTable tt;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <bool F16, int BN>
__device__ __forceinline__ void mma_step(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
    if constexpr (F16) { if constexpr (BN == 128) fused::wgmma_f16_n128(acc, da, db); else fused::wgmma_f16_n8(acc, da, db); }
    else { if constexpr (BN == 128) fused::wgmma_tf32_n128(acc, da, db); else fused::wgmma_tf32_n8(acc, da, db); }
}

template <bool F16, int BN>
__global__ void __launch_bounds__(kThreads) k_modconv(ConvArgs a) {
    constexpr int ES = F16 ? 2 : 4, KCE = kKB / ES, UE = 16 / ES, BTILE = BN * kKB, STAGE = kTileA + BTILE, LBOB = BN * 16;
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const TapTable& tt = a.tt;
    const int ph = blockIdx.z % tt.nphase, n = blockIdx.z / tt.nphase;
    const int owp = tt.ow[ph], mp = tt.oh[ph] * owp, m0 = blockIdx.x * kBM;
    if (m0 >= mp) return;
    const int nb = blockIdx.y, nk = tt.cnt[ph] * a.nchunks, slot0 = tt.base[ph];
    const uint32_t sbase = fused::smem_u32(smem);

    // this thread's im2col row (the same for every K chunk) and its four 16-byte units of that row
    const int lrow = tid & (kBM - 1), lcu0 = tid >> 7;
    const int pix = m0 + lrow;
    const bool prow = pix < mp;
    const int pa = prow ? pix / owp : 0, pb = prow ? pix % owp : 0;
    const unsigned char* xn = a.x + (long long)n * a.sxn * ES;
    const unsigned char* wsb = a.ws + (((size_t)n * a.nnb + nb) * tt.ntaps + slot0) * a.nchunks * (size_t)BTILE;

    auto load_stage = [&](int it, int stage) {
        const int j = it / a.nchunks, q = it % a.nchunks, s = slot0 + j;
        const int iy = pa + tt.dy[s], ix = pb + tt.dx[s];
        const bool valid = prow && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
        const int kvalid = min(KCE, a.Cin - q * KCE) * ES;
        const unsigned char* xrow = xn + ((long long)iy * a.sxh + (long long)ix * a.sxw) * ES;
        const uint32_t sa = sbase + stage * STAGE + (lrow >> 3) * fused::kSBO + (lrow & 7) * 16;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int cu = lcu0 + 2 * i;
            if (cu * 16 >= kvalid) break;
            const long long ch = (long long)q * KCE + cu * UE;
            const uint32_t dst = sa + cu * kLboA;
            if (F16 && a.vec) {
                cp_async16(dst, valid ? (const void*)(xrow + ch * ES) : (const void*)a.x, valid ? 16 : 0);
            } else {
                uint32_t v[4] = {0u, 0u, 0u, 0u};
                if (valid) {
                    if (a.vec) {
                        const uint4 u = __ldg(reinterpret_cast<const uint4*>(xrow + ch * ES));
                        v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w;
                    } else if (F16) {
                        const unsigned short* px = reinterpret_cast<const unsigned short*>(xrow) + ch * a.sxc;
#pragma unroll
                        for (int e = 0; e < 4; ++e) v[e] = (uint32_t)__ldg(px + (2 * e) * a.sxc) | ((uint32_t)__ldg(px + (2 * e + 1) * a.sxc) << 16);
                    } else {
                        const uint32_t* px = reinterpret_cast<const uint32_t*>(xrow) + ch * a.sxc;
#pragma unroll
                        for (int e = 0; e < 4; ++e) v[e] = __ldg(px + e * a.sxc);
                    }
                    if (!F16) {
#pragma unroll
                        for (int e = 0; e < 4; ++e) v[e] = to_tf32(__uint_as_float(v[e]));
                    }
                }
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(dst), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
            }
        }
        const unsigned char* bsrc = wsb + (size_t)it * BTILE;
        const uint32_t sb = sbase + stage * STAGE + kTileA;
        for (int u = tid; u < BTILE / 16; u += kThreads) cp_async16(sb + u * 16, bsrc + u * 16, 16);
    };

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int s = 0; s < kStages - 1; ++s) {
        if (s < nk) load_stage(s, s);
        cp_async_commit();
    }
#pragma unroll 1
    for (int it = 0; it < nk; ++it) {
        cp_async_wait<kStages - 2>();
        fused::fence_proxy_async();
        __syncthreads();
        const int stage = it % kStages, q = it % a.nchunks;
        const int ksteps = min(KCE, a.Cin - q * KCE) * ES / 32;
        const uint32_t sa = sbase + stage * STAGE + wg * 8 * fused::kSBO, sb = sbase + stage * STAGE + kTileA;
        fused::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kKB / 32; ++k)
            if (k < ksteps) mma_step<F16, BN>(acc, fused::wgmma_desc(sa + k * 2 * kLboA, kLboA, fused::kSBO), fused::wgmma_desc(sb + k * 2 * LBOB, LBOB, fused::kSBO));
        fused::wgmma_commit();
        if (it + kStages - 1 < nk) load_stage(it + kStages - 1, (it + kStages - 1) % kStages);
        cp_async_commit();
        fused::wgmma_wait_all();
        fused::fence_operands(acc);
    }

    // epilogue on the fp32 accumulator: + noise, + bias, activation, x gain, clamp, one rounding
    const int stride = tt.stride, oy0 = tt.oy0[ph], ox0 = tt.ox0[ph];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
        const int row = wg * 64 + fused::frag_row(i, lane, warp), co = nb * BN + fused::frag_col(i, lane);
        const int p = m0 + row;
        if (p >= mp || co >= a.Cout) continue;
        const int oy = (p / owp) * stride + oy0, ox = (p % owp) * stride + ox0;
        float v = acc[i];
        if (a.noise) v += a.noise[(long long)n * a.snn + (long long)oy * a.snh + (long long)ox * a.snw];
        if (a.bias) v += F16 ? __half2float(reinterpret_cast<const __half*>(a.bias)[co]) : reinterpret_cast<const float*>(a.bias)[co];
        if (a.act == P3D_ACT_LRELU) v = v > 0.f ? v : v * 0.2f;
        v *= a.gain;
        if (a.clamp >= 0.f) v = (v > -a.clamp && v < a.clamp) ? v : (v >= 0.f ? a.clamp : -a.clamp);
        const long long off = (long long)n * a.syn + (long long)co * a.syc + (long long)oy * a.syh + (long long)ox * a.syw;
        if (F16) reinterpret_cast<__half*>(a.y)[off] = __float2half_rn(v);
        else reinterpret_cast<float*>(a.y)[off] = v;
    }
}

template <bool F16, int BN>
int launch_conv(const ConvArgs& a, dim3 grid, cudaStream_t st) {
    constexpr int kSmem = kStages * (kTileA + BN * kKB);
    P3D_CUDA_TRY(cudaFuncSetAttribute(k_modconv<F16, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));   // per device
    k_modconv<F16, BN><<<grid, kThreads, kSmem, st>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_modconv_supported(const p3d_modconv_params* p) {
    if (!p) return 0;
    const bool k_ok = p->kernel_size == 3 || (p->kernel_size == 1 && p->up == 1);
    const bool dt_ok = p->dtype == P3D_F16 || (p->dtype == P3D_F32 && p->allow_tf32);
    const int nph = p->up == 2 ? 4 : 1;
    return k_ok && (p->up == 1 || p->up == 2) && p->down == 1 && dt_ok && (p->demodulate == 0 || p->demodulate == 1) &&
           p->in_channels > 0 && p->in_channels % 16 == 0 && p->in_channels <= 65536 && p->out_channels >= 1 &&
           p->out_channels <= 4096 && p->batch >= 1 && p->batch * nph <= 65535 && p->in_h >= 1 && p->in_w >= 1 &&
           p->in_h <= 4096 && p->in_w <= 4096;
}

extern "C" int p3d_modconv_out_size(const p3d_modconv_params* p, int32_t* out_h, int32_t* out_w) {
    P3D_REQUIRE(p && out_h && out_w, "p3d_modconv_out_size: NULL pointer");
    P3D_REQUIRE(p3d_modconv_supported(p), "p3d_modconv: unsupported layer (see p3d_modconv_supported)");
    *out_h = p->up == 2 ? 2 * p->in_h + 1 : p->in_h;
    *out_w = p->up == 2 ? 2 * p->in_w + 1 : p->in_w;
    return P3D_OK;
}

extern "C" size_t p3d_modconv_workspace_bytes(const p3d_modconv_params* p) {
    if (!p3d_modconv_supported(p)) return 0;
    const Geometry g = geometry(p);
    return (size_t)p->batch * g.nnb * make_taps(p).ntaps * g.nchunks * g.btile;
}

extern "C" int p3d_modconv_prep(const p3d_modconv_params* p, const float* weight, const float* styles, void* ws, void* stream) {
    P3D_REQUIRE(p3d_modconv_supported(p), "p3d_modconv_prep: unsupported layer (see p3d_modconv_supported)");
    P3D_REQUIRE(weight && styles && ws, "p3d_modconv_prep: NULL pointer");
    P3D_REQUIRE(((uintptr_t)ws & 15) == 0, "p3d_modconv_prep: workspace must be 16-byte aligned");
    const Geometry g = geometry(p);
    PrepArgs a;
    a.weight = weight; a.styles = styles; a.ws = (unsigned char*)ws;
    a.Cin = p->in_channels; a.Cout = p->out_channels; a.kk = p->kernel_size * p->kernel_size;
    a.nnb = g.nnb; a.nchunks = g.nchunks; a.bn = g.bn;
    a.tt = make_taps(p);
    a.ntaps = a.tt.ntaps;
    a.f16 = p->dtype == P3D_F16; a.demod = p->demodulate; a.prenorm = a.f16 && p->demodulate;
    a.cin_pad = g.nchunks * g.kce;
    a.prenorm_c = (float)(1.0 / sqrt((double)p->in_channels * a.kk));
    a.btile = g.btile;
    cudaStream_t st = (cudaStream_t)stream;
    ProfileScope prof(PROF_MODCONV, st);
    k_modconv_prep<<<dim3(g.nnb * g.bn, p->batch), 256, 0, st>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_modconv_forward(const p3d_modconv_params* p, const void* x, const int64_t* x_stride, const void* ws,
                                   const void* bias, const float* noise, const int64_t* noise_stride,
                                   void* y, const int64_t* y_stride, int32_t act, float gain, float clamp, void* stream) {
    P3D_REQUIRE(p3d_modconv_supported(p), "p3d_modconv_forward: unsupported layer (see p3d_modconv_supported)");
    P3D_REQUIRE(x && x_stride && ws && y && y_stride, "p3d_modconv_forward: NULL pointer");
    P3D_REQUIRE(!noise || noise_stride, "p3d_modconv_forward: noise without strides");
    P3D_REQUIRE(act == P3D_ACT_LINEAR || act == P3D_ACT_LRELU, "p3d_modconv_forward: act %d unsupported (linear or lrelu)", act);
    P3D_REQUIRE(((uintptr_t)ws & 15) == 0, "p3d_modconv_forward: workspace must be 16-byte aligned");
    const Geometry g = geometry(p);
    ConvArgs a;
    a.x = (const unsigned char*)x;
    a.sxn = x_stride[0]; a.sxc = x_stride[1]; a.sxh = x_stride[2]; a.sxw = x_stride[3];
    a.ws = (const unsigned char*)ws;
    a.bias = bias; a.noise = noise;
    a.snn = noise ? noise_stride[0] : 0; a.snh = noise ? noise_stride[1] : 0; a.snw = noise ? noise_stride[2] : 0;
    a.y = (unsigned char*)y;
    a.syn = y_stride[0]; a.syc = y_stride[1]; a.syh = y_stride[2]; a.syw = y_stride[3];
    a.Cin = p->in_channels; a.Cout = p->out_channels; a.H = p->in_h; a.W = p->in_w;
    a.nnb = g.nnb; a.nchunks = g.nchunks; a.act = act; a.gain = gain; a.clamp = clamp;
    a.btile = g.btile;
    a.tt = make_taps(p);
    // 16-byte vector loads of A when a pixel's channels are contiguous and every row start is 16-byte aligned
    const long long ue = 16 / g.es;
    a.vec = a.sxc == 1 && ((uintptr_t)x & 15) == 0 && a.sxn % ue == 0 && a.sxh % ue == 0 && a.sxw % ue == 0;
    int mmax = 0;
    for (int ph = 0; ph < a.tt.nphase; ++ph) mmax = max(mmax, a.tt.oh[ph] * a.tt.ow[ph]);
    const dim3 grid((mmax + kBM - 1) / kBM, g.nnb, p->batch * a.tt.nphase);
    cudaStream_t st = (cudaStream_t)stream;
    ProfileScope prof(PROF_MODCONV, st);
    if (p->dtype == P3D_F16) return g.bn == 8 ? launch_conv<true, 8>(a, grid, st) : launch_conv<true, 128>(a, grid, st);
    return g.bn == 8 ? launch_conv<false, 8>(a, grid, st) : launch_conv<false, 128>(a, grid, st);
}
