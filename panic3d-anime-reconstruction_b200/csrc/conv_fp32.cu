// fp32 training convolutions (conv2d_gradfix.conv2d / conv_transpose2d and their weight gradient) as implicit GEMMs on
// Hopper wgmma in 3xTF32: every operand element v is split into big = tf32(v) and small = tf32(v - big), and each K step
// issues small*big, big*small, big*big into one fp32 accumulator (small*small, below 2^-22 of the product, is dropped).
//
//   p3d_conv_forward      GEMM per sample and sub-pixel phase (conv_taps.cuh): M = output pixels of the phase, N = output
//                         channels, K = taps x input channels.  A is gathered from NCHW x per 32-channel chunk of one tap;
//                         B is the weight, first reordered K-major (tap, out channel, in channel) by k_weight_kmajor.
//                         conv_transpose2d runs as a correlation: stride 2 as the four phases of MODE_UP2, stride 1 with
//                         the taps flipped; its weight (Cin, Cout, k, k) is read with the two channel strides swapped.
//   p3d_conv_weight_grad  GEMM M = output channels of the gradient, N = (input channel, tap), K = (sample, pixel) in
//                         32-pixel chunks per sample, both operands gathered from NCHW along K.  conv_transpose2d's weight
//                         gradient is conv2d's with x and dy exchanged.  K is split over gridDim.z when the M x N tiles
//                         alone leave the GPU idle; each split writes its own partial tile and k_split_sum adds the
//                         partials in split order.  No atomics anywhere: outputs repeat bit for bit.
//
// A CTA owns a 128 x 128 tile; two warpgroups own 64 rows each.  Two shared-memory stages: while the tensor cores run on
// one, every thread loads its share of the next chunk into registers, then splits and stores it into the other.
#include "p3d_common.cuh"
#include "fused_common.cuh"
#include "conv_taps.cuh"
#include "../../include/p3d_conv.h"

namespace p3d {
namespace {

constexpr int kBM = 128, kThreads = 256, kKC = 32;   // tile rows (M and N), threads, K elements per chunk (128 B of a row)
// bytes between 16-byte K columns of a tile; the extra 16 put the 32 lanes of a warp that store along K in 32 banks
constexpr int kLbo = kBM * 16 + 16;
constexpr int kTile = 8 * kLbo;                      // one 128 x 32 fp32 operand tile
constexpr int kStage = 4 * kTile;                    // A big, A small, B big, B small
constexpr int kSmem = 2 * kStage;
constexpr int kSplitTarget = 264;                    // weight gradient: CTAs to aim for (two per SM of an H100 SXM)

__device__ __forceinline__ void split_store(unsigned char* st, int tile, int off, float v) {
    const uint32_t b = to_tf32(v);
    *reinterpret_cast<uint32_t*>(st + tile * kTile + off) = b;
    *reinterpret_cast<uint32_t*>(st + (tile + 1) * kTile + off) = to_tf32(v - __uint_as_float(b));
}

// The K loop shared by both GEMMs.  fetch(it) loads chunk it into the caller's registers, store(stage) splits them into
// the stage's four tiles, ksteps(it) is the number of 8-wide K steps chunk it holds (the rest of the tile is zero).
// Each chunk's 3 x ksteps wgmma accumulate into a zeroed register tile `part`, which is then added into `acc` with
// round-to-nearest fp32 adds: the tensor cores' own fp32 accumulation may truncate, and over thousands of steps that
// bias alone would outgrow every other rounding error.
template <class Fetch, class Store, class Ksteps>
__device__ __forceinline__ void mainloop(float (&acc)[64], long long nk, unsigned char* smem, Fetch fetch, Store store, Ksteps ksteps) {
    const int wg = threadIdx.x >> 7;
    const uint32_t sbase = fused::smem_u32(smem);
    float part[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    fetch(0ll);
    store(smem);
#pragma unroll 1
    for (long long it = 0; it < nk; ++it) {
        fused::fence_proxy_async();
        __syncthreads();
        const uint32_t sa = sbase + (uint32_t)(it & 1) * kStage + wg * 8 * fused::kSBO, sb = sbase + (uint32_t)(it & 1) * kStage + 2 * kTile;
        const int ks = ksteps(it);
#pragma unroll
        for (int i = 0; i < 64; ++i) part[i] = 0.f;
        fused::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kKC / 8; ++k)
            if (k < ks) {
                const uint32_t o = k * 2 * kLbo;
                const uint64_t ab = fused::wgmma_desc(sa + o, kLbo, fused::kSBO), as = fused::wgmma_desc(sa + kTile + o, kLbo, fused::kSBO);
                const uint64_t bb = fused::wgmma_desc(sb + o, kLbo, fused::kSBO), bs = fused::wgmma_desc(sb + kTile + o, kLbo, fused::kSBO);
                fused::wgmma_tf32_n128(part, as, bb);
                fused::wgmma_tf32_n128(part, ab, bs);
                fused::wgmma_tf32_n128(part, ab, bb);
            }
        fused::wgmma_commit();
        if (it + 1 < nk) fetch(it + 1);
        fused::wgmma_wait_all();
        fused::fence_operands(part);
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = __fadd_rn(acc[i], part[i]);
        if (it + 1 < nk) store(smem + (int)((it + 1) & 1) * kStage);
    }
}

// ------------------------------------------------------------------------------------------ forward
__global__ void k_weight_kmajor(const float* __restrict__ w, float* __restrict__ wk, int Cout, int Cin, int kk, long long w_co, long long w_ci) {
    const long long total = (long long)kk * Cout * Cin;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(e % Cin);
        const long long r = e / Cin;
        const int co = (int)(r % Cout), t = (int)(r / Cout);
        wk[e] = w[co * w_co + ci * w_ci + t];
    }
}

struct FwdArgs {
    const float* x;
    const float* wk;                     // (tap, Cout, Cin)
    float* y;
    int Cin, Cout, H, W, OH, OW, sin, nchunks;
    TapTable tt;
};

__global__ void __launch_bounds__(kThreads) k_conv_fwd(FwdArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const TapTable& tt = a.tt;
    const int ph = blockIdx.z % tt.nphase, n = blockIdx.z / tt.nphase;
    const int owp = tt.ow[ph], mp = tt.oh[ph] * owp, m0 = blockIdx.x * kBM, co0 = blockIdx.y * kBM;
    if (m0 >= mp) return;
    const long long nk = (long long)tt.cnt[ph] * a.nchunks, hw = (long long)a.H * a.W;
    const int slot0 = tt.base[ph];
    // A: thread = one output pixel (tile row) x four 4-channel units; B: thread = one K column x 16 rows
    const int lrow = tid & (kBM - 1), lcu0 = tid >> 7, kcol = tid & 31, rb0 = tid >> 5;
    const int pix = m0 + lrow;
    const bool prow = pix < mp;
    const int pa = prow ? pix / owp : 0, pb = prow ? pix % owp : 0;
    const float* xn = a.x + (long long)n * a.Cin * hw;
    float ra[16], rb[16];

    auto fetch = [&](long long it) {
        const int j = (int)(it / a.nchunks), q = (int)(it % a.nchunks), s = slot0 + j;
        const int iy = pa * a.sin + tt.dy[s], ix = pb * a.sin + tt.dx[s];
        const bool valid = prow && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
        const float* px = xn + (valid ? (long long)iy * a.W + ix : 0);
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int ci = q * kKC + (lcu0 + 2 * u) * 4 + e;
                ra[4 * u + e] = (valid && ci < a.Cin) ? __ldg(px + ci * hw) : 0.f;
            }
        const int ci = q * kKC + kcol;
        const float* wrow = a.wk + (long long)tt.w[s] * a.Cout * a.Cin + ci;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int co = co0 + rb0 + 8 * i;
            rb[i] = (ci < a.Cin && co < a.Cout) ? __ldg(wrow + (long long)co * a.Cin) : 0.f;
        }
    };
    auto store = [&](unsigned char* st) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            uint32_t b[4], s[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                b[e] = to_tf32(ra[4 * u + e]);
                s[e] = to_tf32(ra[4 * u + e] - __uint_as_float(b[e]));
            }
            const int off = tile_byte(lrow, (lcu0 + 2 * u) * 16, kLbo);
            *reinterpret_cast<uint4*>(st + off) = make_uint4(b[0], b[1], b[2], b[3]);
            *reinterpret_cast<uint4*>(st + kTile + off) = make_uint4(s[0], s[1], s[2], s[3]);
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) split_store(st, 2, tile_byte(rb0 + 8 * i, kcol * 4, kLbo), rb[i]);
    };
    auto ksteps = [&](long long it) { return (min(kKC, a.Cin - (int)(it % a.nchunks) * kKC) + 7) / 8; };

    float acc[64];
    mainloop(acc, nk, smem, fetch, store, ksteps);

    const int stride = tt.stride, oy0 = tt.oy0[ph], ox0 = tt.ox0[ph];
    float* yn = a.y + (long long)n * a.Cout * a.OH * a.OW;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        const int p = m0 + wg * 64 + fused::frag_row(i, lane, warp), co = co0 + fused::frag_col(i, lane);
        if (p >= mp || co >= a.Cout) continue;
        const int oy = (p / owp) * stride + oy0, ox = (p % owp) * stride + ox0;
        yn[((long long)co * a.OH + oy) * a.OW + ox] = acc[i];
    }
}

// ------------------------------------------------------------------------------------------ weight gradient
// dW[cg, cx, t] = sum over (n, a, b) of G[n, cg, a, b] * X[n, cx, a * s + dy[t], b * s + dx[t]]
struct WgradArgs {
    const float* g;                      // (N, CG, HG, WG)
    const float* x;                      // (N, CX, HX, WX)
    float* out;                          // split z's (CG, CX * kk) slab at out + z * slab
    int CG, CX, HG, WG, HX, WX, s, kk, cps, splits;
    long long nk_total, slab;
    TapTable tt;
};

__global__ void __launch_bounds__(kThreads) k_conv_wgrad(WgradArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const TapTable& tt = a.tt;
    const int z = blockIdx.z, m0 = blockIdx.x * kBM, j0 = blockIdx.y * kBM, nj = a.CX * a.kk;
    const long long c0 = a.nk_total * z / a.splits, nk = a.nk_total * (z + 1) / a.splits - c0;
    const long long hwg = (long long)a.HG * a.WG, hwx = (long long)a.HX * a.WX;
    const int kcol = tid & 31, rb0 = tid >> 5;        // thread = one K column (pixel) x 16 rows; rows are warp-uniform
    float ra[16], rb[16];

    auto fetch = [&](long long it) {
        const long long c = c0 + it;
        const long long n = c / a.cps;
        const int p = (int)(c % a.cps) * kKC + kcol;
        const bool pv = p < hwg;
        const int pa = pv ? p / a.WG : 0, pb = pv ? p % a.WG : 0;
        const float* gn = a.g + n * a.CG * hwg + p;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int cg = m0 + rb0 + 8 * i;
            ra[i] = (pv && cg < a.CG) ? __ldg(gn + cg * hwg) : 0.f;
        }
        const float* xn = a.x + n * a.CX * hwx;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int j = j0 + rb0 + 8 * i, cx = j / a.kk, t = j - cx * a.kk;
            const int iy = pa * a.s + tt.dy[t], ix = pb * a.s + tt.dx[t];
            const bool valid = pv && j < nj && iy >= 0 && iy < a.HX && ix >= 0 && ix < a.WX;
            rb[i] = valid ? __ldg(xn + cx * hwx + (long long)iy * a.WX + ix) : 0.f;
        }
    };
    auto store = [&](unsigned char* st) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int off = tile_byte(rb0 + 8 * i, kcol * 4, kLbo);
            split_store(st, 0, off, ra[i]);
            split_store(st, 2, off, rb[i]);
        }
    };
    auto ksteps = [](long long) { return kKC / 8; };

    float acc[64];
    mainloop(acc, nk, smem, fetch, store, ksteps);

    float* out = a.out + z * a.slab;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        const int cg = m0 + wg * 64 + fused::frag_row(i, lane, warp), j = j0 + fused::frag_col(i, lane);
        if (cg < a.CG && j < nj) out[(long long)cg * nj + j] = acc[i];
    }
}

// out[e] = sum over z = 0, 1, ... of parts[z * n + e], in that order
__global__ void k_split_sum(const float* __restrict__ parts, float* __restrict__ out, long long n, int splits) {
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        float s = parts[e];
        for (int z = 1; z < splits; ++z) s += parts[z * n + e];
        out[e] = s;
    }
}

// ------------------------------------------------------------------------------------------ host
void out_size(const p3d_conv_params* p, int& oh, int& ow) {
    const int k = p->kernel_size, s = p->stride, pd = p->padding;
    if (p->transpose) {
        oh = (p->in_h - 1) * s - 2 * pd + k + p->output_padding_h;
        ow = (p->in_w - 1) * s - 2 * pd + k + p->output_padding_w;
    } else {
        oh = (p->in_h + 2 * pd - k) / s + 1;
        ow = (p->in_w + 2 * pd - k) / s + 1;
    }
}

// the conv2d form of the call's (kernel, stride, padding): the weight gradient's taps
int conv2d_mode(const p3d_conv_params* p) { return p->kernel_size == 1 ? MODE_K1 : p->stride == 2 ? MODE_S2 : MODE_K3; }

TapTable forward_taps(const p3d_conv_params* p, int oh, int ow) {
    const bool up2 = p->transpose && p->stride == 2;
    TapTable t = tap_table(up2 ? MODE_UP2 : conv2d_mode(p), p->in_h, p->in_w, p->kernel_size);
    if (p->transpose && p->kernel_size == 3 && p->stride == 1)
        for (int s = 0; s < t.ntaps; ++s) t.w[s] = 8 - t.w[s];      // stride-1 transposed conv = correlation, taps flipped
    for (int ph = 0; ph < t.nphase; ++ph) {
        t.oh[ph] = (oh - t.oy0[ph] + t.stride - 1) / t.stride;
        t.ow[ph] = (ow - t.ox0[ph] + t.stride - 1) / t.stride;
    }
    return t;
}

struct Wgrad {
    int nmt, nnt, cps, splits;
    long long nk_total, slab;
};
Wgrad wgrad_plan(const p3d_conv_params* p) {
    int oh, ow;
    out_size(p, oh, ow);
    const int kk = p->kernel_size * p->kernel_size;
    // conv_transpose2d: G = x, X = dy;  conv2d: G = dy, X = x
    const int cg = p->transpose ? p->in_channels : p->out_channels, cx = p->transpose ? p->out_channels : p->in_channels;
    const long long hwg = p->transpose ? (long long)p->in_h * p->in_w : (long long)oh * ow;
    Wgrad w;
    w.nmt = (cg + kBM - 1) / kBM;
    w.nnt = (cx * kk + kBM - 1) / kBM;
    w.cps = (int)((hwg + kKC - 1) / kKC);
    w.nk_total = (long long)p->batch * w.cps;
    long long s = (kSplitTarget + w.nmt * w.nnt - 1) / (w.nmt * w.nnt);
    s = std::min(s, std::max(1ll, w.nk_total / 4));               // at least four chunks per split
    w.splits = (int)std::min(s, 64ll);
    w.slab = (long long)cg * cx * kk;
    return w;
}

int launch_attr(const void* fn) {
    P3D_CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));   // per device
    return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_conv_supported(const p3d_conv_params* p) {
    if (!p) return 0;
    const int k = p->kernel_size, s = p->stride, pd = p->padding;
    const bool kind = (k == 3 && s == 1 && pd == 1) || (k == 1 && s == 1 && pd == 0) || (k == 3 && s == 2 && pd == 0);
    const bool opad = p->transpose == 1 ? (p->output_padding_h >= 0 && p->output_padding_h < s && p->output_padding_w >= 0 && p->output_padding_w < s)
                                        : (p->transpose == 0 && p->output_padding_h == 0 && p->output_padding_w == 0);
    const int nphase = p->transpose && s == 2 ? 4 : 1;             // the forward grid's z is batch x phases (<= 65535)
    if (!kind || !opad || p->batch < 1 || p->batch > 16384 || p->batch * nphase > 65535 || p->in_channels < 1 || p->in_channels > 8192 ||
        p->out_channels < 1 || p->out_channels > 8192 || p->in_h < 1 || p->in_w < 1 || p->in_h > 4096 || p->in_w > 4096)
        return 0;
    int oh, ow;
    out_size(p, oh, ow);
    const long long lim = 1ll << 31;
    const bool fits = p->transpose || (p->in_h + 2 * pd >= k && p->in_w + 2 * pd >= k);    // conv2d: the kernel fits the padded input
    return fits && oh >= 1 && ow >= 1 &&
           (long long)p->in_channels * p->in_h * p->in_w < lim && (long long)p->out_channels * oh * ow < lim &&
           (long long)p->in_channels * p->out_channels * k * k < lim;
}

extern "C" int p3d_conv_out_size(const p3d_conv_params* p, int32_t* out_h, int32_t* out_w) {
    P3D_REQUIRE(p && out_h && out_w, "p3d_conv_out_size: NULL pointer");
    P3D_REQUIRE(p3d_conv_supported(p), "p3d_conv: unsupported call (see p3d_conv_supported)");
    int oh, ow;
    out_size(p, oh, ow);
    *out_h = oh;
    *out_w = ow;
    return P3D_OK;
}

extern "C" size_t p3d_conv_forward_workspace_bytes(const p3d_conv_params* p) {
    if (!p3d_conv_supported(p)) return 0;
    return (size_t)p->in_channels * p->out_channels * p->kernel_size * p->kernel_size * sizeof(float);
}

extern "C" int p3d_conv_forward(const p3d_conv_params* p, const float* x, const float* w, void* ws, size_t ws_bytes, float* y, void* stream) {
    P3D_REQUIRE(p3d_conv_supported(p), "p3d_conv_forward: unsupported call (see p3d_conv_supported)");
    P3D_REQUIRE(x && w && ws && y, "p3d_conv_forward: NULL pointer");
    P3D_REQUIRE(ws_bytes >= p3d_conv_forward_workspace_bytes(p), "p3d_conv_forward: workspace of %zu bytes, %zu needed", ws_bytes,
                p3d_conv_forward_workspace_bytes(p));
    P3D_REQUIRE(((uintptr_t)ws & 15) == 0, "p3d_conv_forward: workspace must be 16-byte aligned");
    int oh, ow;
    out_size(p, oh, ow);
    const int kk = p->kernel_size * p->kernel_size, cin = p->in_channels, cout = p->out_channels;
    cudaStream_t st = (cudaStream_t)stream;
    // conv2d weight (Cout, Cin, k, k); conv_transpose2d weight (Cin, Cout, k, k)
    const long long w_co = p->transpose ? kk : (long long)cin * kk, w_ci = p->transpose ? (long long)cout * kk : kk;
    const long long total = (long long)kk * cout * cin;
    k_weight_kmajor<<<(unsigned)std::min((total + 255) / 256, 4096ll), 256, 0, st>>>(w, (float*)ws, cout, cin, kk, w_co, w_ci);
    P3D_LAUNCH_CHECK();
    FwdArgs a;
    a.x = x; a.wk = (const float*)ws; a.y = y;
    a.Cin = cin; a.Cout = cout; a.H = p->in_h; a.W = p->in_w; a.OH = oh; a.OW = ow;
    a.sin = (!p->transpose && p->stride == 2) ? 2 : 1;
    a.nchunks = (cin + kKC - 1) / kKC;
    a.tt = forward_taps(p, oh, ow);
    long long mmax = 0;
    for (int ph = 0; ph < a.tt.nphase; ++ph) mmax = std::max(mmax, (long long)a.tt.oh[ph] * a.tt.ow[ph]);
    if (launch_attr((const void*)k_conv_fwd) != P3D_OK) return P3D_ECUDA;
    const dim3 grid((unsigned)((mmax + kBM - 1) / kBM), (cout + kBM - 1) / kBM, p->batch * a.tt.nphase);
    k_conv_fwd<<<grid, kThreads, kSmem, st>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" size_t p3d_conv_weight_grad_workspace_bytes(const p3d_conv_params* p) {
    if (!p3d_conv_supported(p)) return 0;
    const Wgrad g = wgrad_plan(p);
    return g.splits > 1 ? (size_t)g.splits * g.slab * sizeof(float) : 0;
}

extern "C" int p3d_conv_weight_grad(const p3d_conv_params* p, const float* x, const float* dy, void* ws, size_t ws_bytes, float* dw, void* stream) {
    P3D_REQUIRE(p3d_conv_supported(p), "p3d_conv_weight_grad: unsupported call (see p3d_conv_supported)");
    P3D_REQUIRE(x && dy && dw, "p3d_conv_weight_grad: NULL pointer");
    const size_t need = p3d_conv_weight_grad_workspace_bytes(p);
    P3D_REQUIRE(ws_bytes >= need && (need == 0 || ws), "p3d_conv_weight_grad: workspace of %zu bytes, %zu needed", ws_bytes, need);
    P3D_REQUIRE(((uintptr_t)ws & 15) == 0, "p3d_conv_weight_grad: workspace must be 16-byte aligned");
    int oh, ow;
    out_size(p, oh, ow);
    const Wgrad g = wgrad_plan(p);
    const bool tr = p->transpose != 0;
    WgradArgs a;
    a.g = tr ? x : dy;
    a.x = tr ? dy : x;
    a.CG = tr ? p->in_channels : p->out_channels;
    a.CX = tr ? p->out_channels : p->in_channels;
    a.HG = tr ? p->in_h : oh; a.WG = tr ? p->in_w : ow;
    a.HX = tr ? oh : p->in_h; a.WX = tr ? ow : p->in_w;
    a.s = p->stride;
    a.kk = p->kernel_size * p->kernel_size;
    a.cps = g.cps; a.splits = g.splits; a.nk_total = g.nk_total; a.slab = g.slab;
    a.out = g.splits > 1 ? (float*)ws : dw;
    a.tt = tap_table(conv2d_mode(p), a.HG, a.WG, p->kernel_size);
    cudaStream_t st = (cudaStream_t)stream;
    if (launch_attr((const void*)k_conv_wgrad) != P3D_OK) return P3D_ECUDA;
    k_conv_wgrad<<<dim3(g.nmt, g.nnt, g.splits), kThreads, kSmem, st>>>(a);
    P3D_LAUNCH_CHECK();
    if (g.splits > 1) {
        k_split_sum<<<(unsigned)std::min((g.slab + 255) / 256, 4096ll), 256, 0, st>>>((const float*)ws, dw, g.slab, g.splits);
        P3D_LAUNCH_CHECK();
    }
    return P3D_OK;
}
