// upfirdn2d for sm_90a: zero-insert upsample -> pad/crop -> 2-D FIR -> decimate, x gain.
//
//   y[n,c,oy,ox] = gain * sum_{ky,kx} P[oy*downy + ky, ox*downx + kx] * w[ky][kx]
//   P[py,px]     = x[(py-pady0)/upy, (px-padx0)/upx] where both divisions are exact and in range, else 0
//   w[ky][kx]    = flip ? f[ky][kx] : f[fH-1-ky][fW-1-kx]          (reference semantics: ops/upfirdn2d.py:169-213,
//                                                                    kernels ops/upfirdn2d.cu:33-204)
// The op is HBM-bound (read x once, write y once, a handful of FMAs per output), so the kernel is built
// around memory behaviour rather than per-(up,down,filter) template specialisations (the reference has ~100):
//   * tiled path (input rows contiguous along W): a CTA produces a 64x16 output tile of one (n,c) image; the
//     input footprint is staged ONCE in shared memory with coalesced row reads, zero-filled outside the image,
//     so the polyphase inner loop is pure LDS+FFMA with no bounds checks; only the taps whose phase hits a
//     real sample are visited (up>1 never multiplies the inserted zeros);
//   * strided path (channels-last or any other layout): same maths straight from global memory through L1,
//     with threads mapped channel-fastest so channels-last stays coalesced;
//   * fp32 / fp16 / bf16 / fp64 storage, fp32 (fp64) accumulation, 64-bit safe indexing.
#include "p3d_common.cuh"
#include "../../include/p3d_ops.h"

namespace p3d {
namespace {

// a * b + c per component, each rounded once (fma.rn)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

template <typename T> struct Px;
template <> struct Px<float> { using acc = float; static __device__ float ld(float v) { return v; } static __device__ float st(float v) { return v; } };
template <> struct Px<double> { using acc = double; static __device__ double ld(double v) { return v; } static __device__ double st(double v) { return v; } };
template <> struct Px<__half> { using acc = float; static __device__ float ld(__half v) { return __half2float(v); } static __device__ __half st(float v) { return __float2half_rn(v); } };
template <> struct Px<__nv_bfloat16> { using acc = float; static __device__ float ld(__nv_bfloat16 v) { return __bfloat162float(v); } static __device__ __nv_bfloat16 st(float v) { return __float2bfloat16_rn(v); } };

struct UpfirdnParams {
    const void* x;
    const float* f;
    void* y;
    int N, C, inH, inW, outH, outW, fH, fW;
    long long xs[4], ys[4];          // element strides {n, c, h, w}
    long long fsh, fsw;
    int upx, upy, downx, downy, padx0, pady0, flip;
    float gain;
    int tilesX, tilesY, inTileW, inTileH;
};

constexpr int kTileW = 64, kTileH = 16, kThreads = 256, kMaxTaps = 1024;

__device__ __forceinline__ int floor_div(int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }
__device__ __forceinline__ int pos_mod(int a, int b) { int m = a % b; return m < 0 ? m + b : m; }

// ------------------------------------------------------------------------------------------ tiled (W-contiguous input)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_upfirdn2d_tiled(const UpfirdnParams p) {
    using S = typename Px<T>::acc;
    extern __shared__ unsigned char smem_raw[];
    float* s_w = reinterpret_cast<float*>(smem_raw);                         // fH*fW taps (gain, flip folded in)
    S* s_x = reinterpret_cast<S*>(smem_raw + ((p.fH * p.fW * 4 + 15) & ~15));   // inTileH x inTileW
    const int tid = threadIdx.x;
    for (int i = tid; i < p.fH * p.fW; i += kThreads) {
        const int ky = i / p.fW, kx = i - ky * p.fW;
        const int sy = p.flip ? ky : p.fH - 1 - ky, sx = p.flip ? kx : p.fW - 1 - kx;
        s_w[i] = p.f[sy * p.fsh + sx * p.fsw] * p.gain;
    }
    const int tile = blockIdx.x;
    const int tyi = tile / p.tilesX, txi = tile - tyi * p.tilesX;
    const int ox0 = txi * kTileW, oy0 = tyi * kTileH;
    const int ix0 = floor_div(ox0 * p.downx - p.padx0, p.upx);               // first input column/row that can contribute
    const int iy0 = floor_div(oy0 * p.downy - p.pady0, p.upy);
    const T* xp = reinterpret_cast<const T*>(p.x);
    T* yp = reinterpret_cast<T*>(p.y);
    for (long long img = blockIdx.y; img < (long long)p.N * p.C; img += gridDim.y) {
        const int n = (int)(img / p.C), c = (int)(img - (long long)n * p.C);
        const T* xi = xp + n * p.xs[0] + c * p.xs[1];
        __syncthreads();                                                     // previous image's reads are done
        for (int i = tid; i < p.inTileH * p.inTileW; i += kThreads) {
            const int r = i / p.inTileW, q = i - r * p.inTileW;
            const int iy = iy0 + r, ix = ix0 + q;
            S v = (S)0;
            if (iy >= 0 && iy < p.inH && ix >= 0 && ix < p.inW) v = Px<T>::ld(xi[iy * p.xs[2] + ix * p.xs[3]]);
            s_x[i] = v;
        }
        __syncthreads();
        const int tx = tid & (kTileW - 1);
        const int ox = ox0 + tx;
        if (ox < p.outW) {
            const int ux0 = ox * p.downx - p.padx0;                          // up-sampled coordinate of tap kx = 0
            const int kx0 = pos_mod(-ux0, p.upx);
            const int sx0 = (ux0 + kx0) / p.upx - ix0;                       // exact division
#pragma unroll 1
            for (int ty = tid / kTileW; ty < kTileH; ty += kThreads / kTileW) {
                const int oy = oy0 + ty;
                if (oy >= p.outH) break;
                const int uy0 = oy * p.downy - p.pady0;
                const int ky0 = pos_mod(-uy0, p.upy);
                const int sy0 = (uy0 + ky0) / p.upy - iy0;
                S acc = (S)0;
                for (int ky = ky0, sy = sy0; ky < p.fH; ky += p.upy, ++sy) {
                    const S* row = s_x + sy * p.inTileW + sx0;
                    const float* wr = s_w + ky * p.fW;
                    for (int kx = kx0, j = 0; kx < p.fW; kx += p.upx, ++j) acc += row[j] * (S)wr[kx];
                }
                yp[n * p.ys[0] + c * p.ys[1] + oy * p.ys[2] + ox * p.ys[3]] = Px<T>::st(acc);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ fast path (4x4 FIR)
// The shapes panic3d's generator/discriminator hit (SURVEY 8a13): a 4x4 [1,3,3,1]^2 filter at (up,down) = (1,1) blur
// after a transposed conv, (2,1) skip-image upsample, (1,2) discriminator downsample; W-contiguous in and out.
// With 16 fp32 FMAs per output the op sits at the instruction-issue limit long before HBM (16 x 134 M outputs is
// already 60 us of FMA-pipe time against an 82 us HBM floor for fp16), so the kernel is built to minimise issued
// instructions per output as much as bytes:
//   * persistent CTAs walk output tiles (128 x 8*RPT) with a two-stage cp.async pipeline: the input footprint of
//     tile i+1 streams into shared memory as ALIGNED 16-byte vectors while tile i is computed.  Rows of odd-width
//     images (513 x fp16 = 1026 B) are not 16-byte aligned, so each shared row is shifted by the row's own
//     misalignment a_r = (address / sizeof(T)) mod VEC: aligned global vector k of a row lands on aligned shared
//     vector k, and footprint element q sits at column a_r + q.  Vectors that straddle the image border (<= 2 per
//     row) are assembled element-wise, rows above/below the image are zeros.  Row base pointers are computed once
//     per tile (one thread per row, one tile ahead), so a vector costs ~15 instructions to issue;
//   * a thread owns 4 output columns x RPT consecutive rows: up = 1 -> one column in each of four 32-column blocks,
//     up = 2 -> an (even, odd) phase pair in each of two 64-column blocks.  Lanes of a warp therefore read
//     consecutive shared-memory elements (no bank conflicts; the first version's 4 adjacent columns per thread cost
//     4-way conflicts in fp32).  Every input sample of the window is read once and scattered into the accumulators
//     it feeds; tap indices are compile-time (ky = sr*UP - r*DOWN, kx from the polyphase slot), the taps sit in
//     uniform registers, and the FMAs are issued as packed fma.rn.f32x2 (two outputs per instruction);
//   * fp32 accumulation for every storage type, one rounding at the store (the reference's scalar_t=float path).
template <typename T, int UP, int DOWN, int F>
struct FastCfg {
    static constexpr int VEC = 16 / (int)sizeof(T);
    static constexpr int EPT = 4;                                  // outputs per thread and row:
    static constexpr int EA = UP;                                  //   EA adjacent columns (an even/odd phase pair when up = 2)
    static constexpr int NB = EPT / EA;                            //   in NB blocks, BS columns apart - so a warp reads
    static constexpr int TW = 32 * EPT;                            //   consecutive shared-memory words (no bank conflicts)
    static constexpr int BS = TW / NB;
    static constexpr int RPT = (DOWN == 1) ? 8 : (sizeof(T) == 4 ? 2 : 4);
    static constexpr int TH = 8 * RPT;
    static constexpr int IN_W = ((TW - 1) * DOWN + F - 1) / UP + 1;
    static constexpr int IN_H = ((TH - 1) * DOWN + F - 1) / UP + 1;
    static constexpr int NIN = ((EA - 1) * DOWN + F - 1) / UP + 1;             // input columns per block a thread touches per row
    static constexpr int NINROWS = ((RPT - 1) * DOWN + F - 1) / UP + 1;
    static constexpr int NT = (F + UP - 1) / UP;                   // taps per output per dimension (polyphase slots)
    static constexpr int KX_ODD = ((-DOWN) % UP + UP) % UP;        // first tap of an odd output column
    static constexpr int PITCH = (IN_W + VEC - 1 + VEC - 1) / VEC * VEC;
    static constexpr int NV = PITCH / VEC;
    static constexpr size_t kBufBytes = (size_t)IN_H * PITCH * sizeof(T);
    static constexpr size_t kRowPtrOff = 2 * kBufBytes;
    static constexpr size_t kShiftOff = kRowPtrOff + 2 * IN_H * sizeof(void*);
    static constexpr size_t kSmem = kShiftOff + 2 * IN_H * sizeof(int);
    static_assert(F % UP == 0 && (UP == 1 || UP == 2) && (UP == 1 || DOWN == 1), "polyphase slots must be uniform");
    static_assert(IN_H <= 256, "one thread per footprint row");
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <typename T, int UP, int DOWN, int F>
__global__ void __launch_bounds__(kThreads) k_upfirdn2d_fast(const UpfirdnParams p, unsigned total_tiles, int vec_store) {
    using Cfg = FastCfg<T, UP, DOWN, F>;
    using V = uint4;
    constexpr int VEC = Cfg::VEC, PITCH = Cfg::PITCH, NV = Cfg::NV, IN_H = Cfg::IN_H, RPT = Cfg::RPT, NT = Cfg::NT, EPT = Cfg::EPT;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int kBufElems = (int)(Cfg::kBufBytes / sizeof(T));
    T* const s_x = reinterpret_cast<T*>(smem_raw);                              // [2][IN_H][PITCH]; index arithmetic only,
                                                                                // so every access stays an LDS/STS
    const T** const s_rowp = reinterpret_cast<const T**>(smem_raw + Cfg::kRowPtrOff);   // [2][IN_H] footprint row bases
    int* const s_a = reinterpret_cast<int*>(smem_raw + Cfg::kShiftOff);                 // [2][IN_H] row shifts
    const int tid = threadIdx.x;
    const T* xp = reinterpret_cast<const T*>(p.x);
    T* yp = reinterpret_cast<T*>(p.y);

    // taps as (even column, odd column) pairs per polyphase slot: w2[ky][j] = (w[ky][j*UP], w[ky][KX_ODD + j*UP])
    float2 w2[F][NT];
#pragma unroll
    for (int ky = 0; ky < F; ++ky) {
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const int kxe = j * UP, kxo = Cfg::KX_ODD + j * UP;
            const int sy = p.flip ? ky : F - 1 - ky;
            const int sxe = p.flip ? kxe : F - 1 - kxe, sxo = p.flip ? kxo : F - 1 - kxo;
            w2[ky][j] = make_float2(p.f[sy * p.fsh + sxe * p.fsw] * p.gain, p.f[sy * p.fsh + sxo * p.fsw] * p.gain);
        }
    }
    const unsigned tiles_per_img = (unsigned)(p.tilesX * p.tilesY);

    // tile walk: t -> (txi, tyi, c, n) advances by gridDim.x per iteration; the mixed-radix increment is decomposed
    // once, so stepping costs a few adds/compares instead of four integer divisions per tile
    struct Tile { int txi, tyi, c, n; const T* xi; long long yoff; };
    int d_x, d_y, d_c, d_n;
    {
        unsigned g = gridDim.x;
        d_x = (int)(g % (unsigned)p.tilesX); g /= (unsigned)p.tilesX;
        d_y = (int)(g % (unsigned)p.tilesY); g /= (unsigned)p.tilesY;
        d_c = (int)(g % (unsigned)p.C); d_n = (int)(g / (unsigned)p.C);
    }
    auto locate = [&](Tile& tl) { tl.xi = xp + tl.n * p.xs[0] + tl.c * p.xs[1]; tl.yoff = tl.n * p.ys[0] + tl.c * p.ys[1]; };
    auto decode = [&](unsigned t) {
        const unsigned img = t / tiles_per_img;
        const unsigned rem = t - img * tiles_per_img;
        Tile tl;
        tl.tyi = (int)(rem / (unsigned)p.tilesX); tl.txi = (int)(rem - (unsigned)tl.tyi * (unsigned)p.tilesX);
        tl.n = (int)(img / (unsigned)p.C); tl.c = (int)(img - (unsigned)tl.n * (unsigned)p.C);
        locate(tl);
        return tl;
    };
    auto advance = [&](Tile tl) {                                             // tile index + gridDim.x
        tl.txi += d_x; int carry = tl.txi >= p.tilesX; tl.txi -= carry ? p.tilesX : 0;
        tl.tyi += d_y + carry; carry = tl.tyi >= p.tilesY; tl.tyi -= carry ? p.tilesY : 0;
        tl.c += d_c + carry; carry = tl.c >= p.C; tl.c -= carry ? p.C : 0;
        tl.n += d_n + carry;
        locate(tl);
        return tl;
    };
    // footprint row bases of a tile (element q = 0 of each row; nullptr for rows above/below the image)
    auto rows = [&](const Tile& tl, int slot) {
        if (tid < IN_H) {
            const int ix0 = (tl.txi * Cfg::TW * DOWN - p.padx0) / UP, iy = (tl.tyi * Cfg::TH * DOWN - p.pady0) / UP + tid;   // exact
            s_rowp[slot * IN_H + tid] = (iy >= 0 && iy < p.inH) ? tl.xi + (long long)iy * p.xs[2] + ix0 : nullptr;
        }
    };
    auto issue = [&](const Tile& tl, int slot) {
        const int ix0 = (tl.txi * Cfg::TW * DOWN - p.padx0) / UP;
        T* sb = s_x + slot * kBufElems;
        for (int i = tid; i < IN_H * NV; i += kThreads) {
            const int r = i / NV, k = i - r * NV;
            V* dst = reinterpret_cast<V*>(sb + i * VEC);                     // == sb + r*PITCH + k*VEC
            const T* row0 = s_rowp[slot * IN_H + r];
            const int a = (int)((reinterpret_cast<uintptr_t>(row0) / sizeof(T)) & (VEC - 1));
            if (k == 0) s_a[slot * IN_H + r] = a;
            const int ix = ix0 + k * VEC - a;                                // image column of the vector's first element
            const T* src = row0 + (k * VEC - a);                             // 16-byte aligned
            if (row0 != nullptr && ix >= 0 && ix + VEC <= p.inW) {
                cp_async16(dst, src);
            } else if (row0 == nullptr || ix + VEC <= 0 || ix >= p.inW) {
                *dst = make_uint4(0u, 0u, 0u, 0u);
            } else {
                alignas(16) T tmp[VEC];
#pragma unroll
                for (int j = 0; j < VEC; ++j) tmp[j] = (ix + j >= 0 && ix + j < p.inW) ? src[j] : Px<T>::st(0.f);
                *dst = *reinterpret_cast<const V*>(tmp);
            }
        }
    };

    unsigned t = blockIdx.x;
    if (t >= total_tiles) return;
    Tile cur = decode(t);
    rows(cur, 0);
    Tile nxt = cur;
    if (t + gridDim.x < total_tiles) { nxt = advance(cur); rows(nxt, 1); }
    __syncthreads();
    issue(cur, 0);
    cp_async_commit();
    const int tx = tid & 31, tr = tid >> 5;
    constexpr int EA = Cfg::EA, NB = Cfg::NB, BS = Cfg::BS;
    const int y0 = tr * RPT, by = (y0 * DOWN) / UP;
    int bxm[NB];                                                             // first footprint column of each block
#pragma unroll
    for (int m = 0; m < NB; ++m) bxm[m] = ((m * BS + EA * tx) * DOWN) / UP;  // exact: EA*tx and BS are multiples of UP
    int b = 0;
    for (; t < total_tiles; t += gridDim.x, b ^= 1) {
        const bool has_next = t + gridDim.x < total_tiles;
        if (has_next) issue(nxt, b ^ 1);                                     // row bases of nxt were published one sync ago
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        // row bases for the tile after next go into the slot `cur` used (its issue finished an iteration ago)
        Tile nn = nxt;
        if (t + 2ull * gridDim.x < total_tiles) { nn = advance(nxt); rows(nn, b); }

        // acc[r][q]: up = 1 -> columns (block 2q, block 2q+1) at tx; up = 2 -> columns (2tx, 2tx+1) of block q
        float2 acc[RPT][EPT / 2];
#pragma unroll
        for (int r = 0; r < RPT; ++r) acc[r][0] = acc[r][1] = make_float2(0.f, 0.f);
        const T* sb = s_x + b * kBufElems;
#pragma unroll
        for (int sr = 0; sr < Cfg::NINROWS; ++sr) {
            const T* rowp = sb + (by + sr) * PITCH + s_a[b * IN_H + by + sr];
            float v[NB][Cfg::NIN];
#pragma unroll
            for (int m = 0; m < NB; ++m) {
#pragma unroll
                for (int sc = 0; sc < Cfg::NIN; ++sc) v[m][sc] = Px<T>::ld(rowp[bxm[m] + sc]);
            }
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const int ky = sr * UP - r * DOWN;
                if (ky < 0 || ky >= F) continue;
#pragma unroll
                for (int q = 0; q < EPT / 2; ++q) {
#pragma unroll
                    for (int j = 0; j < NT; ++j) {
                        if (UP == 1) {                                       // same tap j, two blocks
                            acc[r][q] = ffma2(make_float2(v[(2 * q) % NB][j], v[(2 * q + 1) % NB][j]), w2[ky][j], acc[r][q]);
                        } else {                                             // even column: tap 2j, input j; odd: tap KX_ODD+2j
                            constexpr int dummy = 0; (void)dummy;
                            const int sco = (DOWN + Cfg::KX_ODD + j * UP) / UP;
                            acc[r][q] = ffma2(make_float2(v[q % NB][j], v[q % NB][sco]), w2[ky][j], acc[r][q]);
                        }
                    }
                }
            }
        }
        {
            const int oxb = cur.txi * Cfg::TW + EA * tx, oy0 = cur.tyi * Cfg::TH + y0;
            T* yi = yp + cur.yoff + oxb;
#pragma unroll
            for (int r = 0; r < RPT; ++r) {
                const int oy = oy0 + r;
                if (oy >= p.outH) break;
                T* dst = yi + (long long)oy * p.ys[2];
                if (UP == 1) {
#pragma unroll
                    for (int m = 0; m < NB; ++m)
                        if (oxb + m * BS < p.outW) dst[m * BS] = Px<T>::st((m & 1) ? acc[r][m / 2].y : acc[r][m / 2].x);
                } else {
#pragma unroll
                    for (int q = 0; q < EPT / 2; ++q) {
                        const int ox = oxb + q * BS;
                        if (vec_store && ox + 1 < p.outW) {
                            struct alignas(2 * sizeof(T)) Pair { T a, b; };
                            *reinterpret_cast<Pair*>(dst + q * BS) = Pair{Px<T>::st(acc[r][q].x), Px<T>::st(acc[r][q].y)};
                        } else {
                            if (ox < p.outW) dst[q * BS] = Px<T>::st(acc[r][q].x);
                            if (ox + 1 < p.outW) dst[q * BS + 1] = Px<T>::st(acc[r][q].y);
                        }
                    }
                }
            }
        }
        __syncthreads();                                                     // buffer b and row slot b^1 are free again
        cur = nxt;
        nxt = nn;
    }
    cp_async_wait<0>();
}

template <typename T, int UP, int DOWN, int F>
int launch_fast(UpfirdnParams p, int n_sm, cudaStream_t stream) {
    using Cfg = FastCfg<T, UP, DOWN, F>;
    static int ctas_per_sm = 0;
    if (!ctas_per_sm) {
        P3D_CUDA_TRY(cudaFuncSetAttribute(k_upfirdn2d_fast<T, UP, DOWN, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem));
        P3D_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, k_upfirdn2d_fast<T, UP, DOWN, F>, kThreads, Cfg::kSmem));
        if (ctas_per_sm < 1) ctas_per_sm = 1;
    }
    p.tilesX = (p.outW + Cfg::TW - 1) / Cfg::TW;
    p.tilesY = (p.outH + Cfg::TH - 1) / Cfg::TH;
    const long long total = (long long)p.N * p.C * p.tilesX * p.tilesY;
    if (total >= 0x7fffffffll) return 1;                          // tile counter is 32-bit: leave it to the generic kernel
    const long long cap = (long long)n_sm * ctas_per_sm;
    const int grid = (int)(total < cap ? total : cap);
    const uintptr_t pa = 2 * sizeof(T) - 1;
    const int pair_store = ((reinterpret_cast<uintptr_t>(p.y) & pa) == 0 && p.ys[0] % 2 == 0 && p.ys[1] % 2 == 0 && p.ys[2] % 2 == 0) ? 1 : 0;
    k_upfirdn2d_fast<T, UP, DOWN, F><<<grid, kThreads, Cfg::kSmem, stream>>>(p, (unsigned)total, pair_store);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

// returns 1 when the shape is not covered by the fast path (0 / negative: launched / error)
template <typename T>
int try_launch_fast(const UpfirdnParams& p, int n_sm, cudaStream_t stream) {
    if (sizeof(T) > 4) return 1;
    if (p.xs[3] != 1 || p.ys[3] != 1 || p.fH != 4 || p.fW != 4 || p.upx != p.upy || p.downx != p.downy) return 1;
    if (p.padx0 % p.upx != 0 || p.pady0 % p.upy != 0) return 1;
    if ((long long)p.outW * p.downx + 8 > 0x3fffffffll || (long long)p.outH * p.downy + 8 > 0x3fffffffll) return 1;
    if (p.upx == 1 && p.downx == 1) return launch_fast<T, 1, 1, 4>(p, n_sm, stream);
    if (p.upx == 2 && p.downx == 1) return launch_fast<T, 2, 1, 4>(p, n_sm, stream);
    if (p.upx == 1 && p.downx == 2) return launch_fast<T, 1, 2, 4>(p, n_sm, stream);
    return 1;
}
template <> int try_launch_fast<double>(const UpfirdnParams&, int, cudaStream_t) { return 1; }

// ------------------------------------------------------------------------------------------ strided (any layout)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_upfirdn2d_strided(const UpfirdnParams p, int c_fastest) {
    using S = typename Px<T>::acc;
    __shared__ float s_w[kMaxTaps];
    const int taps = p.fH * p.fW;
    for (int i = threadIdx.x; i < taps; i += kThreads) {
        const int ky = i / p.fW, kx = i - ky * p.fW;
        const int sy = p.flip ? ky : p.fH - 1 - ky, sx = p.flip ? kx : p.fW - 1 - kx;
        s_w[i] = p.f[sy * p.fsh + sx * p.fsw] * p.gain;
    }
    __syncthreads();
    const T* xp = reinterpret_cast<const T*>(p.x);
    T* yp = reinterpret_cast<T*>(p.y);
    const long long total = (long long)p.N * p.C * p.outH * p.outW;
    for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < total; idx += (long long)gridDim.x * kThreads) {
        int n, c, oy, ox;
        long long r = idx;
        if (c_fastest) { c = (int)(r % p.C); r /= p.C; ox = (int)(r % p.outW); r /= p.outW; oy = (int)(r % p.outH); n = (int)(r / p.outH); }
        else { ox = (int)(r % p.outW); r /= p.outW; oy = (int)(r % p.outH); r /= p.outH; c = (int)(r % p.C); n = (int)(r / p.C); }
        const int ux0 = ox * p.downx - p.padx0, uy0 = oy * p.downy - p.pady0;
        const int kx0 = pos_mod(-ux0, p.upx), ky0 = pos_mod(-uy0, p.upy);
        const T* xi = xp + n * p.xs[0] + c * p.xs[1];
        S acc = (S)0;
        for (int ky = ky0; ky < p.fH; ky += p.upy) {
            const int iy = (uy0 + ky) / p.upy;
            if (iy < 0 || iy >= p.inH) continue;
            for (int kx = kx0; kx < p.fW; kx += p.upx) {
                const int ix = (ux0 + kx) / p.upx;
                if (ix < 0 || ix >= p.inW) continue;
                acc += Px<T>::ld(xi[iy * p.xs[2] + ix * p.xs[3]]) * (S)s_w[ky * p.fW + kx];
            }
        }
        yp[n * p.ys[0] + c * p.ys[1] + oy * p.ys[2] + ox * p.ys[3]] = Px<T>::st(acc);
    }
}

// ------------------------------------------------------------------------------------------ channels-last (C fastest in x and y)
// One thread per (n, oy, ox, 16-byte group of channels): every tap is one aligned 128-bit load of VEC channels, a warp reads
// 512 contiguous bytes per tap, neighbouring outputs re-read their shared taps from L1/L2 - DRAM sees each input once.
template <typename T>
__global__ void __launch_bounds__(kThreads) k_upfirdn2d_cl(const UpfirdnParams p) {
    constexpr int VEC = 16 / (int)sizeof(T);
    __shared__ float s_w[kMaxTaps];
    const int taps = p.fH * p.fW;
    for (int i = threadIdx.x; i < taps; i += kThreads) {
        const int ky = i / p.fW, kx = i - ky * p.fW;
        const int sy = p.flip ? ky : p.fH - 1 - ky, sx = p.flip ? kx : p.fW - 1 - kx;
        s_w[i] = p.f[sy * p.fsh + sx * p.fsw] * p.gain;
    }
    __syncthreads();
    const T* xp = reinterpret_cast<const T*>(p.x);
    T* yp = reinterpret_cast<T*>(p.y);
    const unsigned cv = (unsigned)(p.C / VEC);
    const unsigned total = (unsigned)p.N * (unsigned)p.outH * (unsigned)p.outW * cv;       // < 2^31 (checked by the launcher)
    for (unsigned idx = blockIdx.x * kThreads + threadIdx.x; idx < total; idx += gridDim.x * kThreads) {
        unsigned r = idx;
        const int c = (int)(r % cv) * VEC; r /= cv;
        const int ox = (int)(r % (unsigned)p.outW); r /= (unsigned)p.outW;
        const int oy = (int)(r % (unsigned)p.outH);
        const int n = (int)(r / (unsigned)p.outH);
        const int ux0 = ox * p.downx - p.padx0, uy0 = oy * p.downy - p.pady0;
        const int kx0 = pos_mod(-ux0, p.upx), ky0 = pos_mod(-uy0, p.upy);
        const T* xi = xp + n * p.xs[0] + c;
        float acc[VEC];
#pragma unroll
        for (int e = 0; e < VEC; ++e) acc[e] = 0.f;
        for (int ky = ky0; ky < p.fH; ky += p.upy) {
            const int iy = (uy0 + ky) / p.upy;
            if (iy < 0 || iy >= p.inH) continue;
            for (int kx = kx0; kx < p.fW; kx += p.upx) {
                const int ix = (ux0 + kx) / p.upx;
                if (ix < 0 || ix >= p.inW) continue;
                const uint4 raw = __ldg(reinterpret_cast<const uint4*>(xi + iy * p.xs[2] + ix * p.xs[3]));
                const T* v = reinterpret_cast<const T*>(&raw);
                const float w = s_w[ky * p.fW + kx];
#pragma unroll
                for (int e = 0; e < VEC; ++e) acc[e] = fmaf(Px<T>::ld(v[e]), w, acc[e]);
            }
        }
        alignas(16) T out[VEC];
#pragma unroll
        for (int e = 0; e < VEC; ++e) out[e] = Px<T>::st(acc[e]);
        *reinterpret_cast<uint4*>(yp + n * p.ys[0] + c + oy * p.ys[2] + ox * p.ys[3]) = *reinterpret_cast<const uint4*>(out);
    }
}

template <typename T>
bool channels_last_ok(const UpfirdnParams& p) {
    constexpr int VEC = 16 / (int)sizeof(T);
    if (sizeof(T) > 4 || p.xs[1] != 1 || p.ys[1] != 1 || p.C % VEC != 0 || p.fH * p.fW > kMaxTaps) return false;
    const uintptr_t mask = 15;
    if ((reinterpret_cast<uintptr_t>(p.x) & mask) || (reinterpret_cast<uintptr_t>(p.y) & mask)) return false;
    for (int i : {0, 2, 3})
        if (p.xs[i] % VEC != 0 || p.ys[i] % VEC != 0) return false;
    return (long long)p.N * p.outH * p.outW * (p.C / VEC) < 0x7fffffffll;
}

template <typename T>
int launch_upfirdn2d(UpfirdnParams p, cudaStream_t stream) {
    using S = typename Px<T>::acc;
    static int n_sm = 0;
    if (!n_sm) {
        int dev = 0;
        P3D_CUDA_TRY(cudaGetDevice(&dev));
        P3D_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    {
        const int rc = try_launch_fast<T>(p, n_sm, stream);
        if (rc <= 0) return rc;
    }
    if (channels_last_ok<T>(p)) {
        const long long total = (long long)p.N * p.outH * p.outW * (p.C / (16 / (int)sizeof(T)));
        const long long blocks = (total + kThreads - 1) / kThreads;
        const int grid = (int)(blocks < (long long)n_sm * 32 ? blocks : (long long)n_sm * 32);
        k_upfirdn2d_cl<T><<<grid, kThreads, 0, stream>>>(p);
        P3D_LAUNCH_CHECK();
        return P3D_OK;
    }
    // footprint of a 64x16 output tile in input pixels (+1 for the floor of the first index)
    p.inTileW = (kTileW * p.downx + p.fW - 1 + p.upx - 1) / p.upx + 1;
    p.inTileH = (kTileH * p.downy + p.fH - 1 + p.upy - 1) / p.upy + 1;
    const size_t smem = ((size_t)p.fH * p.fW * 4 + 15 & ~(size_t)15) + (size_t)p.inTileW * p.inTileH * sizeof(S);
    const bool tiled_ok = p.xs[3] == 1 && smem <= 96 * 1024;
    if (tiled_ok) {
        p.tilesX = (p.outW + kTileW - 1) / kTileW;
        p.tilesY = (p.outH + kTileH - 1) / kTileH;
        const long long nc = (long long)p.N * p.C;
        dim3 grid((unsigned)(p.tilesX * p.tilesY), (unsigned)(nc < 32768 ? nc : 32768));
        if (smem > 48 * 1024) P3D_CUDA_TRY(cudaFuncSetAttribute(k_upfirdn2d_tiled<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_upfirdn2d_tiled<T><<<grid, kThreads, smem, stream>>>(p);
        P3D_LAUNCH_CHECK();
        return P3D_OK;
    }
    P3D_REQUIRE(p.fH * p.fW <= kMaxTaps, "filter too large for the strided kernel (%dx%d)", p.fH, p.fW);
    const long long total = (long long)p.N * p.C * p.outH * p.outW;
    const long long blocks = (total + kThreads - 1) / kThreads;
    const int grid = (int)(blocks < (long long)n_sm * 16 ? blocks : (long long)n_sm * 16);
    k_upfirdn2d_strided<T><<<grid, kThreads, 0, stream>>>(p, p.xs[1] == 1 ? 1 : 0);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_upfirdn2d(const void* x, const float* f, void* y, int32_t dtype, int32_t n, int32_t c, int32_t in_h,
                             int32_t in_w, const int64_t* x_stride, int32_t f_h, int32_t f_w, int64_t f_stride_h,
                             int64_t f_stride_w, int32_t out_h, int32_t out_w, const int64_t* y_stride, int32_t upx,
                             int32_t upy, int32_t downx, int32_t downy, int32_t padx0, int32_t padx1, int32_t pady0,
                             int32_t pady1, int32_t flip, float gain, void* stream) {
    P3D_REQUIRE(x && f && y && x_stride && y_stride, "null pointer");
    P3D_REQUIRE(n > 0 && c > 0 && in_h > 0 && in_w > 0, "x has zero size");
    P3D_REQUIRE(f_h >= 1 && f_w >= 1, "f must be at least 1x1");
    P3D_REQUIRE(upx >= 1 && upy >= 1, "upsampling factor must be at least 1");
    P3D_REQUIRE(downx >= 1 && downy >= 1, "downsampling factor must be at least 1");
    const int ow = (in_w * upx + padx0 + padx1 - f_w + downx) / downx;
    const int oh = (in_h * upy + pady0 + pady1 - f_h + downy) / downy;
    P3D_REQUIRE(ow >= 1 && oh >= 1, "output must be at least 1x1");
    P3D_REQUIRE(ow == out_w && oh == out_h, "output size mismatch: expected %dx%d, got %dx%d", oh, ow, out_h, out_w);
    UpfirdnParams p{};
    p.x = x; p.f = f; p.y = y; p.N = n; p.C = c; p.inH = in_h; p.inW = in_w; p.outH = out_h; p.outW = out_w; p.fH = f_h; p.fW = f_w;
    for (int i = 0; i < 4; ++i) { p.xs[i] = x_stride[i]; p.ys[i] = y_stride[i]; }
    p.fsh = f_stride_h; p.fsw = f_stride_w;
    p.upx = upx; p.upy = upy; p.downx = downx; p.downy = downy; p.padx0 = padx0; p.pady0 = pady0; p.flip = flip ? 1 : 0; p.gain = gain;
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case P3D_F32: return launch_upfirdn2d<float>(p, st);
        case P3D_F16: return launch_upfirdn2d<__half>(p, st);
        case P3D_BF16: return launch_upfirdn2d<__nv_bfloat16>(p, st);
        case P3D_F64: return launch_upfirdn2d<double>(p, st);
    }
    set_error("unsupported dtype %d", dtype);
    return P3D_EINVAL;
}
