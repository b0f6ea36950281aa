// PTX wrappers (mbarrier, Hopper wgmma) and the tri-plane gather / decoder helpers shared by the fused tensor-core
// kernels: render_fused_ws3.cu (the renderer) and decode_tc.cu (point / volume decode).
#pragma once
#include "render_device.cuh"

namespace p3d {
namespace fused {

using namespace dev;

constexpr int kSBO = 128;                        // byte distance between 8-row groups of a K-major no-swizzle wgmma operand tile
constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;

// ------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    // (not unrolled: ptxas otherwise replicates the body 16x at each of the ~50 call sites - half of the kernel's code size)
#pragma unroll 1
    for (int it = 0; it < (1 << 17); ++it) {             // ~20 us per try: the cap turns a protocol bug into a trap after ~2 s
        uint32_t ok;
        // the suspend-time hint lets a waiting warp sleep in hardware instead of polling: roles that run ahead of the
        // critical path must not steal issue slots from it
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(addr), "r"(parity), "r"(20000u) : "memory");
        if (ok) return;
    }
    asm volatile("trap;");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// ---- warpgroup MMA (sm_90a).  Operands in shared memory use the K-major, no-swizzle canonical layout of tile_off():
// 8-row x 16-byte core matrices, kSBO bytes between 8-row groups, `lbo` bytes between 8-column (16-byte) groups along K.
// A warpgroup's accumulator fragment of m64nN: element i of thread (warp w, lane l) is row 16 w + l / 4 + 8 ((i / 2) & 1),
// column 8 (i / 4) + 2 (l & 3) + (i & 1) - frag_row / frag_col below.  Columns [16 j, 16 j + 16) of it are, packed in pairs,
// the register A operand of k-step j of the next layer (the accumulator layout equals the A-fragment layout).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void fence_operands(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
    uint64_t d = (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo >> 4) & 0x3FFFu) << 32;
    return d;                                          // base offset 0, layout type 0 (no swizzle)
}
__device__ __forceinline__ int frag_row(int i, int lane, int w) { return 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }
__device__ __forceinline__ void wgmma_ss_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_rs_n8(float (&d)[4], const uint32_t* a, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %9, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0,%1,%2,%3}, {%4,%5,%6,%7}, %8, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_rs_n32(float (&d)[16], const uint32_t* a, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_rs_n48(float (&d)[24], const uint32_t* a, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, {%24,%25,%26,%27}, %28, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float e0, float e1) {
    uint32_t d;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(e1), "f"(e0));
    return d;
}
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    hi = pack_bf16x2(a, b);
    lo = pack_bf16x2(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
}
__device__ __forceinline__ void split1(float x, unsigned short& hi, unsigned short& lo) {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    hi = __bfloat16_as_ushort(h);
    lo = __bfloat16_as_ushort(__float2bfloat16_rn(x - __bfloat162float(h)));
}
__device__ __forceinline__ int tile_off(int row, int k, int lbo) { return (row >> 3) * kSBO + (k >> 3) * lbo + (row & 7) * 16 + (k & 7) * 2; }

// ------------------------------------------------------------------------------------------ gather
// Tap table: one 64 B record per row - chunk 0 = {o[0], o[1], o[2], flags}, chunk 1+p = the four bilinear weights of plane p
// (w00, w01, w10, w11; rows y, y+1 x columns x, x+1) - chunk c of row r stored at position c ^ ((r >> 1) & 3), which makes
// both the lane = row writes and the 8-rows-per-phase reads of the gather conflict-free.  o[p] is the element offset of texel
// (ya, xa) of plane p inside the view's tri-plane, with (ya, xa) CLAMPED to [0, H-2] x [0, W-2]: the 2 x 2 footprint that is
// loaded is always inside the plane, and the weights are moved onto the loaded texels (grid_sample's zero padding,
// renderer.py:68-81: a tap outside the plane contributes nothing, so its weight is dropped; a footprint that hangs over the
// edge by one texel keeps the weights of its inside texels).  flags bit p = plane p has a non-zero weight; the loads of a
// plane whose bit is clear are predicated off (its registers keep older, finite texel values that meet weights of 0).
__device__ __forceinline__ uint32_t tab_off(int row, int chunk) { return (uint32_t)(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4)); }

__device__ __forceinline__ bool plane_taps_rec(const Geom& g, int srow, int scol, int pbase, float ca, float cb, uint32_t& o, float4& w) {
    const float gx = __fmul_rn(ca, g.coord_scale), gy = __fmul_rn(cb, g.coord_scale);
    const float fx = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)g.W), 1.f), 0.5f);
    const float fy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)g.H), 1.f), 0.5f);
    const bool sane = (fx > -2.f) && (fx < (float)g.W + 1.f) && (fy > -2.f) && (fy < (float)g.H + 1.f);   // false for NaN too
    const float x0f = floorf(fx), y0f = floorf(fy);
    const float wx1 = fx - x0f, wy1 = fy - y0f;
    const float wx0 = 1.f - wx1, wy0 = 1.f - wy1;
    const int x0 = sane ? (int)x0f : -4, y0 = sane ? (int)y0f : -4;
    const int xa = min(max(x0, 0), g.W - 2), ya = min(max(y0, 0), g.H - 2);
    const int dx = x0 - xa, dy = y0 - ya;                     // 0 inside, -1 / +1: the footprint hangs over the low / high edge
    const float wl = dx == 0 ? wx0 : (dx == -1 ? wx1 : 0.f), wr = dx == 0 ? wx1 : (dx == 1 ? wx0 : 0.f);
    const float wt = dy == 0 ? wy0 : (dy == -1 ? wy1 : 0.f), wb = dy == 0 ? wy1 : (dy == 1 ? wy0 : 0.f);
    o = (uint32_t)(pbase + ya * srow + xa * scol);
    w = make_float4(wl * wt, wr * wt, wl * wb, wr * wb);
    return ((unsigned)(dx + 1) < 3u) && ((unsigned)(dy + 1) < 3u);
}
// four consecutive channels of one texel (16 B fp32 / 8 B bf16) at addr + IMM bytes, predicated; v keeps its old value when !pred
template <bool BF16, int IMM>
__device__ __forceinline__ void load_quad_p(float (&v)[4], const char* addr, bool pred) {
    if (BF16) {
        uint32_t r0 = 0, r1 = 0;
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p ld.global.nc.v2.u32 {%0,%1}, [%2+%4];\n\t}"
                     : "+r"(r0), "+r"(r1) : "l"(addr), "r"((int)pred), "n"(IMM));
        v[0] = __uint_as_float(r0 << 16); v[1] = __uint_as_float(r0 & 0xffff0000u); v[2] = __uint_as_float(r1 << 16); v[3] = __uint_as_float(r1 & 0xffff0000u);   // zeros when !pred
    } else {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t@p ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+%6];\n\t}"
                     : "+f"(v[0]), "+f"(v[1]), "+f"(v[2]), "+f"(v[3]) : "l"(addr), "r"((int)pred), "n"(IMM));
    }
}
__device__ __forceinline__ void fma4(float (&acc)[4], const float (&v)[4], float w) {
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = fmaf(v[j], w, acc[j]);
}

// ------------------------------------------------------------------------------------------ decoder (one warpgroup, 64 rows)
// Layer 1 of rows [64 half, 64 half + 64) of a 128-row A1 tile (bf16 hi / lo planes, K = 32, `lbo_a` bytes between K groups):
// D1 = A1 W1'^T as 3-pass split bf16 (hi hi + hi lo + lo hi), or hi hi alone when single_pass.
__device__ __forceinline__ void decoder_layer1(float (&d1)[32], uint32_t a1h, uint32_t a1l, int lbo_a, uint32_t w1h, uint32_t w1l,
                                               int lbo_w1, int half, bool single_pass) {
#pragma unroll
    for (int i = 0; i < 32; ++i) d1[i] = 0.f;
    const uint32_t ra = (uint32_t)half * 8 * kSBO;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        const uint32_t ao = ra + ks * 2 * lbo_a, bo = ks * 2 * lbo_w1;
        wgmma_ss_n64(d1, wgmma_desc(a1h + ao, lbo_a, kSBO), wgmma_desc(w1h + bo, lbo_w1, kSBO));
        if (!single_pass) {
            wgmma_ss_n64(d1, wgmma_desc(a1h + ao, lbo_a, kSBO), wgmma_desc(w1l + bo, lbo_w1, kSBO));
            wgmma_ss_n64(d1, wgmma_desc(a1l + ao, lbo_a, kSBO), wgmma_desc(w1h + bo, lbo_w1, kSBO));
        }
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_operands(d1);
}
// softplus2(D1 + b1') -> the bf16 hi / lo register A operands of layer 2 (k-step j = registers [4 j, 4 j + 4)).
// softplus2(x) = max(x, 0) + lg2(1 + 2^-|x|): no overflow for any x, so no threshold select.
__device__ __forceinline__ void decoder_hidden(const float (&d1)[32], const float* b1, int lane, uint32_t (&ah)[16], uint32_t (&al)[16]) {
#pragma unroll
    for (int m = 0; m < 16; ++m) {
        const int c = frag_col(2 * m, lane);
        const float x0 = d1[2 * m] + b1[c], x1 = d1[2 * m + 1] + b1[c + 1];
        const float h0 = fmaxf(x0, 0.f) + lg2_approx(1.f + ex2_approx(-fabsf(x0)));
        const float h1 = fmaxf(x1, 0.f) + lg2_approx(1.f + ex2_approx(-fabsf(x1)));
        split2(h0, h1, ah[m], al[m]);
    }
}
// Layer 2 against an N-row K-major weight tile (hi / lo planes, `lbo_w` bytes between K groups, K = 64).
template <int N>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t* a, uint64_t b_desc) {
    if constexpr (N == 8) wgmma_rs_n8(d, a, b_desc);
    else if constexpr (N == 32) wgmma_rs_n32(d, a, b_desc);
    else wgmma_rs_n48(d, a, b_desc);
}
template <int N>
__device__ __forceinline__ void decoder_layer2_issue(float (&d)[N / 2], const uint32_t (&ah)[16], const uint32_t (&al)[16], uint32_t wh,
                                                     uint32_t wl, int lbo_w, bool single_pass) {
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        const uint32_t bo = ks * 2 * lbo_w;
        wgmma_rs<N>(d, ah + 4 * ks, wgmma_desc(wh + bo, lbo_w, kSBO));
        if (!single_pass) {
            wgmma_rs<N>(d, ah + 4 * ks, wgmma_desc(wl + bo, lbo_w, kSBO));
            wgmma_rs<N>(d, al + 4 * ks, wgmma_desc(wh + bo, lbo_w, kSBO));
        }
    }
}

}  // namespace fused
}  // namespace p3d
