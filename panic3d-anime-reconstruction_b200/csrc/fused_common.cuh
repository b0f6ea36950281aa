// PTX wrappers (mbarrier, Hopper wgmma) and the tri-plane gather / decoder helpers shared by the fused tensor-core
// kernels: render_fused_ws3.cu (the renderer) and decode_tc.cu (point / volume decode).
#pragma once
#include <type_traits>
#include "render_device.cuh"

namespace p3d {
namespace fused {

using namespace dev;

constexpr int kSBO = 128;                        // byte distance between 8-row groups of a K-major no-swizzle wgmma operand tile
constexpr int kLBO_A1 = 2080, kLBO_W1 = 1024;    // byte distance between K groups of the A1 tile (128 x 32) / the W1' tile (64 x 32)
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
// per-warpgroup register budget (every thread of the warpgroup executes it); N a multiple of 8 in [24, 256]
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// ---- bulk copies (TMA without a tensor map): contiguous, 16-byte aligned, sizes a multiple of 16.
// shared -> global, tracked by the issuing thread's bulk groups: wait_read() frees the source, wait_all() completes the writes
__device__ __forceinline__ void bulk_store(void* gdst, uint32_t ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(ssrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// global -> shared, completes `bytes` of the transaction count of `bar`
__device__ __forceinline__ void bulk_load(uint32_t sdst, const void* gsrc, uint32_t bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(sdst), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// ---- L2 residency: per-instruction cache policies (createpolicy -> .L2::cache_hint operands) and line discards.  They
// change which lines L2 keeps, never a value that is read.
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// bulk_load under the L2 policy `pol`
__device__ __forceinline__ void bulk_load_hint(uint32_t sdst, const void* gsrc, uint32_t bytes, unsigned long long* bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(sdst), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(pol) : "memory");
}
// Invalidates the 128 B line at `p` (128-byte aligned) in L2 without writing it back: its contents become undefined.  A
// generic-proxy write; an async-proxy write of the same bytes that must follow it needs fence.proxy.async.global between.
__device__ __forceinline__ void l2_discard_line(const void* p) { asm volatile("discard.global.L2 [%0], 128;" ::"l"(p) : "memory"); }
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

// fp16 / tf32 forms (the modulated convolution, modconv.cu): both operands from shared memory, fp32 accumulation.
// A tf32 K-step (k8) spans the same 32 bytes of a K-major row as an fp16 one (k16), so one tile layout serves both.
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_f16_n8(float (&d)[4], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0,%1,%2,%3}, %4, %5, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_tf32_n8(float (&d)[4], uint64_t a_desc, uint64_t b_desc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0,%1,%2,%3}, %4, %5, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(a_desc), "l"(b_desc), "r"(1));
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

// ------------------------------------------------------------------------------------------ decoder weights
// The tensor-core decoder runs in base 2 (decoder_hidden's softplus2, the epilogues' ex2), so the weights are staged with the
// scale factors folded in:
//   W1' = W1 * gain * log2(e) / 3 (the 1/3 is the plane mean)       b1' = b1 * gain * log2(e)
//   colour rows 1..32 of W2: -W2 * gain                               colour biases: -b2 * gain * log2(e)
//   sigma row 0 of W2: W2 * gain * ln 2                               sigma bias: b2 * gain
// so a colour is rcp(1 + ex2(logit')) and sigma is the plain sum.  Weights are split into bf16 hi / lo K-major tiles.
template <int B>
__device__ __forceinline__ void put_weight(unsigned char (&tile)[2][B], int row, int k, int lbo, float w) {
    unsigned short hi, lo;
    split1(w, hi, lo);
    const int off = tile_off(row, k, lbo);
    *reinterpret_cast<unsigned short*>(tile[0] + off) = hi;
    *reinterpret_cast<unsigned short*>(tile[1] + off) = lo;
}
// W1' (64 x 32) and all biases; threads tid = 0 .. nthreads - 1 share the work
template <int B>
__device__ __forceinline__ void stage_w1_biases(const Geom& g, const float* w1, const float* b1, const float* b2, unsigned char (&sw1)[2][B],
                                                float* sb1, float* sb2c, float& sb2s, int tid, int nthreads) {
    for (int i = tid; i < kHidden * kC; i += nthreads) put_weight(sw1, i / kC, i % kC, kLBO_W1, __fmul_rn(w1[i], g.w1_gain) * (kLog2e / 3.f));
    if (tid < kHidden) sb1[tid] = __fmul_rn(b1[tid], g.b1_gain) * kLog2e;
    if (tid < kRgb) sb2c[tid] = -__fmul_rn(b2[tid + 1], g.b2_gain) * kLog2e;
    if (tid == 0) sb2s = __fmul_rn(b2[0], g.b2_gain);
}
// Layer 2 as one N = 48 wgmma tile: rows 0..31 the colour rows (W2 rows 1..32), row 32 sigma (W2 row 0), rows 33..47 zero -
// so the accumulator holds the 32 colour logits in fragment elements 0..15 and sigma in column 32 (elements 16, 18 of the
// threads with lane % 4 == 0).
constexpr int kD2Cols = 48, kLBO_W2 = 768;
__device__ __forceinline__ int w2_row_n48(int n) { return n < kRgb ? n + 1 : (n == kRgb ? 0 : -1); }
// rows [0, rows) of a layer-2 weight tile (K = 64): tile row n holds W2 row w2_row(n) (0 = sigma, 1..32 = colours, -1 = zeros)
template <int B, class RowMap>
__device__ __forceinline__ void stage_w2(const Geom& g, const float* w2, unsigned char (&tile)[2][B], int rows, int lbo, RowMap w2_row,
                                         int tid, int nthreads) {
    for (int i = tid; i < rows * kHidden; i += nthreads) {
        const int n = i / kHidden, k = i % kHidden, r = w2_row(n);
        float w = 0.f;
        if (r >= 0) {
            const float wg = __fmul_rn(w2[r * kHidden + k], g.w2_gain);
            w = r == 0 ? wg * kLn2 : -wg;
        }
        put_weight(tile, n, k, lbo, w);
    }
}

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

__device__ __forceinline__ bool plane_taps_rec(const Geom& g, int srow, int scol, int pbase, float2 c, uint32_t& o, float4& w) {
    const Footprint f = bilinear_footprint(g, c.x, c.y);
    const int xa = min(max(f.x0, 0), g.W - 2), ya = min(max(f.y0, 0), g.H - 2);
    const int dx = f.x0 - xa, dy = f.y0 - ya;                 // 0 inside, -1 / +1: the footprint hangs over the low / high edge
    const float wl = dx == 0 ? f.wx0 : (dx == -1 ? f.wx1 : 0.f), wr = dx == 0 ? f.wx1 : (dx == 1 ? f.wx0 : 0.f);
    const float wt = dy == 0 ? f.wy0 : (dy == -1 ? f.wy1 : 0.f), wb = dy == 0 ? f.wy1 : (dy == 1 ? f.wy0 : 0.f);
    o = (uint32_t)(pbase + ya * srow + xa * scol);
    w = make_float4(wl * wt, wr * wt, wl * wb, wr * wb);
    return ((unsigned)(dx + 1) < 3u) && ((unsigned)(dy + 1) < 3u);
}
// tap-table row `row` for the point (x, y, z); `view` goes to bits 8.. of the flags word (0 when the caller knows the view)
__device__ __forceinline__ void write_tap_row(unsigned char* tab, int row, const Geom& g, int srow, int scol, int splane, float x, float y,
                                              float z, uint32_t view) {
    uint32_t o0, o1, o2;
    float4 w0, w1, w2;
    const bool f0 = plane_taps_rec(g, srow, scol, 0, plane_coords(g, 0, x, y, z), o0, w0);
    const bool f1 = plane_taps_rec(g, srow, scol, splane, plane_coords(g, 1, x, y, z), o1, w1);
    const bool f2 = plane_taps_rec(g, srow, scol, 2 * splane, plane_coords(g, 2, x, y, z), o2, w2);
    *reinterpret_cast<uint4*>(tab + tab_off(row, 0)) = make_uint4(o0, o1, o2, (f0 ? 1u : 0u) | (f1 ? 2u : 0u) | (f2 ? 4u : 0u) | (view << 8));
    *reinterpret_cast<float4*>(tab + tab_off(row, 1)) = w0;
    *reinterpret_cast<float4*>(tab + tab_off(row, 2)) = w1;
    *reinterpret_cast<float4*>(tab + tab_off(row, 3)) = w2;
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
// The tap table of one gather warp -> rows [32 wt, 32 wt + 32) of an A1 stage (bf16 hi / lo planes a1h / a1l).  8 rounds of 4
// rows: lane (sub, qd) loads channels [4 qd, 4 qd + 4) of the 12 taps of row 4 round + sub - twelve 128-bit loads in flight
// per lane, each warp-wide load covers four whole 128 B texels (one L1 wavefront per texel) - and lerps them with one FMA
// chain.  A row's view starts at `planes` + (flags >> 8) * view_bytes.  SCOL != 0 is the texel stride in elements, which
// makes the x + 1 texel an immediate offset.  v: the caller's texel registers, zeroed once (a plane whose loads are predicated
// off keeps older, finite values, which meet weights of 0).
template <bool BF16, int SCOL>
__device__ __forceinline__ void gather_a1(const unsigned char* tab, const char* planes, long long view_bytes, long long srowB, long long scolB,
                                          float (&v)[12][4], unsigned char* a1h, unsigned char* a1l, int wt, int lane) {
    constexpr int kEsz = BF16 ? 2 : 4;
    constexpr int kImmX4 = SCOL * kEsz;
    const int sub = lane >> 3, qd = lane & 7;
    const char* pq = planes + (long long)(4 * qd) * kEsz;
#pragma unroll 1
    for (int round = 0; round < 8; ++round) {
        const int lrow = round * 4 + sub;
        const uint4 c0 = *reinterpret_cast<const uint4*>(tab + tab_off(lrow, 0));
        const char* vq4 = pq + (long long)(c0.w >> 8) * view_bytes;
        const uint32_t o[3] = {c0.x, c0.y, c0.z};
#pragma unroll
        for (int p = 0; p < 3; ++p) {
            const bool pr = c0.w & (1u << p);
            const char* b = vq4 + (unsigned long long)o[p] * kEsz;
            load_quad_p<BF16, 0>(v[4 * p], b, pr);
            if (SCOL) load_quad_p<BF16, kImmX4>(v[4 * p + 1], b, pr); else load_quad_p<BF16, 0>(v[4 * p + 1], b + scolB, pr);
            load_quad_p<BF16, 0>(v[4 * p + 2], b + srowB, pr);
            if (SCOL) load_quad_p<BF16, kImmX4>(v[4 * p + 3], b + srowB, pr); else load_quad_p<BF16, 0>(v[4 * p + 3], b + srowB + scolB, pr);
        }
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int p = 0; p < 3; ++p) {
            const float4 w = *reinterpret_cast<const float4*>(tab + tab_off(lrow, 1 + p));
            fma4(acc, v[4 * p], w.x); fma4(acc, v[4 * p + 1], w.y); fma4(acc, v[4 * p + 2], w.z); fma4(acc, v[4 * p + 3], w.w);
        }
        uint32_t h[2], l[2];
        split2(acc[0], acc[1], h[0], l[0]);
        split2(acc[2], acc[3], h[1], l[1]);
        const int trow = wt * 32 + lrow;
        const int off = (trow >> 3) * kSBO + (qd >> 1) * kLBO_A1 + (trow & 7) * 16 + (qd & 1) * 8;
        *reinterpret_cast<uint2*>(a1h + off) = make_uint2(h[0], h[1]);
        *reinterpret_cast<uint2*>(a1l + off) = make_uint2(l[0], l[1]);
    }
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

// ------------------------------------------------------------------------------------------ host side of both fused kernels
// SM count of the current device, read once: both kernels run a persistent grid of at most one CTA per SM
inline int sm_count(int* n) {
    static int n_sm = 0;
    if (!n_sm) {
        int dev = 0;
        P3D_CUDA_TRY(cudaGetDevice(&dev));
        P3D_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    *n = n_sm;
    return P3D_OK;
}
// cudaFuncAttributePreferredSharedMemoryCarveout for a kernel with `smem` bytes of dynamic shared memory: the share, in percent
// of the SM's shared-memory maximum, that `smem` and the per-CTA reservation take, rounded down.  The driver rounds the hint
// up to a carve-out that holds the CTA, so this selects the smallest one that does and leaves the rest of the SM's
// 256 KB to L1, instead of leaving the split to the driver.
inline int smem_carveout_percent(size_t smem, int* pct) {
    static int max_sm = 0, reserved = 0;
    if (!max_sm) {
        int dev = 0;
        P3D_CUDA_TRY(cudaGetDevice(&dev));
        P3D_CUDA_TRY(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev));
        P3D_CUDA_TRY(cudaDeviceGetAttribute(&max_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
    }
    const long long share = 100ll * ((long long)smem + reserved) / max_sm;
    *pct = (int)(share < 1 ? 1 : (share > 100 ? 100 : share));
    return P3D_OK;
}
// The texel stride the gather takes as a template argument (SCOL): kC (the layout pre-pass: one plane's texels contiguous),
// 3 kC (a (N,96,H,W) channels_last backbone output consumed zero-copy) or 0 (any other stride, read at run time).
// pick(std::integral_constant<int, SCOL>) returns the kernel instantiation.
template <class Pick>
auto with_texel_stride(const Geom& g, Pick pick) {
    if (g.stride_col == kC) return pick(std::integral_constant<int, kC>{});
    if (g.stride_col == 3 * kC) return pick(std::integral_constant<int, 3 * kC>{});
    return pick(std::integral_constant<int, 0>{});
}
// The tap table holds 32-bit element offsets inside one view's tri-plane and 2 x 2 footprints clamped into the plane
inline bool tap_offsets_fit(const Geom& g) {
    const long long span = 2 * g.stride_plane + (long long)(g.H - 1) * g.stride_row + (long long)(g.W - 1) * g.stride_col + kC;
    return g.H >= 2 && g.W >= 2 && g.stride_plane >= 0 && g.stride_row >= 0 && g.stride_col >= 0 && span < (1ll << 31);
}

}  // namespace p3d
