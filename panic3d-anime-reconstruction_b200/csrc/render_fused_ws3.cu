// The fused renderer: warp-specialised, pipeline depth 3 - THREE ray groups in flight.
//
//   passes C(0) C(1) | F(0) C(2) | F(1) C(3) | ... | F(N-2) F(N-1)          (C = 3 coarse tiles, F = 3 importance tiles)
//
// A tile's colour sigmoids wait for the group's compositing weights (omega), which exist only after its fine pass.  They are
// staged in global memory, in this CTA's own slice of the workspace colour buffers (see colour_area: coarse areas
// CA[n % 3] and one fine area FA, 4 x 48 KB per CTA, ~25 MB on 132 SMs).  The areas are rewritten every few groups, so
// their footprint fits the 50 MB L2, but they share it with the streamed tri-plane gather; how much of the round trip is
// served by L2 rather than HBM has not been measured.  Only
// the COARSE colours of a group have to wait through a whole fine pass; the fine ones are consumed right after the group's
// merge, so all groups share one fine area.  With F(n) followed by C(n+2):
//   * importance(n) has two passes of slack (F(n-1), C(n+1)) before the gather of F(n) needs its depths;
//   * merge(n) + omega(n) run on the RAY warps while the decoder handles the three tiles of C(n+2); colours(n) runs at the
//     top of F(n+1)'s first tile - the last point before F(n+1) overwrites the fine area (C(n+3), which reuses
//     CA[n % 3], comes later still);
//   * the per-group state ring stays 4 deep (groups n .. n+3 alive), the omega slot 2 deep.
//
//   warps  0-11  GATHER    three teams of four warps; team j takes tiles j, j+3, ... of the tile sequence
//   warps 12-19  DECODER   two warpgroups, one per 64-row half of every tile: layer 1 (wgmma, A1 and W1 from shared memory)
//                          -> softplus2 in registers -> layer 2 (wgmma, A from the registers): colour sigmoids -> colour area,
//                          sigma -> group state; colour reduction of a group once its omega is ready
//   warps 20-23  RAY       a warp per ray: importance sampling after a group's coarse pass, merge / transmittance /
//                          omega and the per-ray outputs after its fine pass
#include <stdlib.h>
#include "fused_common.cuh"

namespace p3d {

namespace {

using namespace dev;
using namespace fused;

constexpr int kGW = 12, kEW = 8, kRW = 4, kTeams = 3;   // 24 warps = 6 warpgroups -> 80 registers per thread
constexpr int kWarpsWS = kGW + kEW + kRW;
constexpr int kThreadsWS = kWarpsWS * 32;        // 768
constexpr int kNA = 4;                           // A1 ring depth
constexpr int kStates = 4;                       // per-group state ring
constexpr int kRowsG = 384;                      // rows per pass per group

constexpr int kLBO_A1 = 2080, kLBO_W1 = 1024, kLBO_W2C = 512, kLBO_W2S = 256;


struct GroupState {                               // written by G (t_c, crop), E (sg_*), R (t_f)
    float t_c[kRowsG], sg_c[kRowsG], t_f[kRowsG], sg_f[kRowsG];
    unsigned char crop[2][kRowsG];
};
struct SlotState {                                // written by R (composite), read by E (colours)
    float om[2 * kRowsG];                         // omega per merged position, [ray][2S]
    unsigned short pos[2 * kRowsG];                          // merged position of coarse rows [0,384) and fine rows [384,768)
    float acc[8][kRgb];
    float back[8];
};

struct __align__(1024) WsSmem {
    unsigned char a1[kNA][2][4 * kLBO_A1];
    unsigned char w1[2][4096], w2c[2][4096], w2s[2][2048];
    float b1[kHidden], b2c[kRgb], b2s, pad0[3];
    uint4 tab[kGW][32][4];                        // tap table of a gather warp's 32 rows (see "gather" below)
    GroupState st[kStates];
    SlotState slot[2];
    float rscratch[kRW][768];                      // private scratch of each ray warp (importance / merge)
    unsigned long long a1_full[kNA], a1_empty[kNA];
    unsigned long long fine_ready[kStates], state_free[kStates];
    unsigned long long sigc_ready[kStates], sigf_ready[kStates], omega_ready[2];   // E -> R (sigma in smem), R -> E (omega)
};

static_assert(sizeof(WsSmem) + 1024 <= 232448, "WsSmem + alignment slack exceeds the 227 KB a CTA can opt into");

struct WsArgs {
    Geom g;
    const void* planes;
    const float *w1, *b1, *w2, *b2;
    const float *ro, *rd, *u_c, *u_f;
    const float *ray_t0, *ray_t1;
    unsigned int* bounds;
    float *out_rgb, *out_depth, *out_wsum, *out_xyz;
    float *col_c, *col_f;            // workspace colour buffers: this kernel's colour areas (colour_area)
    long long R;
    int n_groups, single_pass;
    int srow, scol, splane;
    float sigma_cull;
    unsigned long long* timing;      // optional [16] cycle counters (debug: P3D_WS_TIMING=1), nullptr = off
};

// cycle accounting of one gather warp and one epilogue warp of CTA 0 (debug aid, off by default)
struct Tick {
    unsigned long long* dst; long long t0; bool on;
    __device__ Tick(unsigned long long* d, bool enable) : dst(d), t0(0), on(enable && d != nullptr) { if (on) t0 = clock64(); }
    __device__ void lap(int slot) { if (on) { const long long t1 = clock64(); atomicAdd(dst + slot, (unsigned long long)(t1 - t0)); t0 = t1; } }
};

// pass j of a CTA with N groups:  C(0) C(1) | F(0) C(2) | F(1) C(3) | ... | F(N-2) F(N-1)   (N == 1: C(0) F(0))
struct PassDesc { int n, pass; };
__device__ __forceinline__ PassDesc pass_at(int j, int N) {
    if (j == 0) return PassDesc{0, 0};
    if (N == 1) return PassDesc{0, 1};
    if (j == 1) return PassDesc{1, 0};
    const int k = j - 2, body = 2 * (N - 2);
    if (k < body) return (k & 1) ? PassDesc{(k >> 1) + 2, 0} : PassDesc{k >> 1, 1};
    return PassDesc{N - 2 + (k - body), 1};
}
struct TileDesc { int n, pass, k; };
__device__ __forceinline__ TileDesc tile_at(int q, int N) {
    const int j = q / 3;
    const PassDesc p = pass_at(j, N);
    return TileDesc{p.n, p.pass, q - 3 * j};
}

// ------------------------------------------------------------------------------------------
template <bool BF16, int S, int SCOL>
__global__ void __launch_bounds__(kThreadsWS, 1) k_render_ws3(const WsArgs a) {
    constexpr int Sf = S, L = 2 * S;
    constexpr int RPT = S / 3;                   // rows per ray per tile (32 or 16)
    constexpr int GR = 128 / RPT;                // rays per group (4 or 8)
    extern __shared__ unsigned char smem_raw[];
    WsSmem& sm = *reinterpret_cast<WsSmem*>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));   // keeps the shared address space
    const Geom& g = a.g;
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // provably warp-uniform
    const int n_my = (a.n_groups - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // groups of this CTA
    const int T = 6 * n_my;

    // ---------------- setup
    if (tid == 0) {
        for (int i = 0; i < kNA; ++i) { mbar_init(&sm.a1_full[i], 4); mbar_init(&sm.a1_empty[i], kEW); }
        for (int i = 0; i < kStates; ++i) {
            mbar_init(&sm.fine_ready[i], kRW); mbar_init(&sm.state_free[i], 1);
            mbar_init(&sm.sigc_ready[i], kEW); mbar_init(&sm.sigf_ready[i], kEW);
        }
        mbar_init(&sm.omega_ready[0], kRW); mbar_init(&sm.omega_ready[1], kRW);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < kHidden * kC; i += kThreadsWS) {            // W1' = W1 * gain * log2(e)   (64 x 32)
        const int n = i / kC, k = i % kC;
        unsigned short hi, lo;
        split1(__fmul_rn(a.w1[i], g.w1_gain) * (kLog2e / 3.f), hi, lo);      // the 1/3 is the plane mean
        const int off = tile_off(n, k, kLBO_W1);
        *reinterpret_cast<unsigned short*>(sm.w1[0] + off) = hi;
        *reinterpret_cast<unsigned short*>(sm.w1[1] + off) = lo;
    }
    for (int i = tid; i < kRgb * kHidden; i += kThreadsWS) {          // colour rows 1..32 of W2, negated   (32 x 64)
        const int n = i / kHidden, k = i % kHidden;
        unsigned short hi, lo;
        split1(-__fmul_rn(a.w2[(n + 1) * kHidden + k], g.w2_gain), hi, lo);
        const int off = tile_off(n, k, kLBO_W2C);
        *reinterpret_cast<unsigned short*>(sm.w2c[0] + off) = hi;
        *reinterpret_cast<unsigned short*>(sm.w2c[1] + off) = lo;
    }
    for (int i = tid; i < 16 * kHidden; i += kThreadsWS) {            // sigma row 0 of W2 (* ln2) + 15 zero rows (16 x 64)
        const int n = i / kHidden, k = i % kHidden;
        unsigned short hi = 0, lo = 0;
        if (n == 0) split1(__fmul_rn(a.w2[k], g.w2_gain) * kLn2, hi, lo);
        const int off = tile_off(n, k, kLBO_W2S);
        *reinterpret_cast<unsigned short*>(sm.w2s[0] + off) = hi;
        *reinterpret_cast<unsigned short*>(sm.w2s[1] + off) = lo;
    }
    if (tid < kHidden) sm.b1[tid] = __fmul_rn(a.b1[tid], g.b1_gain) * kLog2e;
    if (tid < kRgb) sm.b2c[tid] = -__fmul_rn(a.b2[tid + 1], g.b2_gain) * kLog2e;
    if (tid == 0) sm.b2s = __fmul_rn(a.b2[0], g.b2_gain);
    fence_proxy_async();
    __syncthreads();

    if (warp < kGW) {
        // =========================================================================== GATHER
        const int gw = warp, team = gw >> 2, wt = gw & 3;
        Tick tk_(a.timing, blockIdx.x == 0 && gw == 0 && lane == 0);
        constexpr int kEsz = BF16 ? 2 : 4;
        const long long scolB = (long long)a.scol * kEsz, srowB = (long long)a.srow * kEsz;
        unsigned char* tab = reinterpret_cast<unsigned char*>(sm.tab[gw]);
        float v[6][8];
#pragma unroll
        for (int k = 0; k < 6; ++k)
#pragma unroll
            for (int c = 0; c < 8; ++c) v[k][c] = 0.f;
        int it = 0;
        for (int q = 0; q < T; ++q) {
            const TileDesc td = tile_at(q, n_my);
            const int my_it = it++;
            if (my_it % kTeams != team) continue;
            const int grp = (int)blockIdx.x + td.n * (int)gridDim.x;
            const long long ray0 = (long long)grp * GR;
            GroupState& st = sm.st[td.n & 3];
            tk_.lap(0);
            if (td.pass == 0) mbar_wait(&sm.state_free[td.n & 3], ((td.n >> 2) & 1) ^ 1);
            else mbar_wait(&sm.fine_ready[td.n & 3], (td.n >> 2) & 1);
            tk_.lap(1);                                                   // [1] wait state_free / fine_ready
            const int view = (int)(ray0 / g.M);
            // ---- tap table of this warp's 32 rows: lane = row
            {
                const int trow = wt * 32 + lane;
                const int rl = trow / RPT, s = td.k * RPT + (trow - rl * RPT);
                const int srow = rl * S + s;                               // row in the per-group state arrays
                const long long ray = ray0 + rl;
                const bool live = ray < a.R;
                float tval;
                if (td.pass == 0) {
                    float u = 0.f;
                    if (live) {
                        const long long gidx = ray * S + s;
                        u = a.u_c ? a.u_c[gidx] : philox_uniform(g.seed, (uint64_t)gidx, 0u);
                    }
                    float t0 = 0.f, t1 = 0.f;
                    if (g.ray_mode == P3D_RAYS_AUTOBOX && live) {
                        t0 = a.ray_t0[ray]; t1 = a.ray_t1[ray];
                        if (!(t1 > t0) && a.bounds[4]) { t0 = ordered_to_float(a.bounds[2]); t1 = ordered_to_float(a.bounds[3]); }
                    }
                    tval = coarse_depth(g, s, u, t0, t1);
                    st.t_c[srow] = tval;
                } else {
                    tval = st.t_f[srow];
                }
                float px = 1e30f, py = 1e30f, pz = 1e30f;
                if (live) {
                    const float* o = a.ro + ray * 3;
                    const float* d = a.rd + ray * 3;
                    px = __fadd_rn(o[0], __fmul_rn(tval, d[0]));
                    py = __fadd_rn(o[1], __fmul_rn(tval, d[1]));
                    pz = __fadd_rn(o[2], __fmul_rn(tval, d[2]));
                }
                const bool pm = g.plane_mode == P3D_PLANES_PANIC3D;
                uint32_t o0, o1, o2;
                float4 w0, w1, w2;
                const bool f0 = plane_taps_rec(g, a.srow, a.scol, 0, px, py, o0, w0);
                const bool f1 = plane_taps_rec(g, a.srow, a.scol, a.splane, px, pz, o1, w1);
                const bool f2 = plane_taps_rec(g, a.srow, a.scol, 2 * a.splane, pm ? py : pz, pm ? pz : px, o2, w2);
                *reinterpret_cast<uint4*>(tab + tab_off(lane, 0)) = make_uint4(o0, o1, o2, (f0 ? 1u : 0u) | (f1 ? 2u : 0u) | (f2 ? 4u : 0u));
                *reinterpret_cast<float4*>(tab + tab_off(lane, 1)) = w0;
                *reinterpret_cast<float4*>(tab + tab_off(lane, 2)) = w1;
                *reinterpret_cast<float4*>(tab + tab_off(lane, 3)) = w2;
                st.crop[td.pass][srow] = (g.crop_on && !((fabsf(px) <= g.crop_limit) && (fabsf(pz) <= g.crop_limit))) ? 1 : 0;
            }
            __syncwarp();
            const int stage = my_it % kNA;
            mbar_wait(&sm.a1_empty[stage], ((my_it / kNA) & 1) ^ 1);
            tk_.lap(2);                                                   // [2] taps + wait a1_empty
            unsigned char* a1h = sm.a1[stage][0];
            unsigned char* a1l = sm.a1[stage][1];
            {
                // ---- gather: 8 rounds of 4 rows; lane (sub, qd) loads channels [4 qd, 4 qd + 4) of the 12 taps of row 4 round + sub:
                //      twelve 128-bit loads in flight per lane, each warp-wide load covers four whole 128 B texels (one L1
                //      wavefront per texel)
                const int sub = lane >> 3, qd = lane & 7;
                const char* vq4 = reinterpret_cast<const char*>(a.planes) + ((long long)view * g.stride_view + 4 * qd) * kEsz;
                constexpr int kImmX4 = SCOL * kEsz;
                float (*v4)[4] = reinterpret_cast<float (*)[4]>(&v[0][0]);           // the same 48 registers, as 12 x 4
#pragma unroll 1
                for (int round = 0; round < 8; ++round) {
                    const int lrow = round * 4 + sub;
                    const uint4 c0 = *reinterpret_cast<const uint4*>(tab + tab_off(lrow, 0));
                    const bool p0 = c0.w & 1u, p1 = c0.w & 2u, p2 = c0.w & 4u;
                    const char* b0 = vq4 + (unsigned long long)c0.x * kEsz;
                    const char* b1 = vq4 + (unsigned long long)c0.y * kEsz;
                    const char* b2 = vq4 + (unsigned long long)c0.z * kEsz;
#define P3D_ROW1(base, rbase) (base + srowB)
#define P3D_LD4(k, base, rbase, pr)                                                                                  \
                    load_quad_p<BF16, 0>(v4[k], base, pr);                                                            \
                    if (SCOL) load_quad_p<BF16, kImmX4>(v4[k + 1], base, pr); else load_quad_p<BF16, 0>(v4[k + 1], base + scolB, pr); \
                    load_quad_p<BF16, 0>(v4[k + 2], P3D_ROW1(base, rbase), pr);                                       \
                    if (SCOL) load_quad_p<BF16, kImmX4>(v4[k + 3], P3D_ROW1(base, rbase), pr); else load_quad_p<BF16, 0>(v4[k + 3], P3D_ROW1(base, rbase) + scolB, pr);
                    P3D_LD4(0, b0, r0, p0)
                    P3D_LD4(4, b1, r1, p1)
                    P3D_LD4(8, b2, r2, p2)
#undef P3D_LD4
#undef P3D_ROW1
                    const float4 w0 = *reinterpret_cast<const float4*>(tab + tab_off(lrow, 1));
                    const float4 w1 = *reinterpret_cast<const float4*>(tab + tab_off(lrow, 2));
                    const float4 w2 = *reinterpret_cast<const float4*>(tab + tab_off(lrow, 3));
                    float acc[4] = {0.f, 0.f, 0.f, 0.f};
                    fma4(acc, v4[0], w0.x); fma4(acc, v4[1], w0.y); fma4(acc, v4[2], w0.z); fma4(acc, v4[3], w0.w);
                    fma4(acc, v4[4], w1.x); fma4(acc, v4[5], w1.y); fma4(acc, v4[6], w1.z); fma4(acc, v4[7], w1.w);
                    fma4(acc, v4[8], w2.x); fma4(acc, v4[9], w2.y); fma4(acc, v4[10], w2.z); fma4(acc, v4[11], w2.w);
                    uint32_t h[2], l[2];
                    split2(acc[0], acc[1], h[0], l[0]);
                    split2(acc[2], acc[3], h[1], l[1]);
                    const int trow = wt * 32 + lrow;
                    const int off = (trow >> 3) * kSBO + (qd >> 1) * kLBO_A1 + (trow & 7) * 16 + (qd & 1) * 8;
                    *reinterpret_cast<uint2*>(a1h + off) = make_uint2(h[0], h[1]);
                    *reinterpret_cast<uint2*>(a1l + off) = make_uint2(l[0], l[1]);
                }
            }
            fence_proxy_async();
            __syncwarp();                                                   // also: the tap table is rewritten by the next tile
            if (lane == 0) mbar_arrive(&sm.a1_full[stage]);
            tk_.lap(3);                                                   // [3] gather of one tile (32 rows)
        }
    } else if (warp < kGW + kEW) {
        // =========================================================================== DECODER
        const int e = warp - kGW, quarter = e & 3, chunk = e >> 2;      // chunk = warpgroup = 64-row half of a tile
        const int etid = tid - kGW * 32;                                  // 0..255 inside the decoder group
        // this CTA's colour area of (group n, pass): 384 rows x 32 sigmoids, row = 128 k + row of tile k.  Areas are slices of
        // the workspace colour buffers that belong to this CTA's own first two groups (coarse and fine buffer each), so they
        // exist whenever they are used: CA[0..2] = slices 0..2, FA = slice 3 (slice 1 when the CTA has a single group)
        auto colour_area = [&](int n, int pass) -> float* {
            const int j = pass == 0 ? n % 3 : (n_my >= 2 ? 3 : 1);
            return ((j & 1) ? a.col_f : a.col_c) + ((long long)blockIdx.x + (long long)(j >> 1) * gridDim.x) * (kRowsG * kRgb);
        };
        auto ebar = [] { asm volatile("bar.sync 1, 256;" ::: "memory"); };   // the eight decoder warps
        auto colours = [&](int n) {                                        // sum_j omega_j * rgb_j for group n
            const int slot_i = n & 1;
            SlotState& sl = sm.slot[slot_i];
            mbar_wait(&sm.omega_ready[slot_i], (n >> 1) & 1);              // omega / pos / back of group n (ray warps)
            const int grp = (int)blockIdx.x + n * (int)gridDim.x;
            const long long ray0 = (long long)grp * GR;
            // A warp's 32 rows are the same ray(s) in each of its three tiles, so the per-tile column sums are first added
            // up in a register and published once: every (ray, channel) cell of sl.acc then receives exactly two
            // shared-memory adds (one per chunk), whose order cannot change the rounded sum - the kernel is
            // bit-reproducible run to run and independent of how the rays are batched.
            float part[2] = {0.f, 0.f};
            const int rl_first = (quarter * 32) / RPT;
            for (int i = 0; i < 3; ++i) {
                const int tile6 = chunk + 2 * i;                           // this warp's tiles: {0,2,4} or {1,3,5}
                const int pass = tile6 / 3, k = tile6 - pass * 3;
                const int trow = quarter * 32 + lane;
                const int rl = trow / RPT, s = k * RPT + (trow - rl * RPT);
                const bool live = ray0 + rl < a.R;
                const float om = live ? sl.om[rl * L + sl.pos[pass * kRowsG + rl * S + s]] : 0.f;
                const float ca = g.force_sigmoid ? om : 1.002f * om, cb = g.force_sigmoid ? 0.f : -0.001f * om;
                float v[32];
                const float4* src = reinterpret_cast<const float4*>(colour_area(n, pass) + (k * 128 + trow) * kRgb);
#pragma unroll
                for (int c4 = 0; c4 < 8; ++c4) {
                    const float4 q4 = src[c4];
                    v[4 * c4] = q4.x; v[4 * c4 + 1] = q4.y; v[4 * c4 + 2] = q4.z; v[4 * c4 + 3] = q4.w;
                }
#pragma unroll
                for (int c = 0; c < kRgb; ++c) v[c] = fmaf(v[c], ca, cb);
#pragma unroll
                for (int t2 = 0; t2 < 32 / RPT; ++t2) {
                    const int target = rl_first + t2;
                    float r[32];
#pragma unroll
                    for (int c = 0; c < 32; ++c) r[c] = (RPT == 32 || rl == target) ? v[c] : 0.f;
#pragma unroll
                    for (int off = 16; off >= 1; off >>= 1) {
                        const bool up = (lane & off) != 0;
#pragma unroll
                        for (int j = 0; j < off; ++j) {
                            const float send = up ? r[j] : r[j + off];
                            const float keep = up ? r[j + off] : r[j];
                            r[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                        }
                    }
                    part[t2] += r[0];
                }
            }
#pragma unroll
            for (int t2 = 0; t2 < 32 / RPT; ++t2) atomicAdd(&sl.acc[rl_first + t2][lane], part[t2]);
            ebar();                                                        // all eight decoder warps (also: the areas are read)
            if (etid < GR * kRgb) {
                const int rl = etid >> 5, c = etid & 31;
                const long long ray = ray0 + rl;
                if (ray < a.R) a.out_rgb[ray * kRgb + c] = __fsub_rn(__fmul_rn(__fadd_rn(sl.acc[rl][c], sl.back[rl]), 2.f), 1.f);
            }
            ebar();
            if (etid == 0) mbar_arrive(&sm.state_free[n & 3]);
        };

        // colours(n) needs omega from the ray warps; it runs at the top of the first tile of F(n+1) - three tiles (C(n+2))
        // after the group's last sigma - which is also the last point before F(n+1) overwrites the fine area.
        const uint32_t w1h = smem_u32(sm.w1[0]), w1l = smem_u32(sm.w1[1]);
        const uint32_t w2ch = smem_u32(sm.w2c[0]), w2cl = smem_u32(sm.w2c[1]), w2sh = smem_u32(sm.w2s[0]), w2sl = smem_u32(sm.w2s[1]);
        Tick tk_(a.timing, blockIdx.x == 0 && e == 0 && lane == 0);
        for (int it = 0; it < T; ++it) {
            const TileDesc td = tile_at(it, n_my);
            tk_.lap(4);
            if (td.pass == 1 && td.k == 0 && td.n >= 1) { colours(td.n - 1); tk_.lap(11); }   // [11] colours (incl. wait for omega)
            const int stage = it % kNA;
            mbar_wait(&sm.a1_full[stage], (it / kNA) & 1);
            tk_.lap(5);                                                   // [5] wait a1_full
            float d1[32];
            decoder_layer1(d1, smem_u32(sm.a1[stage][0]), smem_u32(sm.a1[stage][1]), kLBO_A1, w1h, w1l, kLBO_W1, chunk, a.single_pass);
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.a1_empty[stage]);
            uint32_t ah[16], al[16];
            decoder_hidden(d1, sm.b1, lane, ah, al);
            float dc[16], ds[4];
            decoder_layer2_issue<kRgb>(dc, ah, al, w2ch, w2cl, kLBO_W2C, a.single_pass);
            decoder_layer2_issue<8>(ds, ah, al, w2sh, w2sl, kLBO_W2S, a.single_pass);
            wgmma_commit();
            wgmma_wait_all();
            fence_operands(dc);
            fence_operands(ds);
            tk_.lap(6);                                                   // [6] both layers
            // this thread's two rows of the tile (fragment elements 2 rs, 2 rs + 1 of each 8-column block)
            float* area = colour_area(td.n, td.pass) + td.k * 128 * kRgb;
            GroupState& st = sm.st[td.n & 3];
#pragma unroll
            for (int rs = 0; rs < 2; ++rs) {
                const int trow = 64 * chunk + frag_row(2 * rs, lane, quarter);
#pragma unroll
                for (int blk = 0; blk < 4; ++blk) {
                    const int i = 4 * blk + 2 * rs, c = frag_col(i, lane);
                    *reinterpret_cast<float2*>(area + trow * kRgb + c) =
                        make_float2(rcp_approx(1.f + ex2_approx(dc[i] + sm.b2c[c])), rcp_approx(1.f + ex2_approx(dc[i + 1] + sm.b2c[c + 1])));
                }
                if ((lane & 3) == 0) {                                    // column 0 of the sigma accumulator
                    float sg = ds[2 * rs] + sm.b2s;
                    const int rl = trow / RPT, s = td.k * RPT + (trow - rl * RPT);
                    const int srow = rl * S + s;
                    if (st.crop[td.pass][srow]) sg = -1e3f;
                    if (g.binarize_on) sg = sg < a.sigma_cull ? -1e3f : 1e3f;
                    else if (g.cull_on && sg < a.sigma_cull) sg = -1e3f;
                    (td.pass == 0 ? st.sg_c : st.sg_f)[srow] = sg;
                }
            }
            if (td.k == 2) {                                              // the group's pass is complete: hand it to the ray warps
                __threadfence_block();                                    // (its colour-area stores included)
                __syncwarp();
                if (lane == 0) mbar_arrive(td.pass == 0 ? &sm.sigc_ready[td.n & 3] : &sm.sigf_ready[td.n & 3]);
            }
            tk_.lap(8);                                                   // [8] colour / sigma stores
        }
        colours(n_my - 1);
    } else if (warp < kGW + kEW + kRW) {
        // =========================================================================== RAY (one warp per ray)
        const int rw = warp - kGW - kEW;
        float* scr = sm.rscratch[rw];
        constexpr int NC = (S + 31) / 32, nb = S - 3;
        // A single warp has no other warp to hide its latencies behind, so both phases are written for instruction-level
        // parallelism: the 32-lane chunks of a ray are processed as independent chains (per-chunk scans, carries
        // combined afterwards), every search is a fixed-trip branchless bisection, and the importance depths are put in
        // order by sorting the UNIFORMS with a bitonic network (the inverse CDF is monotone, so mapping sorted uniforms
        // yields sorted depths - this replaces the O(S^2) rank sort).
        // ---- importance sampling of ray rl of group n (renderer.py:328-387)
        auto importance_ray = [&](int n, int rl) {
            GroupState& st = sm.st[n & 3];
            const long long ray = (long long)((int)blockIdx.x + n * (int)gridDim.x) * GR + rl;
            const float* tc = st.t_c + rl * S;
            const float* sg = st.sg_c + rl * S;
            float* i_w = scr;                     // [S]
            float* i_cdf = scr + 128;             // [S]
            // uniforms first (global loads / Philox overlap the scans below); 4th chunk = +inf padding to 128
            float us[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int f = c * 32 + lane;
                us[c] = INFINITY;
                if (f < Sf && ray < a.R) us[c] = a.u_f ? a.u_f[ray * Sf + f] : philox_uniform(g.seed, (uint64_t)(ray * Sf + f), 1u);
            }
            float al[NC], inc[NC];
#pragma unroll
            for (int c = 0; c < NC; ++c) {        // alpha and (1 - alpha + 1e-10) per interval
                const int i = c * 32 + lane;
                float alpha = 0.f, fac = 1.f;
                if (i < S - 1) {
                    const float smid = __fsub_rn(__fmul_rn(__fadd_rn(sg[i], sg[i + 1]), 0.5f), 1.f);
                    alpha = 1.f - ex2_approx(-kLog2e * __fmul_rn(softplus_mufu(smid), tc[i + 1] - tc[i]));
                    fac = __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f);
                }
                al[c] = alpha; inc[c] = fac;
            }
#pragma unroll
            for (int c = 0; c < NC; ++c) inc[c] = warp_scan_mul(inc[c], lane);     // independent chains
            float carry = 1.f;
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                const int i = c * 32 + lane;
                float excl = __shfl_up_sync(0xffffffffu, inc[c], 1);
                if (lane == 0) excl = 1.f;
                if (i < S) i_w[i] = al[c] * (carry * excl);
                carry *= __shfl_sync(0xffffffffu, inc[c], 31);
            }
            __syncwarp();
            float my[NC];
            float part = 0.f;
#pragma unroll
            for (int c = 0; c < NC; ++c) {        // max-pool(2) -> avg-pool(2) -> +0.01 -> +1e-5
                const int k = c * 32 + lane;
                float v = 0.f;
                if (k < nb) {
                    const float* w = i_w + k;
                    v = __fadd_rn(__fadd_rn(__fmul_rn(__fadd_rn(fmaxf(w[0], w[1]), fmaxf(w[1], w[2])), 0.5f), 0.01f), 1e-5f);
                }
                my[c] = v; part += v;
            }
            const float total = warp_sum(part);
#pragma unroll
            for (int c = 0; c < NC; ++c) my[c] = warp_scan_add((c * 32 + lane) < nb ? __fdiv_rn(my[c], total) : 0.f, lane);
            float csum = 0.f;
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                const int k = c * 32 + lane;
                const float incl = my[c] + csum;
                if (k < nb) i_cdf[k + 1] = incl;
                csum = __shfl_sync(0xffffffffu, incl, 31);
            }
            if (lane == 0) i_cdf[0] = 0.f;
            // bitonic sort of the 128 (padded) uniforms, element e = c*32 + lane, ascending
#pragma unroll
            for (int k = 2; k <= 128; k <<= 1) {
#pragma unroll
                for (int j = k >> 1; j > 0; j >>= 1) {
                    if (j >= 32) {
                        const int dc = j >> 5;
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            if ((c & dc) == 0) {
                                const bool up = (((c * 32) & k) == 0);         // lane bits are below 32: direction depends on c only
                                const float lo = fminf(us[c], us[c | dc]), hi = fmaxf(us[c], us[c | dc]);
                                us[c] = up ? lo : hi; us[c | dc] = up ? hi : lo;
                            }
                        }
                    } else {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const float other = __shfl_xor_sync(0xffffffffu, us[c], j);
                            const bool up = (((c * 32 + lane) & k) == 0);
                            const bool lower = (lane & j) == 0;
                            us[c] = (lower == up) ? fminf(us[c], other) : fmaxf(us[c], other);
                        }
                    }
                }
            }
            __syncwarp();                         // i_cdf is complete
#pragma unroll
            for (int c = 0; c < NC; ++c) {        // inverse CDF (searchsorted right=True), lerp between bin midpoints
                const int f = c * 32 + lane;
                if (f >= Sf) continue;
                float val = INFINITY;
                if (ray < a.R) {
                    const float u = us[c];
                    int lo = 0;                   // number of cdf[0..nb] entries <= u
#pragma unroll
                    for (int step = 64; step >= 1; step >>= 1) {
                        const int p = lo + step;
                        const float x = i_cdf[min(p, nb + 1) - 1];
                        if (p <= nb + 1 && x <= u) lo = p;
                    }
                    const int below = max(lo - 1, 0), above = min(lo, nb);
                    const float c0 = i_cdf[below], c1 = i_cdf[above];
                    const float b0 = __fmul_rn(0.5f, __fadd_rn(tc[below], tc[below + 1]));
                    const float b1 = __fmul_rn(0.5f, __fadd_rn(tc[above], tc[above + 1]));
                    float den = __fsub_rn(c1, c0);
                    if (den < 1e-5f) den = 1.f;
                    val = __fadd_rn(b0, __fmul_rn(__fdiv_rn(__fsub_rn(u, c0), den), __fsub_rn(b1, b0)));
                }
                st.t_f[rl * Sf + f] = val;
            }
            __syncwarp();
        };
        // ---- merge + transmittance + omega + per-ray outputs of ray rl of group n (renderer.py:289-301, ray_marcher.py:25-57)
        auto composite_ray = [&](int n, int rl) {
            GroupState& st = sm.st[n & 3];
            SlotState& sl = sm.slot[n & 1];
            const long long ray = (long long)((int)blockIdx.x + n * (int)gridDim.x) * GR + rl;
            const float* tc = st.t_c + rl * S;
            const float* tf = st.t_f + rl * Sf;
            float* m_t = scr;                     // [L]
            float* m_sg = scr + 256;              // [L]
            const bool rev = tc[0] > tc[S - 1];
            const float* tca = rev ? tc + (S - 1) : tc;     // ascending view of the coarse depths: tca[m * dir]
            const int dir = rev ? -1 : 1;
            sl.acc[rl][lane] = 0.f;
#pragma unroll
            for (int c = 0; c < L / 32; ++c) {    // merge by rank: position = own index + count of the other list before it
                const int r = c * 32 + lane;
                const bool is_f = r >= S;
                const int i = is_f ? r - S : r;
                const int ci = rev ? S - 1 - i : i;
                const float tv = is_f ? tf[i] : tc[ci];
                int lo = 0;                       // coarse: #fine < tv; fine: #coarse <= tv  (stable: coarse first on ties)
#pragma unroll
                for (int step = 64; step >= 1; step >>= 1) {
                    const int p = lo + step;
                    const int q = min(p, S) - 1;                               // S == Sf
                    const float x = is_f ? tca[q * dir] : tf[q];
                    if (p <= S && (is_f ? (x <= tv) : (x < tv))) lo = p;
                }
                const int pos = i + lo;
                m_t[pos] = tv;
                m_sg[pos] = is_f ? st.sg_f[rl * Sf + i] : st.sg_c[rl * S + ci];
                sl.pos[is_f ? kRowsG + rl * Sf + i : rl * S + ci] = (unsigned short)pos;
            }
            __syncwarp();
            float al[L / 32], inc[L / 32], tm[L / 32];
#pragma unroll
            for (int c = 0; c < L / 32; ++c) {
                const int i = c * 32 + lane;
                float alpha = 0.f, fac = 1.f, tmid = 0.f;
                if (i < L - 1) {
                    const float t0 = m_t[i], t1 = m_t[i + 1];
                    const float smid = __fsub_rn(__fmul_rn(__fadd_rn(m_sg[i], m_sg[i + 1]), 0.5f), 1.f);
                    alpha = 1.f - ex2_approx(-kLog2e * __fmul_rn(softplus_mufu(smid), t1 - t0));
                    fac = __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f);
                    tmid = __fmul_rn(__fadd_rn(t0, t1), 0.5f);
                }
                al[c] = alpha; inc[c] = fac; tm[c] = tmid;
            }
#pragma unroll
            for (int c = 0; c < L / 32; ++c) inc[c] = warp_scan_mul(inc[c], lane);   // independent chains
            float carry = 1.f, acc_w = 0.f, acc_d = 0.f, wprev = 0.f;
#pragma unroll
            for (int c = 0; c < L / 32; ++c) {
                const int i = c * 32 + lane;
                float excl = __shfl_up_sync(0xffffffffu, inc[c], 1);
                if (lane == 0) excl = 1.f;
                const float wi = al[c] * (carry * excl);
                carry *= __shfl_sync(0xffffffffu, inc[c], 31);
                acc_w += wi;
                acc_d = fmaf(wi, tm[c], acc_d);
                float wl = __shfl_up_sync(0xffffffffu, wi, 1);
                if (lane == 0) wl = wprev;
                wprev = __shfl_sync(0xffffffffu, wi, 31);
                sl.om[rl * L + i] = __fmul_rn(__fadd_rn(wl, wi), 0.5f);
            }
            const float wsum = warp_sum(acc_w), dnum = warp_sum(acc_d);
            const float back = g.white_back ? __fsub_rn(1.f, wsum) : 0.f;
            if (ray < a.R) {
                if (lane < 3) {
                    const float v = fmaf(a.ro[ray * 3 + lane], wsum, a.rd[ray * 3 + lane] * dnum);
                    a.out_xyz[ray * 3 + lane] = __fsub_rn(__fmul_rn(__fadd_rn(v, back), 2.f), 1.f);
                }
                if (lane == 0) {
                    a.out_depth[ray] = __fdiv_rn(dnum, wsum);
                    a.out_wsum[ray] = wsum;
                    atomicMin(&a.bounds[0], float_to_ordered(m_t[0]));
                    atomicMax(&a.bounds[1], float_to_ordered(m_t[L - 1]));
                }
            }
            if (lane == 0) sl.back[rl] = back;
            __syncwarp();
        };
        // tasks follow the pass schedule: importance(n) after C(n), merge(n) after F(n)
        Tick tr_(a.timing, blockIdx.x == 0 && rw == 0 && lane == 0);
        for (int j = 0; j < 2 * n_my; ++j) {
            const PassDesc pd = pass_at(j, n_my);
            const int n = pd.n, si = n & 3;
            const uint32_t par = (n >> 2) & 1;
            if (pd.pass == 0) {
                mbar_wait(&sm.sigc_ready[si], par);
                tr_.lap(13);                                                  // [13] wait for coarse sigma
                for (int rl = rw; rl < GR; rl += kRW) importance_ray(n, rl);
                if (lane == 0) mbar_arrive(&sm.fine_ready[si]);
                tr_.lap(9);                                                   // [9] importance
            } else {
                mbar_wait(&sm.sigf_ready[si], par);
                if (n >= 2) mbar_wait(&sm.state_free[(n - 2) & 3], ((n - 2) >> 2) & 1);       // colours(n-2) has released the omega slot
                tr_.lap(14);                                                  // [14] wait for fine sigma / slot
                for (int rl = rw; rl < GR; rl += kRW) composite_ray(n, rl);
                if (lane == 0) mbar_arrive(&sm.omega_ready[n & 1]);
                tr_.lap(10);                                                  // [10] merge / weights
            }
        }
    }
}

}  // namespace

int launch_bounds_init(unsigned int* bounds, cudaStream_t stream);
int launch_ray_limits(const float* ro, const float* rd, long long R, float h, float* t0, float* t1, unsigned int* bounds, cudaStream_t stream);
int launch_depth_finalize(float* depth, long long R, const unsigned int* bounds, cudaStream_t stream);

bool fused_ws3_supported(const Geom& g) {
    if (!((g.S == 96 || g.S == 48) && (g.Sf == g.S) && ((long long)g.M % (384 / g.S) == 0))) return false;
    const long long span = 2 * g.stride_plane + (long long)(g.H - 1) * g.stride_row + (long long)(g.W - 1) * g.stride_col + kC;
    if (g.H < 2 || g.W < 2) return false;
    if ((g.stride_view | g.stride_plane | g.stride_row | g.stride_col) & 7) return false;
    return g.stride_plane >= 0 && g.stride_row >= 0 && g.stride_col >= 0 && span < (1ll << 31);
}

int render_forward_fused_ws3(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                            const float* w2, const float* b2, const float* ro, const float* rd, const float* u_c,
                            const float* u_f, const Workspace& ws, float* out_rgb, float* out_depth, float* out_wsum,
                            float* out_xyz, cudaStream_t stream) {
    if (!fused_ws3_supported(g)) {
        set_error("fused warp-specialised renderer supports depth_resolution == depth_resolution_importance in {48, 96} (got %d, %d)", g.S, g.Sf);
        return P3D_EUNSUPPORTED;
    }
    const long long R = (long long)g.N * g.M;
    int rc;
    if ((rc = launch_bounds_init(ws.bounds, stream))) return rc;
    if (g.ray_mode == P3D_RAYS_AUTOBOX)
        if ((rc = launch_ray_limits(ro, rd, R, g.half_box, ws.ray_t0, ws.ray_t1, ws.bounds, stream))) return rc;
    WsArgs a{};
    a.g = g; a.planes = planes; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2; a.ro = ro; a.rd = rd; a.u_c = u_c; a.u_f = u_f;
    a.ray_t0 = ws.ray_t0; a.ray_t1 = ws.ray_t1; a.bounds = ws.bounds;
    a.out_rgb = out_rgb; a.out_depth = out_depth; a.out_wsum = out_wsum; a.out_xyz = out_xyz;
    a.col_c = ws.rgb_c; a.col_f = ws.rgb_f;
    const int GR = 384 / g.S;
    a.R = R; a.n_groups = (int)((R + GR - 1) / GR);
    a.single_pass = p->mlp_mode == P3D_MLP_TC_BF16;
    a.srow = (int)g.stride_row; a.scol = (int)g.stride_col; a.splane = (int)g.stride_plane;
    if (g.cull_on || g.binarize_on) {
        const double thr = (double)g.cull_thresh;
        a.sigma_cull = thr >= 1.0 ? INFINITY : (thr <= 0.0 ? -INFINITY : (float)(1.0 + log(expm1(-log1p(-thr)))));
    }
    static int n_sm = 0;
    if (!n_sm) {
        int dev = 0;
        P3D_CUDA_TRY(cudaGetDevice(&dev));
        P3D_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    static unsigned long long* d_timing = nullptr;
    static const bool timing_on = getenv("P3D_WS_TIMING") != nullptr;
    if (timing_on) {
        if (!d_timing) P3D_CUDA_TRY(cudaMalloc(&d_timing, 16 * sizeof(unsigned long long)));
        P3D_CUDA_TRY(cudaMemsetAsync(d_timing, 0, 16 * sizeof(unsigned long long), stream));
        a.timing = d_timing;
    }
    const size_t smem = sizeof(WsSmem) + 1024;
    void (*kern)(WsArgs) = nullptr;
    // the x+1 texel is an immediate offset when the texel stride is one of the two layouts the host produces: kC (the layout
    // pre-pass: one plane's texels contiguous) or 3 kC (a (N,96,H,W) channels_last backbone output consumed zero-copy)
    const int sc = g.stride_col == kC ? 1 : (g.stride_col == 3 * kC ? 2 : 0);
#define P3D_PICK(BF, S_) (sc == 1 ? k_render_ws3<BF, S_, kC> : (sc == 2 ? k_render_ws3<BF, S_, 3 * kC> : k_render_ws3<BF, S_, 0>))
    if (g.S == 96) kern = p->planes_bf16 ? P3D_PICK(true, 96) : P3D_PICK(false, 96);
    else kern = p->planes_bf16 ? P3D_PICK(true, 48) : P3D_PICK(false, 48);
#undef P3D_PICK
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = a.n_groups < n_sm ? a.n_groups : n_sm;
    {
        ProfileScope prof(PROF_FUSED, stream);
        kern<<<grid, kThreadsWS, smem, stream>>>(a);
        P3D_LAUNCH_CHECK();
    }
    if (timing_on) {
        unsigned long long h[16];
        P3D_CUDA_TRY(cudaMemcpyAsync(h, d_timing, sizeof(h), cudaMemcpyDeviceToHost, stream));
        P3D_CUDA_TRY(cudaStreamSynchronize(stream));
        const int groups_cta0 = (a.n_groups + grid - 1) / grid;
        fprintf(stderr, "[p3d ws timing, CTA0, cycles/group over %d groups] G(warp0: 1/3 of tiles): wait_dep %.0f wait_ring %.0f gather %.0f | "
                        "D(warp0): wait_a1 %.0f layers %.0f stores %.0f colours(+omega wait) %.0f other %.0f | "
                        "R(warp0): wait_sigc %.0f importance %.0f wait_sigf %.0f merge %.0f\n",
                groups_cta0, (double)h[1] / groups_cta0, (double)h[2] / groups_cta0, (double)h[3] / groups_cta0, (double)h[5] / groups_cta0,
                (double)h[6] / groups_cta0, (double)h[8] / groups_cta0, (double)h[11] / groups_cta0, (double)h[4] / groups_cta0,
                (double)h[13] / groups_cta0, (double)h[9] / groups_cta0, (double)h[14] / groups_cta0, (double)h[10] / groups_cta0);
    }
    if (p->defer_depth_clamp) return P3D_OK;
    return launch_depth_finalize(out_depth, R, ws.bounds, stream);
}

}  // namespace p3d
