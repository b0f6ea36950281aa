// The fused renderer: warp-specialised, pipeline depth 3 - THREE ray groups in flight.
//
//   passes C(0) C(1) | F(0) C(2) | F(1) C(3) | ... | F(N-2) F(N-1)          (C = 3 coarse tiles, F = 3 importance tiles)
//
// A tile's colour sigmoids wait for the group's compositing weights (omega), which exist only after its fine pass.  They are
// staged in global memory, in this CTA's own slices of the workspace colour buffers (see colour_area: coarse areas
// CA[n % 3] and fine areas FA[n & 1], 5 x 48 KB per CTA, ~32 MB on 132 SMs).  They share the 50 MB L2 with the tri-plane
// gather, so the ray warps load them evict-first and discard each line from L2 once its load has landed: a dead line
// leaves without a write-back and without pushing out texels (DESIGN §5).  The decoder's epilogue stages each 8 KB tile half in shared memory
// for one cp.async.bulk store; once a group's fine pass is stored, the ray warps bulk-load their own rays' rows back into
// shared memory (mbarrier complete_tx) and reduce them there (colours(n)), off the decoder's critical path.  With F(n)
// followed by C(n+2):
//   * importance(n) has two passes of slack (F(n-1), C(n+1)) before the gather of F(n) needs its depths;
//   * merge(n) + omega(n) run on the RAY warps while the decoder handles the three tiles of C(n+2); colours(n) follows on
//     the same warps once the decoder signals that F(n)'s stores completed (col_stored, in C(n+2)'s first epilogue);
//   * the decoder stores into an area only after its previous group's colours are done (state_free): C(m) into CA[m % 3]
//     after group m - 3, F(m) into FA[m & 1] after group m - 2, each with several tiles of slack;
//   * the per-group state ring stays 4 deep (groups n .. n+3 alive).
//
//   warps  0-11  GATHER    three teams of four warps; team j takes tiles j, j+3, ... of the tile sequence
//   warps 12-19  DECODER   two warpgroups, one per 64-row half of every tile: layer 1 (wgmma, A1 and W1 from shared memory)
//                          -> softplus2 in registers -> layer 2 (one m64n48 wgmma, A from the registers): colour sigmoids ->
//                          staging tile -> bulk store to the colour area, sigma -> group state
//   warps 20-23  RAY       a warp per ray: importance sampling after a group's coarse pass, merge / transmittance /
//                          omega, the per-ray outputs and the colour reduction of its own rays after its fine pass
#include "fused_common.cuh"

namespace p3d {

namespace {

using namespace dev;
using namespace fused;

constexpr int kGW = 12, kEW = 8, kRW = 4, kTeams = 3;   // 24 warps = 6 warpgroups -> 80 registers per thread
constexpr int kWarpsWS = kGW + kEW + kRW;
constexpr int kThreadsWS = kWarpsWS * 32;        // 768
constexpr int kNA = 3;                           // A1 ring depth: one stage per gather team
// registers per thread by role (launched with 80 = 65536 / 768 rounded down to 8): the decoder warpgroups hold the layer-2
// A operands and accumulators at once and take what the ray warpgroup does not need; 3 x 80 + 2 x kRegE + kRegR <= 6 x 80
constexpr int kRegE = 88, kRegR = 64;
static_assert(3 * 80 + 2 * kRegE + kRegR <= 6 * 80, "per-role registers exceed what the launch allocates");
constexpr int kStates = 4;                       // per-group state ring
constexpr int kRowsG = 384;                      // rows per pass per group
constexpr int kColBufs = 2;                      // colour tiles of a group in shared memory at once (colours())
constexpr int kHalfBytes = 64 * kRgb * 4;        // one decoder warpgroup's 64 rows of colour sigmoids: 8 KB
constexpr int kRowBytes = kRgb * 4;              // one row of colour sigmoids: 128 B


// Per-role cycle accounting, compiled in only with -DP3D_WS3_ROLE_CLOCKS (bench_roles.py): lane 0 of every warp adds
// clock64() deltas into per-CTA counters [role][slot] in shared memory, which the CTA adds into WsArgs::role_clk
// ([CTA][kRoles][kRcSlots], accumulated over launches) at its end.  RC_* slots 1-7 are mbarrier waits, the rest phases of work;
// a role's remainder (RC_TOTAL minus the slots it uses) is untimed bookkeeping.  The default build has no clock reads.
enum RoleClk {
    RC_TOTAL, RC_A1_FULL, RC_A1_EMPTY, RC_STATE_FREE, RC_FINE_READY, RC_SIG_READY, RC_COL_STORED, RC_COL_FULL,
    RC_COLOURS, RC_L1, RC_HIDDEN, RC_L2, RC_EPILOGUE,         // decoder phases (the epilogue includes its state_free wait)
    RC_TAPS, RC_GATHER,                                       // gather phases: tap table, loads + lerp into the A1 stage
    RC_IMPORTANCE,                                            // ray phases: importance sampling, colours() (which includes its
                                                              // col_stored / col_full waits); composite = the rest
    kRcSlots
};
#ifdef P3D_WS3_ROLE_CLOCKS
constexpr int kRoles = 3;                                     // 0 gather, 1 decoder, 2 ray
#define RC_BEGIN(v) const long long v = clock64()
#define RC_END(role, slot, v) do { if (lane == 0) atomicAdd(&sm.rclk[role][slot], (unsigned long long)(clock64() - (v))); } while (0)
// ties register values computed by plain arithmetic to the clock read after them (the compiler may otherwise sink them)
__device__ __forceinline__ void rc_fence_regs(uint32_t (&x)[16], uint32_t (&y)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) asm volatile("" : "+r"(x[i]), "+r"(y[i])::"memory");
}
#define RC_FENCE_REGS(x, y) rc_fence_regs(x, y)
#else
#define RC_BEGIN(v) do {} while (0)
#define RC_END(role, slot, v) do {} while (0)
#define RC_FENCE_REGS(x, y) do {} while (0)
#endif
#define RC_WAIT(role, slot, bar, par) do { RC_BEGIN(rc_t_); mbar_wait(bar, par); RC_END(role, slot, rc_t_); } while (0)

struct GroupState {                               // written by G (t_c, crop), E (sg_*), R (t_f)
    float t_c[kRowsG], sg_c[kRowsG], t_f[kRowsG], sg_f[kRowsG];
    unsigned char crop[2][kRowsG];
};
struct SlotState {                                // written by composite_ray, read by colours() of the same ray warp
    float om[2 * kRowsG];                         // omega per merged position, [ray][2S]
    unsigned short pos[2 * kRowsG];                          // merged position of coarse rows [0,384) and fine rows [384,768)
};

struct __align__(1024) WsSmem {
    unsigned char a1[kNA][2][4 * kLBO_A1];
    float col_stage[2][64 * kRgb];                // per decoder warpgroup: its half of the tile being stored (col_idx layout)
    float col_buf[kColBufs][128 * kRgb];          // colour tiles loaded back for colours(), same layout; each ray warp
                                                  // loads and reads only its own rays' rows
    unsigned char w1[2][4096], w2[2][kD2Cols * 128];
    float b1[kHidden], b2c[kRgb], b2s, pad0[3];
    uint4 tab[kGW][32][4];                        // tap table of a gather warp's 32 rows (see "gather" below)
    GroupState st[kStates];
    SlotState slot;
    float rscratch[kRW][768];                      // private scratch of each ray warp (importance / merge)
    unsigned long long a1_full[kNA], a1_empty[kNA];
    unsigned long long fine_ready[kStates], state_free[kStates];
    unsigned long long sigc_ready[kStates], sigf_ready[kStates];   // E -> R (sigma in smem)
    unsigned long long col_stored[2];             // E -> R: both warpgroups' bulk stores of a group's fine pass completed
    unsigned long long col_full[kRW][kColBufs];   // a ray warp's rows of a col_buf tile have landed (complete_tx)
#ifdef P3D_WS3_ROLE_CLOCKS
    unsigned long long rclk[kRoles][kRcSlots];
#endif
};

// Float index of colour (row, c) in a staged / loaded colour tile: 128 B rows, 16-byte chunk (c / 4) XOR (row % 8).  The
// epilogue's float2 stores (8 rows x 4 column pairs per instruction) and the reduction's lane = channel loads are both
// conflict-free.  The colour areas in global memory are byte copies of the tiles, so they hold the same layout.
__device__ __forceinline__ int col_idx(int row, int c) { return row * kRgb + ((((c >> 2) ^ row) & 7) << 2) + (c & 3); }

// Shared memory and L1 share 256 KB per SM.  At most 196 KB of shared memory (199,680 B for the CTA after the 1 KB the
// system reserves) leaves 60 KB of L1 instead of the 28 KB of the largest carve-out: the gather's texel loads land in L1
// while they are in flight, so L1 bounds how much of that traffic each SM keeps outstanding.  That is what the A1 ring
// (one stage per team) and kColBufs (two colour tiles) are sized for.
constexpr int kSmemWS = (int)sizeof(WsSmem) + 1024;                  // + alignment slack of the extern array
static_assert(kSmemWS <= 199680, "WsSmem + alignment slack exceeds the 196 KB shared-memory carve-out");

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
#ifdef P3D_WS3_ROLE_CLOCKS
    unsigned long long* role_clk;    // [gridDim.x][kRoles][kRcSlots]
#endif
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
    // this CTA's colour area of (group n, pass): 384 rows x 32 sigmoids, row = 128 k + row of tile k, each tile in the
    // col_idx layout (a byte copy of the staged tile).  CA[j] = slice j of the coarse workspace buffer, FA[i] = slice i of
    // the fine one, where slice s is the one of this CTA's group s: they exist whenever they are used (n % 3, n & 1 < n_my).
    auto colour_area = [&](int n, int pass) -> float* {
        const int s = pass == 0 ? n % 3 : n & 1;
        return (pass == 0 ? a.col_c : a.col_f) + ((long long)blockIdx.x + (long long)s * gridDim.x) * (kRowsG * kRgb);
    };

    // ---------------- setup
    if (tid == 0) {
        for (int i = 0; i < kNA; ++i) { mbar_init(&sm.a1_full[i], 4); mbar_init(&sm.a1_empty[i], kEW); }
        for (int i = 0; i < kStates; ++i) {
            mbar_init(&sm.fine_ready[i], kRW); mbar_init(&sm.state_free[i], kRW);
            mbar_init(&sm.sigc_ready[i], kEW); mbar_init(&sm.sigf_ready[i], kEW);
        }
        mbar_init(&sm.col_stored[0], 2); mbar_init(&sm.col_stored[1], 2);
        for (int w = 0; w < kRW; ++w)
            for (int i = 0; i < kColBufs; ++i) mbar_init(&sm.col_full[w][i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    stage_w1_biases(g, a.w1, a.b1, a.b2, sm.w1, sm.b1, sm.b2c, sm.b2s, tid, kThreadsWS);
    stage_w2(g, a.w2, sm.w2, kD2Cols, kLBO_W2, w2_row_n48, tid, kThreadsWS);
#ifdef P3D_WS3_ROLE_CLOCKS
    if (tid < kRoles * kRcSlots) (&sm.rclk[0][0])[tid] = 0ull;
#endif
    fence_proxy_async();
    __syncthreads();

    if (warp < kGW) {
        // =========================================================================== GATHER
        RC_BEGIN(rc_role);
        const int gw = warp, team = gw >> 2, wt = gw & 3;
        constexpr int kEsz = BF16 ? 2 : 4;
        const long long scolB = (long long)a.scol * kEsz, srowB = (long long)a.srow * kEsz;
        unsigned char* tab = reinterpret_cast<unsigned char*>(sm.tab[gw]);
        float v[12][4];
#pragma unroll
        for (int k = 0; k < 12; ++k)
#pragma unroll
            for (int c = 0; c < 4; ++c) v[k][c] = 0.f;
        int it = 0;
        for (int q = 0; q < T; ++q) {
            const TileDesc td = tile_at(q, n_my);
            const int my_it = it++;
            if (my_it % kTeams != team) continue;
            const int grp = (int)blockIdx.x + td.n * (int)gridDim.x;
            const long long ray0 = (long long)grp * GR;
            GroupState& st = sm.st[td.n & 3];
            if (td.pass == 0) RC_WAIT(0, RC_STATE_FREE, &sm.state_free[td.n & 3], ((td.n >> 2) & 1) ^ 1);
            else RC_WAIT(0, RC_FINE_READY, &sm.fine_ready[td.n & 3], (td.n >> 2) & 1);
            const int view = (int)(ray0 / g.M);
            // ---- tap table of this warp's 32 rows: lane = row
            RC_BEGIN(rc_taps);
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
                    tval = coarse_sample_depth(g, s, u, ray, live, a.ray_t0, a.ray_t1, a.bounds);
                    st.t_c[srow] = tval;
                } else {
                    tval = st.t_f[srow];
                }
                float3 pt = make_float3(1e30f, 1e30f, 1e30f);
                if (live) pt = ray_point(a.ro + ray * 3, a.rd + ray * 3, tval);
                write_tap_row(tab, lane, g, a.srow, a.scol, a.splane, pt.x, pt.y, pt.z, 0u);   // the tile lies in one view (M % GR == 0)
                st.crop[td.pass][srow] = (g.crop_on && !((fabsf(pt.x) <= g.crop_limit) && (fabsf(pt.z) <= g.crop_limit))) ? 1 : 0;
            }
            __syncwarp();
            RC_END(0, RC_TAPS, rc_taps);
            const int stage = my_it % kNA;
            RC_WAIT(0, RC_A1_EMPTY, &sm.a1_empty[stage], ((my_it / kNA) & 1) ^ 1);
            RC_BEGIN(rc_gather);
            gather_a1<BF16, SCOL>(tab, reinterpret_cast<const char*>(a.planes) + (long long)view * g.stride_view * kEsz, 0 /* one view */, srowB,
                                  scolB, v, sm.a1[stage][0], sm.a1[stage][1], wt, lane);
            fence_proxy_async();
            __syncwarp();                                                   // also: the tap table is rewritten by the next tile
            RC_END(0, RC_GATHER, rc_gather);
            if (lane == 0) mbar_arrive(&sm.a1_full[stage]);
        }
        RC_END(0, RC_TOTAL, rc_role);
    } else if (warp < kGW + kEW) {
        // =========================================================================== DECODER
        setmaxnreg_inc<kRegE>();
        RC_BEGIN(rc_role);
        const int e = warp - kGW, quarter = e & 3, chunk = e >> 2;      // chunk = warpgroup = 64-row half of a tile
        const int etid = tid - kGW * 32;                                  // 0..255 inside the decoder group
        const bool elect = (etid & 127) == 0;                             // the warpgroup's bulk-copy thread
        auto wgbar = [chunk] { asm volatile("bar.sync %0, 128;" ::"r"(2 + chunk) : "memory"); };   // this warpgroup's four warps
        // The ray warps read a group's colours back once both warpgroups' stores of its fine pass have COMPLETED, not just
        // read their staging tiles: in the epilogue of the next tile (C(n+2)'s first, or F(n+1)'s), and after the tile loop
        // for the last group, the elected thread of each warpgroup waits for all its bulk groups and arrives on
        // col_stored[n & 1].  The chain from these bulk stores to another thread's bulk loads of the same bytes, by the PTX
        // ISA's memory consistency model and its proxy rules:
        //   cp.async.bulk.wait_group 0     the stores (async proxy) are complete: their writes to global memory are performed;
        //   fence.proxy.async.global       orders them before this thread's later generic-proxy operations;
        //   mbarrier.arrive                release.cta by default; the ray warp's mbarrier.try_wait (acquire.cta) that
        //                                  observes the completed phase synchronises with it (colours(), ray warps);
        //   fence.proxy.async.global       on the loading thread: what it acquired is ordered before its own later
        //                                  async-proxy operations;
        //   cp.async.bulk (load)           reads the stored colours.
        int stored = -1, signalled = -1;                                  // last group whose fine pass was stored / signalled
        auto signal_stored = [&] {
            if (elect) {
                bulk_wait_all();
                fence_proxy_async_global();
                mbar_arrive(&sm.col_stored[stored & 1]);
            }
            signalled = stored;
        };
        const uint32_t w1h = smem_u32(sm.w1[0]), w1l = smem_u32(sm.w1[1]), w2h = smem_u32(sm.w2[0]), w2l = smem_u32(sm.w2[1]);
        float* stage_tile = sm.col_stage[chunk];
        for (int it = 0; it < T; ++it) {
            const TileDesc td = tile_at(it, n_my);
            const int stage = it % kNA;
            RC_WAIT(1, RC_A1_FULL, &sm.a1_full[stage], (it / kNA) & 1);
            RC_BEGIN(rc_l1);
            float d1[32];
            decoder_layer1(d1, smem_u32(sm.a1[stage][0]), smem_u32(sm.a1[stage][1]), kLBO_A1, w1h, w1l, kLBO_W1, chunk, a.single_pass);
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.a1_empty[stage]);
            RC_END(1, RC_L1, rc_l1);
            RC_BEGIN(rc_hid);
            uint32_t ah[16], al[16];
            decoder_hidden(d1, sm.b1, lane, ah, al);
            RC_FENCE_REGS(ah, al);
            RC_END(1, RC_HIDDEN, rc_hid);
            RC_BEGIN(rc_l2);
            float d2[kD2Cols / 2];
            decoder_layer2_issue<kD2Cols>(d2, ah, al, w2h, w2l, kLBO_W2, a.single_pass);
            wgmma_commit();
            wgmma_wait_all();
            fence_operands(d2);
            RC_END(1, RC_L2, rc_l2);
            RC_BEGIN(rc_epi);
            // the staging half is free once the bulk store of the previous tile has read it (wait_group 0 includes that)
            if (stored > signalled) signal_stored();
            else if (elect) bulk_wait_read();
            wgbar();
            GroupState& st = sm.st[td.n & 3];
            // this thread's two rows of the half (fragment elements 2 rs, 2 rs + 1 of each 8-column block)
#pragma unroll
            for (int rs = 0; rs < 2; ++rs) {
                const int hrow = frag_row(2 * rs, lane, quarter), trow = 64 * chunk + hrow;
#pragma unroll
                for (int blk = 0; blk < 4; ++blk) {
                    const int i = 4 * blk + 2 * rs, c = frag_col(i, lane);
                    *reinterpret_cast<float2*>(stage_tile + col_idx(hrow, c)) =
                        make_float2(rcp_approx(1.f + ex2_approx(d2[i] + sm.b2c[c])), rcp_approx(1.f + ex2_approx(d2[i + 1] + sm.b2c[c + 1])));
                }
                if ((lane & 3) == 0) {                                    // column 32: sigma
                    float sg = d2[16 + 2 * rs] + sm.b2s;
                    const int rl = trow / RPT, s = td.k * RPT + (trow - rl * RPT);
                    const int srow = rl * S + s;
                    if (st.crop[td.pass][srow]) sg = -1e3f;
                    if (g.binarize_on) sg = sg < a.sigma_cull ? -1e3f : 1e3f;
                    else if (g.cull_on && sg < a.sigma_cull) sg = -1e3f;
                    (td.pass == 0 ? st.sg_c : st.sg_f)[srow] = sg;
                }
            }
            fence_proxy_async();                                          // the staging writes, seen by the bulk store
            wgbar();
            if (elect) {
                // The area was last read by the ray warps' loads for group n - 3 (CA[n % 3]) or n - 2 (FA[n & 1]).  Their
                // colours() have waited for every load to land, and discarded the lines from L2, before arriving on that
                // group's state_free.  The chain from those discards to this thread's bulk stores into the same lines:
                //   discard.global.L2             generic-proxy writes of each ray-warp lane, then __syncwarp (the warp's
                //                                 lanes' writes are ordered before lane 0's later operations);
                //   mbarrier.arrive               lane 0, release.cta (cumulative: includes its warp's discards);
                //   mbarrier.try_wait             here, acquire.cta: observes the completed state_free phase;
                //   fence.proxy.async.global      orders what was acquired before this thread's later async-proxy operations;
                //   cp.async.bulk (store)         cannot be overtaken by a discard, which would leave undefined colours.
                // One fence at tile 0 covers the area: tiles 1 and 2 are stored later by the same thread.
                const int prev = td.n - (td.pass == 0 ? 3 : 2);
                if (td.k == 0 && prev >= 0) {
                    RC_WAIT(1, RC_STATE_FREE, &sm.state_free[prev & 3], (prev >> 2) & 1);
                    fence_proxy_async_global();
                }
                bulk_store(colour_area(td.n, td.pass) + (td.k * 128 + 64 * chunk) * kRgb, smem_u32(stage_tile), kHalfBytes);
                bulk_commit();
            }
            RC_END(1, RC_EPILOGUE, rc_epi);
            if (td.k == 2) {                                              // the group's pass is complete: hand its sigma to the ray warps
                if (td.pass == 1) stored = td.n;
                __syncwarp();
                if (lane == 0) mbar_arrive(td.pass == 0 ? &sm.sigc_ready[td.n & 3] : &sm.sigf_ready[td.n & 3]);
            }
        }
        signal_stored();                                                  // the last group's fine pass
        RC_END(1, RC_TOTAL, rc_role);
    } else if (warp < kGW + kEW + kRW) {
        // =========================================================================== RAY (one warp per ray)
        setmaxnreg_dec<kRegR>();
        RC_BEGIN(rc_role);
        const int rw = warp - kGW - kEW;
        float* scr = sm.rscratch[rw];
        constexpr int NC = (S + 31) / 32, nb = S - 3;
        // A single warp has no other warp to hide its latencies behind, so both phases are written for instruction-level
        // parallelism: the 32-lane chunks of a ray are processed as independent chains (per-chunk scans, carries
        // combined afterwards), every search is a fixed-trip branchless bisection, and the importance depths are put in
        // order by sorting them with a bitonic network after the inverse CDF, as the reference sorts them before the merge.
        // Sorting the uniforms instead would only order the depths when the inverse CDF ascends: descending coarse depths
        // ('auto' limits when no ray of the call hits the box, numeric ray_start > ray_end) give negative weights and a
        // cdf that is neither, and the merge by rank needs ascending fine depths.
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
                us[c] = val;
            }
            // bitonic sort of the 128 (padded) depths, element e = c*32 + lane, ascending
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
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                const int f = c * 32 + lane;
                if (f < Sf) st.t_f[rl * Sf + f] = us[c];
            }
            __syncwarp();
        };
        // ---- merge + transmittance + omega + per-ray outputs of ray rl of group n (renderer.py:289-301, ray_marcher.py:25-57)
        auto composite_ray = [&](int n, int rl) {
            GroupState& st = sm.st[n & 3];
            SlotState& sl = sm.slot;
            const long long ray = (long long)((int)blockIdx.x + n * (int)gridDim.x) * GR + rl;
            const float* tc = st.t_c + rl * S;
            const float* tf = st.t_f + rl * Sf;
            float* m_t = scr;                     // [L]
            float* m_sg = scr + 256;              // [L]
            const bool rev = tc[0] > tc[S - 1];
            const float* tca = rev ? tc + (S - 1) : tc;     // ascending view of the coarse depths: tca[m * dir]
            const int dir = rev ? -1 : 1;
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
            __syncwarp();                         // om / pos are read by the other lanes in colours()
            return back;                          // warp-uniform (warp_sum is a butterfly)
        };
        // ---- colours of this warp's rays of group n: sum_j omega_j * rgb_j over the group's six colour tiles (t = 0..2:
        // coarse tile t, 3..5: fine tile t - 3).  The warp's rows of tile t - a ray's RPT rows of a tile are contiguous in the
        // colour area - are bulk-loaded into the same rows of col_buf[t % kColBufs], which the warp reloads with tile
        // t + kColBufs as soon as all its lanes have read it.
        constexpr int RW = GR / kRW;              // rays of this warp: rw + kRW i, i < RW (1 at S = 96, 2 at S = 48)
        static_assert(RW * RPT == 32, "a ray warp's rows of a tile: one 128 B line per lane");
        // The colour areas are a round trip through L2: each line is read once, by the warp that owns its row, one to three
        // passes after its store.  The loads evict first, and the warp discards its lines once its load has landed, so a
        // dead line leaves L2 without a write-back to HBM and without taking the place of the tri-plane's texels.
        const uint64_t pol_colour = l2_evict_first();
        const int my_row = (rw + kRW * (lane / RPT)) * RPT + lane % RPT;      // this lane's row (line) of a tile
        auto load_tile = [&](int n, int t) {      // lane 0 only
            const int pass = t / 3, k = t - 3 * pass, b = t % kColBufs;
            const float* area = colour_area(n, pass) + k * 128 * kRgb;
            mbar_arrive_expect_tx(&sm.col_full[rw][b], RW * RPT * kRowBytes);
#pragma unroll
            for (int i = 0; i < RW; ++i) {
                const int row = (rw + kRW * i) * RPT;
                bulk_load_hint(smem_u32(sm.col_buf[b] + row * kRgb), area + row * kRgb, RPT * kRowBytes, &sm.col_full[rw][b], pol_colour);
            }
        };
        auto colours = [&](int n, const float (&back)[RW]) {
            RC_BEGIN(rc_col);
            // the decoder's elected threads arrive once their stores of F(n) are complete; the acquire here and the proxy
            // fence below close the chain from those bulk stores to these bulk loads (argued at signal_stored)
            RC_WAIT(2, RC_COL_STORED, &sm.col_stored[n & 1], (n >> 1) & 1);
            if (lane == 0) {
                fence_proxy_async_global();
#pragma unroll 1
                for (int t = 0; t < kColBufs; ++t) load_tile(n, t);
            }
            const SlotState& sl = sm.slot;
            const long long ray0 = (long long)((int)blockIdx.x + n * (int)gridDim.x) * GR;
            // Two chains of 16 rows per tile, lane = channel, each summed over tiles 0..5 in a fixed order: rows [0, 16) and
            // [16, 32) of ray rw at S = 96, rows [0, 16) of rays rw and rw + 4 at S = 48.  The chains of a ray meet on 0
            // (0 + a + b at S = 96), so the result is bit-reproducible run to run and independent of how rays are batched.
            float acc[2] = {0.f, 0.f};
#pragma unroll 1
            for (int t = 0; t < 6; ++t) {
                const int pass = t / 3, k = t - 3 * pass, b = t % kColBufs;
                // The omega of the tile's 32 rows is read before the wait for its colours (the tile may still be landing), and
                // the loops are unrolled, so every load is issued before the first add of the fixed-order sums.
                float omj[2][16];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int rl = rw + kRW * (16 * h / RPT), r0 = 16 * h % RPT;          // chain h: rows r0 .. r0 + 15 of ray rl
                    const bool live = ray0 + rl < a.R;
                    const unsigned short* pos = sl.pos + pass * kRowsG + rl * S + k * RPT;   // pos[r]: merged position of row r
#pragma unroll
                    for (int j = 0; j < 16; ++j) omj[h][j] = live ? sl.om[rl * L + pos[r0 + j]] : 0.f;
                }
                RC_WAIT(2, RC_COL_FULL, &sm.col_full[rw][b], ((6 * n + t) / kColBufs) & 1);
                {
                    // the load of the warp's rows has landed (its reads of global memory are done): drop them from L2.  A
                    // workspace that is not 128-byte aligned keeps its lines (the bulk copies need only 16 bytes).
                    const float* line = colour_area(n, pass) + (k * 128 + my_row) * kRgb;
                    if ((reinterpret_cast<uintptr_t>(line) & 127) == 0) l2_discard_line(line);
                }
                const float* buf = sm.col_buf[b];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int rl = rw + kRW * (16 * h / RPT), r0 = 16 * h % RPT;
                    float& part = acc[h];
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int trow = rl * RPT + r0 + j;
                        const float om = omj[h][j];
                        const float ca = g.force_sigmoid ? om : 1.002f * om, cb = g.force_sigmoid ? 0.f : -0.001f * om;
                        part += fmaf(buf[col_idx(trow, lane)], ca, cb);
                    }
                }
                if (t + kColBufs < 6) {
                    __syncwarp();                 // every lane has read the warp's rows of col_buf[b]
                    if (lane == 0) load_tile(n, t + kColBufs);
                }
            }
#pragma unroll
            for (int i = 0; i < RW; ++i) {
                const long long ray = ray0 + rw + kRW * i;
                const float sum = RW == 1 ? __fadd_rn(__fadd_rn(0.f, acc[0]), acc[1]) : __fadd_rn(0.f, acc[i]);
                if (ray < a.R) a.out_rgb[ray * kRgb + lane] = __fsub_rn(__fmul_rn(__fadd_rn(sum, back[i]), 2.f), 1.f);
            }
            RC_END(2, RC_COLOURS, rc_col);
        };
        // tasks follow the pass schedule: importance(n) after C(n), merge(n) and colours(n) after F(n)
        for (int j = 0; j < 2 * n_my; ++j) {
            const PassDesc pd = pass_at(j, n_my);
            const int n = pd.n, si = n & 3;
            const uint32_t par = (n >> 2) & 1;
            if (pd.pass == 0) {
                RC_WAIT(2, RC_SIG_READY, &sm.sigc_ready[si], par);
                RC_BEGIN(rc_imp);
                for (int rl = rw; rl < GR; rl += kRW) importance_ray(n, rl);
                RC_END(2, RC_IMPORTANCE, rc_imp);
                if (lane == 0) mbar_arrive(&sm.fine_ready[si]);
            } else {
                RC_WAIT(2, RC_SIG_READY, &sm.sigf_ready[si], par);
                float back[RW];
#pragma unroll
                for (int i = 0; i < RW; ++i) back[i] = composite_ray(n, rw + kRW * i);
                colours(n, back);
                __syncwarp();                                          // every lane's discards, before lane 0's release
                if (lane == 0) mbar_arrive(&sm.state_free[si]);       // group state; the colour areas' loads landed, lines discarded
            }
        }
        RC_END(2, RC_TOTAL, rc_role);
    }
#ifdef P3D_WS3_ROLE_CLOCKS
    __syncthreads();
    if (tid < kRoles * kRcSlots) atomicAdd(a.role_clk + (long long)blockIdx.x * (kRoles * kRcSlots) + tid, (&sm.rclk[0][0])[tid]);
#endif
}

#ifdef P3D_WS3_ROLE_CLOCKS
// the role counters of every CTA slot (one per SM), zeroed when first allocated, accumulated by every launch
unsigned long long* g_role_clk = nullptr;
int g_role_clk_ctas = 0;
int role_clocks_buffer(int n_sm, unsigned long long** out) {
    if (!g_role_clk) {
        const size_t bytes = (size_t)n_sm * kRoles * kRcSlots * sizeof(unsigned long long);
        P3D_CUDA_TRY(cudaMalloc(&g_role_clk, bytes));
        P3D_CUDA_TRY(cudaMemset(g_role_clk, 0, bytes));
        g_role_clk_ctas = n_sm;
    }
    *out = g_role_clk;
    return P3D_OK;
}
#endif

}  // namespace

#ifdef P3D_WS3_ROLE_CLOCKS
// Copies the accumulated role counters ([CTA][kRoles][kRcSlots] cycles, at most `cap` values) to `host` after a device
// synchronise and zeroes them when `reset`.  Returns the number of values, or a (negative) P3D error.
extern "C" long long p3d_ws3_role_clocks(unsigned long long* host, long long cap, int reset) {
    int n_sm;
    unsigned long long* buf;
    if (int rc = sm_count(&n_sm)) return rc;
    if (int rc = role_clocks_buffer(n_sm, &buf)) return rc;
    const long long n = (long long)g_role_clk_ctas * kRoles * kRcSlots;
    if (cudaDeviceSynchronize() != cudaSuccess) return P3D_ECUDA;
    if (host && cap >= n && cudaMemcpy(host, buf, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess) return P3D_ECUDA;
    if (reset && cudaMemset(buf, 0, n * sizeof(unsigned long long)) != cudaSuccess) return P3D_ECUDA;
    return n;
}
#endif

bool fused_ws3_supported(const Geom& g) {
    if (!((g.S == 96 || g.S == 48) && (g.Sf == g.S) && ((long long)g.M % (384 / g.S) == 0))) return false;
    if ((g.stride_view | g.stride_plane | g.stride_row | g.stride_col) & 7) return false;
    return tap_offsets_fit(g);
}

int render_forward_fused_ws3(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                            const float* w2, const float* b2, const float* ro, const float* rd, const float* u_c,
                            const float* u_f, const Workspace& ws, float* out_rgb, float* out_depth, float* out_wsum,
                            float* out_xyz, cudaStream_t stream) {
    if (!fused_ws3_supported(g)) {
        set_error("fused warp-specialised renderer supports depth_resolution == depth_resolution_importance in {48, 96}, rays per "
                  "view a multiple of 384 / depth_resolution, planes of at least 2x2 texels and strides that are multiples of "
                  "8 elements (got %d + %d samples, %d rays, stride_col %lld)", g.S, g.Sf, g.M, (long long)g.stride_col);
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
    int n_sm;
    if ((rc = sm_count(&n_sm))) return rc;
#ifdef P3D_WS3_ROLE_CLOCKS
    if ((rc = role_clocks_buffer(n_sm, &a.role_clk))) return rc;
#endif
    const size_t smem = kSmemWS;
    void (*kern)(WsArgs) = with_texel_stride(g, [&](auto sc) -> void (*)(WsArgs) {
        if (g.S == 96) return p->planes_bf16 ? k_render_ws3<true, 96, sc.value> : k_render_ws3<false, 96, sc.value>;
        return p->planes_bf16 ? k_render_ws3<true, 48, sc.value> : k_render_ws3<false, 48, sc.value>;
    });
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int carveout;
    if ((rc = smem_carveout_percent(smem, &carveout))) return rc;
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
    const int grid = a.n_groups < n_sm ? a.n_groups : n_sm;
    {
        ProfileScope prof(PROF_FUSED, stream);
        kern<<<grid, kThreadsWS, smem, stream>>>(a);
        P3D_LAUNCH_CHECK();
    }
    if (p->defer_depth_clamp) return P3D_OK;
    return launch_depth_finalize(out_depth, R, ws.bounds, stream);
}

}  // namespace p3d
