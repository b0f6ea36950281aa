// The fused renderer: warp-specialised, pipeline depth 3 - THREE ray groups in flight.
//
//   passes C(0) C(1) | F(0) C(2) | F(1) C(3) | ... | F(N-2) F(N-1)          (C = 3 coarse tiles, F = 3 importance tiles)
//
// A tile's colour sigmoids wait for the group's compositing weights (omega), which exist only after its fine pass.  They are
// staged in global memory, in this CTA's own slice of the workspace colour buffers (see colour_area: coarse areas
// CA[n % 3] and one fine area FA, 4 x 48 KB per CTA, ~25 MB on 132 SMs).  The areas are rewritten every few groups, so
// their footprint fits the 50 MB L2, but they share it with the streamed tri-plane gather; how much of the round trip is
// served by L2 rather than HBM has not been measured.  Both directions are bulk copies of whole 8 KB tile halves: the
// epilogue stages them in shared memory for one cp.async.bulk store, and a group's tiles come back into shared memory
// buffers (mbarrier complete_tx) while the decoder runs C(n+2), so colours(n) reduces from shared memory.  Only
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
//                          -> softplus2 in registers -> layer 2 (one m64n48 wgmma, A from the registers): colour sigmoids ->
//                          staging tile -> bulk store to the colour area, sigma -> group state; bulk loads of a group's
//                          colours and their reduction once its omega is ready
//   warps 20-23  RAY       a warp per ray: importance sampling after a group's coarse pass, merge / transmittance /
//                          omega and the per-ray outputs after its fine pass
#include "fused_common.cuh"

namespace p3d {

namespace {

using namespace dev;
using namespace fused;

constexpr int kGW = 12, kEW = 8, kRW = 4, kTeams = 3;   // 24 warps = 6 warpgroups -> 80 registers per thread
constexpr int kWarpsWS = kGW + kEW + kRW;
constexpr int kThreadsWS = kWarpsWS * 32;        // 768
constexpr int kNA = 4;                           // A1 ring depth
// registers per thread by role (launched with 80 = 65536 / 768 rounded down to 8): the decoder warpgroups hold the layer-2
// A operands and accumulators at once and take what the ray warpgroup does not need; 3 x 80 + 2 x kRegE + kRegR <= 6 x 80
constexpr int kRegE = 88, kRegR = 64;
static_assert(3 * 80 + 2 * kRegE + kRegR <= 6 * 80, "per-role registers exceed what the launch allocates");
constexpr int kStates = 4;                       // per-group state ring
constexpr int kRowsG = 384;                      // rows per pass per group
constexpr int kColBufs = 3;                      // colour tiles of a group in shared memory at once (colours())
constexpr int kHalfBytes = 64 * kRgb * 4;        // one decoder warpgroup's 64 rows of colour sigmoids: 8 KB


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
    float col_stage[2][64 * kRgb];                // per decoder warpgroup: its half of the tile being stored (col_idx layout)
    float col_buf[kColBufs][128 * kRgb];          // colour tiles loaded back for colours(), same layout
    unsigned char w1[2][4096], w2[2][kD2Cols * 128];
    float b1[kHidden], b2c[kRgb], b2s, pad0[3];
    uint4 tab[kGW][32][4];                        // tap table of a gather warp's 32 rows (see "gather" below)
    GroupState st[kStates];
    SlotState slot[2];
    float rscratch[kRW][768];                      // private scratch of each ray warp (importance / merge)
    unsigned long long a1_full[kNA], a1_empty[kNA];
    unsigned long long fine_ready[kStates], state_free[kStates];
    unsigned long long sigc_ready[kStates], sigf_ready[kStates], omega_ready[2];   // E -> R (sigma in smem), R -> E (omega)
    unsigned long long col_full[kColBufs];        // both warpgroups' halves of a col_buf tile have landed (complete_tx)
};

// Float index of colour (row, c) in a staged / loaded colour tile: 128 B rows, 16-byte chunk (c / 4) XOR (row % 8).  The
// epilogue's float2 stores (8 rows x 4 column pairs per instruction) and the reduction's lane = channel loads are both
// conflict-free.  The colour areas in global memory are byte copies of the tiles, so they hold the same layout.
__device__ __forceinline__ int col_idx(int row, int c) { return row * kRgb + ((((c >> 2) ^ row) & 7) << 2) + (c & 3); }

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
        for (int i = 0; i < kColBufs; ++i) mbar_init(&sm.col_full[i], 2);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    stage_w1_biases(g, a.w1, a.b1, a.b2, sm.w1, sm.b1, sm.b2c, sm.b2s, tid, kThreadsWS);
    stage_w2(g, a.w2, sm.w2, kD2Cols, kLBO_W2, w2_row_n48, tid, kThreadsWS);
    fence_proxy_async();
    __syncthreads();

    if (warp < kGW) {
        // =========================================================================== GATHER
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
            if (td.pass == 0) mbar_wait(&sm.state_free[td.n & 3], ((td.n >> 2) & 1) ^ 1);
            else mbar_wait(&sm.fine_ready[td.n & 3], (td.n >> 2) & 1);
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
            const int stage = my_it % kNA;
            mbar_wait(&sm.a1_empty[stage], ((my_it / kNA) & 1) ^ 1);
            gather_a1<BF16, SCOL>(tab, reinterpret_cast<const char*>(a.planes) + (long long)view * g.stride_view * kEsz, 0 /* one view */, srowB,
                                  scolB, v, sm.a1[stage][0], sm.a1[stage][1], wt, lane);
            fence_proxy_async();
            __syncwarp();                                                   // also: the tap table is rewritten by the next tile
            if (lane == 0) mbar_arrive(&sm.a1_full[stage]);
        }
    } else if (warp < kGW + kEW) {
        // =========================================================================== DECODER
        setmaxnreg_inc<kRegE>();
        const int e = warp - kGW, quarter = e & 3, chunk = e >> 2;      // chunk = warpgroup = 64-row half of a tile
        const int etid = tid - kGW * 32;                                  // 0..255 inside the decoder group
        const bool elect = (etid & 127) == 0;                             // the warpgroup's bulk-copy thread
        // this CTA's colour area of (group n, pass): 384 rows x 32 sigmoids, row = 128 k + row of tile k, each tile in the
        // col_idx layout (a byte copy of the staged tile).  Areas are slices of the workspace colour buffers that belong to this
        // CTA's own first two groups (coarse and fine buffer each), so they exist whenever they are used: CA[0..2] = slices
        // 0..2, FA = slice 3 (slice 1 when the CTA has a single group)
        auto colour_area = [&](int n, int pass) -> float* {
            const int j = pass == 0 ? n % 3 : (n_my >= 2 ? 3 : 1);
            return ((j & 1) ? a.col_f : a.col_c) + ((long long)blockIdx.x + (long long)(j >> 1) * gridDim.x) * (kRowsG * kRgb);
        };
        auto ebar = [] { asm volatile("bar.sync 1, 256;" ::: "memory"); };   // the eight decoder warps
        auto wgbar = [chunk] { asm volatile("bar.sync %0, 128;" ::"r"(2 + chunk) : "memory"); };   // this warpgroup's four warps
        // Colour tile t of a group (t = 0..2: coarse tile t, 3..5: fine tile t - 3) is loaded into col_buf[t % kColBufs].  Each
        // warpgroup loads back the half it stored itself, so the only stores a load depends on are the issuing thread's own.
        auto load_tile = [&](int n, int t) {                             // elected thread only
            const int pass = t / 3, b = t % kColBufs;
            mbar_arrive_expect_tx(&sm.col_full[b], kHalfBytes);
            bulk_load(smem_u32(sm.col_buf[b]) + chunk * kHalfBytes, colour_area(n, pass) + ((t - 3 * pass) * 128 + 64 * chunk) * kRgb,
                      kHalfBytes, &sm.col_full[b]);
        };
        // The first kColBufs tiles of group n are requested once its fine pass is stored: in the epilogue of the next tile,
        // C(n+2)'s first, so they arrive while the decoder runs C(n+2) - or at the top of colours(n) where no C(n+2) exists.
        // A full wait_group (the stores are written, not just read) and the proxy fence make the area readable by the loads.
        int stored = -1, loaded = -1;                                     // last group whose fine pass was stored / first tiles requested
        auto first_loads = [&](int n) {
            if (elect) {
                bulk_wait_all();
                fence_proxy_async_global();
#pragma unroll 1
                for (int t = 0; t < kColBufs; ++t) load_tile(n, t);
            }
            loaded = n;
        };
        auto colours = [&](int n) {                                        // sum_j omega_j * rgb_j for group n
            if (loaded < n) first_loads(n);
            const int slot_i = n & 1;
            SlotState& sl = sm.slot[slot_i];
            mbar_wait(&sm.omega_ready[slot_i], (n >> 1) & 1);              // omega / pos / back of group n (ray warps)
            const int grp = (int)blockIdx.x + n * (int)gridDim.x;
            const long long ray0 = (long long)grp * GR;
            // Warp e sums rows [16 e, 16 e + 16) of each of the six tiles - always one ray, rl - with lane = channel, in a fixed
            // order.  The partial sums of a ray meet in sl.acc as one (S = 48) or two (S = 96: warps 2 rl, 2 rl + 1)
            // shared-memory adds onto 0, whose order cannot change the rounded sum: the kernel is bit-reproducible run to run
            // and independent of how the rays are batched.
            const int rl = 16 * e / RPT;
            const bool live = ray0 + rl < a.R;
            float part = 0.f;
#pragma unroll 1
            for (int t = 0; t < 6; ++t) {
                const int pass = t / 3, k = t - 3 * pass, b = t % kColBufs;
                mbar_wait(&sm.col_full[b], ((6 * n + t) / kColBufs) & 1);
                const float* buf = sm.col_buf[b];
                const unsigned short* pos = sl.pos + pass * kRowsG + rl * S + k * RPT - rl * RPT;   // pos[trow]: the row's merged position
#pragma unroll 4
                for (int j = 0; j < 16; ++j) {
                    const int trow = 16 * e + j;
                    const float om = live ? sl.om[rl * L + pos[trow]] : 0.f;
                    const float ca = g.force_sigmoid ? om : 1.002f * om, cb = g.force_sigmoid ? 0.f : -0.001f * om;
                    part += fmaf(buf[col_idx(trow, lane)], ca, cb);
                }
                if (t + kColBufs < 6) {
                    wgbar();                                               // this warpgroup's half of col_buf[b] is read
                    if (elect) load_tile(n, t + kColBufs);
                }
            }
            atomicAdd(&sl.acc[rl][lane], part);
            ebar();                                                        // all eight decoder warps (also: the buffers are read)
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
        const uint32_t w1h = smem_u32(sm.w1[0]), w1l = smem_u32(sm.w1[1]), w2h = smem_u32(sm.w2[0]), w2l = smem_u32(sm.w2[1]);
        float* stage_tile = sm.col_stage[chunk];
        for (int it = 0; it < T; ++it) {
            const TileDesc td = tile_at(it, n_my);
            if (td.pass == 1 && td.k == 0 && td.n >= 1) colours(td.n - 1);
            const int stage = it % kNA;
            mbar_wait(&sm.a1_full[stage], (it / kNA) & 1);
            float d1[32];
            decoder_layer1(d1, smem_u32(sm.a1[stage][0]), smem_u32(sm.a1[stage][1]), kLBO_A1, w1h, w1l, kLBO_W1, chunk, a.single_pass);
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.a1_empty[stage]);
            uint32_t ah[16], al[16];
            decoder_hidden(d1, sm.b1, lane, ah, al);
            float d2[kD2Cols / 2];
            decoder_layer2_issue<kD2Cols>(d2, ah, al, w2h, w2l, kLBO_W2, a.single_pass);
            wgmma_commit();
            wgmma_wait_all();
            fence_operands(d2);
            // the staging half is free once the bulk store of the previous tile has read it
            if (stored > loaded) first_loads(stored);
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
                bulk_store(colour_area(td.n, td.pass) + (td.k * 128 + 64 * chunk) * kRgb, smem_u32(stage_tile), kHalfBytes);
                bulk_commit();
            }
            if (td.k == 2) {                                              // the group's pass is complete: hand its sigma to the ray warps
                if (td.pass == 1) stored = td.n;
                __syncwarp();
                if (lane == 0) mbar_arrive(td.pass == 0 ? &sm.sigc_ready[td.n & 3] : &sm.sigf_ready[td.n & 3]);
            }
        }
        colours(n_my - 1);
    } else if (warp < kGW + kEW + kRW) {
        // =========================================================================== RAY (one warp per ray)
        setmaxnreg_dec<kRegR>();
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
        for (int j = 0; j < 2 * n_my; ++j) {
            const PassDesc pd = pass_at(j, n_my);
            const int n = pd.n, si = n & 3;
            const uint32_t par = (n >> 2) & 1;
            if (pd.pass == 0) {
                mbar_wait(&sm.sigc_ready[si], par);
                for (int rl = rw; rl < GR; rl += kRW) importance_ray(n, rl);
                if (lane == 0) mbar_arrive(&sm.fine_ready[si]);
            } else {
                mbar_wait(&sm.sigf_ready[si], par);
                if (n >= 2) mbar_wait(&sm.state_free[(n - 2) & 3], ((n - 2) >> 2) & 1);       // colours(n-2) has released the omega slot
                for (int rl = rw; rl < GR; rl += kRW) composite_ray(n, rl);
                if (lane == 0) mbar_arrive(&sm.omega_ready[n & 1]);
            }
        }
    }
}

}  // namespace

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
    const size_t smem = sizeof(WsSmem) + 1024;
    void (*kern)(WsArgs) = with_texel_stride(g, [&](auto sc) -> void (*)(WsArgs) {
        if (g.S == 96) return p->planes_bf16 ? k_render_ws3<true, 96, sc.value> : k_render_ws3<false, 96, sc.value>;
        return p->planes_bf16 ? k_render_ws3<true, 48, sc.value> : k_render_ws3<false, 48, sc.value>;
    });
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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
