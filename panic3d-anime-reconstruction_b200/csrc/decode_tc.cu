// Streaming tensor-core decode of tri-plane points: p3d_decode_points (ImportanceRenderer.run_model, renderer.py:266-280) and
// p3d_volume_query (get_eg3d_volume, _util/eg3d_metrics3d.py:94-183) when mlp_mode is P3D_MLP_TC_*.
//
// The renderer's gather -> tensor-core decoder pipeline without any per-ray phase, so nothing ever waits on a dependency chain:
//
//   warps  0-11  GATHER    three teams of four warps; team j takes tiles j, j+3, ... ; a warp owns 32 points of its tile:
//                          position (given coordinates, or the reference's sheared voxel lattice generated in-kernel) -> tap
//                          table -> 12 x 128-bit loads per lane -> FMA lerp -> bf16 hi/lo A1 tile (4-stage ring)
//   warps 12-19  DECODER   two warpgroups, one per 64-row half of every tile: layer 1 (wgmma, A1 and W1 from shared memory)
//                          -> softplus2 in registers -> layer 2 (wgmma, N = 48: 32 colour logits, sigma, 15 zero rows; A from
//                          the registers) -> sigma / sigmoid colours -> global (and, for the volume query, density with the crop
//                          / cull overwrites and the lattice coordinates, written where the reference's reshape + flip puts them)
//
// A tile is 128 consecutive points; CTA b of the persistent grid takes tiles b, b + grid, ...
#include "fused_common.cuh"

namespace p3d {

namespace {

using namespace dev;
using namespace fused;

constexpr int kGW = 12, kEW = 8, kTeams = 3;
constexpr int kWarpsD = kGW + kEW;
constexpr int kThreadsD = kWarpsD * 32;          // 640
constexpr int kNA = 4;                           // A1 ring depth

struct __align__(1024) DecSmem {
    unsigned char a1[kNA][2][4 * kLBO_A1];
    unsigned char w1[2][4096], w2[2][6144];
    float b1[kHidden], b2c[kRgb], b2s, pad0[3];
    uint4 tab[kGW][32][4];
    unsigned long long a1_full[kNA], a1_empty[kNA];
};

struct DecArgs {
    Geom g;
    const void* planes;
    const float *w1, *b1, *w2, *b2;
    const float* coords;          // points mode: (N, K, 3); volume mode: nullptr
    float *out_sigma, *out_rgb, *out_density, *out_coords;
    long long total, per_view;
    int single_pass, n_tiles;
    int srow, scol, splane;
    VolumeSpec vol;               // volume mode
};

template <bool BF16, bool VOLUME, int SCOL>
__global__ void __launch_bounds__(kThreadsD, 1) k_decode_tc(const DecArgs a) {
    extern __shared__ unsigned char smem_raw[];
    DecSmem& sm = *reinterpret_cast<DecSmem*>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
    const Geom& g = a.g;
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int n_my = (a.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // tiles of this CTA

    if (tid == 0) {
        for (int i = 0; i < kNA; ++i) { mbar_init(&sm.a1_full[i], 4); mbar_init(&sm.a1_empty[i], kEW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    stage_w1_biases(g, a.w1, a.b1, a.b2, sm.w1, sm.b1, sm.b2c, sm.b2s, tid, kThreadsD);
    stage_w2(g, a.w2, sm.w2, kD2Cols, kLBO_W2, w2_row_n48, tid, kThreadsD);
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
        for (int it = team; it < n_my; it += kTeams) {
            const long long tile = (long long)blockIdx.x + (long long)it * gridDim.x;
            // ---- tap table of this warp's 32 points: lane = point
            {
                const long long gidx = tile * 128 + wt * 32 + lane;
                float px = 1e30f, py = 1e30f, pz = 1e30f;
                long long view = 0;
                if (gidx < a.total) {
                    view = gidx / a.per_view;
                    if (VOLUME) volume_point(gidx - view * a.per_view, a.vol.res, a.vol.size, a.vol.origin, px, py, pz);
                    else { px = a.coords[gidx * 3]; py = a.coords[gidx * 3 + 1]; pz = a.coords[gidx * 3 + 2]; }
                }
                write_tap_row(tab, lane, g, a.srow, a.scol, a.splane, px, py, pz, (uint32_t)view);   // a tile may straddle two views
            }
            __syncwarp();
            const int stage = it % kNA;
            mbar_wait(&sm.a1_empty[stage], ((it / kNA) & 1) ^ 1);
            gather_a1<BF16, SCOL>(tab, reinterpret_cast<const char*>(a.planes), g.stride_view * kEsz, srowB, scolB, v, sm.a1[stage][0],
                                  sm.a1[stage][1], wt, lane);
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.a1_full[stage]);
        }
    } else {
        // =========================================================================== DECODER (two warpgroups)
        const int e = warp - kGW, half = e >> 2, w = e & 3;
        const uint32_t w1h = smem_u32(sm.w1[0]), w1l = smem_u32(sm.w1[1]), w2h = smem_u32(sm.w2[0]), w2l = smem_u32(sm.w2[1]);
        for (int it = 0; it < n_my; ++it) {
            const int stage = it % kNA;
            mbar_wait(&sm.a1_full[stage], (it / kNA) & 1);
            float d1[32];
            decoder_layer1(d1, smem_u32(sm.a1[stage][0]), smem_u32(sm.a1[stage][1]), kLBO_A1, w1h, w1l, kLBO_W1, half, a.single_pass);
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.a1_empty[stage]);
            uint32_t ah[16], al[16];
            decoder_hidden(d1, sm.b1, lane, ah, al);
            float d2[kD2Cols / 2];
            decoder_layer2_issue<kD2Cols>(d2, ah, al, w2h, w2l, kLBO_W2, a.single_pass);
            wgmma_commit();
            wgmma_wait_all();
            fence_operands(d2);
            // this thread's two rows (fragment elements 2 rs, 2 rs + 1 of each 8-column block): colours [0, 32) in column
            // pairs, sigma = column 32 (lanes with l % 4 == 0), the volume lattice coordinates from the l % 4 == 1 lanes
            const long long tile = (long long)blockIdx.x + (long long)it * gridDim.x;
#pragma unroll
            for (int rs = 0; rs < 2; ++rs) {
                const long long gidx = tile * 128 + 64 * half + frag_row(2 * rs, lane, w);
                if (gidx >= a.total) continue;
                long long dest = gidx, n = 0;
                if (VOLUME) {
                    const long long view = gidx / a.per_view;
                    n = gidx - view * a.per_view;
                    dest = view * a.per_view + volume_dest(n, a.vol.res);
                }
                if (a.out_rgb) {
#pragma unroll
                    for (int blk = 0; blk < 4; ++blk) {
                        const int i = 4 * blk + 2 * rs, c = frag_col(i, lane);
                        float o[2];
#pragma unroll
                        for (int j = 0; j < 2; ++j) {
                            const float s = rcp_approx(1.f + ex2_approx(d2[i + j] + sm.b2c[c + j]));
                            o[j] = g.force_sigmoid ? s : __fsub_rn(__fmul_rn(s, 1.002f), 0.001f);
                        }
                        *reinterpret_cast<float2*>(a.out_rgb + dest * kRgb + c) = make_float2(o[0], o[1]);
                    }
                }
                if ((lane & 3) == 0) {
                    const float sg = d2[16 + 2 * rs] + sm.b2s;
                    a.out_sigma[dest] = sg;
                    if (VOLUME && a.out_density) {
                        float x, y, z;
                        volume_point(n, a.vol.res, a.vol.size, a.vol.origin, x, y, z);
                        a.out_density[dest] = volume_density(a.vol, sg, x, z);
                    }
                } else if (VOLUME && a.out_coords && (lane & 3) == 1) {
                    float x, y, z;
                    volume_point(n, a.vol.res, a.vol.size, a.vol.origin, x, y, z);
                    a.out_coords[dest * 3 + 0] = x; a.out_coords[dest * 3 + 1] = y; a.out_coords[dest * 3 + 2] = z;
                }
            }
        }
    }
}

template <bool VOLUME>
int launch_decode(const Geom& g, const p3d_render_params* p, DecArgs& a, cudaStream_t stream) {
    int n_sm, rc;
    if ((rc = sm_count(&n_sm))) return rc;
    a.g = g;
    a.single_pass = p->mlp_mode == P3D_MLP_TC_BF16;
    a.srow = (int)g.stride_row; a.scol = (int)g.stride_col; a.splane = (int)g.stride_plane;
    a.n_tiles = (int)((a.total + 127) / 128);
    void (*kern)(DecArgs) = with_texel_stride(g, [&](auto sc) -> void (*)(DecArgs) {
        return p->planes_bf16 ? k_decode_tc<true, VOLUME, sc.value> : k_decode_tc<false, VOLUME, sc.value>;
    });
    const size_t smem = sizeof(DecSmem) + 1024;
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = a.n_tiles < n_sm ? a.n_tiles : n_sm;
    ProfileScope prof(PROF_SAMPLE_DECODE, stream);
    kern<<<grid, kThreadsD, smem, stream>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace

// int tile indices, and the view index in the 24 high bits of a tap row's flags
bool decode_tc_supported(const Geom& g, long long total) {
    return total < (128ll << 31) && g.N < (1 << 24) && tap_offsets_fit(g);
}

int decode_points_tc(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                     const float* w2, const float* b2, const float* coords, long long n_pts, float* out_rgb,
                     float* out_sigma, cudaStream_t stream) {
    DecArgs a{};
    a.planes = planes; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2; a.coords = coords;
    a.out_sigma = out_sigma; a.out_rgb = out_rgb;
    a.total = (long long)g.N * n_pts; a.per_view = n_pts;
    return launch_decode<false>(g, p, a, stream);
}

int volume_query_tc(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                    const float* w2, const float* b2, const VolumeSpec& vol, float* out_sigma, float* out_rgb,
                    float* out_density, float* out_coords, cudaStream_t stream) {
    DecArgs a{};
    a.planes = planes; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2;
    a.out_sigma = out_sigma; a.out_rgb = out_rgb; a.out_density = out_density; a.out_coords = out_coords;
    a.per_view = (long long)vol.res * vol.res * vol.res; a.total = (long long)g.N * a.per_view;
    a.vol = vol;
    return launch_decode<true>(g, p, a, stream);
}

}  // namespace p3d
