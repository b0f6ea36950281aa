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
#include <stdlib.h>
#include "fused_common.cuh"

namespace p3d {

namespace {

using namespace dev;
using namespace fused;

constexpr int kGW = 12, kEW = 8, kTeams = 3;
constexpr int kWarpsD = kGW + kEW;
constexpr int kThreadsD = kWarpsD * 32;          // 640
constexpr int kNA = 4;                           // A1 ring depth
constexpr int kD2Cols = 48;
constexpr int kLBO_A1 = 2080, kLBO_W1 = 1024, kLBO_W2 = 768;

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
    // volume mode (see render_v1.cu: volume_point / volume_dest)
    int vol_res;
    float vol_size, vol_origin, vol_crop, vol_cull;
    int vol_crop_on, vol_cull_on;
};

// point n of the reference's create_samples lattice, bit for bit (eg3d_metrics3d.py:70-92: un-floored float y / x "indices")
__device__ __forceinline__ void volume_point(long long n, int R, float vsize, float vorigin, float& x, float& y, float& z) {
    const float nf = (float)n, Rf = (float)R;
    const float iz = (float)(n % R);
    const float q1 = __fdiv_rn(nf, Rf);
    const float iy = fmodf(q1, Rf);
    const float ix = fmodf(__fdiv_rn(q1, Rf), Rf);
    x = __fadd_rn(__fmul_rn(ix, vsize), vorigin);
    y = __fadd_rn(__fmul_rn(iy, vsize), vorigin);
    z = __fadd_rn(__fmul_rn(iz, vsize), vorigin);
}
__device__ __forceinline__ long long volume_dest(long long n, int R) {
    const long long rr = (long long)R * R;
    const long long a = n / rr, rest = n - a * rr;
    return ((long long)(R - 1) - a) * rr + rest;
}

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
    for (int i = tid; i < kHidden * kC; i += kThreadsD) {             // W1' = W1 * gain * log2(e) / 3   (64 x 32)
        const int n = i / kC, k = i % kC;
        unsigned short hi, lo;
        split1(__fmul_rn(a.w1[i], g.w1_gain) * (kLog2e / 3.f), hi, lo);
        const int off = tile_off(n, k, kLBO_W1);
        *reinterpret_cast<unsigned short*>(sm.w1[0] + off) = hi;
        *reinterpret_cast<unsigned short*>(sm.w1[1] + off) = lo;
    }
    for (int i = tid; i < kD2Cols * kHidden; i += kThreadsD) {        // rows 0..31: -W2 colour rows; row 32: W2 sigma row * ln2; 33..47: 0
        const int n = i / kHidden, k = i % kHidden;
        unsigned short hi = 0, lo = 0;
        if (n < kRgb) split1(-__fmul_rn(a.w2[(n + 1) * kHidden + k], g.w2_gain), hi, lo);
        else if (n == kRgb) split1(__fmul_rn(a.w2[k], g.w2_gain) * kLn2, hi, lo);
        const int off = tile_off(n, k, kLBO_W2);
        *reinterpret_cast<unsigned short*>(sm.w2[0] + off) = hi;
        *reinterpret_cast<unsigned short*>(sm.w2[1] + off) = lo;
    }
    if (tid < kHidden) sm.b1[tid] = __fmul_rn(a.b1[tid], g.b1_gain) * kLog2e;
    if (tid < kRgb) sm.b2c[tid] = -__fmul_rn(a.b2[tid + 1], g.b2_gain) * kLog2e;
    if (tid == 0) sm.b2s = __fmul_rn(a.b2[0], g.b2_gain);
    fence_proxy_async();
    __syncthreads();

    if (warp < kGW) {
        // =========================================================================== GATHER
        const int gw = warp, team = gw >> 2, wt = gw & 3;
        constexpr int kEsz = BF16 ? 2 : 4;
        const long long scolB = (long long)a.scol * kEsz, srowB = (long long)a.srow * kEsz;
        unsigned char* tab = reinterpret_cast<unsigned char*>(sm.tab[gw]);
        float v4[12][4];
#pragma unroll
        for (int k = 0; k < 12; ++k)
#pragma unroll
            for (int c = 0; c < 4; ++c) v4[k][c] = 0.f;
        const int sub = lane >> 3, qd = lane & 7;
        constexpr int kImmX4 = SCOL * kEsz;
        for (int it = team; it < n_my; it += kTeams) {
            const long long tile = (long long)blockIdx.x + (long long)it * gridDim.x;
            // ---- tap table of this warp's 32 points: lane = point
            long long view_w = 0;
            {
                const long long gidx = tile * 128 + wt * 32 + lane;
                float px = 1e30f, py = 1e30f, pz = 1e30f;
                if (gidx < a.total) {
                    const long long view = gidx / a.per_view;
                    if (VOLUME) volume_point(gidx - view * a.per_view, a.vol_res, a.vol_size, a.vol_origin, px, py, pz);
                    else { px = a.coords[gidx * 3]; py = a.coords[gidx * 3 + 1]; pz = a.coords[gidx * 3 + 2]; }
                    view_w = view;
                }
                const bool pm = g.plane_mode == P3D_PLANES_PANIC3D;
                uint32_t o0, o1, o2;
                float4 w0, w1, w2;
                const bool f0 = plane_taps_rec(g, a.srow, a.scol, 0, px, py, o0, w0);
                const bool f1 = plane_taps_rec(g, a.srow, a.scol, a.splane, px, pz, o1, w1);
                const bool f2 = plane_taps_rec(g, a.srow, a.scol, 2 * a.splane, pm ? py : pz, pm ? pz : px, o2, w2);
                // a tile may straddle two views: the view index travels with the row (bits 8.. of the flags word)
                *reinterpret_cast<uint4*>(tab + tab_off(lane, 0)) = make_uint4(o0, o1, o2, (f0 ? 1u : 0u) | (f1 ? 2u : 0u) | (f2 ? 4u : 0u) | ((uint32_t)view_w << 8));
                *reinterpret_cast<float4*>(tab + tab_off(lane, 1)) = w0;
                *reinterpret_cast<float4*>(tab + tab_off(lane, 2)) = w1;
                *reinterpret_cast<float4*>(tab + tab_off(lane, 3)) = w2;
            }
            __syncwarp();
            const int stage = it % kNA;
            mbar_wait(&sm.a1_empty[stage], ((it / kNA) & 1) ^ 1);
            unsigned char* a1h = sm.a1[stage][0];
            unsigned char* a1l = sm.a1[stage][1];
            const char* pq = reinterpret_cast<const char*>(a.planes) + (long long)(4 * qd) * kEsz;
#pragma unroll 1
            for (int round = 0; round < 8; ++round) {
                const int lrow = round * 4 + sub;
                const uint4 c0 = *reinterpret_cast<const uint4*>(tab + tab_off(lrow, 0));
                const bool p0 = c0.w & 1u, p1 = c0.w & 2u, p2 = c0.w & 4u;
                const char* vq4 = pq + (long long)(c0.w >> 8) * g.stride_view * kEsz;
                const char* b0 = vq4 + (unsigned long long)c0.x * kEsz;
                const char* b1 = vq4 + (unsigned long long)c0.y * kEsz;
                const char* b2 = vq4 + (unsigned long long)c0.z * kEsz;
#define P3D_LD4(k, base, pr)                                                                                         \
                load_quad_p<BF16, 0>(v4[k], base, pr);                                                                \
                if (SCOL) load_quad_p<BF16, kImmX4>(v4[k + 1], base, pr); else load_quad_p<BF16, 0>(v4[k + 1], base + scolB, pr); \
                load_quad_p<BF16, 0>(v4[k + 2], base + srowB, pr);                                                    \
                if (SCOL) load_quad_p<BF16, kImmX4>(v4[k + 3], base + srowB, pr); else load_quad_p<BF16, 0>(v4[k + 3], base + srowB + scolB, pr);
                P3D_LD4(0, b0, p0)
                P3D_LD4(4, b1, p1)
                P3D_LD4(8, b2, p2)
#undef P3D_LD4
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
                    dest = view * a.per_view + volume_dest(n, a.vol_res);
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
                        // sigma2density, then the crop / cull overwrites; the reference applies cull_clouds_mask to the DENSITIES
                        // (eg3d_metrics3d.py:155-162 -> renderer.py:150-153): the threshold acts on the twice-transformed value
                        float x, y, z;
                        volume_point(n, a.vol_res, a.vol_size, a.vol_origin, x, y, z);
                        float dens = 1.f - expf(-softplus_t(__fsub_rn(sg, 1.f)));
                        if (a.vol_crop_on && !((fabsf(x) <= a.vol_crop) && (fabsf(z) <= a.vol_crop))) dens = -1e3f;
                        if (a.vol_cull_on && (1.f - expf(-softplus_t(__fsub_rn(dens, 1.f)))) < a.vol_cull) dens = -1e3f;
                        a.out_density[dest] = dens;
                    }
                } else if (VOLUME && a.out_coords && (lane & 3) == 1) {
                    float x, y, z;
                    volume_point(n, a.vol_res, a.vol_size, a.vol_origin, x, y, z);
                    a.out_coords[dest * 3 + 0] = x; a.out_coords[dest * 3 + 1] = y; a.out_coords[dest * 3 + 2] = z;
                }
            }
        }
    }
}

template <bool VOLUME>
int launch_decode(const Geom& g, const p3d_render_params* p, DecArgs& a, cudaStream_t stream) {
    static int n_sm = 0;
    if (!n_sm) {
        int dev = 0;
        P3D_CUDA_TRY(cudaGetDevice(&dev));
        P3D_CUDA_TRY(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    a.g = g;
    a.single_pass = p->mlp_mode == P3D_MLP_TC_BF16;
    a.srow = (int)g.stride_row; a.scol = (int)g.stride_col; a.splane = (int)g.stride_plane;
    a.n_tiles = (int)((a.total + 127) / 128);
    const int sc = g.stride_col == kC ? 1 : (g.stride_col == 3 * kC ? 2 : 0);      // static texel stride: layout pre-pass / zero-copy channels_last
#define P3D_PICK(BF) (sc == 1 ? k_decode_tc<BF, VOLUME, kC> : (sc == 2 ? k_decode_tc<BF, VOLUME, 3 * kC> : k_decode_tc<BF, VOLUME, 0>))
    void (*kern)(DecArgs) = p->planes_bf16 ? P3D_PICK(true) : P3D_PICK(false);
#undef P3D_PICK
    const size_t smem = sizeof(DecSmem) + 1024;
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = a.n_tiles < n_sm ? a.n_tiles : n_sm;
    ProfileScope prof(PROF_SAMPLE_DECODE, stream);
    kern<<<grid, kThreadsD, smem, stream>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace

// 32-bit tap offsets inside one view's tri-plane, 2 x 2 footprints clamped into the plane, 16-byte vector loads
bool decode_tc_supported(const Geom& g, long long total) {
    const long long span = 2 * g.stride_plane + (long long)(g.H - 1) * g.stride_row + (long long)(g.W - 1) * g.stride_col + kC;
    if (g.H < 2 || g.W < 2 || total >= (128ll << 31) || g.N >= (1 << 24)) return false;
    return g.stride_plane >= 0 && g.stride_row >= 0 && g.stride_col >= 0 && span < (1ll << 31);
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
                    const float* w2, const float* b2, int res, double cube_length, double triplane_crop, double cull_clouds,
                    float* out_sigma, float* out_rgb, float* out_density, float* out_coords, cudaStream_t stream) {
    DecArgs a{};
    a.planes = planes; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2;
    a.out_sigma = out_sigma; a.out_rgb = out_rgb; a.out_density = out_density; a.out_coords = out_coords;
    a.per_view = (long long)res * res * res; a.total = (long long)g.N * a.per_view;
    a.vol_res = res;
    a.vol_size = (float)(cube_length / (double)(res - 1));          // python float -> fp32 scalar operand
    a.vol_origin = (float)(0.0 - cube_length / 2.0);
    a.vol_crop = triplane_crop >= 0 ? (float)(p->box_warp / 2.0 - triplane_crop) : -1.f;    // renderer.py:139-148
    a.vol_cull = cull_clouds >= 0 ? (float)cull_clouds : -1.f;
    a.vol_crop_on = triplane_crop >= 0; a.vol_cull_on = cull_clouds >= 0;
    return launch_decode<true>(g, p, a, stream);
}

}  // namespace p3d
