// v1 renderer: multi-kernel SIMT pipeline, fp32 throughout.
//
// This is the parity kernel set (P3D_MLP_FP32_SIMT): every arithmetic step is plain fp32 in
// the same order class as the reference's ATen ops, so it tracks the CPU oracle to ~1e-6.
// Kernels (R = N*M rays):
//   k_ray_limits      'auto' mode only: ray/AABB slab test            math_utils.py:46-98
//   k_sample_decode   stratified depth -> xyz -> tri-plane gather -> OSGDecoder -> masks
//                     one CTA = 128 consecutive samples; gather is cooperative (8 lanes x 16 B
//                     = one 128 B texel per tap), MLP is thread-per-sample FFMA from smem weights
//   k_ray_importance  warp per ray: coarse weights -> smoothed pdf -> inverse CDF -> sorted fine depths
//   k_ray_composite   warp per ray: merge (coarse|fine) by rank, alpha/T scan, weighted colour sum
//   k_depth_finalize  nan_to_num(inf) + clamp to the batch-global [min,max] depth  ray_marcher.py:49-50
#include "render_device.cuh"

namespace p3d {

namespace {

using namespace dev;

constexpr int kTile = 128;          // samples per CTA in k_sample_decode
constexpr int kFeatStride = 33;     // padded feature row (bank-conflict free for thread-per-row reads)
constexpr int kW2Stride = 36;       // W2^T row: 33 outputs padded to 36 floats (float4 broadcast reads)

struct SampleArgs {
    Geom g;
    const void* planes;
    const float *w1, *b1, *w2, *b2;
    const float *ro, *rd;       // (R,3)
    const float* u;             // coarse jitter (R*S) or nullptr
    const float* depth_in;      // fine pass: depths (R*Sf)
    const float* coords;        // points mode: (N,K,3)
    const float *ray_t0, *ray_t1;
    const unsigned int* bounds;
    float* depth_out;           // coarse pass: (R*S)
    float* sigma_out;           // (total)
    float* rgb_out;             // (total,32)
    long long total;            // samples in this launch
    long long per_view;         // samples per view (M*S, M*Sf or K)
    int per_ray;                // S, Sf (or 1 in points mode)
    VolumeSpec vol;             // volume mode (dense grid query): per_view = vol.res^3
    float* density_out;         // (total) or nullptr
    float* coords_out;          // (total,3) or nullptr
};

enum { MODE_COARSE = 0, MODE_FINE = 1, MODE_POINTS = 2, MODE_VOLUME = 3 };
// MODE_VOLUME generates its points and destinations with dev::volume_point / dev::volume_dest (render_device.cuh)


// -------------------------------------------------------------------------------------------
// k_sample_decode
// -------------------------------------------------------------------------------------------
// TRI: multiplane tri-planes (g.D > 1), trilinear gather
template <int MODE, bool BF16, bool TRI>
__global__ void __launch_bounds__(kTile) k_sample_decode(const SampleArgs a) {
    __shared__ __align__(16) float s_w1[kHidden * kC];          // [j][k], gain folded in
    __shared__ __align__(16) float s_w2t[kHidden * kW2Stride];  // [j][m], gain folded in
    __shared__ float s_b1[kHidden];
    __shared__ float s_b2[kW2Stride];
    __shared__ float s_feat[kTile * kFeatStride];               // features in, colours out
    __shared__ float s_xz[kTile * 2];                           // raw x,z for the crop mask

    const Geom& g = a.g;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long tile0 = (long long)blockIdx.x * kTile;

    for (int i = tid; i < kHidden * kC; i += kTile) s_w1[i] = __fmul_rn(a.w1[i], g.w1_gain);
    for (int i = tid; i < kHidden * kOut; i += kTile) {
        const int m = i / kHidden, j = i % kHidden;             // w2 is (out, hidden)
        s_w2t[j * kW2Stride + m] = __fmul_rn(a.w2[i], g.w2_gain);
    }
    if (tid < kHidden) s_b1[tid] = __fmul_rn(a.b1[tid], g.b1_gain);
    if (tid < kOut) s_b2[tid] = __fmul_rn(a.b2[tid], g.b2_gain);

    // ---- phase A: positions + gather; 4 samples per warp per round, 8 lanes per sample
    const int sub = lane >> 3, q = lane & 7;
#pragma unroll 1
    for (int round = 0; round < 8; ++round) {
        const int local = warp * 32 + round * 4 + sub;
        const long long gidx = tile0 + local;
        float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
        float px = 0.f, pz = 0.f;
        if (gidx < a.total) {
            const int view = (int)(gidx / a.per_view);
            float py;
            if (MODE == MODE_POINTS) {
                px = a.coords[gidx * 3 + 0]; py = a.coords[gidx * 3 + 1]; pz = a.coords[gidx * 3 + 2];
            } else if (MODE == MODE_VOLUME) {
                volume_point(gidx - (long long)view * a.per_view, a.vol.res, a.vol.size, a.vol.origin, px, py, pz);
            } else {
                const long long ray = gidx / a.per_ray;
                const int s = (int)(gidx - ray * a.per_ray);
                float t;
                if (MODE == MODE_COARSE) {
                    const float u = a.u ? a.u[gidx] : philox_uniform(g.seed, (uint64_t)gidx, 0u);
                    t = coarse_sample_depth(g, s, u, ray, true, a.ray_t0, a.ray_t1, a.bounds);
                    if (q == 0) a.depth_out[gidx] = t;
                } else {
                    t = a.depth_in[gidx];
                }
                const float3 pt = ray_point(a.ro + ray * 3, a.rd + ray * 3, t);
                px = pt.x; py = pt.y; pz = pt.z;
            }
            f = gather_features<BF16, TRI>(a.planes, g, view, px, py, pz, q);
        }
        float* dst = s_feat + local * kFeatStride + 4 * q;
        dst[0] = f.x; dst[1] = f.y; dst[2] = f.z; dst[3] = f.w;
        if (q == 0) { s_xz[local * 2] = px; s_xz[local * 2 + 1] = pz; }
    }
    __syncthreads();

    // ---- phase B: OSGDecoder, one sample per thread.  triplane.py:528-544
    float x[kC];
#pragma unroll
    for (int k = 0; k < kC; ++k) x[k] = s_feat[tid * kFeatStride + k];
    float o[kW2Stride];
#pragma unroll
    for (int m = 0; m < kW2Stride; ++m) o[m] = m < kOut ? s_b2[m] : 0.f;
#pragma unroll 2
    for (int j = 0; j < kHidden; ++j) {
        const float4* wrow = reinterpret_cast<const float4*>(s_w1 + j * kC);
        float h = s_b1[j];
#pragma unroll
        for (int k4 = 0; k4 < kC / 4; ++k4) {
            const float4 w = wrow[k4];
            h = fmaf(x[4 * k4 + 0], w.x, h);
            h = fmaf(x[4 * k4 + 1], w.y, h);
            h = fmaf(x[4 * k4 + 2], w.z, h);
            h = fmaf(x[4 * k4 + 3], w.w, h);
        }
        h = softplus_t(h);
        const float4* w2row = reinterpret_cast<const float4*>(s_w2t + j * kW2Stride);
#pragma unroll
        for (int m4 = 0; m4 < kW2Stride / 4; ++m4) {
            const float4 w = w2row[m4];
            o[4 * m4 + 0] = fmaf(h, w.x, o[4 * m4 + 0]);
            o[4 * m4 + 1] = fmaf(h, w.y, o[4 * m4 + 1]);
            o[4 * m4 + 2] = fmaf(h, w.z, o[4 * m4 + 2]);
            o[4 * m4 + 3] = fmaf(h, w.w, o[4 * m4 + 3]);
        }
    }
    const long long gidx = tile0 + tid;
    float sigma = o[0];
    if (MODE == MODE_COARSE || MODE == MODE_FINE) sigma = apply_masks(g, sigma, s_xz[tid * 2], s_xz[tid * 2 + 1]);
    if (MODE == MODE_VOLUME) {
        if (gidx < a.total) {
            const int view = (int)(gidx / a.per_view);
            const long long n = gidx - (long long)view * a.per_view;
            const long long dest = (long long)view * a.per_view + volume_dest(n, a.vol.res);
            a.sigma_out[dest] = sigma;
            if (a.density_out) a.density_out[dest] = volume_density(a.vol, sigma, s_xz[tid * 2], s_xz[tid * 2 + 1]);
            if (a.coords_out) {
                float x, y, z;
                volume_point(n, a.vol.res, a.vol.size, a.vol.origin, x, y, z);
                a.coords_out[dest * 3 + 0] = x; a.coords_out[dest * 3 + 1] = y; a.coords_out[dest * 3 + 2] = z;
            }
        }
    } else if (gidx < a.total) a.sigma_out[gidx] = sigma;
    __syncthreads();                       // everyone has consumed its feature row
#pragma unroll
    for (int c = 0; c < kRgb; ++c) {
        float v = sigmoid_t(o[1 + c]);
        if (!g.force_sigmoid) v = __fsub_rn(__fmul_rn(v, 1.002f), 0.001f);
        s_feat[tid * kFeatStride + c] = v;
    }
    __syncthreads();
    // coalesced colour store: 128 rows x 32 floats
    if (MODE == MODE_VOLUME && a.rgb_out == nullptr) return;
    for (int i = tid; i < kTile * kRgb; i += kTile) {
        const int row = i >> 5, col = i & 31;
        long long gi = tile0 + row;
        if (gi >= a.total) continue;
        if (MODE == MODE_VOLUME) {
            const long long view = gi / a.per_view, n = gi - view * a.per_view;
            gi = view * a.per_view + volume_dest(n, a.vol.res);
        }
        a.rgb_out[gi * kRgb + col] = s_feat[row * kFeatStride + col];
    }
}

// -------------------------------------------------------------------------------------------
// k_ray_limits: math_utils.get_ray_limits_box (:46-98) + validity reduction (renderer.py:165-170)
// An axis-parallel ray (a direction component of +-0, inv = +-inf) whose origin lies exactly on that axis's box face gets
// 0 * inf = NaN there.  torch.max / torch.min propagate it, so the reference returns a NaN limit, fails t1 > t0 and
// renders the ray with the batch's fallback limits; max_nan / min_nan keep that NaN where fmaxf / fminf would drop it.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ float max_nan(float a, float b) { return (isnan(a) || isnan(b)) ? __int_as_float(0x7fffffff) : fmaxf(a, b); }
__device__ __forceinline__ float min_nan(float a, float b) { return (isnan(a) || isnan(b)) ? __int_as_float(0x7fffffff) : fminf(a, b); }

__global__ void k_ray_limits(const float* ro, const float* rd, long long R, float h, float* t0o, float* t1o,
                             unsigned int* bounds) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    float tmin = 0.f, tmax = 0.f;
    bool valid = true;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
        const float o = ro[r * 3 + ax], inv = __fdiv_rn(1.f, rd[r * 3 + ax]);
        const bool neg = inv < 0.f;
        const float lo = __fmul_rn(__fsub_rn(neg ? h : -h, o), inv);
        const float hi = __fmul_rn(__fsub_rn(neg ? -h : h, o), inv);
        if (ax == 0) { tmin = lo; tmax = hi; }
        else {
            if (tmin > hi || lo > tmax) valid = false;
            tmin = max_nan(tmin, lo);
            tmax = min_nan(tmax, hi);
        }
    }
    if (!valid) { tmin = -1.f; tmax = -2.f; }
    t0o[r] = tmin; t1o[r] = tmax;
    if (tmax > tmin) {
        atomicMin(&bounds[2], float_to_ordered(tmin));
        atomicMax(&bounds[3], float_to_ordered(tmin));
        atomicOr(&bounds[4], 1u);
    }
}

__global__ void k_init_bounds(unsigned int* bounds) {
    if (threadIdx.x == 0) {
        bounds[0] = 0xffffffffu; bounds[1] = 0u; bounds[2] = 0xffffffffu; bounds[3] = 0u; bounds[4] = 0u;
    }
}


// -------------------------------------------------------------------------------------------
struct ImportanceArgs {
    Geom g;
    const float *depth_c, *sigma_c, *u_fine;
    float* depth_f;
    unsigned int* bounds;
    long long R;
    int sort_pow2;     // next power of two >= Sf
};

__global__ void __launch_bounds__(128) k_ray_importance(const ImportanceArgs a) {
    extern __shared__ float smem[];
    const Geom& g = a.g;
    const int S = g.S, Sf = g.Sf, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long ray = (long long)blockIdx.x * 4 + warp;
    if (ray >= a.R) return;
    const int per_warp = 4 * S + a.sort_pow2;
    float* t = smem + warp * per_warp;      // S
    float* sg = t + S;                      // S
    float* w = sg + S;                      // S   (weights, S-1 used; later pooled pdf)
    float* cdf = w + S;                     // S   (S-2 used)
    float* fine = cdf + S;                  // sort_pow2

    for (int i = lane; i < S; i += 32) { t[i] = a.depth_c[ray * S + i]; sg[i] = a.sigma_c[ray * S + i]; }
    __syncwarp();
    importance_ray(g, t, sg, w, cdf, fine, a.sort_pow2, a.u_fine ? a.u_fine + ray * Sf : nullptr,
                   (unsigned long long)(ray * Sf), lane);
    for (int f = lane; f < Sf; f += 32) a.depth_f[ray * Sf + f] = fine[f];
}

// -------------------------------------------------------------------------------------------
// k_ray_composite: unify_samples (renderer.py:289-301) + final MipRayMarcher2 (ray_marcher.py:25-57)
// on the 32 colour channels and, analytically, on xyz (the marcher is linear in the colours and
// xyz_j = o + t_j d, so  sum_i w_i xyz_mid_i = o*sum(w) + d*sum(w_i t_mid_i)).
// -------------------------------------------------------------------------------------------
struct CompositeArgs {
    Geom g;
    const float *depth_c, *sigma_c, *rgb_c, *depth_f, *sigma_f, *rgb_f, *ro, *rd;
    float *out_rgb, *out_depth, *out_wsum, *out_xyz;
    unsigned int* bounds;
    long long R;
};

__global__ void __launch_bounds__(128) k_ray_composite(const CompositeArgs a) {
    extern __shared__ float smem[];
    const Geom& g = a.g;
    const int S = g.S, Sf = g.Sf, L = S + Sf, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long ray = (long long)blockIdx.x * 4 + warp;
    if (ray >= a.R) return;
    float* t = smem + warp * (4 * L);       // merged depths
    float* sg = t + L;                      // merged densities
    float* w = sg + L;                      // interval weights (L-1), then per-sample omegas
    int* src = reinterpret_cast<int*>(w + L);   // merged position -> colour row

    const float* tc = a.depth_c + ray * S;
    const float* tf = a.depth_f + ray * Sf;
    float wsum, dnum;
    composite_weights(tc, a.sigma_c + ray * S, tf, a.sigma_f + ray * Sf, S, Sf, t, sg, w, src, lane, wsum, dnum);
    float acc = 0.f;                        // lane = colour channel
    for (int j = 0; j < L; ++j) {
        const int s = src[j];
        const float c = s < S ? a.rgb_c[(ray * S + s) * kRgb + lane] : a.rgb_f[(ray * Sf + (s - S)) * kRgb + lane];
        acc = fmaf(w[j], c, acc);
    }
    const float back = g.white_back ? __fsub_rn(1.f, wsum) : 0.f;
    a.out_rgb[ray * kRgb + lane] = __fsub_rn(__fmul_rn(__fadd_rn(acc, back), 2.f), 1.f);
    if (lane < 3) {
        const float v = fmaf(a.ro[ray * 3 + lane], wsum, a.rd[ray * 3 + lane] * dnum);
        a.out_xyz[ray * 3 + lane] = __fsub_rn(__fmul_rn(__fadd_rn(v, back), 2.f), 1.f);
    }
    if (lane == 0) {
        a.out_depth[ray] = __fdiv_rn(dnum, wsum);      // 0/0 -> NaN, fixed up by k_depth_finalize
        a.out_wsum[ray] = wsum;
        atomicMin(&a.bounds[0], float_to_ordered(t[0]));
        atomicMax(&a.bounds[1], float_to_ordered(t[L - 1]));
    }
}

// nan_to_num(nan=inf) then clamp(min(depths), max(depths)) over the whole batch.  ray_marcher.py:49-50.  The bounds are the
// workspace's ordered uints (bounds[0..1]), or two floats from the caller when the clamp was deferred (defer_depth_clamp).
__device__ __forceinline__ float depth_bound(unsigned int b) { return ordered_to_float(b); }
__device__ __forceinline__ float depth_bound(float b) { return b; }
template <typename B>
__global__ void k_depth_finalize(float* depth, long long R, const B* bounds) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const float lo = depth_bound(bounds[0]), hi = depth_bound(bounds[1]);
    float d = depth[r];
    if (isnan(d)) d = INFINITY;
    depth[r] = fminf(fmaxf(d, lo), hi);
}

__global__ void k_bounds_to_float(const unsigned int* bounds, float* out2) {
    if (threadIdx.x < 2) out2[threadIdx.x] = ordered_to_float(bounds[threadIdx.x]);
}

template <int MODE>
int launch_sample_decode(const SampleArgs& a, bool bf16, cudaStream_t stream) {
    if (a.total <= 0) return P3D_OK;
    const long long blocks = (a.total + kTile - 1) / kTile;
    P3D_REQUIRE(blocks < (1ll << 31), "too many samples for one launch (%lld)", a.total);
    ProfileScope prof(PROF_SAMPLE_DECODE, stream);
    if (a.g.D > 1) {
        if (bf16) k_sample_decode<MODE, true, true><<<(unsigned)blocks, kTile, 0, stream>>>(a);
        else k_sample_decode<MODE, false, true><<<(unsigned)blocks, kTile, 0, stream>>>(a);
    } else {
        if (bf16) k_sample_decode<MODE, true, false><<<(unsigned)blocks, kTile, 0, stream>>>(a);
        else k_sample_decode<MODE, false, false><<<(unsigned)blocks, kTile, 0, stream>>>(a);
    }
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace

int launch_bounds_init(unsigned int* bounds, cudaStream_t stream) {
    k_init_bounds<<<1, 32, 0, stream>>>(bounds);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
int launch_ray_limits(const float* ro, const float* rd, long long R, float h, float* t0, float* t1, unsigned int* bounds, cudaStream_t stream) {
    k_ray_limits<<<(unsigned)((R + 255) / 256), 256, 0, stream>>>(ro, rd, R, h, t0, t1, bounds);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
int launch_bounds_to_float(const unsigned int* bounds, float* out2, cudaStream_t stream) {
    k_bounds_to_float<<<1, 32, 0, stream>>>(bounds, out2);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
int launch_depth_finalize_f(float* depth, long long R, const float* bounds2, cudaStream_t stream) {
    k_depth_finalize<<<(unsigned)((R + 255) / 256), 256, 0, stream>>>(depth, R, bounds2);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}
int launch_depth_finalize(float* depth, long long R, const unsigned int* bounds, cudaStream_t stream) {
    k_depth_finalize<<<(unsigned)((R + 255) / 256), 256, 0, stream>>>(depth, R, bounds);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

// -------------------------------------------------------------------------------------------
int render_forward_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                      const float* w2, const float* b2, const float* ro, const float* rd, const float* u_c,
                      const float* u_f, const Workspace& ws, float* out_rgb, float* out_depth, float* out_wsum,
                      float* out_xyz, cudaStream_t stream) {
    const long long R = (long long)g.N * g.M;
    P3D_REQUIRE(g.S >= 2 && g.S <= 256, "depth_resolution must be in [2,256], got %d", g.S);
    P3D_REQUIRE(g.Sf == 0 || g.S >= 4, "importance sampling needs depth_resolution >= 4");
    P3D_REQUIRE(g.Sf >= 0 && g.S + g.Sf <= 512, "depth_resolution + depth_resolution_importance must be <= 512");

    int rc;
    if ((rc = launch_bounds_init(ws.bounds, stream))) return rc;
    if (g.ray_mode == P3D_RAYS_AUTOBOX)
        if ((rc = launch_ray_limits(ro, rd, R, g.half_box, ws.ray_t0, ws.ray_t1, ws.bounds, stream))) return rc;
    SampleArgs sa{};
    sa.g = g; sa.planes = planes; sa.w1 = w1; sa.b1 = b1; sa.w2 = w2; sa.b2 = b2; sa.ro = ro; sa.rd = rd;
    sa.ray_t0 = ws.ray_t0; sa.ray_t1 = ws.ray_t1; sa.bounds = ws.bounds;
    // coarse pass
    sa.u = u_c; sa.depth_out = ws.depth_c; sa.sigma_out = ws.sigma_c; sa.rgb_out = ws.rgb_c;
    sa.total = R * g.S; sa.per_view = (long long)g.M * g.S; sa.per_ray = g.S;
    if ((rc = launch_sample_decode<MODE_COARSE>(sa, p->planes_bf16 != 0, stream))) return rc;
    if (g.Sf > 0) {
        ImportanceArgs ia{};
        ia.g = g; ia.depth_c = ws.depth_c; ia.sigma_c = ws.sigma_c; ia.u_fine = u_f; ia.depth_f = ws.depth_f;
        ia.bounds = ws.bounds; ia.R = R;
        int p2 = 1; while (p2 < g.Sf) p2 <<= 1;
        ia.sort_pow2 = p2;
        const size_t smem = (size_t)4 * (4 * g.S + p2) * sizeof(float);
        {
            ProfileScope prof(PROF_IMPORTANCE, stream);
            k_ray_importance<<<(unsigned)((R + 3) / 4), 128, smem, stream>>>(ia);
            P3D_LAUNCH_CHECK();
        }
        sa.u = nullptr; sa.depth_in = ws.depth_f; sa.depth_out = nullptr; sa.sigma_out = ws.sigma_f; sa.rgb_out = ws.rgb_f;
        sa.total = R * g.Sf; sa.per_view = (long long)g.M * g.Sf; sa.per_ray = g.Sf;
        rc = launch_sample_decode<MODE_FINE>(sa, p->planes_bf16 != 0, stream);
        if (rc) return rc;
    }
    CompositeArgs ca{};
    ca.g = g; ca.depth_c = ws.depth_c; ca.sigma_c = ws.sigma_c; ca.rgb_c = ws.rgb_c; ca.depth_f = ws.depth_f;
    ca.sigma_f = ws.sigma_f; ca.rgb_f = ws.rgb_f; ca.ro = ro; ca.rd = rd; ca.out_rgb = out_rgb; ca.out_depth = out_depth;
    ca.out_wsum = out_wsum; ca.out_xyz = out_xyz; ca.bounds = ws.bounds; ca.R = R;
    const size_t smem = (size_t)4 * 4 * (g.S + g.Sf) * sizeof(float);
    {
        ProfileScope prof(PROF_COMPOSITE, stream);
        k_ray_composite<<<(unsigned)((R + 3) / 4), 128, smem, stream>>>(ca);
        P3D_LAUNCH_CHECK();
    }
    if (p->defer_depth_clamp) return P3D_OK;
    return launch_depth_finalize(out_depth, R, ws.bounds, stream);
}

int decode_points_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                     const float* w2, const float* b2, const float* coords, long long n_pts, float* out_rgb,
                     float* out_sigma, cudaStream_t stream) {
    SampleArgs sa{};
    sa.g = g; sa.planes = planes; sa.w1 = w1; sa.b1 = b1; sa.w2 = w2; sa.b2 = b2; sa.coords = coords;
    sa.sigma_out = out_sigma; sa.rgb_out = out_rgb;
    sa.total = (long long)g.N * n_pts; sa.per_view = n_pts; sa.per_ray = 1;
    return launch_sample_decode<MODE_POINTS>(sa, p->planes_bf16 != 0, stream);
}

int volume_query_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                    const float* w2, const float* b2, const VolumeSpec& vol, float* out_sigma, float* out_rgb,
                    float* out_density, float* out_coords, cudaStream_t stream) {
    SampleArgs sa{};
    sa.g = g; sa.planes = planes; sa.w1 = w1; sa.b1 = b1; sa.w2 = w2; sa.b2 = b2;
    sa.sigma_out = out_sigma; sa.rgb_out = out_rgb; sa.density_out = out_density; sa.coords_out = out_coords;
    sa.per_view = (long long)vol.res * vol.res * vol.res; sa.total = (long long)g.N * sa.per_view; sa.per_ray = 1;
    sa.vol = vol;
    return launch_sample_decode<MODE_VOLUME>(sa, p->planes_bf16 != 0, stream);
}

}  // namespace p3d
