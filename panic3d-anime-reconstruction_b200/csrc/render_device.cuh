// Device functions shared by the v1 (multi-kernel SIMT) and the fused tensor-core renderer.
#pragma once
#include "render_internal.cuh"

namespace p3d {
namespace dev {

// -------------------------------------------------------------------------------------------
// depth of coarse sample s of a ray.  renderer.py:303-326 (+ math_utils.linspace :101-118)
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ float coarse_depth(const Geom& g, int s, float u, float t0, float t1) {
    const int S = g.S;
    if (g.ray_mode == P3D_RAYS_AUTOBOX) {
        float step = __fdiv_rn((float)s, (float)(S - 1));
        float span = __fsub_rn(t1, t0);
        float base = __fadd_rn(t0, __fmul_rn(step, span));
        float delta = __fdiv_rn(span, (float)(S - 1));
        return __fadd_rn(base, __fmul_rn(u, delta));
    }
    if (g.disparity) {
        float st = __fdiv_rn(1.0f, (float)(S - 1));
        float lin = (s < S / 2) ? __fmul_rn(st, (float)s) : __fsub_rn(1.0f, __fmul_rn(st, (float)(S - 1 - s)));
        float t = __fadd_rn(lin, __fmul_rn(u, g.disp_delta));
        float den = __fadd_rn(__fmul_rn(g.inv_start, __fsub_rn(1.0f, t)), __fmul_rn(g.inv_end, t));
        return __fdiv_rn(1.0f, den);
    }
    float lin = (s < S / 2) ? __fadd_rn(g.ray_start, __fmul_rn(g.lin_step, (float)s))
                            : __fsub_rn(g.ray_end, __fmul_rn(g.lin_step, (float)(S - 1 - s)));
    return __fadd_rn(lin, __fmul_rn(u, g.depth_delta));
}

// -------------------------------------------------------------------------------------------
// Grid point n of the reference's create_samples (eg3d_metrics3d.py:70-92), bit for bit: the z index is the integer
// n % R, but the y and x "indices" come from FLOAT divisions that are never floored - (float(n)/R) % R and
// ((float(n)/R)/R) % R - so the lattice is sheared by a fraction of a voxel.  Meshes downstream were extracted from
// exactly these points, so the shear is part of the contract.  Used by the v1 and tensor-core volume queries and by
// the mesh's colour lookup (marching_cubes.cu).
// -------------------------------------------------------------------------------------------
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
// where sample n of a view lands in the returned volume: reshape (R,R,R) by flat index, first axis flipped.  The map is
// its own inverse, so it also gives the sample n of volume element (a, b, c).
__device__ __forceinline__ long long volume_dest(long long n, int R) {
    const long long rr = (long long)R * R;
    const long long a = n / rr, rest = n - a * rr;
    return ((long long)(R - 1) - a) * rr + rest;
}

// -------------------------------------------------------------------------------------------
// Tri-plane bilinear gather for one sample, channels [4q, 4q+4).  renderer.py:52-81:
//   grid = coord * (2/box_warp); texel = ((grid+1)*size - 1)/2  (align_corners=False);
//   taps outside the plane contribute zero (padding_mode='zeros'); mean over the 3 planes.
// Every tap is one contiguous 128 B (fp32) / 64 B (bf16) texel: the 8 lanes of a sample read
// 16 B (8 B) each, so a warp-wide load touches 4 lines.
// -------------------------------------------------------------------------------------------
template <bool BF16>
__device__ __forceinline__ float4 load_quad(const void* planes, long long elem_off) {
    if (BF16) {
        const uint2 raw = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(planes) + elem_off));
        float4 r;
        r.x = __uint_as_float(raw.x << 16);
        r.y = __uint_as_float(raw.x & 0xffff0000u);
        r.z = __uint_as_float(raw.y << 16);
        r.w = __uint_as_float(raw.y & 0xffff0000u);
        return r;
    } else {
        return ldg128(reinterpret_cast<const float*>(planes) + elem_off);
    }
}

struct Tap4 {
    long long off[4];
    float w[4];
};

__device__ __forceinline__ Tap4 plane_taps(const Geom& g, long long base, float ca, float cb) {
    Tap4 t;
    const float gx = __fmul_rn(ca, g.coord_scale), gy = __fmul_rn(cb, g.coord_scale);
    const float fx = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)g.W), 1.f), 0.5f);
    const float fy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)g.H), 1.f), 0.5f);
    const bool sane = (fx > -2.f) && (fx < (float)g.W + 1.f) && (fy > -2.f) && (fy < (float)g.H + 1.f);  // false for NaN too
    const float x0f = floorf(fx), y0f = floorf(fy);
    const float wx1 = fx - x0f, wy1 = fy - y0f;
    const float wx0 = 1.f - wx1, wy0 = 1.f - wy1;
    const int x0 = sane ? (int)x0f : -4, y0 = sane ? (int)y0f : -4;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int xi = x0 + (k & 1), yi = y0 + (k >> 1);
        const bool ok = (xi >= 0) && (xi < g.W) && (yi >= 0) && (yi < g.H);
        const float wgt = ((k & 1) ? wx1 : wx0) * ((k >> 1) ? wy1 : wy0);
        t.w[k] = ok ? wgt : 0.f;
        t.off[k] = base + (ok ? (long long)yi * g.stride_row + (long long)xi * g.stride_col : 0ll);
    }
    return t;
}

template <bool BF16>
__device__ __forceinline__ float4 gather_features(const void* planes, const Geom& g, int view, float x, float y, float z, int q) {
    const long long vbase = (long long)view * g.stride_view + 4 * q;
    const float a2 = g.plane_mode == P3D_PLANES_PANIC3D ? y : z;
    const float b2 = g.plane_mode == P3D_PLANES_PANIC3D ? z : x;
    Tap4 t0 = plane_taps(g, vbase, x, y);
    Tap4 t1 = plane_taps(g, vbase + g.stride_plane, x, z);
    Tap4 t2 = plane_taps(g, vbase + 2 * g.stride_plane, a2, b2);
    float4 v[12];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        v[k] = load_quad<BF16>(planes, t0.off[k]);
        v[4 + k] = load_quad<BF16>(planes, t1.off[k]);
        v[8 + k] = load_quad<BF16>(planes, t2.off[k]);
    }
    float4 f[3];
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        const Tap4& t = p == 0 ? t0 : (p == 1 ? t1 : t2);
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            a.x = fmaf(v[4 * p + k].x, t.w[k], a.x);
            a.y = fmaf(v[4 * p + k].y, t.w[k], a.y);
            a.z = fmaf(v[4 * p + k].z, t.w[k], a.z);
            a.w = fmaf(v[4 * p + k].w, t.w[k], a.w);
        }
        f[p] = a;
    }
    float4 r;
    r.x = __fdiv_rn(__fadd_rn(__fadd_rn(f[0].x, f[1].x), f[2].x), 3.f);
    r.y = __fdiv_rn(__fadd_rn(__fadd_rn(f[0].y, f[1].y), f[2].y), 3.f);
    r.z = __fdiv_rn(__fadd_rn(__fadd_rn(f[0].z, f[1].z), f[2].z), 3.f);
    r.w = __fdiv_rn(__fadd_rn(__fadd_rn(f[0].w, f[1].w), f[2].w), 3.f);
    return r;
}

// crop + cull/binarize on a raw density.  renderer.py:138-153, :187-198
__device__ __forceinline__ float apply_masks(const Geom& g, float sigma, float x, float z) {
    if (g.crop_on && !((fabsf(x) <= g.crop_limit) && (fabsf(z) <= g.crop_limit))) sigma = -1e3f;
    if (g.binarize_on || g.cull_on) {
        const float alpha = 1.f - expf(-softplus_t(sigma - 1.f));
        const bool m = alpha < g.cull_thresh;
        if (g.binarize_on) sigma = m ? -1e3f : 1e3f;
        else if (m) sigma = -1e3f;
    }
    return sigma;
}

// -------------------------------------------------------------------------------------------
// per-ray compositing weights.  ray_marcher.py:25-44
//   alpha_i = 1 - exp(-softplus((s_i+s_{i+1})/2 - 1) * (t_{i+1}-t_i)),
//   w_i = alpha_i * prod_{k<i} (1 - alpha_k + 1e-10)
// t, sg: L sorted samples in shared memory; writes w[0..L-2]; returns (sum w, sum w*t_mid) on all lanes.
// -------------------------------------------------------------------------------------------
// FAST: MUFU ex2/lg2 based softplus/exp (abs err ~1e-7) for the fused kernel; false: libm-accurate (v1).
template <bool FAST = false>
__device__ __forceinline__ void ray_weights(const float* t, const float* sg, float* w, int L, int lane,
                                            float& wsum, float& dnum) {
    float carry = 1.f, acc_w = 0.f, acc_d = 0.f;
    for (int base = 0; base < L - 1; base += 32) {
        const int i = base + lane;
        float alpha = 0.f, factor = 1.f, tmid = 0.f;
        if (i < L - 1) {
            const float delta = t[i + 1] - t[i];
            const float smid = __fsub_rn(__fmul_rn(__fadd_rn(sg[i], sg[i + 1]), 0.5f), 1.f);
            if (FAST) alpha = 1.f - ex2_approx(-1.4426950408889634f * __fmul_rn(softplus_mufu(smid), delta));
            else alpha = 1.f - expf(-__fmul_rn(softplus_t(smid), delta));
            factor = __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f);
            tmid = __fmul_rn(__fadd_rn(t[i], t[i + 1]), 0.5f);
        }
        const float incl = warp_scan_mul(factor, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        const float T = carry * excl;
        const float wi = alpha * T;
        if (i < L - 1) { w[i] = wi; acc_w += wi; acc_d = fmaf(wi, tmid, acc_d); }
        carry *= __shfl_sync(0xffffffffu, incl, 31);
    }
    wsum = warp_sum(acc_w);
    dnum = warp_sum(acc_d);
}

// -------------------------------------------------------------------------------------------
// importance_ray: sample_importance + sample_pdf for ONE ray, executed by one warp.  renderer.py:328-387
//   t, sg   : S coarse depths / densities (shared memory)
//   w, cdf  : scratch, S floats each
//   fine    : out, sort_pow2 floats; the first Sf entries are the importance depths, ascending
//   u_fine  : Sf injected uniforms for this ray (global) or nullptr -> Philox(seed, rng_base + f)
// -------------------------------------------------------------------------------------------
template <bool FAST = false>
__device__ __forceinline__ void importance_ray(const Geom& g, const float* t, const float* sg, float* w, float* cdf,
                                               float* fine, int sort_pow2, const float* u_fine,
                                               unsigned long long rng_base, int lane) {
    const int S = g.S, Sf = g.Sf;
    float wsum, dnum;
    ray_weights<FAST>(t, sg, w, S, lane, wsum, dnum);
    __syncwarp();
    // max_pool1d(k=2,s=1,pad=1) -> avg_pool1d(k=2,s=1) -> +0.01 ; keep [1:-1] ; +eps     (:336-343, :360)
    // pooled[i] = (max(w[i-1],w[i]) + max(w[i],w[i+1]))/2 , i in [1, S-3]
    const int nb = S - 3;                   // pdf bins
    float my[8];                            // up to 256 coarse samples per ray
    float part = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int k = c * 32 + lane;
        float v = 0.f;
        if (k < nb) {
            const int i = k + 1;
            const float wl = w[i - 1], wc = w[i], wr = w[i + 1];
            const float pooled = __fmul_rn(__fadd_rn(fmaxf(wl, wc), fmaxf(wc, wr)), 0.5f);
            v = __fadd_rn(__fadd_rn(pooled, 0.01f), 1e-5f);
        }
        my[c] = v;
        part += v;
    }
    const float total = warp_sum(part);
    // cdf[0] = 0, cdf[k+1] = cumsum(pdf)[k]
    float carry = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        if (c * 32 < nb) {
            const int k = c * 32 + lane;
            const float pdf = k < nb ? __fdiv_rn(my[c], total) : 0.f;
            const float incl = warp_scan_add(pdf, lane) + carry;
            if (k < nb) cdf[k + 1] = incl;
            carry = __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    if (lane == 0) cdf[0] = 0.f;
    __syncwarp();
    // inverse CDF.  searchsorted(right=True): first index with cdf[idx] > u
    for (int f = lane; f < sort_pow2; f += 32) {
        float val = INFINITY;
        if (f < Sf) {
            const float u = u_fine ? u_fine[f] : philox_uniform(g.seed, rng_base + (unsigned long long)f, 1u);
            int lo = 0, hi = nb + 1;            // cdf has nb+1 entries
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
            }
            const int below = max(lo - 1, 0), above = min(lo, nb);
            const float c0 = cdf[below], c1 = cdf[above];
            const float b0 = __fmul_rn(0.5f, __fadd_rn(t[below], t[below + 1]));
            const float b1 = __fmul_rn(0.5f, __fadd_rn(t[above], t[above + 1]));
            float den = __fsub_rn(c1, c0);
            if (den < 1e-5f) den = 1.f;
            val = __fadd_rn(b0, __fmul_rn(__fdiv_rn(__fsub_rn(u, c0), den), __fsub_rn(b1, b0)));
        }
        fine[f] = val;
    }
    __syncwarp();
    // bitonic sort ascending (per ray); the merged composite is order independent, sorting here
    // lets the composite merge by rank instead of running a global sort (renderer.py:289-301)
    for (int k = 2; k <= sort_pow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < sort_pow2; i += 32) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const float x = fine[i], y = fine[ixj];
                    const bool up = (i & k) == 0;
                    if ((x > y) == up) { fine[i] = y; fine[ixj] = x; }
                }
            }
            __syncwarp();
        }
    }
}

// -------------------------------------------------------------------------------------------
// composite_weights: unify_samples (renderer.py:289-301) + the weight part of the final
// MipRayMarcher2 pass (ray_marcher.py:25-44) for ONE ray, executed by one warp.
//   tc, sc : S coarse depths/densities   tf, sf : Sf fine depths (ascending) / densities
//   t, sg, w : scratch of L = S+Sf floats each; src : L ints
// On return w[j] holds omega_j = (w_{j-1}+w_j)/2 for merged position j and src[j] names its
// sample (i < S: coarse i, else fine i-S), so  sum_i w_i (c_i+c_{i+1})/2 == sum_j omega_j c_j.
// -------------------------------------------------------------------------------------------
template <bool FAST = false>
__device__ __forceinline__ void composite_weights(const float* tc, const float* sc, const float* tf, const float* sf,
                                                  int S, int Sf, float* t, float* sg, float* w, int* src, int lane,
                                                  float& wsum, float& dnum) {
    const int L = S + Sf;
    // merge by rank; ties keep coarse before fine (stable sort of cat([coarse, fine])).
    // Coarse depths ascend except for the degenerate 'auto' case where no ray hits the box
    // (t0=-1 > t1=-2, renderer.py:166-170 leaves them untouched): then they descend -> read reversed.
    const bool rev = tc[0] > tc[S - 1];
    for (int i = lane; i < S; i += 32) {
        const int ci = rev ? S - 1 - i : i;
        const float v = tc[ci];
        int lo = 0, hi = Sf;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (tf[mid] < v) lo = mid + 1; else hi = mid; }
        const int pos = i + lo;
        t[pos] = v; sg[pos] = sc[ci]; src[pos] = ci;
    }
    for (int j = lane; j < Sf; j += 32) {
        const float v = tf[j];
        int lo = 0, hi = S;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (tc[rev ? S - 1 - mid : mid] <= v) lo = mid + 1; else hi = mid; }
        const int pos = j + lo;
        t[pos] = v; sg[pos] = sf[j]; src[pos] = S + j;
    }
    __syncwarp();
    ray_weights<FAST>(t, sg, w, L, lane, wsum, dnum);
    __syncwarp();
    float om[16];                           // up to 512 merged samples per ray
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        const int j = c * 32 + lane;
        float v = 0.f;
        if (j < L) {
            const float wl = j > 0 ? w[j - 1] : 0.f, wr = j < L - 1 ? w[j] : 0.f;
            v = __fmul_rn(__fadd_rn(wl, wr), 0.5f);
        }
        om[c] = v;
    }
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        const int j = c * 32 + lane;
        if (j < L) w[j] = om[c];
    }
    __syncwarp();
}

}  // namespace dev
}  // namespace p3d
