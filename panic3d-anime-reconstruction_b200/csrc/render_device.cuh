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
// coarse_depth with the ray's 'auto' limits: a ray that misses the box takes the smallest and largest valid start of the
// whole batch (bounds[2..3], when bounds[4] says there is one).  renderer.py:165-170.  A dead row (live == false) reads
// no limits.
// Deviation from the reference: a NaN limit (k_ray_limits: an axis-parallel ray starting on a box face) in a batch where no
// ray hits the box takes the miss limits (-1, -2).  The reference renders NaN depths there; NaN depths would break the
// rank merge (merge_by_rank's comparisons are all false), leaving merged slots whose colour row index is never written.
__device__ __forceinline__ float coarse_sample_depth(const Geom& g, int s, float u, long long ray, bool live, const float* ray_t0,
                                                     const float* ray_t1, const unsigned int* bounds) {
    float t0 = 0.f, t1 = 0.f;
    if (g.ray_mode == P3D_RAYS_AUTOBOX && live) {
        t0 = ray_t0[ray]; t1 = ray_t1[ray];
        if (!(t1 > t0)) {
            if (bounds[4]) { t0 = ordered_to_float(bounds[2]); t1 = ordered_to_float(bounds[3]); }
            else if (isnan(t0) || isnan(t1)) { t0 = -1.f; t1 = -2.f; }
        }
    }
    return coarse_depth(g, s, u, t0, t1);
}

// o + t d, rounded per operation like the reference's ATen ops (no FMA contraction)
__device__ __forceinline__ float3 ray_point(const float* o, const float* d, float t) {
    return make_float3(__fadd_rn(o[0], __fmul_rn(t, d[0])), __fadd_rn(o[1], __fmul_rn(t, d[1])), __fadd_rn(o[2], __fmul_rn(t, d[2])));
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
// The volume query's density at a lattice point (x, z): sigma2density (eg3d_metrics3d.py:65-69), then crop / cull write -1e3
// (:155-162).  The reference hands the DENSITIES to cull_clouds_mask, which applies softplus(. - 1) -> 1 - exp(-.) once more
// (renderer.py:150-153): the threshold acts on the twice-transformed value.
__device__ __forceinline__ float volume_density(const VolumeSpec& v, float sigma, float x, float z) {
    float dens = 1.f - expf(-softplus_t(__fsub_rn(sigma, 1.f)));
    if (v.crop_on && !((fabsf(x) <= v.crop) && (fabsf(z) <= v.crop))) dens = -1e3f;
    if (v.cull_on && (1.f - expf(-softplus_t(__fsub_rn(dens, 1.f)))) < v.cull) dens = -1e3f;
    return dens;
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

// Coordinates (a, b) of a point on plane p: (x, y), (x, z), then (y, z) for P3D_PLANES_PANIC3D or (z, x) otherwise.
__device__ __forceinline__ float2 plane_coords(const Geom& g, int p, float x, float y, float z) {
    const bool pm = g.plane_mode == P3D_PLANES_PANIC3D;
    return make_float2(p == 2 ? (pm ? y : z) : x, p == 0 ? y : (p == 1 ? z : (pm ? z : x)));
}

// grid_sample's bilinear footprint of plane coordinates (ca, cb): the top-left texel (x0, y0) and the 1-D weights of columns
// x0, x0 + 1 and rows y0, y0 + 1.  A point that is NaN or lies more than a texel outside the plane gets x0 = y0 = -4, so all
// four taps fall outside.  The forward gathers (plane_taps, fused::write_tap_row) and the backward scatter (plane_texels)
// all take their taps from here, so the gradients land on exactly the texels and weights the forward used.
struct Footprint {
    int x0, y0;
    float wx0, wx1, wy0, wy1;
};
__device__ __forceinline__ Footprint bilinear_footprint(const Geom& g, float ca, float cb) {
    const float gx = __fmul_rn(ca, g.coord_scale), gy = __fmul_rn(cb, g.coord_scale);
    const float fx = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)g.W), 1.f), 0.5f);
    const float fy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)g.H), 1.f), 0.5f);
    const bool sane = (fx > -2.f) && (fx < (float)g.W + 1.f) && (fy > -2.f) && (fy < (float)g.H + 1.f);  // false for NaN too
    const float x0f = floorf(fx), y0f = floorf(fy);
    Footprint f;
    f.wx1 = fx - x0f; f.wy1 = fy - y0f;
    f.wx0 = 1.f - f.wx1; f.wy0 = 1.f - f.wy1;
    f.x0 = sane ? (int)x0f : -4; f.y0 = sane ? (int)y0f : -4;
    return f;
}

// -------------------------------------------------------------------------------------------
// Multiplane tri-planes (triplane_depth D > 1).  renderer.py:84-94: each plane is a stack of D slabs sampled by a 5-D
// grid_sample (trilinear, zero padding, align_corners=False).  project_onto_planes keeps all three components of
// coordinates @ inv(plane_axes); the third indexes the slabs.  Slab d of plane p of a view starts at
// p * stride_plane + d * H * stride_row.
// -------------------------------------------------------------------------------------------
// The slab (normal-axis) coordinate of plane p: z, y, then x for P3D_PLANES_PANIC3D or y otherwise.
__device__ __forceinline__ float plane_normal(const Geom& g, int p, float x, float y, float z) {
    const bool pm = g.plane_mode == P3D_PLANES_PANIC3D;
    return p == 0 ? z : (p == 1 ? y : (pm ? x : y));
}

// grid_sample's footprint along the normal: the first slab z0 and the weights of slabs z0 and z0 + 1.  Slabs outside
// [0, D) contribute zero; a NaN or far-away normal coordinate gets z0 = -4.
struct SlabFootprint {
    int z0;
    float wz0, wz1;
};
__device__ __forceinline__ SlabFootprint slab_footprint(const Geom& g, float cn) {
    const float gz = __fmul_rn(cn, g.coord_scale);
    const float fz = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gz, 1.f), (float)g.D), 1.f), 0.5f);
    const bool sane = (fz > -2.f) && (fz < (float)g.D + 1.f);
    const float z0f = floorf(fz);
    SlabFootprint s;
    s.wz1 = fz - z0f;
    s.wz0 = 1.f - s.wz1;
    s.z0 = sane ? (int)z0f : -4;
    return s;
}

// -------------------------------------------------------------------------------------------
// The taps of one plane: 4 bilinear ones, or for multiplane planes (TRI) 8 = those 4 in slab z0, then in slab z0 + 1.
// plane_tap gives tap k: texel (x0 + (k & 1), y0 + ((k >> 1) & 1), z0 + (k >> 2)) (z = 0 on one-slab planes), its weight
// (wx wy) wz and whether it lies inside the plane.  The forward's element offsets (plane_taps) and the backward's scatter
// list (plane_texels) both take their taps from it, so the gradients land on exactly the texels and weights the forward read.
// -------------------------------------------------------------------------------------------
template <bool TRI> constexpr int kPlaneTaps = TRI ? 8 : 4;

template <bool TRI>
__device__ __forceinline__ bool plane_tap(const Geom& g, const Footprint& f, const SlabFootprint& s, int k, int& x, int& y, int& z,
                                          float& w) {
    x = f.x0 + (k & 1); y = f.y0 + ((k >> 1) & 1); z = TRI ? s.z0 + (k >> 2) : 0;
    w = ((k & 1) ? f.wx1 : f.wx0) * (((k >> 1) & 1) ? f.wy1 : f.wy0);
    if constexpr (TRI) w = w * ((k >> 2) ? s.wz1 : s.wz0);
    return (x >= 0) && (x < g.W) && (y >= 0) && (y < g.H) && (!TRI || ((z >= 0) && (z < g.D)));
}

// element offsets (base + slab + row + column) and weights of plane coordinates c; cn, the normal coordinate, is read for TRI
template <bool TRI>
struct Taps {
    long long off[kPlaneTaps<TRI>];
    float w[kPlaneTaps<TRI>];
};
template <bool TRI>
__device__ __forceinline__ Taps<TRI> plane_taps(const Geom& g, long long base, float2 c, float cn) {
    const Footprint f = bilinear_footprint(g, c.x, c.y);
    const SlabFootprint s = TRI ? slab_footprint(g, cn) : SlabFootprint{};
    const long long slab = (long long)g.H * g.stride_row;
    Taps<TRI> r;
#pragma unroll
    for (int k = 0; k < kPlaneTaps<TRI>; ++k) {
        int x, y, z;
        float w;
        const bool ok = plane_tap<TRI>(g, f, s, k, x, y, z, w);
        long long o = (long long)y * g.stride_row + (long long)x * g.stride_col;
        if constexpr (TRI) o += (long long)z * slab;
        r.w[k] = ok ? w : 0.f;
        r.off[k] = base + (ok ? o : 0ll);
    }
    return r;
}

// texel indices ((p * D + z) * H + y) * W + x in the backward's (N,3,D,H,W,C) gradient (D = 1 on one-slab planes), or -1,
// and the weight bits of plane p's taps; cn is read for TRI
template <bool TRI>
__device__ __forceinline__ void plane_texels(const Geom& g, int plane, float2 c, float cn, int2* out) {
    const Footprint f = bilinear_footprint(g, c.x, c.y);
    const SlabFootprint s = TRI ? slab_footprint(g, cn) : SlabFootprint{};
#pragma unroll
    for (int k = 0; k < kPlaneTaps<TRI>; ++k) {
        int x, y, z;
        float w;
        const bool ok = plane_tap<TRI>(g, f, s, k, x, y, z, w);
        const int pz = TRI ? plane * g.D + z : plane;
        out[k] = make_int2(ok ? (pz * g.H + y) * g.W + x : -1, __float_as_int(ok ? w : 0.f));
    }
}

// channels [4q, 4q+4) of the plane mean at (x, y, z); TRI: multiplane planes (Geom::D > 1), trilinear per plane.  The loads
// of all three planes go out together on one-slab planes (12 taps), while multiplane planes (24 taps) are gathered one plane
// at a time: with all 24 loads in flight, k_sample_backward<*, true> took 11 % longer (H100 80GB HBM3, 700 W power limit).
template <bool BF16, bool TRI = false>
__device__ __forceinline__ float4 gather_features(const void* planes, const Geom& g, int view, float x, float y, float z, int q) {
    constexpr int NT = kPlaneTaps<TRI>, PB = TRI ? 1 : 3;
    const long long vbase = (long long)view * g.stride_view + 4 * q;
    float4 f[3];
#pragma unroll
    for (int p0 = 0; p0 < 3; p0 += PB) {
        Taps<TRI> t[PB];
#pragma unroll
        for (int p = 0; p < PB; ++p) {
            const int pl = p0 + p;
            t[p] = plane_taps<TRI>(g, vbase + pl * g.stride_plane, plane_coords(g, pl, x, y, z), plane_normal(g, pl, x, y, z));
        }
        float4 v[PB][NT];
#pragma unroll
        for (int k = 0; k < NT; ++k)
#pragma unroll
            for (int p = 0; p < PB; ++p) v[p][k] = load_quad<BF16>(planes, t[p].off[k]);
#pragma unroll
        for (int p = 0; p < PB; ++p) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < NT; ++k) {
                a.x = fmaf(v[p][k].x, t[p].w[k], a.x);
                a.y = fmaf(v[p][k].y, t[p].w[k], a.y);
                a.z = fmaf(v[p][k].z, t[p].w[k], a.z);
                a.w = fmaf(v[p][k].w, t[p].w[k], a.w);
            }
            f[p0 + p] = a;
        }
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
// KEEP (the backward's k_ray_backward): also writes alpha_i, 1 - alpha_i + 1e-10 and T_i to al, fc and Tr.
// -------------------------------------------------------------------------------------------
template <bool KEEP = false>
__device__ __forceinline__ void ray_weights(const float* t, const float* sg, float* w, int L, int lane,
                                            float& wsum, float& dnum, float* al = nullptr, float* fc = nullptr, float* Tr = nullptr) {
    float carry = 1.f, acc_w = 0.f, acc_d = 0.f;
    for (int base = 0; base < L - 1; base += 32) {
        const int i = base + lane;
        float alpha = 0.f, factor = 1.f, tmid = 0.f;
        if (i < L - 1) {
            const float delta = t[i + 1] - t[i];
            const float smid = __fsub_rn(__fmul_rn(__fadd_rn(sg[i], sg[i + 1]), 0.5f), 1.f);
            alpha = 1.f - expf(-__fmul_rn(softplus_t(smid), delta));
            factor = __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f);
            tmid = __fmul_rn(__fadd_rn(t[i], t[i + 1]), 0.5f);
        }
        const float incl = warp_scan_mul(factor, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        const float T = carry * excl;
        const float wi = alpha * T;
        if (i < L - 1) {
            w[i] = wi;
            if constexpr (KEEP) { al[i] = alpha; fc[i] = factor; Tr[i] = T; }
            acc_w += wi; acc_d = fmaf(wi, tmid, acc_d);
        }
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
__device__ __forceinline__ void importance_ray(const Geom& g, const float* t, const float* sg, float* w, float* cdf,
                                               float* fine, int sort_pow2, const float* u_fine,
                                               unsigned long long rng_base, int lane) {
    const int S = g.S, Sf = g.Sf;
    float wsum, dnum;
    ray_weights(t, sg, w, S, lane, wsum, dnum);
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
// merge_by_rank: unify_samples (renderer.py:289-301) for ONE ray, executed by one warp.  Writes the S + Sf merged depths t,
// densities sg and sources src (i < S: coarse i, else fine i - S).  Ties keep coarse before fine (stable sort of
// cat([coarse, fine])).  Coarse depths ascend except for the degenerate 'auto' case where no ray hits the box (t0=-1 > t1=-2,
// renderer.py:166-170 leaves them untouched): then they descend -> read reversed.  The backward rebuilds the forward's
// order with this same function.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ void merge_by_rank(const float* tc, const float* sc, const float* tf, const float* sf, int S, int Sf,
                                              float* t, float* sg, int* src, int lane) {
    const bool rev = tc[0] > tc[S - 1];
    // (not unrolled: a lane makes a few trips at most, and unrolled copies of the searches only cost registers)
#pragma unroll 1
    for (int i = lane; i < S; i += 32) {
        const int ci = rev ? S - 1 - i : i;
        const float v = tc[ci];
        int lo = 0, hi = Sf;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (tf[mid] < v) lo = mid + 1; else hi = mid; }
        const int pos = i + lo;
        t[pos] = v; sg[pos] = sc[ci]; src[pos] = ci;
    }
#pragma unroll 1
    for (int j = lane; j < Sf; j += 32) {
        const float v = tf[j];
        int lo = 0, hi = S;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (tc[rev ? S - 1 - mid : mid] <= v) lo = mid + 1; else hi = mid; }
        const int pos = j + lo;
        t[pos] = v; sg[pos] = sf[j]; src[pos] = S + j;
    }
    __syncwarp();
}

// -------------------------------------------------------------------------------------------
// composite_weights: unify_samples (renderer.py:289-301) + the weight part of the final
// MipRayMarcher2 pass (ray_marcher.py:25-44) for ONE ray, executed by one warp.
//   tc, sc : S coarse depths/densities   tf, sf : Sf fine depths (ascending) / densities
//   t, sg, w : scratch of L = S+Sf floats each; src : L ints
// On return w[j] holds omega_j = (w_{j-1}+w_j)/2 for merged position j and src[j] names its
// sample (i < S: coarse i, else fine i-S), so  sum_i w_i (c_i+c_{i+1})/2 == sum_j omega_j c_j.
// -------------------------------------------------------------------------------------------
__device__ __forceinline__ void composite_weights(const float* tc, const float* sc, const float* tf, const float* sf,
                                                  int S, int Sf, float* t, float* sg, float* w, int* src, int lane,
                                                  float& wsum, float& dnum) {
    const int L = S + Sf;
    merge_by_rank(tc, sc, tf, sf, S, Sf, t, sg, src, lane);
    ray_weights(t, sg, w, L, lane, wsum, dnum);
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
