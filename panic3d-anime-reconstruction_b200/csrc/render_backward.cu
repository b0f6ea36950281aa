// Backward of ImportanceRenderer.forward (first order; what the ecrutileE training loop needs:
// loss_orthocondA.py:171,279,343,426 call G.f -> renderer under autograd; R1's double-backward flows
// through the discriminator only - SURVEY.md section 3.3).
//
// Differentiated: tri-plane features and the four OSGDecoder tensors.  Constants, exactly as in the
// reference graph: ray origins/directions, stratified depths, the importance depths
// (sample_importance runs under torch.no_grad, renderer.py:332) and every density that a crop/cull/binarize
// mask overwrote in place (renderer.py:187-198 - the assignment cuts the graph).
//
// Recompute-based, fp32, two kernels on top of the v1 forward's scratch (depths, masked densities, colours):
//   k_ray_backward     warp per ray: rebuild the merged order and (alpha, T, w); from the incoming
//                      (d_rgb, d_depth, d_wsum, d_xyz) form dL/dw_i, then dL/dalpha_i via a suffix scan,
//                      dL/dsigma_j and omega_j per sample  (ray_marcher.py:25-57 differentiated by hand)
//   k_sample_backward  CTA of 128 samples: re-gather features, re-run the decoder keeping pre-activations
//                      in smem, back-propagate; weight gradients reduced per CTA in smem then one
//                      red.global per element; feature gradients scattered to the channels-last
//                      tri-plane gradient with 128-bit vector atomics (one per tap per 4 channels).
#include "render_device.cuh"

namespace p3d {
namespace {

using namespace dev;

constexpr int kT = 128;

struct RayBwdArgs {
    Geom g;
    const float *depth_c, *sigma_c, *rgb_c, *depth_f, *sigma_f, *rgb_f, *ro, *rd;
    const float *g_rgb, *g_depth, *g_wsum, *g_xyz;      // incoming gradients (N*M, 32 | 1 | 1 | 3)
    const float* out_depth;                              // forward's final (clamped) depth
    const unsigned int* bounds;
    float *dsig_c, *om_c, *dsig_f, *om_f;                // per-sample outputs
    long long R;
};

__global__ void __launch_bounds__(128) k_ray_backward(const RayBwdArgs a) {
    extern __shared__ float smem[];
    const Geom& g = a.g;
    const int S = g.S, Sf = g.Sf, L = S + Sf, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long ray = (long long)blockIdx.x * 4 + warp;
    if (ray >= a.R) return;
    float* t = smem + warp * (8 * L);
    float* sg = t + L;
    float* w = sg + L;            // interval weights w_i
    float* al = w + L;            // alpha_i
    float* fc = al + L;           // 1 - alpha_i + 1e-10
    float* Tr = fc + L;           // transmittance T_i
    float* q = Tr + L;            // g_rgb . c_j per merged sample, later dL/dsigmabar_i
    int* src = reinterpret_cast<int*>(q + L);

    merge_by_rank(a.depth_c + ray * S, a.sigma_c + ray * S, a.depth_f + ray * Sf, a.sigma_f + ray * Sf, S, Sf, t, sg, src, lane);
    float W, D;                   // the forward's wsum and dnum, bit for bit
    ray_weights<true>(t, sg, w, L, lane, W, D, al, fc, Tr);
    __syncwarp();
    // q_j = g_rgb . c_j   (lane = channel)
    const float grgb = a.g_rgb[ray * kRgb + lane];
    for (int j = 0; j < L; ++j) {
        const int s = src[j];
        const float c = s < S ? a.rgb_c[(ray * S + s) * kRgb + lane] : a.rgb_f[(ray * Sf + (s - S)) * kRgb + lane];
        const float d = warp_sum(grgb * c);
        if (lane == 0) q[j] = d;
    }
    const float grgb_sum = warp_sum(grgb);
    float gx_o = 0.f, gx_d = 0.f, gx_sum = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float gk = a.g_xyz[ray * 3 + k];
        gx_o = fmaf(gk, a.ro[ray * 3 + k], gx_o); gx_d = fmaf(gk, a.rd[ray * 3 + k], gx_d); gx_sum += gk;
    }
    // depth = clamp(nan_to_num(D/W)): gradient only where the value is finite and strictly inside the clamp range
    const float lo_b = ordered_to_float(a.bounds[0]), hi_b = ordered_to_float(a.bounds[1]);
    const float depth_raw = D / W;
    const bool depth_live = (W != 0.f) && !isnan(depth_raw) && depth_raw >= lo_b && depth_raw <= hi_b;
    const float gdep = depth_live ? a.g_depth[ray] : 0.f;
    const float gW = a.g_wsum[ray];
    const float back = g.white_back ? 1.f : 0.f;
    const float common = gW - 2.f * back * (grgb_sum + gx_sum) + 2.f * gx_o;
    __syncwarp();
    // dL/dw_i = P_i ; prefix sums of w_i P_i for the suffix term
    float pcarry = 0.f;
    float total = 0.f;
    for (int pass = 0; pass < 2; ++pass) {
        pcarry = 0.f;
        for (int base = 0; base < L - 1; base += 32) {
            const int i = base + lane;
            float P = 0.f, wP = 0.f;
            if (i < L - 1) {
                const float tmid = __fmul_rn(__fadd_rn(t[i], t[i + 1]), 0.5f);
                P = (q[i] + q[i + 1]) + 2.f * gx_d * tmid + common + (depth_live ? gdep * (tmid - depth_raw) / W : 0.f);
                wP = w[i] * P;
            }
            const float incl = warp_scan_add(wP, lane) + pcarry;
            pcarry = __shfl_sync(0xffffffffu, incl, 31);
            if (pass == 1 && i < L - 1) {
                const float suffix = total - incl;                              // sum_{k>i} w_k P_k
                const float dalpha = Tr[i] * P - suffix / fc[i];
                const float smid = __fsub_rn(__fmul_rn(__fadd_rn(sg[i], sg[i + 1]), 0.5f), 1.f);
                const float dsp = smid > 20.f ? 1.f : sigmoid_t(smid);          // d softplus
                al[i] = dalpha * (1.f - al[i]) * (t[i + 1] - t[i]) * dsp;       // dL/dsigmabar_i (reuse al[])
            }
        }
        if (pass == 0) total = pcarry;
    }
    __syncwarp();
    // per sample: dsigma_j = (dsb_{j-1} + dsb_j)/2 ; omega_j = (w_{j-1} + w_j)/2
    for (int j = lane; j < L; j += 32) {
        const float dl = j > 0 ? al[j - 1] : 0.f, dr = j < L - 1 ? al[j] : 0.f;
        const float wl = j > 0 ? w[j - 1] : 0.f, wr = j < L - 1 ? w[j] : 0.f;
        const float ds = 0.5f * (dl + dr), om = 0.5f * (wl + wr);
        const int s = src[j];
        if (s < S) { a.dsig_c[ray * S + s] = ds; a.om_c[ray * S + s] = om; }
        else { a.dsig_f[ray * Sf + (s - S)] = ds; a.om_f[ray * Sf + (s - S)] = om; }
    }
}

// ------------------------------------------------------------------------------------------------
struct SampleBwdArgs {
    Geom g;
    const void* planes;
    const float *w1, *b1, *w2, *b2;
    const float *ro, *rd;
    const float* depth;          // (R*per_ray) depths of this pass
    const float* dsig;           // dL/dsigma (post-mask) per sample
    const float* omega;          // omega per sample
    const float* g_rgb;          // (R,32)
    float* d_planes;             // (N,3,H,W,32) contiguous fp32 gradient (its own canonical strides)
    float *d_w1, *d_b1, *d_w2, *d_b2;   // gradients w.r.t. the RAW parameters (gains folded in)
    long long total;
    int per_ray;
    // point-query mode (run_model backward, renderer.py:266-280): positions come from `coords` (N,K,3), the incoming
    // gradients are per point - dsig = g_sigma (N,K), g_col = g_rgb (N,K,32) - and there are no masks and no omega
    const float* coords;
    const float* g_col;
    long long per_view;
};

constexpr int kXs = 33, kHs = 65, kDs = 36;
// taps per sample: 4 per plane, 8 per plane for multiplane tri-planes (TRI)
template <bool TRI> constexpr int kTaps = 3 * kPlaneTaps<TRI>;
template <bool TRI> constexpr size_t kBwdSmemFloats = (size_t)kHidden * kC + kOut * kHidden + kHidden + 36 +
                                                      (size_t)kT * (kXs + kHs + kHs + kDs + kHs + kXs) + kT * kTaps<TRI> * 2 + kT * 2 + kT;

// TRI: multiplane tri-planes (g.D > 1): trilinear re-gather, 8 taps per plane scattered to the (N,3,D,H,W,C) gradient
template <bool BF16, bool TRI>
__global__ void __launch_bounds__(kT) k_sample_backward(const SampleBwdArgs a) {
    constexpr int NT = kTaps<TRI>, PT = NT / 3;
    extern __shared__ float sm[];
    float* s_w1 = sm;                        // [64][32]  effective (gain folded)
    float* s_w2 = s_w1 + kHidden * kC;       // [33][64]
    float* s_b1 = s_w2 + kOut * kHidden;     // [64]
    float* s_b2 = s_b1 + kHidden;            // [36]
    float* s_x = s_b2 + 36;                  // [128][33] features
    float* s_pre = s_x + kT * kXs;           // [128][65] pre-activations
    float* s_hs = s_pre + kT * kHs;          // [128][65] softplus(pre)
    float* s_do = s_hs + kT * kHs;           // [128][36] d_logits
    float* s_dp = s_do + kT * kDs;           // [128][65] d_pre
    float* s_dx = s_dp + kT * kHs;           // [128][33] d_features (already / 3)
    int2* s_tap = reinterpret_cast<int2*>(s_dx + kT * kXs);   // [128][NT]
    float* s_xz = reinterpret_cast<float*>(s_tap + kT * NT);  // [128][2]
    int* s_view = reinterpret_cast<int*>(s_xz + kT * 2);      // [128]

    const Geom& g = a.g;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long tile0 = (long long)blockIdx.x * kT;
    for (int i = tid; i < kHidden * kC; i += kT) s_w1[i] = __fmul_rn(a.w1[i], g.w1_gain);
    for (int i = tid; i < kOut * kHidden; i += kT) s_w2[i] = __fmul_rn(a.w2[i], g.w2_gain);
    if (tid < kHidden) s_b1[tid] = __fmul_rn(a.b1[tid], g.b1_gain);
    if (tid < kOut) s_b2[tid] = __fmul_rn(a.b2[tid], g.b2_gain);

    // ---- A) positions, tap records (for the scatter), features
    {
        const int sub = lane >> 3, qd = lane & 7;
        for (int round = 0; round < 8; ++round) {
            const int local = warp * 32 + round * 4 + sub;
            const long long gidx = tile0 + local;
            float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
            float px = 0.f, pz = 0.f;
            int view = 0;
            const bool ok = gidx < a.total;
            float py = 0.f;
            if (ok) {
                if (a.coords) {
                    view = (int)(gidx / a.per_view);
                    px = a.coords[gidx * 3]; py = a.coords[gidx * 3 + 1]; pz = a.coords[gidx * 3 + 2];
                } else {
                    const long long ray = gidx / a.per_ray;
                    view = (int)(ray / g.M);
                    const float3 pt = ray_point(a.ro + ray * 3, a.rd + ray * 3, a.depth[gidx]);
                    px = pt.x; py = pt.y; pz = pt.z;
                }
                f = gather_features<BF16, TRI>(a.planes, g, view, px, py, pz, qd);
            }
            if (qd < 3) {                                         // lanes 0..2 of a sample record plane qd's taps
                if (ok) {
                    plane_texels<TRI>(g, qd, plane_coords(g, qd, px, py, pz), plane_normal(g, qd, px, py, pz), s_tap + local * NT + qd * PT);
                } else {
#pragma unroll
                    for (int k = 0; k < PT; ++k) s_tap[local * NT + qd * PT + k] = make_int2(-1, 0);
                }
            }
            float* dst = s_x + local * kXs + 4 * qd;
            dst[0] = f.x; dst[1] = f.y; dst[2] = f.z; dst[3] = f.w;
            if (qd == 0) { s_xz[local * 2] = px; s_xz[local * 2 + 1] = pz; s_view[local] = view; }
        }
    }
    __syncthreads();
    // ---- B) decoder forward, thread per sample; C) d_logits; D) back through the two layers
    {
        const long long gidx = tile0 + tid;
        const bool live = gidx < a.total;
        float o[kOut];
#pragma unroll
        for (int m = 0; m < kOut; ++m) o[m] = s_b2[m];
        float x[kC];
#pragma unroll
        for (int k = 0; k < kC; ++k) x[k] = s_x[tid * kXs + k];
        for (int j = 0; j < kHidden; ++j) {
            float h = s_b1[j];
#pragma unroll
            for (int k = 0; k < kC; ++k) h = fmaf(x[k], s_w1[j * kC + k], h);
            const float hs = softplus_t(h);
            s_pre[tid * kHs + j] = h;
            s_hs[tid * kHs + j] = hs;
#pragma unroll
            for (int m = 0; m < kOut; ++m) o[m] = fmaf(hs, s_w2[m * kHidden + j], o[m]);
        }
        float dsg = 0.f, om = 0.f;
        long long ray = 0;
        const bool pts = a.coords != nullptr;
        if (live) { dsg = a.dsig[gidx]; if (!pts) { om = a.omega[gidx]; ray = gidx / a.per_ray; } }
        // a density overwritten by a crop/cull/binarize mask is a constant of the reference graph (run_model has no masks)
        if (!pts && apply_masks(g, o[0], s_xz[tid * 2], s_xz[tid * 2 + 1]) != o[0]) dsg = 0.f;
        float dlog[kOut];
        dlog[0] = dsg;
#pragma unroll
        for (int c = 0; c < kRgb; ++c) {
            const float sgm = sigmoid_t(o[1 + c]);
            const float dcol = !live ? 0.f : (pts ? a.g_col[gidx * kRgb + c] : 2.f * om * a.g_rgb[ray * kRgb + c]);   // d rgb / d c_j = 2 * omega_j
            dlog[1 + c] = dcol * (g.force_sigmoid ? 1.f : 1.002f) * sgm * (1.f - sgm);
        }
#pragma unroll
        for (int m = 0; m < kOut; ++m) s_do[tid * kDs + m] = dlog[m];
        float dx[kC];
#pragma unroll
        for (int k = 0; k < kC; ++k) dx[k] = 0.f;
        for (int j = 0; j < kHidden; ++j) {
            float dh = 0.f;
#pragma unroll
            for (int m = 0; m < kOut; ++m) dh = fmaf(dlog[m], s_w2[m * kHidden + j], dh);
            const float pre = s_pre[tid * kHs + j];
            const float dpre = dh * (pre > 20.f ? 1.f : sigmoid_t(pre));
            s_dp[tid * kHs + j] = dpre;
#pragma unroll
            for (int k = 0; k < kC; ++k) dx[k] = fmaf(dpre, s_w1[j * kC + k], dx[k]);
        }
#pragma unroll
        for (int k = 0; k < kC; ++k) s_dx[tid * kXs + k] = dx[k] * (1.f / 3.f);            // d(mean over 3 planes)
    }
    __syncthreads();
    // ---- E) parameter gradients: two small GEMMs over the CTA's 128 samples, register-blocked 4x4 per thread (8 shared
    //         loads feed 16 FMAs; the first version's 2 loads per FMA made this phase the whole kernel's bottleneck),
    //         then one red.global per element
    {
        // dW2[m][j] = sum_s dlog[s][m] * hs[s][j]: 9 x 16 blocks of 4x4 (rows 33..35 of the last block are padding)
        for (int blk = tid; blk < 9 * 16; blk += kT) {
            const int mb = blk >> 4, jb = blk & 15;
            float acc[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
            for (int sidx = 0; sidx < kT; ++sidx) {
                const float4 d4 = *reinterpret_cast<const float4*>(s_do + sidx * kDs + 4 * mb);
                const float dl[4] = {d4.x, d4.y, d4.z, d4.w};
                float hv[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) hv[j] = s_hs[sidx * kHs + 4 * jb + j];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(dl[i], hv[j], acc[i][j]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int m = 4 * mb + i;
                if (m >= kOut) continue;
#pragma unroll
                for (int j = 0; j < 4; ++j) atomicAdd(a.d_w2 + m * kHidden + 4 * jb + j, acc[i][j] * g.w2_gain);
            }
        }
        // dW1[j][k] = sum_s dpre[s][j] * x[s][k]: 16 x 8 blocks of 4x4, one per thread
        {
            const int jb = tid >> 3, kb = tid & 7;
            float acc[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
            for (int sidx = 0; sidx < kT; ++sidx) {
                float dp[4], xv[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) { dp[i] = s_dp[sidx * kHs + 4 * jb + i]; xv[i] = s_x[sidx * kXs + 4 * kb + i]; }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(dp[i], xv[j], acc[i][j]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) atomicAdd(a.d_w1 + (4 * jb + i) * kC + 4 * kb + j, acc[i][j] * g.w1_gain);
        }
    }
    if (tid < kOut) {
        float acc = 0.f;
        for (int sidx = 0; sidx < kT; ++sidx) acc += s_do[sidx * kDs + tid];
        atomicAdd(a.d_b2 + tid, acc * g.b2_gain);
    }
    if (tid >= 64 && tid < 64 + kHidden) {
        const int j = tid - 64;
        float acc = 0.f;
        for (int sidx = 0; sidx < kT; ++sidx) acc += s_dp[sidx * kHs + j];
        atomicAdd(a.d_b1 + j, acc * g.b1_gain);
    }
    // ---- F) scatter d_features to the tri-plane gradient: 8 lanes x float4 per tap
    {
        const int sub = lane >> 3, qd = lane & 7;
        const long long plane_elems = (long long)3 * (TRI ? g.D : 1) * g.H * g.W * kC;
        for (int round = 0; round < 8; ++round) {
            const int local = warp * 32 + round * 4 + sub;
            if (tile0 + local >= a.total) continue;
            const float* dxr = s_dx + local * kXs + 4 * qd;
            const float4 dv = make_float4(dxr[0], dxr[1], dxr[2], dxr[3]);
            float* base = a.d_planes + (long long)s_view[local] * plane_elems + 4 * qd;
#pragma unroll
            for (int k = 0; k < NT; ++k) {
                const int2 tp = s_tap[local * NT + k];
                if (tp.x < 0) continue;
                const float wgt = __int_as_float(tp.y);
                atomicAdd(reinterpret_cast<float4*>(base + (long long)tp.x * kC), make_float4(dv.x * wgt, dv.y * wgt, dv.z * wgt, dv.w * wgt));
            }
        }
    }
}

// the k_sample_backward instance for these planes and its dynamic shared memory (bytes)
using SampleBwdKernel = void (*)(const SampleBwdArgs);
SampleBwdKernel sample_backward_kernel(const Geom& g, const p3d_render_params* p, size_t* smem) {
    if (g.D > 1) {
        *smem = kBwdSmemFloats<true> * sizeof(float);
        return p->planes_bf16 ? k_sample_backward<true, true> : k_sample_backward<false, true>;
    }
    *smem = kBwdSmemFloats<false> * sizeof(float);
    return p->planes_bf16 ? k_sample_backward<true, false> : k_sample_backward<false, false>;
}

}  // namespace

int render_backward_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                       const float* w2, const float* b2, const float* ro, const float* rd, const Workspace& ws,
                       const float* out_depth, const float* g_rgb, const float* g_depth, const float* g_wsum,
                       const float* g_xyz, void* scratch, size_t scratch_bytes, float* d_planes, float* d_w1, float* d_b1,
                       float* d_w2, float* d_b2, cudaStream_t stream) {
    const long long R = (long long)g.N * g.M;
    const size_t per = (size_t)R * (g.S + g.Sf) * sizeof(float);
    if (scratch_bytes < 2 * per + 1024) { set_error("backward scratch too small: need %zu bytes", 2 * per + 1024); return P3D_EWORKSPACE; }
    float* dsig_c = reinterpret_cast<float*>(scratch);
    float* dsig_f = dsig_c + (size_t)R * g.S;
    float* om_c = dsig_f + (size_t)R * g.Sf;
    float* om_f = om_c + (size_t)R * g.S;
    RayBwdArgs ra{};
    ra.g = g; ra.depth_c = ws.depth_c; ra.sigma_c = ws.sigma_c; ra.rgb_c = ws.rgb_c; ra.depth_f = ws.depth_f; ra.sigma_f = ws.sigma_f;
    ra.rgb_f = ws.rgb_f; ra.ro = ro; ra.rd = rd; ra.g_rgb = g_rgb; ra.g_depth = g_depth; ra.g_wsum = g_wsum; ra.g_xyz = g_xyz;
    ra.out_depth = out_depth; ra.bounds = ws.bounds; ra.dsig_c = dsig_c; ra.om_c = om_c; ra.dsig_f = dsig_f; ra.om_f = om_f; ra.R = R;
    const size_t smem_ray = (size_t)4 * 8 * (g.S + g.Sf) * sizeof(float);
    if (smem_ray > 48 * 1024) P3D_CUDA_TRY(cudaFuncSetAttribute(k_ray_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ray));
    k_ray_backward<<<(unsigned)((R + 3) / 4), 128, smem_ray, stream>>>(ra);
    P3D_LAUNCH_CHECK();
    size_t smem;
    auto kern = sample_backward_kernel(g, p, &smem);
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int pass = 0; pass < 2; ++pass) {
        const int per_ray = pass == 0 ? g.S : g.Sf;
        if (per_ray == 0) continue;
        SampleBwdArgs sa{};
        sa.g = g; sa.planes = planes; sa.w1 = w1; sa.b1 = b1; sa.w2 = w2; sa.b2 = b2; sa.ro = ro; sa.rd = rd;
        sa.depth = pass == 0 ? ws.depth_c : ws.depth_f; sa.dsig = pass == 0 ? dsig_c : dsig_f; sa.omega = pass == 0 ? om_c : om_f;
        sa.g_rgb = g_rgb; sa.d_planes = d_planes; sa.d_w1 = d_w1; sa.d_b1 = d_b1; sa.d_w2 = d_w2; sa.d_b2 = d_b2;
        sa.total = R * per_ray; sa.per_ray = per_ray;
        const long long blocks = (sa.total + kT - 1) / kT;
        kern<<<(unsigned)blocks, kT, smem, stream>>>(sa);
        P3D_LAUNCH_CHECK();
    }
    return P3D_OK;
}

int decode_points_backward_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                              const float* w2, const float* b2, const float* coords, long long n_pts, const float* g_rgb,
                              const float* g_sigma, float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2,
                              cudaStream_t stream) {
    size_t smem;
    auto kern = sample_backward_kernel(g, p, &smem);
    P3D_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SampleBwdArgs sa{};
    sa.g = g; sa.planes = planes; sa.w1 = w1; sa.b1 = b1; sa.w2 = w2; sa.b2 = b2;
    sa.coords = coords; sa.dsig = g_sigma; sa.g_col = g_rgb; sa.per_view = n_pts; sa.per_ray = 1;
    sa.d_planes = d_planes; sa.d_w1 = d_w1; sa.d_b1 = d_b1; sa.d_w2 = d_w2; sa.d_b2 = d_b2;
    sa.total = (long long)g.N * n_pts;
    const long long blocks = (sa.total + kT - 1) / kT;
    kern<<<(unsigned)blocks, kT, smem, stream>>>(sa);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

}  // namespace p3d
