// extern "C" surface of libp3d.so (see include/p3d_render.h) + small utility kernels.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <vector>

#include "render_internal.cuh"

namespace p3d {

std::atomic<uint64_t> g_launches{0};
static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ------------------------------------------------------------------------------------------
// profiler
// ------------------------------------------------------------------------------------------
struct ProfRec { int slot; cudaEvent_t a, b; };
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof_pending;
static std::vector<cudaEvent_t> g_prof_pool;
static double g_prof_ms[PROF_SLOTS] = {0};
static uint64_t g_prof_n[PROF_SLOTS] = {0};
static cudaEvent_t g_prof_open[PROF_SLOTS] = {nullptr};

bool profile_enabled() { return g_prof_on; }
static cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
}
void profile_begin(int slot, cudaStream_t stream) {
    std::lock_guard<std::mutex> l(g_prof_mu);
    cudaEvent_t e = prof_event();
    cudaEventRecord(e, stream);
    g_prof_open[slot] = e;
}
void profile_end(int slot, cudaStream_t stream) {
    std::lock_guard<std::mutex> l(g_prof_mu);
    cudaEvent_t e = prof_event();
    cudaEventRecord(e, stream);
    g_prof_pending.push_back({slot, g_prof_open[slot], e});
    g_prof_open[slot] = nullptr;
}

// ------------------------------------------------------------------------------------------
// derived scalars: computed in double from the Python-side doubles, then rounded to fp32 once,
// exactly where the reference's Python scalars meet an fp32 tensor.
// ------------------------------------------------------------------------------------------
int make_geom(const p3d_render_params* p, Geom* g) {
    P3D_REQUIRE(p != nullptr, "params is NULL");
    P3D_REQUIRE(p->channels == kC && p->hidden == kHidden && p->out_dim == kOut,
                "decoder shape %d->%d->%d unsupported (built for %d->%d->%d)", p->channels, p->hidden, p->out_dim, kC,
                kHidden, kOut);
    P3D_REQUIRE(p->n_views >= 0 && p->n_rays >= 0 && p->plane_h > 0 && p->plane_w > 0, "bad sizes");
    P3D_REQUIRE(p->box_warp > 0, "box_warp must be > 0");
    memset(g, 0, sizeof(*g));
    g->N = p->n_views; g->M = p->n_rays; g->S = p->n_coarse; g->Sf = p->n_fine; g->H = p->plane_h; g->W = p->plane_w;
    g->stride_view = p->stride_view; g->stride_plane = p->stride_plane; g->stride_row = p->stride_row; g->stride_col = p->stride_col;
    // quads of 4 channels: 16 B (fp32) / 8 B (bf16) vector loads
    P3D_REQUIRE(p->stride_view % 4 == 0 && p->stride_plane % 4 == 0 && p->stride_row % 4 == 0 && p->stride_col % 4 == 0,
                "plane strides must be multiples of 4 elements");
    // multiplane tri-planes: D slabs per plane, slab d at d * plane_h * stride_row inside its plane
    P3D_REQUIRE(p->plane_depth >= 0, "plane_depth must be >= 0, got %d", p->plane_depth);
    g->D = p->plane_depth > 1 ? p->plane_depth : 1;
    if (g->D > 1) {
        P3D_REQUIRE(p->stride_plane >= (int64_t)g->D * p->plane_h * p->stride_row,
                    "stride_plane %lld is shorter than plane_depth * plane_h * stride_row = %lld", (long long)p->stride_plane,
                    (long long)g->D * p->plane_h * p->stride_row);
        P3D_REQUIRE(p->stride_view == 0 || p->stride_view >= 3 * p->stride_plane,
                    "stride_view %lld is shorter than 3 * stride_plane = %lld", (long long)p->stride_view,
                    3 * (long long)p->stride_plane);
    }
    g->coord_scale = (float)(2.0 / p->box_warp);
    g->half_box = (float)(p->box_warp / 2.0);
    g->ray_mode = p->ray_mode; g->disparity = p->disparity; g->white_back = p->white_back; g->plane_mode = p->plane_mode;
    if (p->ray_mode == P3D_RAYS_NUMERIC) {
        g->ray_start = (float)p->ray_start; g->ray_end = (float)p->ray_end;
        const int S = p->n_coarse > 1 ? p->n_coarse : 2;
        g->lin_step = (g->ray_end - g->ray_start) / (float)(S - 1);                  // torch.linspace: fp32 step
        g->depth_delta = (float)((p->ray_end - p->ray_start) / (double)(S - 1));      // python double -> fp32
        g->inv_start = (float)(1.0 / p->ray_start); g->inv_end = (float)(1.0 / p->ray_end);
        g->disp_delta = (float)(1.0 / (double)(S - 1));
    }
    g->crop_on = p->triplane_crop > 0; g->crop_limit = (float)(p->box_warp / 2.0 - p->triplane_crop);
    g->binarize_on = p->binarize_clouds > 0; g->cull_on = !g->binarize_on && p->cull_clouds > 0;
    g->cull_thresh = (float)(g->binarize_on ? p->binarize_clouds : p->cull_clouds);
    g->force_sigmoid = p->force_sigmoid;
    g->w1_gain = p->w1_gain; g->b1_gain = p->b1_gain; g->w2_gain = p->w2_gain; g->b2_gain = p->b2_gain;
    g->seed = p->seed;
    return P3D_OK;
}

static size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

size_t workspace_layout(const p3d_render_params* p, void* base, Workspace* ws) {
    const size_t R = (size_t)p->n_views * (size_t)p->n_rays;
    const size_t S = (size_t)p->n_coarse, Sf = (size_t)p->n_fine;
    size_t off = 0;
    char* b = reinterpret_cast<char*>(base);
    auto take = [&](size_t bytes) { void* ptr = b ? b + off : nullptr; off += align_up(bytes); return ptr; };
    Workspace w;
    w.bounds = (unsigned int*)take(64);
    w.depth_c = (float*)take(R * S * 4);
    w.sigma_c = (float*)take(R * S * 4);
    w.rgb_c = (float*)take(R * S * kRgb * 4);
    w.depth_f = (float*)take(R * Sf * 4);
    w.sigma_f = (float*)take(R * Sf * 4);
    w.rgb_f = (float*)take(R * Sf * kRgb * 4);
    w.ray_t0 = (float*)take(R * 4);
    w.ray_t1 = (float*)take(R * 4);
    if (ws) *ws = w;
    return off;
}

// ------------------------------------------------------------------------------------------
// layout pre-pass: (n_planes, C, H, W) fp32 -> (n_planes, H, W, C) fp32|bf16.  32x32 smem transpose.
// ------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void k_planes_to_cl(const float* __restrict__ in, void* __restrict__ out, int C, long long HW) {
    __shared__ float tile[32][33];
    const long long plane = blockIdx.z;
    const long long p0 = (long long)blockIdx.x * 32;     // pixel tile
    const int c0 = blockIdx.y * 32;                      // channel tile
    const int tx = threadIdx.x, ty = threadIdx.y;        // 32 x 8
    for (int r = ty; r < 32; r += 8) {
        const int c = c0 + r;
        const long long px = p0 + tx;
        tile[r][tx] = (c < C && px < HW) ? in[(plane * C + c) * HW + px] : 0.f;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const long long px = p0 + r;
        const int c = c0 + tx;
        if (c < C && px < HW) {
            const long long o = (plane * HW + px) * C + c;
            if (BF16) reinterpret_cast<__nv_bfloat16*>(out)[o] = __float2bfloat16_rn(tile[tx][r]);
            else reinterpret_cast<float*>(out)[o] = tile[tx][r];
        }
    }
}

// C == 32 fast path: a CTA moves a 32-channel x 128-pixel tile with 128-bit accesses on both sides.  Loads: a warp reads
// 4 channels x 32 pixels (four 128-byte rows); the transposed tile tileT[pixel][channel] has pitch 33, which makes both
// the scalar transposing stores (bank = 4q + j + c) and the channel-vector reads (bank = px + 4c4 + i) conflict-free;
// stores: a warp writes 4 pixels x 32 channels = 512 contiguous bytes (256 for bf16).
template <bool BF16>
__global__ void __launch_bounds__(256) k_planes_to_cl32(const float* __restrict__ in, void* __restrict__ out, long long HW) {
    __shared__ float tileT[128 * 33];
    const long long plane = blockIdx.y;
    const long long p0 = (long long)blockIdx.x * 128;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    {
        const int c_sub = lane >> 3, q = lane & 7;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int task = warp + 8 * i, cg = task & 7, seg = task >> 3;
            const long long px = p0 + 32 * seg + 4 * q;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (px < HW) v = *reinterpret_cast<const float4*>(in + (plane * 32 + 4 * cg + c_sub) * HW + px);   // HW % 4 == 0
            float* dst = tileT + (32 * seg + 4 * q) * 33 + 4 * cg + c_sub;
            dst[0] = v.x; dst[33] = v.y; dst[66] = v.z; dst[99] = v.w;
        }
    }
    __syncthreads();
    {
        const int c4 = lane & 7, px_sub = lane >> 3;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int pl = (warp + 8 * i) * 4 + px_sub;
            const long long px = p0 + pl;
            if (px >= HW) continue;
            const float* src = tileT + pl * 33 + 4 * c4;
            const float4 v = make_float4(src[0], src[1], src[2], src[3]);
            const long long o = (plane * HW + px) * 32 + 4 * c4;
            if (BF16) {
                __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
                *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + o) =
                    make_uint2(*reinterpret_cast<unsigned*>(&lo), *reinterpret_cast<unsigned*>(&hi));
            } else {
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + o) = v;
            }
        }
    }
}

// RaySampler.forward, ray_sampler.py:24-63
__global__ void k_raygen_pinhole(const float* __restrict__ c2w, const float* __restrict__ K, int N, int R,
                                 float* __restrict__ ro, float* __restrict__ rd) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long M = (long long)R * R;
    if (idx >= (long long)N * M) return;
    const int n = (int)(idx / M);
    const int m = (int)(idx - (long long)n * M);
    const int row = m / R, col = m - row * R;
    const float* k = K + n * 9;
    const float* c = c2w + n * 16;
    const float fx = k[0], sk = k[1], cx = k[2], fy = k[4], cy = k[5];
    const float inv_r = __fdiv_rn(1.f, (float)R), half = __fdiv_rn(0.5f, (float)R);
    const float xc = __fadd_rn(__fmul_rn((float)col, inv_r), half);
    const float yc = __fadd_rn(__fmul_rn((float)row, inv_r), half);
    // (x - cx + cy*sk/fy - sk*y/fy) / fx , (y - cy) / fy      (z_cam = 1)
    float xl = __fsub_rn(xc, cx);
    xl = __fadd_rn(xl, __fdiv_rn(__fmul_rn(cy, sk), fy));
    xl = __fsub_rn(xl, __fdiv_rn(__fmul_rn(sk, yc), fy));
    xl = __fdiv_rn(xl, fx);
    const float yl = __fdiv_rn(__fsub_rn(yc, cy), fy);
    float d[3], o[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float w = fmaf(c[i * 4 + 0], xl, fmaf(c[i * 4 + 1], yl, c[i * 4 + 2])) + c[i * 4 + 3];
        o[i] = c[i * 4 + 3];
        d[i] = __fsub_rn(w, o[i]);
    }
    const float nrm = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);   // F.normalize eps
#pragma unroll
    for (int i = 0; i < 3; ++i) { ro[idx * 3 + i] = o[i]; rd[idx * 3 + i] = __fdiv_rn(d[i], nrm); }
}

// get_rays_ortho, lustrous_renders_v1.py:78-104
__global__ void k_raygen_ortho(const float* __restrict__ rot, const float* __restrict__ dist, int N, int R, float bw,
                               float* __restrict__ ro, float* __restrict__ rd) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long M = (long long)R * R;
    if (idx >= (long long)N * M) return;
    const int n = (int)(idx / M);
    const int m = (int)(idx - (long long)n * M);
    const int row = m / R, col = m - row * R;
    const float half = __fdiv_rn(bw, 2.f);
    const float gx = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)col, 0.5f), (float)R), bw), half);
    const float gy = -__fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)row, 0.5f), (float)R), bw), half);
    const float z0 = dist[n], z1 = __fadd_rn(-1.f, dist[n]);
    const float* r = rot + n * 9;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float a = r[i * 3 + 0] * gx + r[i * 3 + 1] * gy;
        const float p0 = a + r[i * 3 + 2] * z0, p1 = a + r[i * 3 + 2] * z1;
        ro[idx * 3 + i] = p0;
        rd[idx * 3 + i] = __fsub_rn(p1, p0);
    }
}

// pairs[2*(i+1)], pairs[2*(i+1)+1] = (min, max) of view i  ->  pairs[0], pairs[1] = batch-wide (min, max)
__global__ void k_merge_bounds(float* pairs, int n) {
    float lo = INFINITY, hi = -INFINITY;
    for (int i = threadIdx.x; i < n; i += 32) { lo = fminf(lo, pairs[2 * (i + 1)]); hi = fmaxf(hi, pairs[2 * (i + 1) + 1]); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if (threadIdx.x == 0) { pairs[0] = lo; pairs[1] = hi; }
}

// ------------------------------------------------------------------------------------------
// host arena for the *_host entry point
// ------------------------------------------------------------------------------------------
struct Arena {
    std::mutex mu;
    std::vector<std::pair<void*, size_t>> bufs;   // slot -> (ptr, bytes)
    cudaStream_t stream = nullptr, copy_in = nullptr, copy_out = nullptr;
    std::vector<cudaEvent_t> events;
    int event(size_t i, cudaEvent_t* out) {
        while (events.size() <= i) {
            cudaEvent_t e;
            P3D_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            events.push_back(e);
        }
        *out = events[i];
        return P3D_OK;
    }
    int get(size_t slot, size_t bytes, void** out) {
        if (bufs.size() <= slot) bufs.resize(slot + 1, {nullptr, 0});
        if (bufs[slot].second < bytes) {
            if (bufs[slot].first) cudaFree(bufs[slot].first);
            bufs[slot] = {nullptr, 0};
            P3D_CUDA_TRY(cudaMalloc(&bufs[slot].first, bytes));
            bufs[slot].second = bytes;
        }
        *out = bufs[slot].first;
        return P3D_OK;
    }
    void release() {
        for (auto& b : bufs) if (b.first) cudaFree(b.first);
        bufs.clear();
        for (auto& e : events) cudaEventDestroy(e);
        events.clear();
        if (stream) { cudaStreamDestroy(stream); stream = nullptr; }
        if (copy_in) { cudaStreamDestroy(copy_in); copy_in = nullptr; }
        if (copy_out) { cudaStreamDestroy(copy_out); copy_out = nullptr; }
    }
};
static Arena g_arena;

}  // namespace p3d

using namespace p3d;

extern "C" {

const char* p3d_version(void) { return "p3d-render-b200 0.1 (sm_90a)"; }
const char* p3d_last_error(void) { return g_err; }
uint64_t p3d_launch_count(void) { return g_launches.load(); }

int p3d_planes_to_channels_last(const float* planes_nchw, void* planes_cl, int64_t n_planes, int32_t channels,
                                int32_t h, int32_t w, int32_t out_bf16, void* stream) {
    P3D_REQUIRE(n_planes >= 0 && n_planes < 65536 && channels > 0 && h > 0 && w > 0, "bad plane sizes");
    if (n_planes == 0) return P3D_OK;                       // empty batch: nothing to do, pointers may be NULL
    P3D_REQUIRE(planes_nchw && planes_cl, "null plane pointer");
    const long long HW = (long long)h * w;
    dim3 grid((unsigned)((HW + 31) / 32), (unsigned)((channels + 31) / 32), (unsigned)n_planes), block(32, 8);
    ProfileScope prof(PROF_LAYOUT, (cudaStream_t)stream);
    if (channels == 32 && HW % 4 == 0 && ((reinterpret_cast<uintptr_t>(planes_nchw) | reinterpret_cast<uintptr_t>(planes_cl)) & 15) == 0) {
        dim3 g32((unsigned)((HW + 127) / 128), (unsigned)n_planes);
        if (out_bf16) k_planes_to_cl32<true><<<g32, 256, 0, (cudaStream_t)stream>>>(planes_nchw, planes_cl, HW);
        else k_planes_to_cl32<false><<<g32, 256, 0, (cudaStream_t)stream>>>(planes_nchw, planes_cl, HW);
        P3D_LAUNCH_CHECK();
        return P3D_OK;
    }
    if (out_bf16) k_planes_to_cl<true><<<grid, block, 0, (cudaStream_t)stream>>>(planes_nchw, planes_cl, channels, HW);
    else k_planes_to_cl<false><<<grid, block, 0, (cudaStream_t)stream>>>(planes_nchw, planes_cl, channels, HW);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

int p3d_raygen_pinhole(const float* cam2world, const float* intrinsics, int32_t n_views, int32_t resolution,
                       float* ray_origins, float* ray_dirs, void* stream) {
    P3D_REQUIRE(cam2world && intrinsics && ray_origins && ray_dirs, "null pointer");
    P3D_REQUIRE(n_views >= 0 && resolution > 0, "bad sizes");
    const long long total = (long long)n_views * resolution * resolution;
    if (total == 0) return P3D_OK;
    ProfileScope prof(PROF_RAYGEN, (cudaStream_t)stream);
    k_raygen_pinhole<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(cam2world, intrinsics, n_views,
                                                                                        resolution, ray_origins, ray_dirs);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

int p3d_raygen_ortho(const float* rot, const float* dist, int32_t n_views, int32_t resolution, double box_warp,
                     float* ray_origins, float* ray_dirs, void* stream) {
    P3D_REQUIRE(rot && dist && ray_origins && ray_dirs, "null pointer");
    P3D_REQUIRE(n_views >= 0 && resolution > 0, "bad sizes");
    const long long total = (long long)n_views * resolution * resolution;
    if (total == 0) return P3D_OK;
    k_raygen_ortho<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rot, dist, n_views, resolution,
                                                                                      (float)box_warp, ray_origins, ray_dirs);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

void p3d_profile_enable(int on) {
    std::lock_guard<std::mutex> l(g_prof_mu);
    g_prof_on = on != 0;
}

int p3d_profile_read(double* ms_by_slot, uint64_t* launches_by_slot, int n_slots, int reset) {
    std::lock_guard<std::mutex> l(g_prof_mu);
    for (auto& r : g_prof_pending) {
        P3D_CUDA_TRY(cudaEventSynchronize(r.b));
        float ms = 0.f;
        P3D_CUDA_TRY(cudaEventElapsedTime(&ms, r.a, r.b));
        g_prof_ms[r.slot] += ms; g_prof_n[r.slot] += 1;
        g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b);
    }
    g_prof_pending.clear();
    for (int i = 0; i < n_slots && i < PROF_SLOTS; ++i) {
        if (ms_by_slot) ms_by_slot[i] = g_prof_ms[i];
        if (launches_by_slot) launches_by_slot[i] = g_prof_n[i];
    }
    if (reset) for (int i = 0; i < PROF_SLOTS; ++i) { g_prof_ms[i] = 0; g_prof_n[i] = 0; }
    return P3D_OK;
}

size_t p3d_render_workspace_bytes(const p3d_render_params* p) {
    if (!p) return 0;
    return workspace_layout(p, nullptr, nullptr);
}

int p3d_render_fused_supported(const p3d_render_params* p) {
    Geom g;
    if (!p || make_geom(p, &g) || g.D > 1) return 0;      // multiplane planes: fp32 SIMT kernels only
    return fused_ws3_supported(g) ? 1 : 0;
}

int p3d_decode_tc_supported(const p3d_render_params* p, int64_t n_points_total) {
    Geom g;
    if (!p || make_geom(p, &g) || g.D > 1) return 0;
    return decode_tc_supported(g, n_points_total) ? 1 : 0;
}

// an explicit tensor-core request for multiplane planes fails: only the fp32 SIMT kernels gather trilinearly
static int refuse_tc_multiplane(const Geom& g, const p3d_render_params* p) {
    if (g.D > 1 && (p->mlp_mode == P3D_MLP_TC_3XBF16 || p->mlp_mode == P3D_MLP_TC_BF16)) {
        set_error("plane_depth %d (multiplane tri-planes) has no tensor-core kernel; use mlp_mode P3D_MLP_FP32_SIMT", g.D);
        return P3D_EUNSUPPORTED;
    }
    return P3D_OK;
}

int p3d_render_forward(const p3d_render_params* p, const void* planes, const float* w1, const float* b1, const float* w2,
                       const float* b2, const float* ray_origins, const float* ray_dirs, const float* u_coarse,
                       const float* u_fine, void* workspace, size_t workspace_bytes, float* out_rgb, float* out_depth,
                       float* out_wsum, float* out_xyz, void* stream) {
    Geom g;
    int rc = make_geom(p, &g);
    if (rc) return rc;
    P3D_REQUIRE(p->ray_mode == P3D_RAYS_NUMERIC || p->ray_mode == P3D_RAYS_AUTOBOX, "bad ray_mode %d", p->ray_mode);
    P3D_REQUIRE(!(p->ray_mode == P3D_RAYS_AUTOBOX && p->disparity), "disparity sampling needs numeric ray limits");
    if ((rc = refuse_tc_multiplane(g, p))) return rc;
    if ((long long)g.N * g.M == 0) return P3D_OK;           // empty batch: empty outputs, pointers may be NULL
    P3D_REQUIRE(planes && w1 && b1 && w2 && b2 && ray_origins && ray_dirs, "null input pointer");
    P3D_REQUIRE(out_rgb && out_depth && out_wsum && out_xyz, "null output pointer");
    Workspace ws;
    const size_t need = workspace_layout(p, workspace, &ws);
    if (!workspace || workspace_bytes < need) {
        set_error("workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
        return P3D_EWORKSPACE;
    }
    if (p->mlp_mode == P3D_MLP_FP32_SIMT)
        return render_forward_v1(g, p, planes, w1, b1, w2, b2, ray_origins, ray_dirs, u_coarse, u_fine, ws, out_rgb,
                                 out_depth, out_wsum, out_xyz, (cudaStream_t)stream);
    if (p->mlp_mode == P3D_MLP_TC_3XBF16 || p->mlp_mode == P3D_MLP_TC_BF16) {
        return render_forward_fused_ws3(g, p, planes, w1, b1, w2, b2, ray_origins, ray_dirs, u_coarse, u_fine, ws, out_rgb,
                                        out_depth, out_wsum, out_xyz, (cudaStream_t)stream);     // P3D_EUNSUPPORTED without a kernel
    }
    set_error("mlp_mode %d has no kernel in this build", p->mlp_mode);
    return P3D_EUNSUPPORTED;
}

size_t p3d_render_backward_scratch_bytes(const p3d_render_params* p) {
    if (!p) return 0;
    return (size_t)2 * p->n_views * p->n_rays * ((size_t)p->n_coarse + p->n_fine) * sizeof(float) + 1024;
}

int p3d_render_backward(const p3d_render_params* p, const void* planes, const float* w1, const float* b1, const float* w2,
                        const float* b2, const float* ray_origins, const float* ray_dirs, const void* fwd_workspace,
                        size_t fwd_workspace_bytes, const float* out_depth, const float* g_rgb, const float* g_depth,
                        const float* g_wsum, const float* g_xyz, void* scratch, size_t scratch_bytes, float* d_planes,
                        float* d_w1, float* d_b1, float* d_w2, float* d_b2, void* stream) {
    Geom g;
    int rc = make_geom(p, &g);
    if (rc) return rc;
    P3D_REQUIRE(planes && w1 && b1 && w2 && b2 && ray_origins && ray_dirs && fwd_workspace && out_depth, "null input pointer");
    P3D_REQUIRE(g_rgb && g_depth && g_wsum && g_xyz, "null gradient pointer (pass zeros for unused outputs)");
    P3D_REQUIRE(scratch && d_planes && d_w1 && d_b1 && d_w2 && d_b2, "null output pointer");
    if ((long long)g.N * g.M == 0) return P3D_OK;
    Workspace ws;
    const size_t need = workspace_layout(p, const_cast<void*>(fwd_workspace), &ws);
    if (fwd_workspace_bytes < need) { set_error("forward workspace too small: need %zu bytes", need); return P3D_EWORKSPACE; }
    return render_backward_v1(g, p, planes, w1, b1, w2, b2, ray_origins, ray_dirs, ws, out_depth, g_rgb, g_depth, g_wsum, g_xyz,
                              scratch, scratch_bytes, d_planes, d_w1, d_b1, d_w2, d_b2, (cudaStream_t)stream);
}

// an empty batch of the deterministic backward still writes every output: zeros
static int det_zero(const DetPlan& d, float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2, cudaStream_t st) {
    P3D_CUDA_TRY(cudaMemsetAsync(d_planes, 0, (size_t)d.texels * kC * sizeof(float), st));
    P3D_CUDA_TRY(cudaMemsetAsync(d_w1, 0, (size_t)kHidden * kC * sizeof(float), st));
    P3D_CUDA_TRY(cudaMemsetAsync(d_b1, 0, (size_t)kHidden * sizeof(float), st));
    P3D_CUDA_TRY(cudaMemsetAsync(d_w2, 0, (size_t)kOut * kHidden * sizeof(float), st));
    P3D_CUDA_TRY(cudaMemsetAsync(d_b2, 0, (size_t)kOut * sizeof(float), st));
    return P3D_OK;
}

size_t p3d_render_backward_det_scratch_bytes(const p3d_render_params* p) {
    Geom g;
    DetPlan d;
    if (make_geom(p, &g) || det_plan(g, -1, &d)) return 0;
    return det_layout(d, p3d_render_backward_scratch_bytes(p), nullptr, nullptr);
}

int p3d_render_backward_det(const p3d_render_params* p, const void* planes, const float* w1, const float* b1, const float* w2,
                            const float* b2, const float* ray_origins, const float* ray_dirs, const void* fwd_workspace,
                            size_t fwd_workspace_bytes, const float* out_depth, const float* g_rgb, const float* g_depth,
                            const float* g_wsum, const float* g_xyz, void* scratch, size_t scratch_bytes, float* d_planes,
                            float* d_w1, float* d_b1, float* d_w2, float* d_b2, void* stream) {
    Geom g;
    DetPlan d;
    int rc = make_geom(p, &g);
    if (rc || (rc = det_plan(g, -1, &d))) return rc;
    P3D_REQUIRE(planes && w1 && b1 && w2 && b2 && ray_origins && ray_dirs && fwd_workspace && out_depth, "null input pointer");
    P3D_REQUIRE(g_rgb && g_depth && g_wsum && g_xyz, "null gradient pointer (pass zeros for unused outputs)");
    P3D_REQUIRE(scratch && d_planes && d_w1 && d_b1 && d_w2 && d_b2, "null output pointer");
    if (d.samples == 0) return det_zero(d, d_planes, d_w1, d_b1, d_w2, d_b2, (cudaStream_t)stream);
    Workspace ws;
    const size_t need = workspace_layout(p, const_cast<void*>(fwd_workspace), &ws);
    if (fwd_workspace_bytes < need) { set_error("forward workspace too small: need %zu bytes", need); return P3D_EWORKSPACE; }
    return render_backward_v1(g, p, planes, w1, b1, w2, b2, ray_origins, ray_dirs, ws, out_depth, g_rgb, g_depth, g_wsum, g_xyz,
                              scratch, scratch_bytes, d_planes, d_w1, d_b1, d_w2, d_b2, (cudaStream_t)stream, &d);
}

int p3d_render_depth_bounds(const void* workspace, float* bounds2, void* stream) {
    P3D_REQUIRE(workspace && bounds2, "null pointer");
    return launch_bounds_to_float(reinterpret_cast<const unsigned int*>(workspace), bounds2, (cudaStream_t)stream);   // bounds live at offset 0
}

int p3d_depth_finalize(float* depth, int64_t n_rays, const float* bounds2, void* stream) {
    P3D_REQUIRE(depth && bounds2 && n_rays >= 0, "bad arguments");
    if (n_rays == 0) return P3D_OK;
    return launch_depth_finalize_f(depth, n_rays, bounds2, (cudaStream_t)stream);
}

int p3d_decode_points(const p3d_render_params* p, const void* planes, const float* w1, const float* b1, const float* w2,
                      const float* b2, const float* coords, int64_t n_points_per_view, float* out_rgb, float* out_sigma,
                      void* stream) {
    Geom g;
    int rc = make_geom(p, &g);
    if (rc) return rc;
    P3D_REQUIRE(n_points_per_view >= 0, "negative point count");
    if ((rc = refuse_tc_multiplane(g, p))) return rc;
    if ((long long)g.N * n_points_per_view == 0) return P3D_OK;
    P3D_REQUIRE(planes && w1 && b1 && w2 && b2 && coords && out_rgb && out_sigma, "null pointer");
    if (p->mlp_mode == P3D_MLP_TC_3XBF16 || p->mlp_mode == P3D_MLP_TC_BF16) {
        if (!decode_tc_supported(g, (long long)g.N * n_points_per_view)) {
            set_error("tensor-core point decode needs planes of at least 2x2 texels with non-negative strides below 2^31 elements per view");
            return P3D_EUNSUPPORTED;
        }
        return decode_points_tc(g, p, planes, w1, b1, w2, b2, coords, n_points_per_view, out_rgb, out_sigma, (cudaStream_t)stream);
    }
    return decode_points_v1(g, p, planes, w1, b1, w2, b2, coords, n_points_per_view, out_rgb, out_sigma, (cudaStream_t)stream);
}

int p3d_decode_points_backward(const p3d_render_params* p, const void* planes, const float* w1, const float* b1, const float* w2,
                               const float* b2, const float* coords, int64_t n_points_per_view, const float* g_rgb,
                               const float* g_sigma, float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2,
                               void* stream) {
    Geom g;
    int rc = make_geom(p, &g);
    if (rc) return rc;
    P3D_REQUIRE(n_points_per_view >= 0, "negative point count");
    if ((long long)g.N * n_points_per_view == 0) return P3D_OK;
    P3D_REQUIRE(planes && w1 && b1 && w2 && b2 && coords && g_rgb && g_sigma, "null input pointer (pass zeros for an unused gradient)");
    P3D_REQUIRE(d_planes && d_w1 && d_b1 && d_w2 && d_b2, "null output pointer");
    return decode_points_backward_v1(g, p, planes, w1, b1, w2, b2, coords, n_points_per_view, g_rgb, g_sigma, d_planes, d_w1,
                                     d_b1, d_w2, d_b2, (cudaStream_t)stream);
}

size_t p3d_decode_points_backward_det_scratch_bytes(const p3d_render_params* p, int64_t n_points_per_view) {
    Geom g;
    DetPlan d;
    if (make_geom(p, &g)) return 0;
    if (n_points_per_view < 0) { set_error("negative point count"); return 0; }
    if (det_plan(g, n_points_per_view, &d)) return 0;
    return det_layout(d, 0, nullptr, nullptr);
}

int p3d_decode_points_backward_det(const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                                   const float* w2, const float* b2, const float* coords, int64_t n_points_per_view,
                                   const float* g_rgb, const float* g_sigma, void* scratch, size_t scratch_bytes, float* d_planes,
                                   float* d_w1, float* d_b1, float* d_w2, float* d_b2, void* stream) {
    Geom g;
    DetPlan d;
    int rc = make_geom(p, &g);
    if (rc) return rc;
    P3D_REQUIRE(n_points_per_view >= 0, "negative point count");
    if ((rc = det_plan(g, n_points_per_view, &d))) return rc;
    P3D_REQUIRE(planes && w1 && b1 && w2 && b2 && coords && g_rgb && g_sigma, "null input pointer (pass zeros for an unused gradient)");
    P3D_REQUIRE(scratch && d_planes && d_w1 && d_b1 && d_w2 && d_b2, "null output pointer");
    if (d.samples == 0) return det_zero(d, d_planes, d_w1, d_b1, d_w2, d_b2, (cudaStream_t)stream);
    return decode_points_backward_v1(g, p, planes, w1, b1, w2, b2, coords, n_points_per_view, g_rgb, g_sigma, d_planes, d_w1,
                                     d_b1, d_w2, d_b2, (cudaStream_t)stream, &d, scratch, scratch_bytes);
}

int p3d_volume_query(const p3d_render_params* p, const void* planes, const float* w1, const float* b1, const float* w2,
                     const float* b2, int32_t resolution, double cube_length, double triplane_crop, double cull_clouds,
                     float* out_sigma, float* out_rgb, float* out_density, float* out_coords, void* stream) {
    Geom g;
    int rc = make_geom(p, &g);
    if (rc) return rc;
    P3D_REQUIRE(resolution >= 2 && resolution <= 1024, "resolution must be in [2, 1024], got %d", resolution);
    P3D_REQUIRE(cube_length > 0, "cube_length must be > 0");
    if ((rc = refuse_tc_multiplane(g, p))) return rc;
    if (g.N == 0) return P3D_OK;
    P3D_REQUIRE(planes && w1 && b1 && w2 && b2 && out_sigma, "null pointer");
    VolumeSpec vol;
    vol.res = resolution;
    vol.size = (float)(cube_length / (double)(resolution - 1));          // python float -> fp32 scalar operand
    vol.origin = (float)(0.0 - cube_length / 2.0);
    vol.crop = triplane_crop >= 0 ? (float)(p->box_warp / 2.0 - triplane_crop) : -1.f;    // renderer.py:139-148
    vol.cull = cull_clouds >= 0 ? (float)cull_clouds : -1.f;
    vol.crop_on = triplane_crop >= 0; vol.cull_on = cull_clouds >= 0;
    if (p->mlp_mode == P3D_MLP_TC_3XBF16 || p->mlp_mode == P3D_MLP_TC_BF16) {
        if (!decode_tc_supported(g, (long long)g.N * resolution * resolution * resolution)) {
            set_error("tensor-core volume query needs planes of at least 2x2 texels with non-negative strides below 2^31 elements per view");
            return P3D_EUNSUPPORTED;
        }
        return volume_query_tc(g, p, planes, w1, b1, w2, b2, vol, out_sigma, out_rgb, out_density, out_coords, (cudaStream_t)stream);
    }
    return volume_query_v1(g, p, planes, w1, b1, w2, b2, vol, out_sigma, out_rgb, out_density, out_coords, (cudaStream_t)stream);
}

int p3d_render_forward_host(const p3d_render_params* p_in, const float* planes_nchw, const float* w1, const float* b1,
                            const float* w2, const float* b2, const float* cam2world, const float* intrinsics,
                            int32_t resolution, const float* u_coarse, const float* u_fine, float* out_rgb,
                            float* out_depth, float* out_wsum, float* out_xyz) {
    // Host-resident inputs -> host-resident outputs.  The step is PCIe-bound (a view's tri-planes are 100 MB of
    // fp32 against ~1 ms of rendering), so views are pipelined over three streams: H2D of view v+1 overlaps layout +
    // rendering of view v, whose rgb / weights / xyz start their D2H while view v+1 renders.  Each view is one
    // p3d_render_forward call with defer_depth_clamp; the batch-wide depth clamp (ray_marcher.py:50) is applied once
    // at the end from the merged per-view bounds, so results equal the one-shot call on the whole batch.  That holds for
    // numeric ray limits only: with 'auto' limits the reference fills the rays that miss the box with the min / max start
    // of the WHOLE batch (renderer.py:167-170), a second batch-wide reduction this per-view pipeline does not carry -
    // P3D_RAYS_AUTOBOX is rejected here (use p3d_render_forward on device buffers for it).
    P3D_REQUIRE(p_in && planes_nchw && w1 && b1 && w2 && b2 && cam2world && intrinsics, "null input pointer");
    P3D_REQUIRE(out_rgb && out_depth && out_wsum && out_xyz, "null output pointer");
    p3d_render_params p = *p_in;
    if (p.plane_depth > 1) {
        set_error("p3d_render_forward_host takes one-slab NCHW tri-planes; render multiplane tri-planes (plane_depth %d) with "
                  "p3d_render_forward on device buffers", p.plane_depth);
        return P3D_EUNSUPPORTED;
    }
    P3D_REQUIRE(p.n_rays == resolution * resolution, "n_rays must equal resolution^2");
    if (p.ray_mode == P3D_RAYS_AUTOBOX) {
        set_error("p3d_render_forward_host renders view by view and cannot reproduce the batch-wide fill of 'auto' ray limits "
                  "(renderer.py:167-170); pass numeric ray_start / ray_end or call p3d_render_forward on the whole batch");
        return P3D_EUNSUPPORTED;
    }
    P3D_REQUIRE(p.n_views >= 0, "bad sizes");
    if ((long long)p.n_views * p.n_rays == 0) return P3D_OK;
    std::lock_guard<std::mutex> lock(g_arena.mu);
    if (!g_arena.stream) P3D_CUDA_TRY(cudaStreamCreateWithFlags(&g_arena.stream, cudaStreamNonBlocking));
    if (!g_arena.copy_in) P3D_CUDA_TRY(cudaStreamCreateWithFlags(&g_arena.copy_in, cudaStreamNonBlocking));
    if (!g_arena.copy_out) P3D_CUDA_TRY(cudaStreamCreateWithFlags(&g_arena.copy_out, cudaStreamNonBlocking));
    cudaStream_t st = g_arena.stream, sin = g_arena.copy_in, sout = g_arena.copy_out;
    const size_t N = p.n_views, M = p.n_rays, C = p.channels, HW = (size_t)p.plane_h * p.plane_w;
    const size_t view_elems = 3 * C * HW;
    const size_t esz = p.planes_bf16 ? 2 : 4;
    p.stride_col = C; p.stride_row = (int64_t)p.plane_w * C; p.stride_plane = (int64_t)HW * C; p.stride_view = 3 * p.stride_plane;
    p3d_render_params pv = p;                      // one view per launch
    pv.n_views = 1;
    pv.defer_depth_clamp = 1;
    void *d_nchw, *d_cl, *d_w, *d_cam, *d_rays, *d_u, *d_out, *d_ws, *d_bounds;
    int rc;
    if ((rc = g_arena.get(0, N * view_elems * 4, &d_nchw))) return rc;
    if ((rc = g_arena.get(1, N * view_elems * esz, &d_cl))) return rc;
    const size_t nw = (size_t)p.hidden * C + p.hidden + (size_t)p.out_dim * p.hidden + p.out_dim;
    if ((rc = g_arena.get(2, nw * 4, &d_w))) return rc;
    if ((rc = g_arena.get(3, N * 25 * 4, &d_cam))) return rc;
    if ((rc = g_arena.get(4, N * M * 6 * 4, &d_rays))) return rc;
    const size_t nu = (u_coarse ? N * M * p.n_coarse : 0) + (u_fine ? N * M * p.n_fine : 0);
    if ((rc = g_arena.get(5, (nu + 1) * 4, &d_u))) return rc;
    const size_t out_per_ray = (size_t)(p.out_dim - 1) + 1 + 1 + 3;
    if ((rc = g_arena.get(6, N * M * out_per_ray * 4, &d_out))) return rc;
    const size_t ws_bytes = p3d_render_workspace_bytes(&pv);
    if ((rc = g_arena.get(7, ws_bytes, &d_ws))) return rc;
    if ((rc = g_arena.get(8, (N + 1) * 2 * 4, &d_bounds))) return rc;

    cudaEvent_t ev_small, ev_rays;
    if ((rc = g_arena.event(0, &ev_small)) || (rc = g_arena.event(1, &ev_rays))) return rc;
    float* dw1 = (float*)d_w; float* db1 = dw1 + (size_t)p.hidden * C; float* dw2 = db1 + p.hidden; float* db2 = dw2 + (size_t)p.out_dim * p.hidden;
    P3D_CUDA_TRY(cudaMemcpyAsync(dw1, w1, (size_t)p.hidden * C * 4, cudaMemcpyHostToDevice, sin));
    P3D_CUDA_TRY(cudaMemcpyAsync(db1, b1, (size_t)p.hidden * 4, cudaMemcpyHostToDevice, sin));
    P3D_CUDA_TRY(cudaMemcpyAsync(dw2, w2, (size_t)p.out_dim * p.hidden * 4, cudaMemcpyHostToDevice, sin));
    P3D_CUDA_TRY(cudaMemcpyAsync(db2, b2, (size_t)p.out_dim * 4, cudaMemcpyHostToDevice, sin));
    float* dc2w = (float*)d_cam; float* dK = dc2w + N * 16;
    P3D_CUDA_TRY(cudaMemcpyAsync(dc2w, cam2world, N * 16 * 4, cudaMemcpyHostToDevice, sin));
    P3D_CUDA_TRY(cudaMemcpyAsync(dK, intrinsics, N * 9 * 4, cudaMemcpyHostToDevice, sin));
    P3D_CUDA_TRY(cudaEventRecord(ev_small, sin));
    P3D_CUDA_TRY(cudaStreamWaitEvent(st, ev_small, 0));
    float* dro = (float*)d_rays; float* drd = dro + N * M * 3;
    if ((rc = p3d_raygen_pinhole(dc2w, dK, p.n_views, resolution, dro, drd, st))) return rc;
    float* duc_all = u_coarse ? (float*)d_u : nullptr;
    float* duf_all = u_fine ? (float*)d_u + (u_coarse ? N * M * p.n_coarse : 0) : nullptr;
    float* drgb = (float*)d_out; float* ddepth = drgb + N * M * (p.out_dim - 1); float* dwsum = ddepth + N * M; float* dxyz = dwsum + N * M;
    float* dbounds = (float*)d_bounds;
    const size_t rgb_v = M * (size_t)(p.out_dim - 1);
    for (size_t v = 0; v < N; ++v) {
        cudaEvent_t ev_in, ev_done;
        if ((rc = g_arena.event(2 + 2 * v, &ev_in)) || (rc = g_arena.event(3 + 2 * v, &ev_done))) return rc;
        float* nchw_v = (float*)d_nchw + v * view_elems;
        P3D_CUDA_TRY(cudaMemcpyAsync(nchw_v, planes_nchw + v * view_elems, view_elems * 4, cudaMemcpyHostToDevice, sin));
        float *duc = nullptr, *duf = nullptr;
        if (u_coarse) { duc = duc_all + v * M * p.n_coarse; P3D_CUDA_TRY(cudaMemcpyAsync(duc, u_coarse + v * M * p.n_coarse, M * p.n_coarse * 4, cudaMemcpyHostToDevice, sin)); }
        if (u_fine) { duf = duf_all + v * M * p.n_fine; P3D_CUDA_TRY(cudaMemcpyAsync(duf, u_fine + v * M * p.n_fine, M * p.n_fine * 4, cudaMemcpyHostToDevice, sin)); }
        P3D_CUDA_TRY(cudaEventRecord(ev_in, sin));
        P3D_CUDA_TRY(cudaStreamWaitEvent(st, ev_in, 0));
        void* cl_v = (char*)d_cl + v * view_elems * esz;
        if ((rc = p3d_planes_to_channels_last(nchw_v, cl_v, 3, p.channels, p.plane_h, p.plane_w, p.planes_bf16, st))) return rc;
        pv.seed = p.seed + v * 0x9E3779B97F4A7C15ull;          // independent Philox stream per view (used when u_* are NULL)
        if ((rc = p3d_render_forward(&pv, cl_v, dw1, db1, dw2, db2, dro + v * M * 3, drd + v * M * 3, duc, duf, d_ws, ws_bytes,
                                     drgb + v * rgb_v, ddepth + v * M, dwsum + v * M, dxyz + v * M * 3, st))) return rc;
        if ((rc = p3d_render_depth_bounds(d_ws, dbounds + 2 * (v + 1), st))) return rc;
        P3D_CUDA_TRY(cudaEventRecord(ev_done, st));
        P3D_CUDA_TRY(cudaStreamWaitEvent(sout, ev_done, 0));
        P3D_CUDA_TRY(cudaMemcpyAsync(out_rgb + v * rgb_v, drgb + v * rgb_v, rgb_v * 4, cudaMemcpyDeviceToHost, sout));
        P3D_CUDA_TRY(cudaMemcpyAsync(out_wsum + v * M, dwsum + v * M, M * 4, cudaMemcpyDeviceToHost, sout));
        P3D_CUDA_TRY(cudaMemcpyAsync(out_xyz + v * M * 3, dxyz + v * M * 3, M * 3 * 4, cudaMemcpyDeviceToHost, sout));
    }
    k_merge_bounds<<<1, 32, 0, st>>>(dbounds, (int)N);
    P3D_LAUNCH_CHECK();
    if ((rc = p3d_depth_finalize(ddepth, (int64_t)(N * M), dbounds, st))) return rc;
    P3D_CUDA_TRY(cudaMemcpyAsync(out_depth, ddepth, N * M * 4, cudaMemcpyDeviceToHost, st));
    P3D_CUDA_TRY(cudaStreamSynchronize(sout));
    P3D_CUDA_TRY(cudaStreamSynchronize(st));
    return P3D_OK;
}

int p3d_ipc_alloc(size_t bytes, void** dptr, unsigned char* handle64) {
    P3D_REQUIRE(dptr && handle64 && bytes > 0, "bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    P3D_CUDA_TRY(cudaMalloc(dptr, bytes));
    P3D_CUDA_TRY(cudaMemset(*dptr, 0, bytes));
    cudaIpcMemHandle_t h;
    P3D_CUDA_TRY(cudaIpcGetMemHandle(&h, *dptr));
    memcpy(handle64, &h, 64);
    return P3D_OK;
}

int p3d_ipc_open(const unsigned char* handle64, void** dptr) {
    P3D_REQUIRE(dptr && handle64, "bad arguments");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    P3D_CUDA_TRY(cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
    return P3D_OK;
}

int p3d_ipc_close(void* dptr) {
    if (dptr) P3D_CUDA_TRY(cudaIpcCloseMemHandle(dptr));
    return P3D_OK;
}

int p3d_ipc_free(void* dptr) {
    if (dptr) P3D_CUDA_TRY(cudaFree(dptr));
    return P3D_OK;
}

int p3d_copy_async(void* dst, const void* src, size_t bytes, void* stream) {
    P3D_REQUIRE(dst && src, "null pointer");
    P3D_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return P3D_OK;
}

void p3d_host_arena_release(void) {
    std::lock_guard<std::mutex> lock(g_arena.mu);
    g_arena.release();
}

}  // extern "C"
