// Front-view paste (SURVEY 8f-3): the reference's paste_front (training/triplane.py:608-691) as one kernel at output
// resolution.  Per output pixel the reference's ~35 eager ops read and write five full-resolution mask images, an
// up-sampled xyz image (three times) and two grid_sample results; here each output pixel is computed once from the
// low-resolution render outputs (L1/L2 resident: 3 x 128 x 128 floats per view) and the only HBM traffic is the
// compulsory one: image and front image in, image / paste / masks out.
//
// HBM-bound elementwise work: no tensor cores.  One CTA = a 32 x 8 output tile; the up-sampled xyz of the tile plus a
// one-pixel halo (the Sobel footprint, replicate-padded like kornia) is staged once in shared memory.
#include "p3d_common.cuh"
#include "../../include/p3d_paste.h"

namespace p3d {
namespace {

constexpr int TW = 32, TH = 8, NT = TW * TH;

struct PasteArgs {
    const float *image, *xyz, *wts, *front, *occ, *ro, *rd, *eroded;
    float *o_image, *o_paste, *o_mask, *o_parts;
    int N, R, S, Rf, normalize;
    float inv_bw, half_bw;
    float t_w, t_e, t_o, t_d;
    float scale;       // (float)R / S : torch's area_pixel_compute_scale for size-given interpolate
};

// F.interpolate(mode='bilinear', align_corners=False): source index / weights of one output coordinate
// (aten UpSample.h: area_pixel_compute_source_index + guard_index_and_lambda)
struct Lin { unsigned i0, i1; float l0, l1; };   // unsigned: a 32-bit offset folds into one IMAD.WIDE.U32 per access
__device__ __forceinline__ Lin lin_src(int dst, float scale, int in) {
    float s = scale * ((float)dst + 0.5f) - 0.5f;
    s = s < 0.f ? 0.f : s;
    int i0 = min((int)s, in - 1);
    Lin r;
    r.i0 = (unsigned)i0;
    r.i1 = (unsigned)min(i0 + 1, in - 1);
    r.l1 = fminf(fmaxf(s - (float)i0, 0.f), 1.f);
    r.l0 = 1.f - r.l1;
    return r;
}
__device__ __forceinline__ float bilerp(const float* __restrict__ img, int R, Lin y, Lin x) {
    float a = __ldg(img + y.i0 * R + x.i0), b = __ldg(img + y.i0 * R + x.i1);
    float c = __ldg(img + y.i1 * R + x.i0), d = __ldg(img + y.i1 * R + x.i1);
    return y.l0 * (x.l0 * a + x.l1 * b) + y.l1 * (x.l0 * c + x.l1 * d);
}

// sample_orthofront's grid coordinate of one world coordinate (triplane.py:557,560), then grid_sample's
// un-normalisation (align_corners=False) and border clipping (aten GridSampler.h)
struct Tap { unsigned i0; float f; float gmul; };     // floor index, fraction, d(index)/d(world coordinate) (0 where clipped)
__device__ __forceinline__ Tap ortho_tap(float v, float half_bw, float inv_bw, int size) {
    float vij = 1.f - (v + half_bw) * inv_bw;            // torch's CUDA div-by-scalar multiplies by the reciprocal
    float g = vij * 2.f - 1.f;
    float ix = ((g + 1.f) * (float)size - 1.f) * 0.5f;
    float mul = -(float)size * inv_bw;
    float hi = (float)(size - 1);
    if (ix <= 0.f) { ix = 0.f; mul = 0.f; }
    else if (ix >= hi) { ix = hi; mul = 0.f; }
    Tap t;
    float fl = floorf(ix);
    t.i0 = (unsigned)(int)fl;
    t.f = ix - fl;
    t.gmul = mul;
    return t;
}

// ---------------------------------------------------------------- forward
__global__ void __launch_bounds__(NT) k_paste_front(PasteArgs a) {
    __shared__ float s_up[3][TH + 2][TW + 2 + 1];
    __shared__ Lin s_row[TH + 2], s_col[TW + 2];          // source rows / columns + weights of the tile's halo, computed once
    const int n = blockIdx.z, tx0 = blockIdx.x * TW, ty0 = blockIdx.y * TH;
    const unsigned R = a.R, S = a.S;
    const float* xyz = a.xyz + (size_t)n * 3 * R * R;
    if (threadIdx.x < TH + 2) s_row[threadIdx.x] = lin_src(min(max(ty0 + (int)threadIdx.x - 1, 0), a.S - 1), a.scale, a.R);   // replicate pad
    else if (threadIdx.x >= 64 && threadIdx.x < 64 + TW + 2) s_col[threadIdx.x - 64] = lin_src(min(max(tx0 + (int)threadIdx.x - 65, 0), a.S - 1), a.scale, a.R);
    __syncthreads();
    for (int idx = threadIdx.x; idx < (TH + 2) * (TW + 2); idx += NT) {
        int hy = idx / (TW + 2), hx = idx - hy * (TW + 2);
        const Lin ly = s_row[hy], lx = s_col[hx];
        const unsigned h00 = ly.i0 * R + lx.i0, h01 = ly.i0 * R + lx.i1, h10 = ly.i1 * R + lx.i0, h11 = ly.i1 * R + lx.i1;
#pragma unroll
        for (unsigned c = 0; c < 3; ++c) {
            const float* pc = xyz + c * R * R;
            float v0 = lx.l0 * __ldg(pc + h00) + lx.l1 * __ldg(pc + h01);
            float v1 = lx.l0 * __ldg(pc + h10) + lx.l1 * __ldg(pc + h11);
            s_up[c][hy][hx] = ly.l0 * v0 + ly.l1 * v1;
        }
    }
    __syncthreads();
    const int lx_ = threadIdx.x & (TW - 1), ly_ = threadIdx.x / TW;
    const unsigned ox = tx0 + lx_, oy = ty0 + ly_;
    if (ox >= S || oy >= S) return;
    // 32-bit offsets inside one view (the host checks 5 * N * S * S < 2^31): one IMAD.WIDE per access instead of 64-bit chains
    const unsigned pix = oy * S + ox, plane = S * S;
    const Lin by = s_row[ly_ + 1], bx = s_col[lx_ + 1];
    const unsigned o00 = by.i0 * R + bx.i0, o01 = by.i0 * R + bx.i1, o10 = by.i1 * R + bx.i0, o11 = by.i1 * R + bx.i1;

    // mask 1: visible weights (triplane.py:625-629)
    const float* wv = a.wts + (size_t)n * R * R;
    float qw = by.l0 * (bx.l0 * __ldg(wv + o00) + bx.l1 * __ldg(wv + o01)) + by.l1 * (bx.l0 * __ldg(wv + o10) + bx.l1 * __ldg(wv + o11));
    float wmask = qw > a.t_w ? 1.f : 0.f;

    // mask 2: deep crevasses - normalised Sobel magnitude of the up-sampled xyz, L2 norm over channels (:632-637)
    float q2 = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float(*p)[TW + 3] = s_up[c];
        int y = ly_ + 1, x = lx_ + 1;
        float gx = ((p[y - 1][x + 1] - p[y - 1][x - 1]) + 2.f * (p[y][x + 1] - p[y][x - 1]) + (p[y + 1][x + 1] - p[y + 1][x - 1])) * 0.125f;
        float gy = ((p[y + 1][x - 1] - p[y - 1][x - 1]) + 2.f * (p[y + 1][x] - p[y - 1][x]) + (p[y + 1][x + 1] - p[y - 1][x + 1])) * 0.125f;
        q2 += gx * gx + gy * gy + 1e-6f;                       // = magnitude_c^2
    }
    float smask = sqrtf(q2) < a.t_e ? 1.f : 0.f;

    // mask 3: occlusion seen from the front - threshold at render resolution, THEN bilinear up-sampling (:640-641)
    float fmask;
    {
        const float* o = a.occ + (size_t)n * R * R;
        float v00 = __ldg(o + o00) < a.t_o ? 1.f : 0.f, v01 = __ldg(o + o01) < a.t_o ? 1.f : 0.f;
        float v10 = __ldg(o + o10) < a.t_o ? 1.f : 0.f, v11 = __ldg(o + o11) < a.t_o ? 1.f : 0.f;
        fmask = by.l0 * (bx.l0 * v00 + bx.l1 * v01) + by.l1 * (bx.l0 * v10 + bx.l1 * v11);
    }

    // mask 4: distance of the rendered point from its own ray, nearest up-sampling (:644-646, get_xyz_discrepancy
    // :601-606).  The subtraction cancels ~6 digits against a 5e-6 threshold: every operation is rounded separately
    // (no fma contraction), in the order the eager ops apply them.
    float dmask;
    {
        const unsigned sy = min((unsigned)(int)floorf((float)oy * a.scale), R - 1), sx = min((unsigned)(int)floorf((float)ox * a.scale), R - 1);
        const unsigned o = sy * R + sx, st = R * R;
        const float* ro = a.ro + (size_t)n * 3 * R * R, *rd = a.rd + (size_t)n * 3 * R * R;
        float d0 = __fsub_rn(-__ldg(xyz + o), __ldg(ro + o));
        float d1 = __fsub_rn(__ldg(xyz + o + st), __ldg(ro + o + st));
        float d2 = __fsub_rn(-__ldg(xyz + o + 2 * st), __ldg(ro + o + 2 * st));
        float n0 = __ldg(rd + o), n1 = __ldg(rd + o + st), n2 = __ldg(rd + o + 2 * st);
        float dot = __fadd_rn(__fadd_rn(__fmul_rn(d0, n0), __fmul_rn(d1, n1)), __fmul_rn(d2, n2));
        float r0 = __fsub_rn(d0, __fmul_rn(dot, n0)), r1 = __fsub_rn(d1, __fmul_rn(dot, n1)), r2 = __fsub_rn(d2, __fmul_rn(dot, n2));
        const float q2 = __fadd_rn(__fadd_rn(__fmul_rn(r0, r0), __fmul_rn(r1, r1)), __fmul_rn(r2, r2));
        const float q = q2 > 0.f ? sqrtf(q2) : 0.f;              // a point exactly on its ray: keep zero off sqrtf's slow path
        dmask = q < a.t_d ? 1.f : 0.f;
    }

    // the front image at this pixel's world (y, x): sample_orthofront (:555-564) - rows follow y, columns follow x
    const float vx = s_up[0][ly_ + 1][lx_ + 1], vy = s_up[1][ly_ + 1][lx_ + 1];

    // mask 5: eroded front weights looked up the same way (:648-662); 1 when front_weight_erosion < 1
    float fwmask = 1.f;
    if (a.Rf > 0) {
        Tap tr = ortho_tap(vy, a.half_bw, a.inv_bw, a.Rf), tc = ortho_tap(vx, a.half_bw, a.inv_bw, a.Rf);
        const float* e = a.eroded + (size_t)n * a.Rf * a.Rf;
        const unsigned r1 = min(tr.i0 + 1, (unsigned)a.Rf - 1), c1 = min(tc.i0 + 1, (unsigned)a.Rf - 1);   // weight is 0 where the neighbour is outside
        float nw = (1.f - tr.f) * (1.f - tc.f), ne = tr.f * (1.f - tc.f), sw = (1.f - tr.f) * tc.f, se = tr.f * tc.f;
        fwmask = __ldg(e + tr.i0 * a.Rf + tc.i0) * nw + __ldg(e + r1 * a.Rf + tc.i0) * ne + __ldg(e + tr.i0 * a.Rf + c1) * sw +
                 __ldg(e + r1 * a.Rf + c1) * se;
    }
    const float mask = wmask * smask * fmask * dmask * fwmask;

    // paste + blend (:670-679); torch.lerp's two-sided formula
    Tap tr = ortho_tap(vy, a.half_bw, a.inv_bw, S), tc = ortho_tap(vx, a.half_bw, a.inv_bw, S);
    const unsigned r1 = min(tr.i0 + 1, S - 1), c1 = min(tc.i0 + 1, S - 1);
    float nw = (1.f - tr.f) * (1.f - tc.f), ne = tr.f * (1.f - tc.f), sw = (1.f - tr.f) * tc.f, se = tr.f * tc.f;
    const size_t view3 = (size_t)n * 3 * plane;
    const float* fv = a.front + view3, *iv = a.image + view3;
    float* opv = a.o_paste + view3, *oiv = a.o_image + view3;
    const unsigned t00 = tr.i0 * S + tc.i0, t10 = r1 * S + tc.i0, t01 = tr.i0 * S + c1, t11 = r1 * S + c1;
#pragma unroll
    for (unsigned c = 0; c < 3; ++c) {
        const float* f = fv + c * plane;
        float f00 = __ldg(f + t00), f10 = __ldg(f + t10), f01 = __ldg(f + t01), f11 = __ldg(f + t11);
        if (a.normalize) { f00 = f00 * 2.f - 1.f; f10 = f10 * 2.f - 1.f; f01 = f01 * 2.f - 1.f; f11 = f11 * 2.f - 1.f; }
        float paste = f00 * nw + f10 * ne + f01 * sw + f11 * se;
        const unsigned o = c * plane + pix;
        float img = __ldg(iv + o);
        float diff = paste - img;
        opv[o] = paste;
        oiv[o] = mask < 0.5f ? img + mask * diff : paste - diff * (1.f - mask);
    }
    a.o_mask[(size_t)n * plane + pix] = mask;
    if (a.o_parts) {
        float* pv = a.o_parts + (size_t)n * plane;
        const unsigned st = (unsigned)a.N * plane;                  // 5 * N * S * S < 2^31 (checked by the host)
        pv[pix] = wmask; pv[st + pix] = smask; pv[2 * st + pix] = fmask; pv[3 * st + pix] = dmask; pv[4 * st + pix] = fwmask;
    }
}

// ---------------------------------------------------------------- backward
struct PasteBwdArgs {
    const float *xyz, *front, *mask, *g_image, *g_paste;
    float *d_image, *d_xyz;
    int N, R, S, normalize;
    float inv_bw, half_bw, scale;
    float* g_v;        // DET: (N,2,S,S) gradients of the up-sampled x and y, gathered into d_xyz by k_paste_dxyz_gather
};

// DET (torch.use_deterministic_algorithms): record each pixel's gradients of the up-sampled (x, y) instead of scattering them
template <bool DET>
__global__ void __launch_bounds__(NT) k_paste_front_bwd(PasteBwdArgs a) {
    const int n = blockIdx.z, ox = blockIdx.x * TW + (threadIdx.x & (TW - 1)), oy = blockIdx.y * TH + threadIdx.x / TW;
    const int R = a.R, S = a.S;
    if (ox >= S || oy >= S) return;
    const size_t pix = (size_t)oy * S + ox, plane = (size_t)S * S;
    const float m = __ldg(a.mask + (size_t)n * plane + pix);
    float gp[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        size_t o = ((size_t)n * 3 + c) * plane + pix;
        float g = __ldg(a.g_image + o);
        a.d_image[o] = g * (1.f - m);                              // lerp: d/d start
        gp[c] = g * m + (a.g_paste ? __ldg(a.g_paste + o) : 0.f);  // d/d end (+ a gradient arriving at the 'paste' output)
    }
    if (!a.d_xyz) return;
    const Lin by = lin_src(oy, a.scale, R), bx = lin_src(ox, a.scale, R);
    const float* xyz = a.xyz + (size_t)n * 3 * R * R;
    const float vx = bilerp(xyz, R, by, bx), vy = bilerp(xyz + R * R, R, by, bx);
    Tap tr = ortho_tap(vy, a.half_bw, a.inv_bw, S), tc = ortho_tap(vx, a.half_bw, a.inv_bw, S);
    int r1 = min(tr.i0 + 1, S - 1), c1 = min(tc.i0 + 1, S - 1);
    float g_r = 0.f, g_c = 0.f;                                    // d loss / d (row index), d (column index)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float* f = a.front + ((size_t)n * 3 + c) * plane;
        float f00 = __ldg(f + (size_t)tr.i0 * S + tc.i0), f10 = __ldg(f + (size_t)r1 * S + tc.i0);
        float f01 = __ldg(f + (size_t)tr.i0 * S + c1), f11 = __ldg(f + (size_t)r1 * S + c1);
        if (a.normalize) { f00 *= 2.f; f10 *= 2.f; f01 *= 2.f; f11 *= 2.f; }              // the -1 drops out of differences
        g_r += gp[c] * ((f10 - f00) * (1.f - tc.f) + (f11 - f01) * tc.f);
        g_c += gp[c] * ((f01 - f00) * (1.f - tr.f) + (f11 - f10) * tr.f);
    }
    const float g_vy = g_r * tr.gmul, g_vx = g_c * tc.gmul;          // rows follow world y, columns world x
    if constexpr (DET) {
        a.g_v[(size_t)n * 2 * plane + pix] = g_vx;
        a.g_v[((size_t)n * 2 + 1) * plane + pix] = g_vy;
        return;
    }
    float* d = a.d_xyz + (size_t)n * 3 * R * R;
    const float w00 = by.l0 * bx.l0, w01 = by.l0 * bx.l1, w10 = by.l1 * bx.l0, w11 = by.l1 * bx.l1;
    if (g_vx != 0.f) {
        atomicAdd(d + by.i0 * R + bx.i0, g_vx * w00); atomicAdd(d + by.i0 * R + bx.i1, g_vx * w01);
        atomicAdd(d + by.i1 * R + bx.i0, g_vx * w10); atomicAdd(d + by.i1 * R + bx.i1, g_vx * w11);
    }
    if (g_vy != 0.f) {
        d += R * R;
        atomicAdd(d + by.i0 * R + bx.i0, g_vy * w00); atomicAdd(d + by.i0 * R + bx.i1, g_vy * w01);
        atomicAdd(d + by.i1 * R + bx.i0, g_vy * w10); atomicAdd(d + by.i1 * R + bx.i1, g_vy * w11);
    }
}

// first output coordinate in [0, size) whose up-sampling source (i1 if HI, else i0) is >= src; both are monotone in it
template <bool HI>
__device__ __forceinline__ int first_dst(int src, float scale, int in, int size) {
    int lo = 0, hi = size;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const Lin l = lin_src(mid, scale, in);
        if ((int)(HI ? l.i1 : l.i0) < src) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// Deterministic d_xyz: texel (row, col) of view n sums, in a fixed order, every contribution the scatter would add to it -
// output pixels (oy, ox) ascending row-major over the static stencil whose bilinear footprint covers the texel, and per pixel
// its taps (i0,i0), (i0,i1), (i1,i0), (i1,i1) that land here: acc = fl(acc + fl(g * fl(ly * lx))), zero gradients skipped
// as the scatter skips them.  The z channel gets no gradient and is written as zero.
__global__ void __launch_bounds__(256) k_paste_dxyz_gather(const float* __restrict__ g_v, float* __restrict__ d_xyz, int R, int S,
                                                           float scale) {
    const int n = blockIdx.y, t = blockIdx.x * 256 + threadIdx.x;
    if (t >= R * R) return;
    const int row = t / R, col = t - row * R;
    const int y0 = first_dst<true>(row, scale, R, S), y1 = first_dst<false>(row + 1, scale, R, S);
    const int x0 = first_dst<true>(col, scale, R, S), x1 = first_dst<false>(col + 1, scale, R, S);
    const size_t plane = (size_t)S * S;
    const float* gx = g_v + (size_t)n * 2 * plane;
    const float* gy = gx + plane;
    float ax = 0.f, ay = 0.f;
    for (int oy = y0; oy < y1; ++oy) {
        const Lin by = lin_src(oy, scale, R);
        for (int ox = x0; ox < x1; ++ox) {
            const Lin bx = lin_src(ox, scale, R);
            const float vx = __ldg(gx + (size_t)oy * S + ox), vy = __ldg(gy + (size_t)oy * S + ox);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const unsigned ry = (k >> 1) ? by.i1 : by.i0, cx = (k & 1) ? bx.i1 : bx.i0;
                if (ry != (unsigned)row || cx != (unsigned)col) continue;
                const float w = __fmul_rn((k >> 1) ? by.l1 : by.l0, (k & 1) ? bx.l1 : bx.l0);
                if (vx != 0.f) ax = __fadd_rn(ax, __fmul_rn(vx, w));
                if (vy != 0.f) ay = __fadd_rn(ay, __fmul_rn(vy, w));
            }
        }
    }
    float* d = d_xyz + (size_t)n * 3 * R * R + t;
    d[0] = ax;
    d[(size_t)R * R] = ay;
    d[(size_t)2 * R * R] = 0.f;
}

// ---------------------------------------------------------------- small kernels
__global__ void k_occlusion_rays(const float* __restrict__ xyz, float* __restrict__ ro, float* __restrict__ rd, int64_t total,
                                 int64_t hw, float shift) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int c = (int)((i / hw) % 3);
    float v = xyz[i];
    ro[i] = c == 1 ? v : (c == 0 ? -v : __fsub_rn(-v, shift));
    rd[i] = c == 2 ? 1.f : 0.f;
}

__global__ void k_erode(const float* __restrict__ src, float* __restrict__ dst, int n, int h, int w, int e, float thresh) {
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y, b = blockIdx.z;
    if (x >= w || y >= h) return;
    const float* s = src + (size_t)b * h * w;
    const int o = e / 2;
    float v = 1.f;
    for (int dy = 0; dy < e; ++dy) {
        int yy = y + dy - o;
        if (yy < 0 || yy >= h) continue;                            // geodesic border: outside never lowers the minimum
        for (int dx = 0; dx < e; ++dx) {
            int xx = x + dx - o;
            if (xx < 0 || xx >= w) continue;
            if (!(__ldg(s + (size_t)yy * w + xx) > thresh)) v = 0.f;
        }
    }
    dst[(size_t)b * h * w + (size_t)y * w + x] = v;
}

int check_params(const p3d_paste_params* p) {
    P3D_REQUIRE(p != nullptr, "p3d_paste: params is NULL");
    P3D_REQUIRE(p->n_views > 0 && p->n_views <= 65535, "p3d_paste: n_views %d out of range", p->n_views);
    P3D_REQUIRE(p->res_render > 0 && p->res_image > 0 && p->res_front >= 0, "p3d_paste: bad resolutions R=%d S=%d Rf=%d",
                p->res_render, p->res_image, p->res_front);
    P3D_REQUIRE(p->res_image <= 16384 && p->res_render <= 16384 && p->res_front <= 16384, "p3d_paste: resolution above 16384");
    P3D_REQUIRE(p->box_warp > 0, "p3d_paste: box_warp must be positive");
    P3D_REQUIRE(5ll * p->n_views * p->res_image * p->res_image < (1ll << 31) && 3ll * p->n_views * p->res_render * p->res_render < (1ll << 31),
                "p3d_paste: batch too large for 32-bit offsets (N=%d S=%d R=%d): split the views", p->n_views, p->res_image, p->res_render);
    return P3D_OK;
}

}  // namespace
}  // namespace p3d

using namespace p3d;

extern "C" int p3d_paste_occlusion_rays(const float* image_xyz, int32_t n_views, int32_t res, double ray_start, double offset,
                                        float* ray_origins, float* ray_dirs, void* stream) {
    P3D_REQUIRE(image_xyz && ray_origins && ray_dirs, "p3d_paste_occlusion_rays: NULL pointer");
    P3D_REQUIRE(n_views > 0 && res > 0, "p3d_paste_occlusion_rays: bad shape N=%d R=%d", n_views, res);
    int64_t hw = (int64_t)res * res, total = hw * 3 * n_views;
    k_occlusion_rays<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(image_xyz, ray_origins, ray_dirs, total, hw,
                                                                                      (float)(ray_start - offset));
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_paste_erode(const float* frontw, int32_t n, int32_t h, int32_t w, int32_t e, double thresh, float* eroded,
                               void* stream) {
    P3D_REQUIRE(frontw && eroded, "p3d_paste_erode: NULL pointer");
    P3D_REQUIRE(n > 0 && n <= 65535 && h > 0 && w > 0 && e >= 1 && e <= 255, "p3d_paste_erode: bad shape n=%d h=%d w=%d e=%d", n, h, w, e);
    dim3 blk(32, 8), grd((w + 31) / 32, (h + 7) / 8, n);
    k_erode<<<grd, blk, 0, (cudaStream_t)stream>>>(frontw, eroded, n, h, w, e, (float)thresh);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_paste_front(const p3d_paste_params* p, const float* image, const float* image_xyz, const float* image_weights,
                               const float* front_rgb, const float* occ_weights, const float* ray_origins, const float* ray_dirs,
                               const float* front_eroded, float* out_image, float* out_paste, float* out_mask, float* out_parts,
                               void* stream) {
    if (int rc = check_params(p)) return rc;
    P3D_REQUIRE(image && image_xyz && image_weights && front_rgb && occ_weights && ray_origins && ray_dirs,
                "p3d_paste_front: NULL input pointer");
    P3D_REQUIRE(out_image && out_paste && out_mask, "p3d_paste_front: NULL output pointer");
    P3D_REQUIRE((p->res_front > 0) == (front_eroded != nullptr), "p3d_paste_front: front_eroded must be given exactly when res_front > 0");
    PasteArgs a;
    a.image = image; a.xyz = image_xyz; a.wts = image_weights; a.front = front_rgb; a.occ = occ_weights;
    a.ro = ray_origins; a.rd = ray_dirs; a.eroded = front_eroded;
    a.o_image = out_image; a.o_paste = out_paste; a.o_mask = out_mask; a.o_parts = out_parts;
    a.N = p->n_views; a.R = p->res_render; a.S = p->res_image; a.Rf = p->res_front; a.normalize = p->normalize_images;
    a.inv_bw = 1.f / (float)p->box_warp; a.half_bw = (float)(p->box_warp / 2);
    a.t_w = (float)p->thresh_weight; a.t_e = (float)p->thresh_edges; a.t_o = (float)p->thresh_occ; a.t_d = (float)p->thresh_dxyz;
    a.scale = (float)p->res_render / (float)p->res_image;
    dim3 grd((a.S + TW - 1) / TW, (a.S + TH - 1) / TH, a.N);
    ProfileScope prof(PROF_OTHER, (cudaStream_t)stream);
    k_paste_front<<<grd, NT, 0, (cudaStream_t)stream>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" int p3d_paste_front_backward(const p3d_paste_params* p, const float* image_xyz, const float* front_rgb, const float* mask,
                                        const float* g_image, const float* g_paste, float* d_image, float* d_xyz, void* stream) {
    if (int rc = check_params(p)) return rc;
    P3D_REQUIRE(image_xyz && front_rgb && mask && g_image && d_image, "p3d_paste_front_backward: NULL pointer");
    PasteBwdArgs a;
    a.xyz = image_xyz; a.front = front_rgb; a.mask = mask; a.g_image = g_image; a.g_paste = g_paste;
    a.d_image = d_image; a.d_xyz = d_xyz;
    a.N = p->n_views; a.R = p->res_render; a.S = p->res_image; a.normalize = p->normalize_images;
    a.inv_bw = 1.f / (float)p->box_warp; a.half_bw = (float)(p->box_warp / 2);
    a.scale = (float)p->res_render / (float)p->res_image;
    dim3 grd((a.S + TW - 1) / TW, (a.S + TH - 1) / TH, a.N);
    k_paste_front_bwd<false><<<grd, NT, 0, (cudaStream_t)stream>>>(a);
    P3D_LAUNCH_CHECK();
    return P3D_OK;
}

extern "C" size_t p3d_paste_front_backward_det_scratch_bytes(const p3d_paste_params* p) {
    if (check_params(p)) return 0;
    return (size_t)2 * p->n_views * p->res_image * p->res_image * sizeof(float);
}

extern "C" int p3d_paste_front_backward_det(const p3d_paste_params* p, const float* image_xyz, const float* front_rgb, const float* mask,
                                            const float* g_image, const float* g_paste, void* scratch, size_t scratch_bytes,
                                            float* d_image, float* d_xyz, void* stream) {
    if (int rc = check_params(p)) return rc;
    P3D_REQUIRE(image_xyz && front_rgb && mask && g_image && d_image, "p3d_paste_front_backward_det: NULL pointer");
    const size_t need = p3d_paste_front_backward_det_scratch_bytes(p);
    if (d_xyz && (!scratch || scratch_bytes < need)) {
        set_error("p3d_paste_front_backward_det: scratch too small: need %zu bytes, got %zu", need, scratch_bytes);
        return P3D_EWORKSPACE;
    }
    PasteBwdArgs a;
    a.xyz = image_xyz; a.front = front_rgb; a.mask = mask; a.g_image = g_image; a.g_paste = g_paste;
    a.d_image = d_image; a.d_xyz = d_xyz; a.g_v = reinterpret_cast<float*>(scratch);
    a.N = p->n_views; a.R = p->res_render; a.S = p->res_image; a.normalize = p->normalize_images;
    a.inv_bw = 1.f / (float)p->box_warp; a.half_bw = (float)(p->box_warp / 2);
    a.scale = (float)p->res_render / (float)p->res_image;
    cudaStream_t st = (cudaStream_t)stream;
    ProfileScope prof(PROF_OTHER, st);
    dim3 grd((a.S + TW - 1) / TW, (a.S + TH - 1) / TH, a.N);
    k_paste_front_bwd<true><<<grd, NT, 0, st>>>(a);
    P3D_LAUNCH_CHECK();
    if (d_xyz) {
        k_paste_dxyz_gather<<<dim3((unsigned)((a.R * a.R + 255) / 256), (unsigned)a.N), 256, 0, st>>>(a.g_v, d_xyz, a.R, a.S, a.scale);
        P3D_LAUNCH_CHECK();
    }
    return P3D_OK;
}
