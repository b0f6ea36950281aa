// Internal (non-ABI) declarations shared by the renderer translation units.
#pragma once
#include "p3d_common.cuh"

namespace p3d {

constexpr int kC = 32;        // features per plane
constexpr int kHidden = 64;   // OSGDecoder hidden width
constexpr int kOut = 33;      // sigma + 32 colour features
constexpr int kRgb = 32;

// Everything a kernel needs that is derived from p3d_render_params (host-computed, fp32-rounded
// the way the reference's Python scalars get rounded when they meet an fp32 tensor).
struct Geom {
    int N, M, S, Sf, H, W;
    long long stride_view, stride_plane, stride_row, stride_col;
    float coord_scale;        // float(2 / box_warp)                          renderer.py:77
    float half_box;           // float(box_warp / 2)                          math_utils.py:58-59
    float ray_start, ray_end; // float(ray_start), float(ray_end)
    float lin_step;           // fp32 (end - start) / (S - 1)   torch.linspace step
    float depth_delta;        // float((ray_end - ray_start) / (S - 1))        renderer.py:323
    float inv_start, inv_end; // float(1/ray_start), float(1/ray_end)          renderer.py:313
    float disp_delta;         // float(1 / (S - 1))                            renderer.py:311
    float crop_limit;         // float(box_warp / 2 - triplane_crop)           renderer.py:143
    float cull_thresh;        // float(cull_clouds or binarize_clouds)
    int ray_mode, disparity, white_back, plane_mode;
    int crop_on, cull_on, binarize_on;
    int force_sigmoid;
    float w1_gain, b1_gain, w2_gain, b2_gain;
    int D;                    // slabs per plane (plane_depth; 1 unless multiplane).  Fills the padding before seed, so the
                              // struct keeps its size and every other field its offset
    unsigned long long seed;
};

struct Workspace {
    float* depth_c;   // R*S      coarse depths
    float* sigma_c;   // R*S      coarse densities (after crop/cull)
    float* rgb_c;     // R*S*32   coarse colours
    float* depth_f;   // R*Sf     importance depths, ascending per ray
    float* sigma_f;   // R*Sf
    float* rgb_f;     // R*Sf*32
    float* ray_t0;    // R        'auto' limits
    float* ray_t1;    // R
    unsigned int* bounds;  // [0] min depth, [1] max depth (ordered-uint), [2] min valid t0, [3] max valid t0, [4] any valid
};

// The volume query's scalars, each rounded to fp32 once where the reference's Python floats meet an fp32 tensor
// (_util/eg3d_metrics3d.py:70-183).
struct VolumeSpec {
    int res;                  // grid side R: R^3 points per view
    float size, origin;       // voxel size cube / (R - 1) and corner -cube / 2
    float crop, cull;         // crop limit box_warp / 2 - triplane_crop (< 0 crops everything, as there) / cull threshold
    int crop_on, cull_on;
};

// Sizes of a deterministic backward (render_backward.cu, DESIGN.md section 4.3): samples of the call, NT = 3 planes x taps
// entries per sample, CTAs of the sample kernel, texels of the gradient, radix-sort key bits and CUB's temporary bytes.
struct DetPlan {
    long long samples, entries, ctas, texels, texels_view;
    int nt, key_bits;
    size_t sort_bytes;
};
// its scratch: sample feature gradients, entry weights, keys and ids (two buffers each for the sort), CTA partials, the
// pairwise levels over them and the sort's temporaries
struct DetBufs {
    float *dx, *w, *part, *part2;
    unsigned *key0, *key1, *id0, *id1;
    void* sort_tmp;
};
// n_pts < 0: a render of g's rays, else a point query of n_pts points per view.  P3D_EINVAL past the 2^31 - 1 entry / texel envelope
int det_plan(const Geom& g, long long n_pts, DetPlan* d);
size_t det_layout(const DetPlan& d, size_t head, void* base, DetBufs* b);

int make_geom(const p3d_render_params* p, Geom* g);
size_t workspace_layout(const p3d_render_params* p, void* base, Workspace* ws);

// v1: multi-kernel SIMT pipeline (fp32 exact); always available.
int render_forward_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                      const float* w2, const float* b2, const float* ro, const float* rd, const float* u_c,
                      const float* u_f, const Workspace& ws, float* out_rgb, float* out_depth, float* out_wsum,
                      float* out_xyz, cudaStream_t stream);
int render_backward_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                       const float* w2, const float* b2, const float* ro, const float* rd, const Workspace& ws,
                       const float* out_depth, const float* g_rgb, const float* g_depth, const float* g_wsum,
                       const float* g_xyz, void* scratch, size_t scratch_bytes, float* d_planes, float* d_w1, float* d_b1,
                       float* d_w2, float* d_b2, cudaStream_t stream, const DetPlan* det = nullptr);
// small launches of render_v1.cu shared by both renderers
int launch_bounds_init(unsigned int* bounds, cudaStream_t stream);
int launch_ray_limits(const float* ro, const float* rd, long long R, float h, float* t0, float* t1, unsigned int* bounds,
                      cudaStream_t stream);
int launch_depth_finalize(float* depth, long long R, const unsigned int* bounds, cudaStream_t stream);
int launch_bounds_to_float(const unsigned int* bounds, float* out2, cudaStream_t stream);
int launch_depth_finalize_f(float* depth, long long R, const float* bounds2, cudaStream_t stream);
// warp-specialised fused renderer (render_fused_ws3.cu): gather / wgmma decoder / ray roles, three ray groups in flight
bool fused_ws3_supported(const Geom& g);
int render_forward_fused_ws3(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                             const float* w2, const float* b2, const float* ro, const float* rd, const float* u_c,
                             const float* u_f, const Workspace& ws, float* out_rgb, float* out_depth, float* out_wsum,
                             float* out_xyz, cudaStream_t stream);
int decode_points_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                     const float* w2, const float* b2, const float* coords, long long n_pts, float* out_rgb,
                     float* out_sigma, cudaStream_t stream);
// streaming tensor-core decode (decode_tc.cu): the gather -> wgmma decoder pipeline of the renderer without per-ray phases
bool decode_tc_supported(const Geom& g, long long total);
int decode_points_tc(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                     const float* w2, const float* b2, const float* coords, long long n_pts, float* out_rgb,
                     float* out_sigma, cudaStream_t stream);
int volume_query_tc(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                    const float* w2, const float* b2, const VolumeSpec& vol, float* out_sigma, float* out_rgb,
                    float* out_density, float* out_coords, cudaStream_t stream);
int decode_points_backward_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                              const float* w2, const float* b2, const float* coords, long long n_pts, const float* g_rgb,
                              const float* g_sigma, float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2,
                              cudaStream_t stream, const DetPlan* det = nullptr, void* scratch = nullptr, size_t scratch_bytes = 0);
int volume_query_v1(const Geom& g, const p3d_render_params* p, const void* planes, const float* w1, const float* b1,
                    const float* w2, const float* b2, const VolumeSpec& vol, float* out_sigma, float* out_rgb,
                    float* out_density, float* out_coords, cudaStream_t stream);

}  // namespace p3d
