/*
 * p3d_render.h - C ABI of the H100-native tri-plane volumetric renderer.
 *
 * Drop-in boundary for the hot path of panic3d's EG3D-derived ray-marcher.  The
 * reference has NO native code on this path (it is ~60 eager PyTorch ops per
 * pass, SURVEY.md section 2.2); each entry point below names the reference
 * Python interface it replaces (paths relative to
 * /root/reference/_train/eg3dc/src/training/).  Everything is plain C: device
 * (or, for the *_host entry points, host) pointers + sizes + a cudaStream_t
 * passed as void*.  No torch types cross this boundary.
 *
 * Conventions
 *   - all tensors fp32 unless stated; "device pointer" means memory of the
 *     CUDA device that is current on the calling thread;
 *   - every function returns 0 on success, a negative P3D_E* code otherwise;
 *     p3d_last_error() returns a thread-local human-readable message
 *     (the Python host turns it into RuntimeError, matching TORCH_CHECK);
 *   - kernels are enqueued on `stream` and the call returns without
 *     synchronising, except the *_host entry points which synchronise.
 */
#ifndef P3D_RENDER_H_
#define P3D_RENDER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define P3D_OK            0
#define P3D_EINVAL       -1   /* bad argument (shape, null pointer, unsupported option) */
#define P3D_ECUDA        -2   /* CUDA runtime error (message has cudaGetErrorString) */
#define P3D_EWORKSPACE   -3   /* workspace too small */
#define P3D_EUNSUPPORTED -4   /* configuration has no kernel (caller must not fall back silently) */

/* third tri-plane convention: generate_planes(use_triplane), volumetric_rendering/renderer.py:26-50 */
#define P3D_PLANES_EG3D     0  /* planes read (x,y), (x,z), (z,x) */
#define P3D_PLANES_PANIC3D  1  /* planes read (x,y), (x,z), (y,z)   [use_triplane=True] */

/* ray limit mode: rendering_options['ray_start'/'ray_end'], renderer.py:165-174 */
#define P3D_RAYS_NUMERIC 0
#define P3D_RAYS_AUTOBOX 1     /* 'auto': math_utils.get_ray_limits_box, math_utils.py:46-98 */

/* decoder arithmetic */
#define P3D_MLP_FP32_SIMT   0  /* scalar FFMA, bit-for-bit-class fp32 (parity reference kernel) */
#define P3D_MLP_TC_3XBF16   1  /* wgmma bf16 tensor cores, 3-pass split operands (fp32-class accuracy) */
#define P3D_MLP_TC_BF16     2  /* wgmma bf16 single pass (fast mode; ~1e-2 abs) */

typedef struct p3d_render_params {
    /* problem size */
    int32_t n_views;          /* N */
    int32_t n_rays;           /* M rays per view */
    int32_t n_coarse;         /* S  = rendering_options['depth_resolution'] */
    int32_t n_fine;           /* Sf = rendering_options['depth_resolution_importance'] (0 = no importance pass) */
    int32_t channels;         /* C features per plane (32) */
    int32_t plane_h, plane_w; /* H, W of each plane */
    int32_t hidden;           /* OSGDecoder hidden width (64) */
    int32_t out_dim;          /* 1 + decoder_output_dim (33): [sigma, rgb...] */
    /* plane addressing, in ELEMENTS; channel stride must be 1 (channels-last texels).
       stride_view may be 0 (all views share one tri-plane). */
    int64_t stride_view, stride_plane, stride_row, stride_col;
    int32_t planes_bf16;      /* 0: planes are fp32, 1: planes are bf16 (fast mode storage) */
    /* rendering_options (doubles: the reference holds them as Python floats and rounds derived
       scalars such as 2/box_warp or (ray_end-ray_start)/(S-1) to fp32 only after computing them
       in double; the library does the same) */
    double  box_warp;
    double  ray_start, ray_end;
    int32_t ray_mode;         /* P3D_RAYS_* */
    int32_t disparity;        /* disparity_space_sampling */
    int32_t white_back;
    int32_t plane_mode;       /* P3D_PLANES_* */
    /* per-call flags of ImportanceRenderer.forward (renderer.py:162) ; <= 0 disables */
    double  triplane_crop, cull_clouds, binarize_clouds;
    /* decoder (triplane.py:516-548): gains of FullyConnectedLayer (networks_stylegan2.py:115-128) */
    float   w1_gain, b1_gain, w2_gain, b2_gain;
    int32_t force_sigmoid;
    int32_t mlp_mode;         /* P3D_MLP_* */
    /* jitter: when the u_* pointers passed to the call are NULL, uniforms come from Philox(seed) */
    uint64_t seed;
    /* multi-GPU exactness: the reference clamps composite depth to [min, max] of ALL depths of the batch
       (ray_marcher.py:50).  With defer_depth_clamp != 0 p3d_render_forward leaves out_depth un-clamped
       (NaN where the ray accumulated no weight) and stores this rank's (min, max) as two floats at the start of
       out-of-band device memory `depth_bounds` (see p3d_render_depth_bounds); the host all-reduces them
       (MIN, MAX) and calls p3d_depth_finalize. */
    int32_t defer_depth_clamp;
    /* multiplane tri-planes (rendering_kwargs['triplane_depth'] = D > 1; sample_from_planes, renderer.py:84-94): each plane
       is D slabs of (H, W, C) texels, sampled trilinearly (zero padding, align_corners=False) at the point's two plane
       coordinates and, across the slabs, its third component of project_onto_planes: z, y, then y (P3D_PLANES_EG3D) or
       x (P3D_PLANES_PANIC3D).  0 and 1 mean one slab.  Slab d of plane p of view v starts at element
       v*stride_view + p*stride_plane + d*plane_h*stride_row; texels stay channels-last (channel stride 1).  For D > 1:
         - stride_plane >= D*plane_h*stride_row and stride_view (unless 0) >= 3*stride_plane, else P3D_EINVAL;
         - only the fp32 SIMT kernels have a trilinear gather: p3d_render_fused_supported and p3d_decode_tc_supported
           return 0, an explicit P3D_MLP_TC_* request fails with P3D_EUNSUPPORTED, and so does p3d_render_forward_host;
         - the gradients of p3d_render_backward and p3d_decode_points_backward are (N,3,D,H,W,C) contiguous fp32. */
    int32_t plane_depth;
} p3d_render_params;

const char* p3d_version(void);
const char* p3d_last_error(void);

/* planes (N*3, C, H, W) fp32 NCHW  ->  (N*3, H, W, C) channels-last texels, fp32 or bf16.
   Replaces nothing in the reference (it samples NCHW through F.grid_sample, renderer.py:68-81);
   this is the layout pre-pass that makes every bilinear tap one contiguous 128 B (64 B) line. */
int p3d_planes_to_channels_last(const float* planes_nchw, void* planes_cl, int64_t n_planes,
                                int32_t channels, int32_t h, int32_t w, int32_t out_bf16, void* stream);

/* RaySampler.forward, volumetric_rendering/ray_sampler.py:24-63.
   cam2world (N,4,4), intrinsics (N,3,3) -> ray_origins, ray_dirs (N, R*R, 3). */
int p3d_raygen_pinhole(const float* cam2world, const float* intrinsics, int32_t n_views, int32_t resolution,
                       float* ray_origins, float* ray_dirs, void* stream);

/* get_rays_ortho, /root/reference/_databacks/lustrous_renders_v1.py:78-104.
   rot (N,3,3) row-major rotation (scipy Rotation 'xyz' [-elev, azim, 0] built by the host),
   dist (N) -> ray_origins, ray_dirs (N, R*R, 3). */
int p3d_raygen_ortho(const float* rot, const float* dist, int32_t n_views, int32_t resolution, double box_warp,
                     float* ray_origins, float* ray_dirs, void* stream);

/* Scratch needed by p3d_render_forward for these params (bytes). */
size_t p3d_render_workspace_bytes(const p3d_render_params* p);

/* 1 when the fused tensor-core renderer (mlp_mode P3D_MLP_TC_*) has a kernel for these params
   (depth_resolution == depth_resolution_importance in {48, 96}, C=32, hidden 64, out 33, rays per view a multiple of
   384/S, 32-bit tap offsets), else 0: such configurations run on the fp32 SIMT kernels (P3D_MLP_FP32_SIMT).  The host
   mirror (ImportanceRenderer.mlp_mode = 'auto') uses this to pick the tensor-core path whenever it exists; an
   explicit P3D_MLP_TC_* request for an unsupported configuration still fails with P3D_EUNSUPPORTED. */
int p3d_render_fused_supported(const p3d_render_params* p);

/* ImportanceRenderer.forward, volumetric_rendering/renderer.py:162-264
   (= sample_stratified :303-326, run_model :266-280 [sample_from_planes :68-81 + OSGDecoder
   triplane.py:528-544], crop/cull masks :138-153, MipRayMarcher2 ray_marcher.py:25-57,
   sample_importance :328-387, unify_samples :289-301, final composite :250-253).
     planes      channels-last texels addressed by the strides in *p
     w1 (hidden,C)  b1 (hidden)  w2 (out_dim,hidden)  b2 (out_dim)     raw parameters; gains in *p
     ray_origins, ray_dirs (N,M,3)
     u_coarse (N,M,S) or NULL, u_fine (N*M,Sf) or NULL                  injected U[0,1) jitter
     out_rgb (N,M,out_dim-1)  out_depth (N,M)  out_wsum (N,M)  out_xyz (N,M,3)                   */
int p3d_render_forward(const p3d_render_params* p, const void* planes,
                       const float* w1, const float* b1, const float* w2, const float* b2,
                       const float* ray_origins, const float* ray_dirs,
                       const float* u_coarse, const float* u_fine,
                       void* workspace, size_t workspace_bytes,
                       float* out_rgb, float* out_depth, float* out_wsum, float* out_xyz, void* stream);

/* Backward of p3d_render_forward (first order) - the autograd counterpart the training loop needs
   (loss_orthocondA.py:171,279,343,426 -> G.f -> ImportanceRenderer under autograd).  Gradients flow to the
   tri-plane features and the four decoder tensors; rays, stratified and importance depths (no_grad in the
   reference, renderer.py:332) and mask-overwritten densities are constants.
     fwd_workspace   the workspace of the matching p3d_render_forward call with mlp_mode = P3D_MLP_FP32_SIMT,
                     untouched since (it holds depths, masked densities and colours of every sample)
     out_depth       that call's out_depth;   g_*  incoming gradients (N,M,32) (N,M) (N,M) (N,M,3)
     d_planes        (N,3,H,W,C) contiguous fp32, d_w1 (hidden,C), d_b1, d_w2 (out,hidden), d_b2: ZERO-INITIALISED
                     by the caller, accumulated with atomics; parameter gradients are w.r.t. the raw tensors. */
size_t p3d_render_backward_scratch_bytes(const p3d_render_params* p);
int p3d_render_backward(const p3d_render_params* p, const void* planes,
                        const float* w1, const float* b1, const float* w2, const float* b2,
                        const float* ray_origins, const float* ray_dirs,
                        const void* fwd_workspace, size_t fwd_workspace_bytes, const float* out_depth,
                        const float* g_rgb, const float* g_depth, const float* g_wsum, const float* g_xyz,
                        void* scratch, size_t scratch_bytes,
                        float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2, void* stream);

/* Deterministic p3d_render_backward (torch.use_deterministic_algorithms): the same gradients, bit-identical from run to run
   whatever the GPU, grid or timing.  The outputs are WRITTEN, not accumulated (no zero-fill needed).  Instead of float atomics:
     d_planes  every tap is recorded as (texel, entry = (sample, plane, tap)); the entries are stably radix-sorted by texel and
               each texel sums its run in entry order, acc = fl(acc + fl(weight * feature gradient)); samples are numbered
               coarse pass first, then fine, each ray-major
     d_w1 .. d_b2  each 128-sample CTA writes its partial sums; they are added over CTA index by adjacent pairs, level by level
   At most 2^31 - 1 entries (views x rays x samples x 3 planes x 4 taps, 8 for multiplane planes) and texels; past that the
   scratch query returns 0 and the call P3D_EINVAL.  scratch: p3d_render_backward_det_scratch_bytes(p) device bytes. */
size_t p3d_render_backward_det_scratch_bytes(const p3d_render_params* p);
int p3d_render_backward_det(const p3d_render_params* p, const void* planes,
                            const float* w1, const float* b1, const float* w2, const float* b2,
                            const float* ray_origins, const float* ray_dirs,
                            const void* fwd_workspace, size_t fwd_workspace_bytes, const float* out_depth,
                            const float* g_rgb, const float* g_depth, const float* g_wsum, const float* g_xyz,
                            void* scratch, size_t scratch_bytes,
                            float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2, void* stream);

/* After a p3d_render_forward with defer_depth_clamp: write this call's (min depth, max depth) as 2 floats to
   device memory `bounds2` (from the call's workspace). */
int p3d_render_depth_bounds(const void* workspace, float* bounds2, void* stream);

/* nan_to_num(nan=inf) + clamp(depth, bounds2[0], bounds2[1]) in place, n rays.  ray_marcher.py:49-50. */
int p3d_depth_finalize(float* depth, int64_t n_rays, const float* bounds2, void* stream);

/* ImportanceRenderer.run_model, renderer.py:266-280 (used by TriPlaneGenerator.sample /
   sample_mixed, triplane.py:254-298, and the 256^3 grid query of _util/eg3d_metrics3d.py:94-183).
     coords (N,K,3) -> out_rgb (N,K,out_dim-1), out_sigma (N,K).  Uses n_views and the plane /
     decoder fields of *p; ray fields are ignored. */
int p3d_decode_points(const p3d_render_params* p, const void* planes,
                      const float* w1, const float* b1, const float* w2, const float* b2,
                      const float* coords, int64_t n_points_per_view,
                      float* out_rgb, float* out_sigma, void* stream);

/* 1 when p3d_decode_points / p3d_volume_query have a tensor-core kernel for these params (mlp_mode P3D_MLP_TC_*: the
   renderer's gather -> wgmma decoder pipeline streamed over the points; any point count), else 0 (fp32 SIMT kernels).
   The host mirror's mlp_mode = 'auto' uses it like p3d_render_fused_supported. */
int p3d_decode_tc_supported(const p3d_render_params* p, int64_t n_points_total);

/* Backward of p3d_decode_points (first order): what the density-regularisation phase of the training loop needs
   (loss_orthocondA.py:579-600: G.sample_mixed(...)['sigma'] -> TVloss.backward(); triplane.py:283-298 -> run_model).
   Gradients flow to the tri-plane features and the four decoder tensors; the coordinates are constants (they carry
   no grad in the reference's call).  planes: channels-last texels addressed by the strides in *p (read only);
     g_rgb (N,K,out_dim-1), g_sigma (N,K)   incoming gradients (pass zeros for an output the loss does not use)
     d_planes (N,3,H,W,C) contiguous fp32, d_w1, d_b1, d_w2, d_b2: ZERO-INITIALISED by the caller, accumulated with
     atomics; parameter gradients are w.r.t. the raw tensors (gains folded in). */
int p3d_decode_points_backward(const p3d_render_params* p, const void* planes,
                               const float* w1, const float* b1, const float* w2, const float* b2,
                               const float* coords, int64_t n_points_per_view,
                               const float* g_rgb, const float* g_sigma,
                               float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2, void* stream);

/* Deterministic p3d_decode_points_backward: written outputs and fixed summation orders as p3d_render_backward_det, sample
   index = view * n_points_per_view + point.  scratch: p3d_decode_points_backward_det_scratch_bytes(p, n) device bytes (0 and
   p3d_last_error past the 2^31 - 1 entry envelope or for a negative count). */
size_t p3d_decode_points_backward_det_scratch_bytes(const p3d_render_params* p, int64_t n_points_per_view);
int p3d_decode_points_backward_det(const p3d_render_params* p, const void* planes,
                                   const float* w1, const float* b1, const float* w2, const float* b2,
                                   const float* coords, int64_t n_points_per_view,
                                   const float* g_rgb, const float* g_sigma, void* scratch, size_t scratch_bytes,
                                   float* d_planes, float* d_w1, float* d_b1, float* d_w2, float* d_b2, void* stream);

/* Dense sigma / colour grid for mesh extraction: the renderer-level part of get_eg3d_volume
   (_util/eg3d_metrics3d.py:94-183), which the reference evaluates as 168 host-side chunks of 100k points through
   G.sample_mixed -> ImportanceRenderer.run_model with a .cpu() round trip per chunk.  One launch here:
     * point n of view v (0 <= n < resolution^3) is the reference's create_samples point (eg3d_metrics3d.py:70-92),
       reproduced bit for bit INCLUDING its un-floored float y/x indices, for cube_length = box_warp;
     * results are written where the reference's reshape(R,R,R,.).flip(dims=(1,)) puts them: element (a,b,c) of view v
       is point n = ((R-1-a)*R + b)*R + c.  out_sigma (N,R,R,R); out_rgb (N,R,R,R,out_dim-1) or NULL;
       out_coords (N,R,R,R,3) or NULL; out_density (N,R,R,R) or NULL = sigma2density(sigma) with -1e3 where
       triplane_crop (>= 0; negative = None) crops the point or where cull_clouds (>= 0; negative = None) culls it -
       the cull test is applied to the density exactly as the reference does (cull_clouds_mask on densities,
       eg3d_metrics3d.py:160-162).
   Uses n_views, the plane / decoder fields and box_warp of *p; ray fields are ignored. */
int p3d_volume_query(const p3d_render_params* p, const void* planes,
                     const float* w1, const float* b1, const float* w2, const float* b2,
                     int32_t resolution, double cube_length, double triplane_crop, double cull_clouds,
                     float* out_sigma, float* out_rgb, float* out_density, float* out_coords, void* stream);

/* End-to-end entry point with HOST buffers (what a non-torch caller binds): copies the
   NCHW fp32 tri-planes, decoder and cameras to the device, generates pinhole rays, renders and
   copies (rgb, depth, wsum, xyz) back.  Device buffers are cached between calls in a
   process-wide arena; p3d_host_arena_release() frees it.  planes_nchw (N,3,C,H,W);
   stride fields of *p are ignored (set internally). u_* may be NULL (Philox). Synchronises. */
int p3d_render_forward_host(const p3d_render_params* p, const float* planes_nchw,
                            const float* w1, const float* b1, const float* w2, const float* b2,
                            const float* cam2world, const float* intrinsics, int32_t resolution,
                            const float* u_coarse, const float* u_fine,
                            float* out_rgb, float* out_depth, float* out_wsum, float* out_xyz);
void p3d_host_arena_release(void);

/* Peer-to-peer delivery of rendered images between the per-GPU processes of one box (views.PeerGather): the consumer rank
   allocates a device buffer and exports it; every other rank opens the handle ON ITS OWN device (peer access over NVLink is
   enabled lazily by the driver) and copies its shard into it with the copy engines - no SM, so the transfer runs under the
   persistent renderer of the next step, which an NCCL kernel cannot.
     p3d_ipc_alloc   cudaMalloc + cudaIpcGetMemHandle; handle64 receives the 64-byte cudaIpcMemHandle_t
     p3d_ipc_open    cudaIpcOpenMemHandle(cudaIpcMemLazyEnablePeerAccess) on the current device
     p3d_ipc_close / p3d_ipc_free   undo the above
     p3d_copy_async  cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, stream) */
int p3d_ipc_alloc(size_t bytes, void** dptr, unsigned char* handle64);
int p3d_ipc_open(const unsigned char* handle64, void** dptr);
int p3d_ipc_close(void* dptr);
int p3d_ipc_free(void* dptr);
int p3d_copy_async(void* dst, const void* src, size_t bytes, void* stream);

/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
uint64_t p3d_launch_count(void);

/* Per-kernel device timing for bench.py's roofline leg.  When enabled, launch sites bracket their
   kernel with CUDA events on the launching stream.  Slots: 0 sample_decode (gather+MLP), 1 importance,
   2 composite, 3 layout pre-pass, 4 raygen, 5 fused renderer, 6 other.  p3d_profile_read waits for the
   recorded events, adds them up per slot (milliseconds, launch counts) and optionally resets. */
void p3d_profile_enable(int on);
int  p3d_profile_read(double* ms_by_slot, uint64_t* launches_by_slot, int n_slots, int reset);

#ifdef __cplusplus
}
#endif
#endif /* P3D_RENDER_H_ */
