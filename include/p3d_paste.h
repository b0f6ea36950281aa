/*
 * p3d_paste.h - C ABI of the front-view paste (SURVEY.md 8f-3).
 *
 * The reference has no native code here: `paste_front` (/root/reference/_train/eg3dc/src/training/triplane.py:608-691)
 * is ~35 eager PyTorch / kornia ops over five full-resolution mask images per view, called by `TriPlaneGenerator.f`
 * (triplane.py:498-502) for every view of the eval sweep (_scripts/eval/generate.py:59-65) and, in the training modes
 * 'A' / 'Agrad', for every generated image (loss_orthocondA.py:131-150).  Here the five masks, the front-image lookup
 * and the blend are ONE kernel at output resolution; the two extra renders paste_front asks for stay calls of the
 * renderer (p3d_render.h), only their ray construction / erosion are small kernels below.
 *
 * All tensors fp32, contiguous NCHW, device pointers; return codes / p3d_last_error() as in p3d_render.h.
 */
#ifndef P3D_PASTE_H_
#define P3D_PASTE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct p3d_paste_params {
    int32_t n_views;            /* N */
    int32_t res_render;         /* R: side of image_xyz / image_weights / the occlusion render / the rays */
    int32_t res_image;          /* S: side of the output image = front_rgb.shape[-1] (triplane.py:627) */
    int32_t res_front;          /* side of the eroded front-weight image (0: front_weight_erosion < 1, mask = 1) */
    int32_t normalize_images;   /* x['normalize_images']: the pasted colours are front_rgb*2-1 (triplane.py:671) */
    int32_t reserved0;
    double  box_warp;           /* G.rendering_kwargs['box_warp'] */
    /* thresholds: Python floats in the reference, compared against fp32 tensors (the library rounds them to fp32) */
    double  thresh_weight, thresh_edges, thresh_occ, thresh_dxyz;
} p3d_paste_params;

/* get_front_occlusion's ray construction, triplane.py:565-570:
   ray_origins = image_xyz * (-1, 1, -1) with z -= ray_start - offset;  ray_dirs = (0, 0, 1).   All (N,3,R,R). */
int p3d_paste_occlusion_rays(const float* image_xyz, int32_t n_views, int32_t res, double ray_start, double offset,
                             float* ray_origins, float* ray_dirs, void* stream);

/* kornia.morphology.erosion((frontw > thresh).float(), ones(e, e)), triplane.py:650-655 (kornia 0.6.5: structuring
   element anchored at (e/2, e/2), geodesic border).  frontw, eroded: (N,1,H,W). */
int p3d_paste_erode(const float* frontw, int32_t n, int32_t h, int32_t w, int32_t e, double thresh, float* eroded,
                    void* stream);

/* paste_front's masks + paste + blend, triplane.py:620-679.
     image          (N,3,S,S)  out['image']
     image_xyz      (N,3,R,R)  out['image_xyz']
     image_weights  (N,1,R,R)  out['image_weights']
     front_rgb      (N,3,S,S)  x['cond']['image_ortho_front'] (or force_image)
     occ_weights    (N,1,R,R)  image_weights of the occlusion render (get_front_occlusion)
     ray_origins/ray_dirs (N,3,R,R)  x['force_rays']
     front_eroded   (N,1,res_front,res_front) from p3d_paste_erode, or NULL when res_front == 0
   outputs (caller-allocated)
     out_image, out_paste (N,3,S,S); out_mask (N,1,S,S);
     out_parts (5,N,1,S,S) = mask_weights, mask_edges, mask_occ, mask_dxyz, mask_frontweight - or NULL (not stored). */
int p3d_paste_front(const p3d_paste_params* p, const float* image, const float* image_xyz, const float* image_weights,
                    const float* front_rgb, const float* occ_weights, const float* ray_origins, const float* ray_dirs,
                    const float* front_eroded, float* out_image, float* out_paste, float* out_mask, float* out_parts,
                    void* stream);

/* Backward of the blend and (grad_sample=True, triplane.py:674-679) of the front-image lookup; the masks carry no
   gradient (computed under no_grad in the reference).
     g_image (N,3,S,S) gradient of out_image; g_paste (N,3,S,S) gradient of out_paste or NULL;
     d_image (N,3,S,S) <- g_image * (1 - mask)
     d_xyz   (N,3,R,R) <- through sample_orthofront and the bilinear up-sampling (ACCUMULATED: zero it first), or NULL
                          when grad_sample is off. */
int p3d_paste_front_backward(const p3d_paste_params* p, const float* image_xyz, const float* front_rgb, const float* mask,
                             const float* g_image, const float* g_paste, float* d_image, float* d_xyz, void* stream);

/* Deterministic p3d_paste_front_backward (torch.use_deterministic_algorithms): the same gradients, bit-identical from run to
   run.  d_image as above.  d_xyz is WRITTEN, not accumulated: each texel gathers, in a fixed order, the contributions the
   scatter above adds atomically (output pixels row-major, then the pixel's taps (i0,i0), (i0,i1), (i1,i0), (i1,i1); the z
   channel is zero).  scratch: p3d_paste_front_backward_det_scratch_bytes(p) device bytes (0 and p3d_last_error for bad
   params), needed when d_xyz is not NULL. */
size_t p3d_paste_front_backward_det_scratch_bytes(const p3d_paste_params* p);
int p3d_paste_front_backward_det(const p3d_paste_params* p, const float* image_xyz, const float* front_rgb, const float* mask,
                                 const float* g_image, const float* g_paste, void* scratch, size_t scratch_bytes,
                                 float* d_image, float* d_xyz, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* P3D_PASTE_H_ */
