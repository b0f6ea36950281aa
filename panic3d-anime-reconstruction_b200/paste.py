"""Front-view paste - the H100 replacement for ``paste_front`` and its helpers
(reference ``_train/eg3dc/src/training/triplane.py:555-691``; SURVEY.md section 8f-3).

``TriPlaneGenerator.f`` (triplane.py:498-502) calls ``paste_front(self, x, ret, **x['paste_params'])`` for every view
of the eval sweep (``_scripts/eval/generate.py:59-65``) and, in the training modes 'A' / 'Agrad'
(``loss_orthocondA.py:131-150``), for every generated image.  The reference builds five full-resolution masks with
~35 eager PyTorch / kornia ops; here

    ``get_front_occlusion`` / ``get_front_weights``   same two extra ``G.f`` renders (they run on the fused renderer),
                                                      ray construction / erosion = ``p3d_paste_occlusion_rays`` /
                                                      ``p3d_paste_erode``
    ``paste_front``                                   ONE launch of ``p3d_paste_front`` (masks + lookup + blend), with
                                                      a hand-written backward (``p3d_paste_front_backward``: the blend,
                                                      and with ``grad_sample=True`` the lookup back to ``image_xyz``)
    ``sample_orthofront`` / ``get_xyz_discrepancy``   kept for callers that use them stand-alone (plain torch ops on
                                                      the caller's device; not on the hot path)

Same names, arguments, defaults and returned keys as the reference.  ``dropin.install_paste()`` rebinds the reference
module's ``paste_front`` to this one, so ``G.f`` is unchanged.  No CPU path: tensors must live on a CUDA device (the
PyTorch restatement is ``oracle/paste_oracle.py``, tests only).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


class PasteParams(C.Structure):
    """Mirror of ``p3d_paste_params`` (include/p3d_paste.h) - field order and types must match."""
    _fields_ = [
        ('n_views', C.c_int32), ('res_render', C.c_int32), ('res_image', C.c_int32), ('res_front', C.c_int32),
        ('normalize_images', C.c_int32), ('reserved0', C.c_int32),
        ('box_warp', C.c_double),
        ('thresh_weight', C.c_double), ('thresh_edges', C.c_double), ('thresh_occ', C.c_double), ('thresh_dxyz', C.c_double),
    ]


_VP = C.c_void_p
_lib.register_protos({
    'p3d_paste_occlusion_rays': (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_double, C.c_double, _VP, _VP, _VP]),
    'p3d_paste_erode': (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, _VP, _VP]),
    'p3d_paste_front': (C.c_int, [C.POINTER(PasteParams)] + [_VP] * 8 + [_VP] * 4 + [_VP]),
    'p3d_paste_front_backward': (C.c_int, [C.POINTER(PasteParams)] + [_VP] * 7 + [_VP]),
    'p3d_paste_front_backward_det_scratch_bytes': (C.c_size_t, [C.POINTER(PasteParams)]),
    'p3d_paste_front_backward_det': (C.c_int, [C.POINTER(PasteParams)] + [_VP] * 5 + [_VP, C.c_size_t] + [_VP] * 2 + [_VP]),
})


class _AttrDict(dict):
    """Item + attribute access, like the ``uutil.Dict`` (addict) the reference returns."""
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


def _f32(t, name, shape=None):
    if not (torch.is_tensor(t) and t.is_cuda):
        raise RuntimeError(f'panic3d_b200.paste: {name} must be a CUDA tensor (there is no CPU path)')
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise RuntimeError(f'panic3d_b200.paste: {name} has shape {tuple(t.shape)}, expected {tuple(shape)}')
    return t.detach().float().contiguous()


# ---------------------------------------------------------------- stand-alone helpers (reference call surface)
def sample_orthofront(front_rgb, view_xyz, bw):
    """triplane.py:555-564.  Off the hot path (``paste_front`` fuses it); plain torch ops for stand-alone callers."""
    vij = 1 - (view_xyz[:, [1, 0]] + bw / 2) / bw
    return torch.nn.functional.grid_sample(front_rgb.permute(0, 1, 3, 2), vij.permute(0, 2, 3, 1) * 2 - 1, padding_mode='border',
                                           mode='bilinear', align_corners=False)


def get_xyz_discrepancy(xyz, rays):
    """triplane.py:601-606.  Off the hot path (fused into ``paste_front``)."""
    a, n = rays['ray_origins'], rays['ray_directions']
    p = xyz * torch.tensor([-1, 1, -1], device=xyz.device)[None, :, None, None]
    return ((p - a) - ((p - a) * n).sum(dim=1, keepdims=True) * n).norm(2, dim=1, keepdim=True)


def occlusion_rays(image_xyz, ray_start, offset=0.01):
    """Rays of ``get_front_occlusion`` (triplane.py:565-570): origins just in front of the visible surface, direction +z."""
    xyz = _f32(image_xyz, 'image_xyz')
    N, c, R, R2 = xyz.shape
    if c != 3 or R != R2:
        raise RuntimeError(f'panic3d_b200.paste: image_xyz must be (N,3,R,R), got {tuple(xyz.shape)}')
    ro, rd = torch.empty_like(xyz), torch.empty_like(xyz)
    with torch.cuda.device(xyz.device):
        _lib.check(_lib.lib().p3d_paste_occlusion_rays(xyz.data_ptr(), N, R, float(ray_start), float(offset), ro.data_ptr(),
                                                      rd.data_ptr(), _lib.stream_ptr(xyz.device)))
    return ro, rd


# Opt-in (``dropin.install_paste(reuse_triplane=True)``): the occlusion render needs only ``image_weights``, and ``G.f`` hands the
# tri-planes of the view back in ``out['triplane']`` (triplane.py:233-240) - so render from them directly instead of going through
# ``G.f`` again, which re-runs the 29 M-parameter backbone and the super-resolution head just to throw their outputs away.
# A deliberate deviation, like the plane memo: the reference's second ``G.f`` redraws the backbone's layer noise (noise_mode defaults
# to 'random', networks_stylegan2.py:334-343), so ITS occlusion render sees slightly different tri-planes than the view it belongs to;
# with const / no noise the two routes give the same weights.  Off by default.
REUSE_TRIPLANE = False


def get_front_occlusion(G, x, out, offset=0.01):
    """triplane.py:565-580: render along +z from the visible surface; returns that render's ``image_weights``."""
    ro, rd = occlusion_rays(out['image_xyz'], G.rendering_kwargs['ray_start'], offset)
    if REUSE_TRIPLANE and out.get('triplane') is not None and hasattr(G, 'renderer'):
        N, _, R, _ = ro.shape
        flat = lambda t: t.permute(0, 2, 3, 1).reshape(N, R * R, 3)
        _, _, weights, _ = G.renderer(out['triplane'], G.decoder, flat(ro), flat(rd), G.rendering_kwargs,
                                      triplane_crop=x.get('triplane_crop'), cull_clouds=x.get('cull_clouds'),
                                      binarize_clouds=x.get('binarize_clouds'))
        return weights.permute(0, 2, 1).reshape(N, 1, R, R)
    xin = {**x}
    xin['paste_params'] = None
    xin['force_rays'] = {'ray_origins': ro, 'ray_directions': rd}
    return G.f(xin, return_more=True)['image_weights']


def get_front_weights(G, x):
    """triplane.py:581-600: ``image_weights`` of the orthographic front view."""
    device = x['cond']['image_ortho_front'].device
    xin = {k: v for k, v in x.items() if k not in ['paste_params', 'camera_params', 'conditioning_params', 'force_rays']}
    xin['elevations'] = torch.zeros(1).to(device)
    xin['azimuths'] = torch.zeros(1).to(device)
    xin['fovs'] = -torch.ones(1).to(device)
    return G.f(xin, return_more=True)['image_weights']


def erode_front_weights(frontw, e, thresh=0.5):
    """``kornia.morphology.erosion((frontw > thresh).float(), ones(e, e))`` (triplane.py:650-655) on the GPU."""
    fw = _f32(frontw, 'frontw')
    if fw.dim() != 4 or fw.shape[1] != 1:
        raise RuntimeError(f'panic3d_b200.paste: frontw must be (N,1,H,W), got {tuple(fw.shape)}')
    out = torch.empty_like(fw)
    with torch.cuda.device(fw.device):
        _lib.check(_lib.lib().p3d_paste_erode(fw.data_ptr(), fw.shape[0], fw.shape[2], fw.shape[3], int(e), float(thresh),
                                             out.data_ptr(), _lib.stream_ptr(fw.device)))
    return out


# ---------------------------------------------------------------- the fused op
class _PasteFunction(torch.autograd.Function):
    """(image, image_xyz) -> (image_out, paste, mask, parts): p3d_paste_front / p3d_paste_front_backward, or
    p3d_paste_front_backward_det under ``torch.use_deterministic_algorithms(True)``."""

    @staticmethod
    def forward(ctx, image, image_xyz, consts, p, grad_sample, want_parts):
        weights, front, occ, ro, rd, eroded = consts
        dev = image.device
        N, S = p.n_views, p.res_image
        img, xyz = image.detach().float().contiguous(), image_xyz.detach().float().contiguous()
        o_img = torch.empty((N, 3, S, S), device=dev, dtype=torch.float32)
        o_paste = torch.empty_like(o_img)
        o_mask = torch.empty((N, 1, S, S), device=dev, dtype=torch.float32)
        o_parts = torch.empty((5, N, 1, S, S), device=dev, dtype=torch.float32) if want_parts else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().p3d_paste_front(C.byref(p), img.data_ptr(), xyz.data_ptr(), weights.data_ptr(), front.data_ptr(),
                                                 occ.data_ptr(), ro.data_ptr(), rd.data_ptr(), _lib.ptr(eroded), o_img.data_ptr(),
                                                 o_paste.data_ptr(), o_mask.data_ptr(), _lib.ptr(o_parts), _lib.stream_ptr(dev)))
        ctx.p, ctx.grad_sample = p, bool(grad_sample)
        ctx.xyz_shape = tuple(image_xyz.shape)
        ctx.save_for_backward(xyz, front, o_mask)
        ctx.mark_non_differentiable(o_mask)
        if o_parts is not None:
            ctx.mark_non_differentiable(o_parts)
            return o_img, o_paste, o_mask, o_parts
        return o_img, o_paste, o_mask

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_img, g_paste, *_):
        xyz, front, mask = ctx.saved_tensors
        dev = xyz.device
        g_img = torch.zeros_like(mask).expand(-1, 3, -1, -1).contiguous() if g_img is None else g_img.float().contiguous()
        want_xyz = ctx.grad_sample and ctx.needs_input_grad[1]
        g_paste = None if (g_paste is None or not ctx.grad_sample) else g_paste.float().contiguous()
        d_img = torch.empty_like(g_img)
        L = _lib.lib()
        if torch.are_deterministic_algorithms_enabled():
            d_xyz = torch.empty(ctx.xyz_shape, device=dev, dtype=torch.float32) if want_xyz else None
            scratch = torch.empty(int(L.p3d_paste_front_backward_det_scratch_bytes(C.byref(ctx.p))) if want_xyz else 0,
                                  dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                _lib.check(L.p3d_paste_front_backward_det(C.byref(ctx.p), xyz.data_ptr(), front.data_ptr(), mask.data_ptr(),
                                                          g_img.data_ptr(), _lib.ptr(g_paste), _lib.ptr(scratch if want_xyz else None),
                                                          scratch.numel(), d_img.data_ptr(), _lib.ptr(d_xyz), _lib.stream_ptr(dev)))
            return d_img, d_xyz, None, None, None, None
        d_xyz = torch.zeros(ctx.xyz_shape, device=dev, dtype=torch.float32) if want_xyz else None
        with torch.cuda.device(dev):
            _lib.check(L.p3d_paste_front_backward(C.byref(ctx.p), xyz.data_ptr(), front.data_ptr(), mask.data_ptr(),
                                                          g_img.data_ptr(), _lib.ptr(g_paste), d_img.data_ptr(), _lib.ptr(d_xyz),
                                                          _lib.stream_ptr(dev)))
        return d_img, d_xyz, None, None, None, None


def paste_front_fused(image, image_xyz, image_weights, front_rgb, occ_weights, ray_origins, ray_directions, box_warp,
                      front_eroded=None, normalize_images=False, thresh_weight=0.95, thresh_edges=0.02, thresh_occ=0.05,
                      thresh_dxyz=0.01, grad_sample=False, want_parts=True):
    """The mask / lookup / blend part of ``paste_front`` on explicit tensors (everything but the two extra renders).
    Returns (image, paste, mask, parts) with parts (5,N,1,S,S) = weights, edges, occ, dxyz, frontweight masks or None."""
    N, _, S, _ = front_rgb.shape
    R = image_xyz.shape[-1]
    image_in = image if torch.is_tensor(image) and image.is_cuda else _f32(image, 'image')
    if tuple(image_in.shape) != (N, 3, S, S):
        raise RuntimeError(f'panic3d_b200.paste: image must be {(N, 3, S, S)} like the front image, got {tuple(image_in.shape)}')
    if not image_xyz.is_cuda:
        raise RuntimeError('panic3d_b200.paste: image_xyz must be a CUDA tensor (there is no CPU path)')
    if tuple(image_xyz.shape) != (N, 3, R, R):
        raise RuntimeError(f'panic3d_b200.paste: image_xyz must be (N,3,R,R), got {tuple(image_xyz.shape)}')
    consts = (_f32(image_weights, 'image_weights', (N, 1, R, R)), _f32(front_rgb, 'front_rgb', (N, 3, S, S)),
              _f32(occ_weights, 'occ_weights', (N, 1, R, R)), _f32(ray_origins, 'ray_origins', (N, 3, R, R)),
              _f32(ray_directions, 'ray_directions', (N, 3, R, R)),
              None if front_eroded is None else _f32(front_eroded, 'front_eroded'))
    p = PasteParams()
    p.n_views, p.res_render, p.res_image = N, R, S
    p.res_front = 0 if front_eroded is None else int(front_eroded.shape[-1])
    if front_eroded is not None and tuple(front_eroded.shape) != (N, 1, p.res_front, p.res_front):
        raise RuntimeError(f'panic3d_b200.paste: front_eroded must be (N,1,Rf,Rf), got {tuple(front_eroded.shape)}')
    p.normalize_images = int(bool(normalize_images))
    p.box_warp = float(box_warp)
    p.thresh_weight, p.thresh_edges, p.thresh_occ, p.thresh_dxyz = float(thresh_weight), float(thresh_edges), float(thresh_occ), float(thresh_dxyz)
    res = _PasteFunction.apply(image_in, image_xyz, consts, p, grad_sample, want_parts)
    return res if want_parts else (*res, None)


def paste_front(G, x, out, mode='default', thresh_weight=0.95, thresh_edges=0.02, thresh_occ=0.05, offset_occ=0.01,
                thresh_dxyz=0.01, front_weight_erosion=0, grad_sample=False, force_image=None, **kwargs):
    """Drop-in for the reference ``paste_front`` (triplane.py:608-691): same arguments, same returned keys
    (``image, paste, mask, mask_weights, mask_edges, mask_occ, mask_dxyz, mask_frontweight, frontweight``)."""
    del mode, kwargs
    front_rgb = x['cond']['image_ortho_front']
    with torch.no_grad():
        occ = get_front_occlusion(G, x, out, offset=offset_occ)
        if front_weight_erosion >= 1:
            frontw = get_front_weights(G, x)
            eroded = erode_front_weights(frontw, int(front_weight_erosion))
        else:
            frontw = eroded = None
    tocopy = front_rgb if force_image is None else force_image.t()[None,].to(front_rgb.device)
    normalize = bool(x['normalize_images']) and force_image is None
    rays = x['force_rays']
    image, paste, mask, parts = paste_front_fused(
        out['image'], out['image_xyz'], out['image_weights'], tocopy, occ, rays['ray_origins'], rays['ray_directions'],
        G.rendering_kwargs['box_warp'], front_eroded=eroded, normalize_images=normalize, thresh_weight=thresh_weight,
        thresh_edges=thresh_edges, thresh_occ=thresh_occ, thresh_dxyz=thresh_dxyz, grad_sample=grad_sample)
    return _AttrDict({'image': image, 'paste': paste if grad_sample else paste.detach(), 'mask': mask, 'mask_weights': parts[0],
                      'mask_edges': parts[1], 'mask_occ': parts[2], 'mask_dxyz': parts[3], 'mask_frontweight': parts[4],
                      'frontweight': frontw})
