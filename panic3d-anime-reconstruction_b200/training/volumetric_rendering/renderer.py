"""Drop-in for ``training/volumetric_rendering/renderer.py`` of the reference
(/root/reference/_train/eg3dc/src/training/volumetric_rendering/renderer.py).

Same names, argument meaning and return shapes as the reference module; the whole of
``ImportanceRenderer.forward`` (renderer.py:162-264) is one call into the CUDA library
(``p3d_render_forward``, include/p3d_render.h) instead of ~60 eager PyTorch ops.
No CPU path: tensors must live on a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import torch

from ... import _lib
from .ray_marcher import MipRayMarcher2


def generate_planes(use_triplane: bool = False) -> torch.Tensor:
    """Axis triplets of the three planes (reference renderer.py:26-50).  Kept for API
    compatibility (``renderer.plane_axes``); the kernels use the equivalent ``plane_mode``."""
    third = [[0, 1, 0], [0, 0, 1], [1, 0, 0]] if use_triplane else [[0, 0, 1], [1, 0, 0], [0, 1, 0]]
    return torch.tensor([[[1, 0, 0], [0, 1, 0], [0, 0, 1]],
                         [[1, 0, 0], [0, 0, 1], [0, 1, 0]],
                         third], dtype=torch.float32)


def project_onto_planes(planes: torch.Tensor, coordinates: torch.Tensor) -> torch.Tensor:
    """(n_planes,3,3), (N,M,3) -> (N*n_planes, M, 3).  Reference renderer.py:52-66.
    Host-side helper only; the CUDA gather selects the two components directly."""
    N, M, _ = coordinates.shape
    n_planes = planes.shape[0]
    inv = torch.linalg.inv(planes)
    out = torch.einsum('nmc,pcd->npmd', coordinates, inv)
    return out.reshape(N * n_planes, M, 3)


def triplane_crop_mask(xyz_unformatted, thresh, boxwarp, allow_bottom=True):
    """True where density is forced to -1e3 (reference renderer.py:138-149)."""
    lim = boxwarp / 2 - thresh
    return ~((xyz_unformatted[:, :, [0, 2]].abs() <= lim).all(dim=-1, keepdim=True))


def cull_clouds_mask(denities, thresh):
    """Reference renderer.py:150-153."""
    return (1 - torch.exp(-torch.nn.functional.softplus(denities - 1))) < thresh


def _decoder_params(decoder):
    """Pull the four tensors + gains out of an OSGDecoder-like module (ours or the reference's:
    triplane.py:516-548 with FullyConnectedLayer, networks_stylegan2.py:101-136)."""
    fc1, fc2 = decoder.net[0], decoder.net[2]
    return (fc1.weight, fc1.bias, fc2.weight, fc2.bias,
            float(fc1.weight_gain), float(fc1.bias_gain), float(fc2.weight_gain), float(fc2.bias_gain),
            bool(getattr(decoder, 'force_sigmoid', False)))


def _multiplane_texels(planes: torch.Tensor, depth: int) -> torch.Tensor:
    """(N,3,C*D,H,W) -> (N,3,D,H,W,C) contiguous: channel c*D + d of the input is feature c of slab d (the reference's
    view as (N*3,C,D,H,W), renderer.py:84-94), laid out as the D slabs of channels-last texels p3d_render_params'
    plane_depth addresses."""
    N, P, CD, H, W = planes.shape
    return planes.view(N, P, CD // depth, depth, H, W).permute(0, 1, 3, 4, 5, 2).contiguous()


def _check_depth(planes: torch.Tensor, depth: int) -> int:
    if depth < 1 or planes.shape[2] % depth:
        raise ValueError(f'triplane_depth {depth} does not divide the {planes.shape[2]} plane channels')
    if depth > 1 and planes.shape[2] // depth != 32:
        # the kernels are built for 32 features per texel (p3d_render_params.channels); a multiplane model with another
        # width per slab (e.g. triplane_width 16 at triplane_depth 2) has no accelerated path
        raise NotImplementedError(f'triplane_depth {depth} splits {planes.shape[2]} plane channels into {planes.shape[2] // depth} '
                                  'features per slab; multiplane tri-planes are rendered with 32 features per slab only')
    return depth


class _PlaneCache:
    """Channels-last copy of the most recent tri-plane tensor (keyed on storage + version), so the
    16 views of one subject (generate.py:108-130) pay for the layout pre-pass once."""

    def __init__(self):
        self.key = None
        self.buf = None
        self.src = None        # strong ref: while cached, the source storage cannot be freed and its address reused

    def get(self, planes: torch.Tensor, bf16: bool, depth: int = 1):
        key = (planes.data_ptr(), planes._version, tuple(planes.shape), tuple(planes.stride()), planes.device, bf16, depth)
        if key != self.key:
            if depth > 1:
                buf = _multiplane_texels(planes, depth).to(torch.bfloat16 if bf16 else torch.float32)
            else:
                N, P, Cc, H, W = planes.shape
                src = planes if planes.is_contiguous() else planes.contiguous()
                buf = torch.empty((N, P, H, W, Cc), device=planes.device, dtype=torch.bfloat16 if bf16 else torch.float32)
                _lib.check(_lib.lib().p3d_planes_to_channels_last(src.data_ptr(), buf.data_ptr(), N * P, Cc, H, W,
                                                                 1 if bf16 else 0, _lib.stream_ptr(planes.device)))
            self.key, self.buf, self.src = key, buf, planes
        return self.buf


def _fp32_texels(planes: torch.Tensor, p) -> torch.Tensor:
    """The training path's fp32 channels-last copy of the planes, (N,3,H,W,C) or (N,3,D,H,W,C) for multiplane planes; the
    backward scatters into a buffer of the same layout.  Sets the plane strides of p."""
    src = planes.detach().float()
    if p.plane_depth > 1:
        planes_cl = _multiplane_texels(src, p.plane_depth)
        sv, sp, _, sr, sc, _ = planes_cl.stride()
    else:
        planes_cl = torch.empty((p.n_views, 3, p.plane_h, p.plane_w, p.channels), device=planes.device, dtype=torch.float32)
        srcc = src if src.is_contiguous() else src.contiguous()
        _lib.check(_lib.lib().p3d_planes_to_channels_last(srcc.data_ptr(), planes_cl.data_ptr(), p.n_views * 3, p.channels,
                                                         p.plane_h, p.plane_w, 0, _lib.stream_ptr(planes.device)))
        sv, sp, sr, sc, _ = planes_cl.stride()
    p.stride_view, p.stride_plane, p.stride_row, p.stride_col, p.planes_bf16 = sv, sp, sr, sc, 0
    return planes_cl


def _planes_grad(d_planes: torch.Tensor, dtype) -> torch.Tensor:
    """(N,3,H,W,C) or (N,3,D,H,W,C) gradient of the texels -> the (N,3,C[*D],H,W) indexing of the input planes."""
    if d_planes.dim() == 6:
        N, P, D, H, W, Cc = d_planes.shape
        return d_planes.permute(0, 1, 5, 2, 3, 4).reshape(N, P, Cc * D, H, W).to(dtype)
    return d_planes.permute(0, 1, 4, 2, 3).to(dtype)


class _RenderFunction(torch.autograd.Function):
    """Training path: fp32 SIMT forward (keeps its per-sample scratch) + p3d_render_backward.  Gradients reach
    the tri-planes and the four decoder tensors; rays and the (no_grad) importance depths are constants, as in
    the reference graph (renderer.py:332)."""

    @staticmethod
    def forward(ctx, renderer, planes, w1, b1, w2, b2, ro, rd, p, noise):
        dev = planes.device
        L = _lib.lib()
        N, M = p.n_views, p.n_rays
        # the backward scatters into a canonical (N,3,[D,]H,W,C) buffer, so the forward reads the same layout
        planes_cl = _fp32_texels(planes, p)
        p.mlp_mode = _lib.P3D_MLP_FP32_SIMT
        wt = [t.detach().float().contiguous() for t in (w1, b1, w2, b2)]
        ro, rd = ro.detach().float().contiguous(), rd.detach().float().contiguous()
        u_c, u_f = noise
        out = [torch.empty(sh, device=dev, dtype=torch.float32) for sh in ((N, M, p.out_dim - 1), (N, M, 1), (N, M, 1), (N, M, 3))]
        ws = torch.empty(int(L.p3d_render_workspace_bytes(C.byref(p))), dtype=torch.uint8, device=dev)
        _lib.check(L.p3d_render_forward(C.byref(p), planes_cl.data_ptr(), *[t.data_ptr() for t in wt], ro.data_ptr(), rd.data_ptr(),
                                        _lib.ptr(u_c), _lib.ptr(u_f), ws.data_ptr(), ws.numel(), *[o.data_ptr() for o in out],
                                        _lib.stream_ptr(dev)))
        if p.defer_depth_clamp:
            b2_ = torch.empty(2, device=dev, dtype=torch.float32)
            _lib.check(L.p3d_render_depth_bounds(ws.data_ptr(), b2_.data_ptr(), _lib.stream_ptr(dev)))
            renderer.depth_bounds_reduce(b2_)
            _lib.check(L.p3d_depth_finalize(out[1].data_ptr(), N * M, b2_.data_ptr(), _lib.stream_ptr(dev)))
        ctx.save_for_backward(planes_cl, *wt, ro, rd, ws, out[1])
        ctx.p = p
        ctx.in_dtypes = (planes.dtype, w1.dtype, b1.dtype, w2.dtype, b2.dtype)
        return tuple(out)

    @staticmethod
    @torch.autograd.function.once_differentiable     # hand-written first-order backward: a double backward must raise, not silently treat it as constant
    def backward(ctx, g_rgb, g_depth, g_wsum, g_xyz):
        planes_cl, w1, b1, w2, b2, ro, rd, ws, depth = ctx.saved_tensors
        p, dev, L = ctx.p, planes_cl.device, _lib.lib()
        N, M = p.n_views, p.n_rays
        z = lambda g_, sh: (torch.zeros(sh, device=dev, dtype=torch.float32) if g_ is None else g_.float().contiguous())
        g_rgb, g_depth, g_wsum, g_xyz = z(g_rgb, (N, M, p.out_dim - 1)), z(g_depth, (N, M, 1)), z(g_wsum, (N, M, 1)), z(g_xyz, (N, M, 3))
        d_planes = torch.zeros_like(planes_cl)
        d_w = [torch.zeros_like(t) for t in (w1, b1, w2, b2)]
        scratch = torch.empty(int(L.p3d_render_backward_scratch_bytes(C.byref(p))), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.p3d_render_backward(C.byref(p), planes_cl.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                             ro.data_ptr(), rd.data_ptr(), ws.data_ptr(), ws.numel(), depth.data_ptr(),
                                             g_rgb.data_ptr(), g_depth.data_ptr(), g_wsum.data_ptr(), g_xyz.data_ptr(),
                                             scratch.data_ptr(), scratch.numel(), d_planes.data_ptr(), *[t.data_ptr() for t in d_w],
                                             _lib.stream_ptr(dev)))
        dts = ctx.in_dtypes
        return (None, _planes_grad(d_planes, dts[0]), d_w[0].to(dts[1]), d_w[1].to(dts[2]), d_w[2].to(dts[3]),
                d_w[3].to(dts[4]), None, None, None, None)


class _PointsFunction(torch.autograd.Function):
    """run_model under autograd (the Greg phase: loss_orthocondA.py:579-600 back-propagates a TV loss on
    G.sample_mixed(...)['sigma']; triplane.py:283-298 -> renderer.run_model).  Forward = p3d_decode_points, backward =
    p3d_decode_points_backward: gradients reach the tri-planes and the four decoder tensors; the query coordinates are
    constants (they carry no grad in the reference's call)."""

    @staticmethod
    def forward(ctx, planes, w1, b1, w2, b2, coords, p):
        dev = planes.device
        L = _lib.lib()
        N, K = coords.shape[0], coords.shape[1]
        planes_cl = _fp32_texels(planes, p)
        wt = [t.detach().float().contiguous() for t in (w1, b1, w2, b2)]
        coords = coords.detach().float().contiguous()
        rgb = torch.empty((N, K, p.out_dim - 1), device=dev, dtype=torch.float32)
        sigma = torch.empty((N, K, 1), device=dev, dtype=torch.float32)
        _lib.check(L.p3d_decode_points(C.byref(p), planes_cl.data_ptr(), *[t.data_ptr() for t in wt], coords.data_ptr(), K,
                                       rgb.data_ptr(), sigma.data_ptr(), _lib.stream_ptr(dev)))
        ctx.save_for_backward(planes_cl, *wt, coords)
        ctx.p = p
        ctx.in_dtypes = (planes.dtype, w1.dtype, b1.dtype, w2.dtype, b2.dtype)
        return rgb, sigma

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_rgb, g_sigma):
        planes_cl, w1, b1, w2, b2, coords = ctx.saved_tensors
        p, dev, L = ctx.p, planes_cl.device, _lib.lib()
        N, K = coords.shape[0], coords.shape[1]
        g_rgb = torch.zeros((N, K, p.out_dim - 1), device=dev) if g_rgb is None else g_rgb.float().contiguous()
        g_sigma = torch.zeros((N, K, 1), device=dev) if g_sigma is None else g_sigma.float().contiguous()
        d_planes = torch.zeros_like(planes_cl)
        d_w = [torch.zeros_like(t) for t in (w1, b1, w2, b2)]
        with torch.cuda.device(dev):
            _lib.check(L.p3d_decode_points_backward(C.byref(p), planes_cl.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                                    b2.data_ptr(), coords.data_ptr(), K, g_rgb.data_ptr(), g_sigma.data_ptr(),
                                                    d_planes.data_ptr(), *[t.data_ptr() for t in d_w], _lib.stream_ptr(dev)))
        dts = ctx.in_dtypes
        return (_planes_grad(d_planes, dts[0]), d_w[0].to(dts[1]), d_w[1].to(dts[2]), d_w[2].to(dts[3]), d_w[3].to(dts[4]),
                None, None)


class ImportanceRenderer(torch.nn.Module):
    """Reference: renderer.py:156-387.  Parameter-free, like the reference."""

    def __init__(self, use_triplane: bool = False):
        super().__init__()
        self.ray_marcher = MipRayMarcher2()
        self.use_triplane = bool(use_triplane)
        self.plane_axes = generate_planes(use_triplane=use_triplane)
        # decoder arithmetic (include/p3d_render.h).  'auto' (default): the fused tensor-core kernel in its fp32-class 3-pass
        # mode wherever it exists (p3d_render_fused_supported: depth_resolution == depth_resolution_importance in
        # {48, 96} - the reference's training and eval settings), the fp32 SIMT kernels for every other sample count.
        # An explicit _lib.P3D_MLP_* value forces that mode and raises if it has no kernel.
        self.mlp_mode = 'auto'
        self.planes_bf16 = False                   # fast-mode plane storage
        self.injected_noise = None                 # (u_coarse (N,M,S[,1]), u_fine (N*M,Sf)) for parity tests
        # multi-GPU: callable(bounds2: cuda float tensor [min,max]) reducing the depth-clamp bounds across ranks in
        # place (panic3d_b200.views.all_reduce_depth_bounds) so a sharded batch clamps like the whole batch would
        self.depth_bounds_reduce = None
        self._planes = _PlaneCache()
        self._workspace = None

    # ------------------------------------------------------------------ helpers
    def _params(self, planes_cl, N, M, opts, decoder, triplane_crop, cull_clouds, binarize_clouds, n_points=None):
        if opts.get('density_noise', 0) > 0:
            raise NotImplementedError('density_noise > 0 is outside the accelerated path')
        if opts.get('clamp_mode', 'softplus') != 'softplus':
            raise AssertionError('MipRayMarcher only supports `clamp_mode`=`softplus`!')
        w1, b1, w2, b2, g1, gb1, g2, gb2, force_sigmoid = _decoder_params(decoder)
        p = _lib.RenderParams()
        p.n_views, p.n_rays = N, M
        p.n_coarse = int(opts.get('depth_resolution', 2))
        p.n_fine = int(opts.get('depth_resolution_importance', 0) or 0)
        if planes_cl.dim() == 6:                         # multiplane (N,3,D,H,W,C): slab d at d * H * stride_row
            _, _, D, H, W, Cc = planes_cl.shape
            sv, sp, ss, sr, sc, s1 = planes_cl.stride()
            assert ss == H * sr
            p.plane_depth = D
        else:
            _, _, H, W, Cc = planes_cl.shape
            sv, sp, sr, sc, s1 = planes_cl.stride()
        assert s1 == 1
        p.channels, p.plane_h, p.plane_w = Cc, H, W
        p.hidden, p.out_dim = w1.shape[0], w2.shape[0]
        p.stride_view, p.stride_plane, p.stride_row, p.stride_col = sv, sp, sr, sc
        p.planes_bf16 = 1 if planes_cl.dtype == torch.bfloat16 else 0
        p.box_warp = float(opts['box_warp'])
        rs, re = opts.get('ray_start', 'auto'), opts.get('ray_end', 'auto')
        if rs == 'auto' and re == 'auto':
            p.ray_mode = _lib.P3D_RAYS_AUTOBOX
        else:
            p.ray_mode, p.ray_start, p.ray_end = _lib.P3D_RAYS_NUMERIC, float(rs), float(re)
        p.disparity = 1 if opts.get('disparity_space_sampling', False) else 0
        p.white_back = 1 if opts.get('white_back', False) else 0
        p.plane_mode = _lib.P3D_PLANES_PANIC3D if self.use_triplane else _lib.P3D_PLANES_EG3D
        p.triplane_crop = float(triplane_crop or 0)
        p.cull_clouds = float(cull_clouds or 0)
        p.binarize_clouds = float(binarize_clouds or 0)
        p.w1_gain, p.b1_gain, p.w2_gain, p.b2_gain = g1, gb1, g2, gb2
        p.force_sigmoid = 1 if force_sigmoid else 0
        if self.mlp_mode == 'auto':
            p.mlp_mode = _lib.P3D_MLP_TC_3XBF16
            ok = (_lib.lib().p3d_render_fused_supported(C.byref(p)) if n_points is None      # ray rendering
                  else _lib.lib().p3d_decode_tc_supported(C.byref(p), int(n_points)))       # point / volume decode
            if not ok:
                p.mlp_mode = _lib.P3D_MLP_FP32_SIMT
        else:
            p.mlp_mode = int(self.mlp_mode)
        p.seed = int(torch.empty((), dtype=torch.int64).random_().item()) & 0xFFFFFFFFFFFFFFFF
        return p, (w1, b1, w2, b2)

    def _planes_cl(self, planes: torch.Tensor, depth: int = 1) -> torch.Tensor:
        """Channels-last texels of (N,3,C*depth,H,W) planes: (N,3,H,W,C), or (N,3,depth,H,W,C) for multiplane planes."""
        if planes.dim() != 5 or planes.shape[1] != 3:
            raise ValueError(f'planes must be (N,3,C,H,W), got {tuple(planes.shape)}')
        depth = _check_depth(planes, depth)
        want = torch.bfloat16 if self.planes_bf16 else torch.float32
        if depth > 1:
            return self._planes.get(planes if planes.dtype == torch.float32 else planes.float(), self.planes_bf16, depth)
        if planes.stride(2) == 1 and planes.dtype == want:
            return planes.permute(0, 1, 3, 4, 2)            # already channels-last texels: zero-copy view
        if planes.dtype != torch.float32:
            planes = planes.float()
        return self._planes.get(planes, self.planes_bf16)

    @staticmethod
    def _shape_probe(planes: torch.Tensor, opts) -> torch.Tensor:
        """A meta tensor with the shape of _planes_cl's result, for _params on the autograd paths."""
        N, _, CD, H, W = planes.shape
        D = _check_depth(planes, int(opts.get('triplane_depth', 1)))
        return torch.empty((N, 3, D, H, W, CD // D) if D > 1 else (N, 3, H, W, CD), device='meta')

    @staticmethod
    def _require_cuda(*tensors):
        for t in tensors:
            if t is not None and not t.is_cuda:
                raise RuntimeError('panic3d_b200.ImportanceRenderer has no CPU path: tensors must be on a CUDA device')

    def _get_workspace(self, nbytes: int, device):
        ws = self._workspace
        if ws is None or ws.numel() < nbytes or ws.device != device:
            self._workspace = ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        return ws

    # ------------------------------------------------------------------ forward
    def forward(self, planes, decoder, ray_origins, ray_directions, rendering_options,
                triplane_crop=None, cull_clouds=None, binarize_clouds=None):
        """-> rgb (N,M,32), depth (N,M,1), weights_sum (N,M,1), xyz (N,M,3).  Reference renderer.py:162-264."""
        self._require_cuda(planes, ray_origins, ray_directions)
        dev = planes.device
        self.plane_axes = self.plane_axes.to(dev)
        N, M, _ = ray_origins.shape
        if torch.is_grad_enabled() and (planes.requires_grad or any(q.requires_grad for q in decoder.parameters())):
            return self._forward_autograd(planes, decoder, ray_origins, ray_directions, rendering_options, triplane_crop,
                                          cull_clouds, binarize_clouds)
        with torch.cuda.device(dev):
            planes_cl = self._planes_cl(planes.detach(), int(rendering_options.get('triplane_depth', 1)))
            p, (w1, b1, w2, b2) = self._params(planes_cl, N, M, rendering_options, decoder, triplane_crop, cull_clouds,
                                               binarize_clouds)
            ro = ray_origins.detach().float().contiguous()
            rd = ray_directions.detach().float().contiguous()
            u_c = u_f = None
            if self.injected_noise is not None:
                u_c, u_f = self.injected_noise
                u_c = u_c.to(dev, torch.float32).contiguous()
                assert u_c.numel() == N * M * p.n_coarse, 'u_coarse shape'
                if p.n_fine > 0:
                    u_f = u_f.to(dev, torch.float32).contiguous()
                    assert u_f.numel() == N * M * p.n_fine, 'u_fine shape'
                else:
                    u_f = None
            rgb = torch.empty((N, M, p.out_dim - 1), device=dev, dtype=torch.float32)
            depth = torch.empty((N, M, 1), device=dev, dtype=torch.float32)
            wsum = torch.empty((N, M, 1), device=dev, dtype=torch.float32)
            xyz = torch.empty((N, M, 3), device=dev, dtype=torch.float32)
            L = _lib.lib()
            nbytes = int(L.p3d_render_workspace_bytes(C.byref(p)))
            ws = self._get_workspace(nbytes, dev)
            wt = [t.detach().float().contiguous() for t in (w1, b1, w2, b2)]
            p.defer_depth_clamp = 1 if self.depth_bounds_reduce is not None else 0
            _lib.check(L.p3d_render_forward(C.byref(p), planes_cl.data_ptr(), wt[0].data_ptr(), wt[1].data_ptr(),
                                            wt[2].data_ptr(), wt[3].data_ptr(), ro.data_ptr(), rd.data_ptr(),
                                            _lib.ptr(u_c), _lib.ptr(u_f), ws.data_ptr(), ws.numel(),
                                            rgb.data_ptr(), depth.data_ptr(), wsum.data_ptr(), xyz.data_ptr(),
                                            _lib.stream_ptr(dev)))
            if self.depth_bounds_reduce is not None:
                b2 = torch.empty(2, device=dev, dtype=torch.float32)
                _lib.check(L.p3d_render_depth_bounds(ws.data_ptr(), b2.data_ptr(), _lib.stream_ptr(dev)))
                self.depth_bounds_reduce(b2)
                _lib.check(L.p3d_depth_finalize(depth.data_ptr(), N * M, b2.data_ptr(), _lib.stream_ptr(dev)))
        return rgb, depth, wsum, xyz

    def _noise(self, dev, N, M, p):
        if self.injected_noise is None:
            return None, None
        u_c, u_f = self.injected_noise
        u_c = u_c.to(dev, torch.float32).contiguous()
        assert u_c.numel() == N * M * p.n_coarse, 'u_coarse shape'
        if p.n_fine > 0:
            u_f = u_f.to(dev, torch.float32).contiguous()
            assert u_f.numel() == N * M * p.n_fine, 'u_fine shape'
        else:
            u_f = None
        return u_c, u_f

    def _forward_autograd(self, planes, decoder, ray_origins, ray_directions, rendering_options, triplane_crop, cull_clouds,
                          binarize_clouds):
        dev = planes.device
        N, M, _ = ray_origins.shape
        if planes.dim() != 5 or planes.shape[1] != 3:
            raise ValueError(f'planes must be (N,3,C,H,W), got {tuple(planes.shape)}')
        with torch.cuda.device(dev):
            shape_probe = self._shape_probe(planes, rendering_options)
            p, (w1, b1, w2, b2) = self._params(shape_probe, N, M, rendering_options, decoder, triplane_crop, cull_clouds, binarize_clouds)
            p.defer_depth_clamp = 1 if self.depth_bounds_reduce is not None else 0
            return _RenderFunction.apply(self, planes, w1, b1, w2, b2, ray_origins, ray_directions, p, self._noise(dev, N, M, p))

    # ------------------------------------------------------------------ point queries
    def run_model(self, planes, decoder, sample_coordinates, sample_directions, options):
        """-> {'rgb' (N,K,32), 'sigma' (N,K,1), 'xyz'}.  Reference renderer.py:266-280."""
        self._require_cuda(planes, sample_coordinates)
        dev = planes.device
        N, K, _ = sample_coordinates.shape
        if torch.is_grad_enabled() and sample_coordinates.requires_grad:
            raise NotImplementedError('run_model: gradients w.r.t. the query coordinates are not implemented (no caller of the '
                                      'reference needs them; planes and decoder parameters are differentiable)')
        if torch.is_grad_enabled() and (planes.requires_grad or any(q.requires_grad for q in decoder.parameters())):
            if planes.dim() != 5 or planes.shape[1] != 3:
                raise ValueError(f'planes must be (N,3,C,H,W), got {tuple(planes.shape)}')
            with torch.cuda.device(dev):
                opts = dict(options)
                opts.setdefault('depth_resolution', 2)
                shape_probe = self._shape_probe(planes, opts)
                p, (w1, b1, w2, b2) = self._params(shape_probe, N, 0, opts, decoder, None, None, None)
                rgb, sigma = _PointsFunction.apply(planes, w1, b1, w2, b2, sample_coordinates, p)
            return {'rgb': rgb, 'sigma': sigma, 'xyz': sample_coordinates}
        with torch.cuda.device(dev):
            opts = dict(options)
            opts.setdefault('depth_resolution', 2)
            planes_cl = self._planes_cl(planes.detach(), int(opts.get('triplane_depth', 1)))
            p, (w1, b1, w2, b2) = self._params(planes_cl, N, 0, opts, decoder, None, None, None, n_points=N * K)
            coords = sample_coordinates.detach().float().contiguous()
            rgb = torch.empty((N, K, p.out_dim - 1), device=dev, dtype=torch.float32)
            sigma = torch.empty((N, K, 1), device=dev, dtype=torch.float32)
            wt = [t.detach().float().contiguous() for t in (w1, b1, w2, b2)]
            _lib.check(_lib.lib().p3d_decode_points(C.byref(p), planes_cl.data_ptr(), wt[0].data_ptr(), wt[1].data_ptr(),
                                                    wt[2].data_ptr(), wt[3].data_ptr(), coords.data_ptr(), K,
                                                    rgb.data_ptr(), sigma.data_ptr(), _lib.stream_ptr(dev)))
        return {'rgb': rgb, 'sigma': sigma, 'xyz': sample_coordinates}
