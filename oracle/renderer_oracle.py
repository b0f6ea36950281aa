"""CPU oracle for the tri-plane volumetric renderer hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is product code: only
``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl
reference`` legs of ``bench.py`` may import it, and there only as the checker
(or as the timed CPU baseline), never as the thing shipped.  The product path
(``panic3d_b200``) never imports this module and has no CPU fallback.

What it is: a plain torch-CPU fp32 restatement of the reference algorithm
(paths relative to ``/root/reference/_train/eg3dc/src/training``):

* ``ray_sampler``            <- volumetric_rendering/ray_sampler.py:24-63
* ``rays_ortho``             <- /root/reference/_databacks/lustrous_renders_v1.py:78-104
* ``stratified_depths``      <- volumetric_rendering/renderer.py:303-326
* ``plane_coords``           <- volumetric_rendering/renderer.py:26-66 (generate_planes + project_onto_planes)
* ``sample_planes``          <- volumetric_rendering/renderer.py:68-81
* ``decode``                 <- triplane.py:528-544, networks_stylegan2.py:120-133
* ``crop_mask/cull_mask``    <- volumetric_rendering/renderer.py:138-153
* ``march``                  <- volumetric_rendering/ray_marcher.py:25-57
* ``importance_depths``      <- volumetric_rendering/renderer.py:328-387
* ``render``                 <- volumetric_rendering/renderer.py:162-264
* ``run_model``              <- volumetric_rendering/renderer.py:266-280

Randomness is explicit: every function that the reference feeds from
``torch.rand_like`` / ``torch.rand`` takes the uniform noise as an argument, so
the same numbers can be injected into the reference (tests/golden/make_golden.py
patches ``torch.rand*``), into this oracle and into the CUDA kernels.

Pinning status: PINNED.  The reference ships no tests or golden vectors
(SURVEY.md section 4), so the pins are outputs of the reference itself, imported and
run in the build container by ``tests/golden/make_golden.py`` and committed as
``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks this file against
every one of them.

Two gather implementations are provided: ``gather='manual'`` (independent
restatement of bilinear/zero-pad/align_corners=False, the one parity tests use)
and ``gather='aten'`` (``F.grid_sample`` - the same ATen op the reference calls,
used when this oracle is *timed* as the CPU baseline so the baseline is not
handicapped by a slow Python gather).

The decode path (``sample_planes``, ``decode``, ``run_model``) allocates on the device and in the dtype of its inputs, so
the GPU tests run it in fp64 on the device at sizes the CPU could not reach in time (tests/test_decode_tc_depth_gpu.py,
which pins that run to this CPU fp32 one).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


# --------------------------------------------------------------------------
# rays
# --------------------------------------------------------------------------
def ray_sampler(cam2world: Tensor, intrinsics: Tensor, resolution: int) -> Tuple[Tensor, Tensor]:
    """Pinhole rays through pixel centres. ray_sampler.py:24-63.

    Pixel m = row*R + col; u = (col+.5)/R is x, v = (row+.5)/R is y (the
    reference's meshgrid('ij') + flip(0) makes x the fastest-varying index).
    """
    N = cam2world.shape[0]
    R = int(resolution)
    dev = cam2world.device
    fx, fy = intrinsics[:, 0, 0], intrinsics[:, 1, 1]
    cx, cy = intrinsics[:, 0, 2], intrinsics[:, 1, 2]
    sk = intrinsics[:, 0, 1]
    idx = torch.arange(R, dtype=torch.float32, device=dev) * (1.0 / R) + (0.5 / R)
    x_cam = idx.repeat(R)[None].expand(N, -1)               # col fastest
    y_cam = idx.repeat_interleave(R)[None].expand(N, -1)    # row slowest
    fx, fy, cx, cy, sk = (t[:, None] for t in (fx, fy, cx, cy, sk))
    x_lift = (x_cam - cx + cy * sk / fy - sk * y_cam / fy) / fx
    y_lift = (y_cam - cy) / fy
    ones = torch.ones_like(x_lift)
    pts = torch.stack((x_lift, y_lift, ones, ones), dim=-1)             # N,M,4
    world = torch.bmm(cam2world, pts.permute(0, 2, 1)).permute(0, 2, 1)[:, :, :3]
    origin = cam2world[:, :3, 3]
    dirs = F.normalize(world - origin[:, None, :], dim=2)
    return origin[:, None, :].expand(-1, R * R, -1).contiguous(), dirs


def euler_xyz_matrix(ax_deg: float, ay_deg: float, az_deg: float) -> Tensor:
    """scipy Rotation.from_euler('xyz', [ax,ay,az], degrees=True).as_matrix():
    extrinsic rotations about x, then y, then z  ==>  R = Rz @ Ry @ Rx."""
    ax, ay, az = (math.radians(a) for a in (ax_deg, ay_deg, az_deg))
    cx_, sx_ = math.cos(ax), math.sin(ax)
    cy_, sy_ = math.cos(ay), math.sin(ay)
    cz_, sz_ = math.cos(az), math.sin(az)
    Rx = torch.tensor([[1, 0, 0], [0, cx_, -sx_], [0, sx_, cx_]], dtype=torch.float64)
    Ry = torch.tensor([[cy_, 0, sy_], [0, 1, 0], [-sy_, 0, cy_]], dtype=torch.float64)
    Rz = torch.tensor([[cz_, -sz_, 0], [sz_, cz_, 0], [0, 0, 1]], dtype=torch.float64)
    return Rz @ Ry @ Rx


def camera_params_to_matrix(elev: float, azim: float, dist: float, fov: float) -> Tuple[Tensor, Tensor]:
    """'eg3d_lustrousB' camera. lustrous_renders_v1.py:33-75. Returns (cam2world 4x4, K 3x3)."""
    focal = 0.5 / math.tan((fov / 2) * math.pi / 180)
    K = torch.tensor([[focal, 0, 0.5], [0, focal, 0.5], [0, 0, 1]], dtype=torch.float32)
    R = torch.eye(4, dtype=torch.float64)
    R[:3, :3] = euler_xyz_matrix(elev, azim, 0.0).T
    R[[0, 2]] *= -1
    R[2, -1] = -dist
    A = torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0], dtype=torch.float64))
    B = torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0], dtype=torch.float64))
    extr = A @ torch.linalg.inv(R) @ B
    return extr.float(), K


def rays_ortho(elev: float, azim: float, dist: float, boxwarp: float, resolution: int) -> Tuple[Tensor, Tensor]:
    """Orthographic rays over the box_warp square. lustrous_renders_v1.py:78-104.
    Returns (origins, dirs) each (1, 3, R, R) like the reference's force_rays."""
    r, bw = int(resolution), float(boxwarp)
    lin = (torch.arange(r, dtype=torch.float32) + 0.5) / r * bw - bw / 2
    gx = lin[None, :].expand(r, r)           # x varies along columns
    gy = (-lin)[:, None].expand(r, r)        # y varies along rows, flipped
    gz = torch.zeros(r, r)
    p0 = torch.stack([gx, gy, gz + dist])
    p1 = torch.stack([gx, gy, gz - 1.0 + dist])
    rot = euler_xyz_matrix(-elev, azim, 0.0).float()
    t0 = torch.einsum('ij,jhw->ihw', rot, p0)
    t1 = torch.einsum('ij,jhw->ihw', rot, p1)
    return t0[None], (t1 - t0)[None]


# --------------------------------------------------------------------------
# sampling along rays
# --------------------------------------------------------------------------
def stratified_depths(u: Tensor, ray_start, ray_end, disparity: bool = False) -> Tensor:
    """renderer.py:303-326.  u: (N,M,S,1) uniform [0,1)."""
    N, M, S, _ = u.shape
    if disparity:
        t = torch.linspace(0, 1, S, dtype=u.dtype, device=u.device).reshape(1, 1, S, 1) + u * (1.0 / (S - 1))
        return 1.0 / (1.0 / ray_start * (1.0 - t) + 1.0 / ray_end * t)
    if isinstance(ray_start, torch.Tensor):          # per-ray limits ('auto' mode)
        steps = (torch.arange(S, dtype=u.dtype, device=u.device) / (S - 1)).reshape(1, 1, S, 1)
        base = ray_start[:, :, None, :] + steps * (ray_end - ray_start)[:, :, None, :]
        delta = (ray_end - ray_start) / (S - 1)
        return base + u * delta[..., None]
    base = torch.linspace(ray_start, ray_end, S, dtype=u.dtype, device=u.device).reshape(1, 1, S, 1)
    return base + u * ((ray_end - ray_start) / (S - 1))


def ray_limits_box(ro: Tensor, rd: Tensor, box_side: float) -> Tuple[Tensor, Tensor]:
    """Slab-test ray/AABB limits. math_utils.py:46-98. (N,M,1) each; (-1,-2) when missed."""
    shape = ro.shape
    o, d = ro.reshape(-1, 3), rd.reshape(-1, 3)
    h = box_side / 2
    inv = 1 / d
    neg = inv < 0
    lo = torch.where(neg, torch.full_like(o, h), torch.full_like(o, -h))
    hi = torch.where(neg, torch.full_like(o, -h), torch.full_like(o, h))
    t0 = (lo - o) * inv
    t1 = (hi - o) * inv
    tmin, tmax = t0[:, 0], t1[:, 0]
    valid = ~((tmin > t1[:, 1]) | (t0[:, 1] > tmax))
    tmin, tmax = torch.max(tmin, t0[:, 1]), torch.min(tmax, t1[:, 1])
    valid &= ~((tmin > t1[:, 2]) | (t0[:, 2] > tmax))
    tmin, tmax = torch.max(tmin, t0[:, 2]), torch.min(tmax, t1[:, 2])
    tmin = torch.where(valid, tmin, torch.full_like(tmin, -1))
    tmax = torch.where(valid, tmax, torch.full_like(tmax, -2))
    return tmin.reshape(*shape[:-1], 1), tmax.reshape(*shape[:-1], 1)


# --------------------------------------------------------------------------
# tri-plane lookup
# --------------------------------------------------------------------------
def plane_coords(xyz: Tensor, use_triplane: bool) -> Tensor:
    """Which two world components each plane reads. renderer.py:26-66.

    ``project_onto_planes`` right-multiplies the coordinates by inv(plane_axes)
    and ``sample_from_planes`` keeps ``[..., :2]``.  For the permutation matrices
    of ``generate_planes`` that selects (x,y) for plane 0, (x,z) for plane 1 and
    (y,z) for plane 2 when ``use_triplane`` (panic3d) or (z,x) otherwise (EG3D
    default).  Returned (N,3,K,2): [..., 0] is the grid x (width/column)
    coordinate, [..., 1] the grid y (height/row) coordinate.  The third plane is
    derived numerically from the axis matrix so both variants stay faithful.
    """
    x, y, z = xyz[..., 0], xyz[..., 1], xyz[..., 2]
    p0 = torch.stack([x, y], -1)
    p1 = torch.stack([x, z], -1)
    return torch.stack([p0, p1, _third_plane(xyz, use_triplane)], dim=1)


def _third_plane(xyz: Tensor, use_triplane: bool) -> Tensor:
    axes = torch.tensor([[0, 1, 0], [0, 0, 1], [1, 0, 0]] if use_triplane else
                        [[0, 0, 1], [1, 0, 0], [0, 1, 0]], dtype=xyz.dtype, device=xyz.device)
    inv = torch.linalg.inv(axes)
    return (xyz @ inv)[..., :2]


def _bilinear_zero_pad(plane: Tensor, gx: Tensor, gy: Tensor) -> Tensor:
    """plane (C,H,W); gx,gy (K,) normalised [-1,1] grid coords, align_corners=False,
    zero padding.  Returns (K,C).  Independent restatement of F.grid_sample."""
    C, H, W = plane.shape
    fx = ((gx + 1) * W - 1) * 0.5
    fy = ((gy + 1) * H - 1) * 0.5
    x0f, y0f = torch.floor(fx), torch.floor(fy)
    wx1, wy1 = fx - x0f, fy - y0f
    wx0, wy0 = 1 - wx1, 1 - wy1
    x0, y0 = x0f.long(), y0f.long()
    flat = plane.reshape(C, H * W)
    out = torch.zeros(gx.shape[0], C, dtype=plane.dtype, device=plane.device)
    for dy, wy in ((0, wy0), (1, wy1)):
        for dx, wx in ((0, wx0), (1, wx1)):
            xi, yi = x0 + dx, y0 + dy
            ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
            lin = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1))
            tap = flat[:, lin].t()                                  # K,C
            out += tap * (wx * wy * ok.to(plane.dtype))[:, None]
    return out


def sample_planes(planes: Tensor, xyz: Tensor, box_warp: float, use_triplane: bool,
                  gather: str = 'manual') -> Tensor:
    """renderer.py:68-81.  planes (N,3,C,H,W), xyz (N,K,3) -> (N,3,K,C)."""
    N, P, C, H, W = planes.shape
    grid = plane_coords((2.0 / box_warp) * xyz, use_triplane)       # N,3,K,2
    if gather == 'aten':
        g = grid.reshape(N * P, 1, -1, 2)
        o = F.grid_sample(planes.reshape(N * P, C, H, W), g, mode='bilinear',
                          padding_mode='zeros', align_corners=False)
        return o.permute(0, 3, 2, 1).reshape(N, P, -1, C)
    out = torch.empty(N, P, xyz.shape[1], C, dtype=planes.dtype, device=planes.device)
    for n in range(N):
        for p in range(P):
            out[n, p] = _bilinear_zero_pad(planes[n, p], grid[n, p, :, 0], grid[n, p, :, 1])
    return out


# --------------------------------------------------------------------------
# decoder
# --------------------------------------------------------------------------
def decode(feat: Tensor, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor,
           lr_mul: float = 1.0, force_sigmoid: bool = False) -> Tuple[Tensor, Tensor]:
    """OSGDecoder.forward, triplane.py:528-544 with FullyConnectedLayer
    (networks_stylegan2.py:120-133): weight_gain = lr_mul/sqrt(in), bias_gain = lr_mul.
    feat (N,3,K,C) -> rgb (N,K,32), sigma (N,K,1)."""
    x = feat.mean(1)
    N, K, C = x.shape
    x = x.reshape(N * K, C)
    g1 = lr_mul / math.sqrt(w1.shape[1])
    g2 = lr_mul / math.sqrt(w2.shape[1])
    h = F.softplus(torch.addmm((b1 * lr_mul)[None], x, (w1 * g1).t()))
    o = torch.addmm((b2 * lr_mul)[None], h, (w2 * g2).t()).reshape(N, K, -1)
    rgb = torch.sigmoid(o[..., 1:])
    if not force_sigmoid:
        rgb = rgb * (1 + 2 * 0.001) - 0.001
    return rgb, o[..., 0:1]


def crop_mask(xyz: Tensor, thresh: float, box_warp: float) -> Tensor:
    """True where sigma must be forced to -1e3. renderer.py:138-149 (the
    allow_bottom clause ORs in a subset of the first clause, so it is a no-op)."""
    lim = box_warp / 2 - thresh
    inside = (xyz[:, :, [0, 2]].abs() <= lim).all(dim=-1, keepdim=True)
    return ~inside


def cull_mask(sigma: Tensor, thresh: float) -> Tensor:
    """renderer.py:150-153."""
    return (1 - torch.exp(-F.softplus(sigma - 1))) < thresh


def apply_masks(sigma: Tensor, xyz: Tensor, box_warp: float, triplane_crop, cull_clouds, binarize_clouds,
                mask: Optional[Tensor] = None) -> Tensor:
    """renderer.py:187-198 / :227-238 (order: crop, then binarize XOR cull).  `mask` (bool, like sigma), when given, replaces
    the decision: True where the density is forced to -1e3; under binarize every other density is forced to 1e3."""
    sigma = sigma.clone()
    if mask is not None:
        if triplane_crop or cull_clouds or binarize_clouds:
            sigma[mask] = -1e3
            if binarize_clouds:
                sigma[~mask] = 1e3
        return sigma
    if triplane_crop:
        sigma[crop_mask(xyz, triplane_crop, box_warp)] = -1e3
    if binarize_clouds:
        m = cull_mask(sigma, binarize_clouds)
        sigma[m] = -1e3
        sigma[~m] = 1e3
    elif cull_clouds:
        sigma[cull_mask(sigma, cull_clouds)] = -1e3
    return sigma


# --------------------------------------------------------------------------
# compositing
# --------------------------------------------------------------------------
def march(colors: Tensor, sigma: Tensor, depths: Tensor, white_back: bool,
          depth_lo: Optional[Tensor] = None, depth_hi: Optional[Tensor] = None,
          alpha_eps: Optional[Tensor] = None, left_colours: bool = False
          ) -> Tuple[Tensor, Tensor, Tensor]:
    """MipRayMarcher2.run_forward, ray_marcher.py:25-57.
    colors (N,M,S,Cc), sigma (N,M,S,1), depths (N,M,S,1), depth sorted along S.

    For tests only: `alpha_eps` (N,M,S-1,1) is added to every interval's alpha (a perturbation to differentiate against;
    adding zeros changes nothing), and `left_colours` weights each interval by its first sample's colour instead of the
    mean of its two (a deliberately wrong variant for negative controls)."""
    delta = depths[:, :, 1:] - depths[:, :, :-1]
    c_mid = colors[:, :, :-1] if left_colours else (colors[:, :, :-1] + colors[:, :, 1:]) / 2
    s_mid = F.softplus((sigma[:, :, :-1] + sigma[:, :, 1:]) / 2 - 1)
    d_mid = (depths[:, :, :-1] + depths[:, :, 1:]) / 2
    alpha = 1 - torch.exp(-(s_mid * delta))
    if alpha_eps is not None:
        alpha = alpha + alpha_eps
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :, :1]), 1 - alpha + 1e-10], -2), -2)[:, :, :-1]
    w = alpha * trans
    rgb = (w * c_mid).sum(-2)
    wsum = w.sum(2)
    depth = (w * d_mid).sum(-2) / wsum
    depth = torch.nan_to_num(depth, float('inf'))
    lo = depths.min() if depth_lo is None else depth_lo
    hi = depths.max() if depth_hi is None else depth_hi
    depth = torch.clamp(depth, lo, hi)
    if white_back:
        rgb = rgb + 1 - wsum
    return rgb * 2 - 1, depth, w


def importance_depths(z: Tensor, w: Tensor, u: Tensor, eps: float = 1e-5, floor: float = 0.01,
                      cdf_eps: Optional[Tensor] = None) -> Tensor:
    """sample_importance + sample_pdf, renderer.py:328-387.
    z (R,S) coarse depths, w (R,S-1) coarse weights, u (R,Sf) uniforms -> (R,Sf).

    For tests only: `floor` is the pdf floor the reference adds (0.01), and `cdf_eps` (R,S-2) is added to the cdf (a
    perturbation to differentiate against; adding zeros changes nothing)."""
    R, S = z.shape
    wp = F.max_pool1d(w[:, None, :], 2, 1, padding=1)          # R,1,S
    wp = F.avg_pool1d(wp, 2, 1)[:, 0] + floor                  # R,S-1
    bins = 0.5 * (z[:, :-1] + z[:, 1:])                        # R,S-1
    wi = wp[:, 1:-1] + eps                                     # R,S-3
    pdf = wi / wi.sum(-1, keepdim=True)
    cdf = torch.cat([torch.zeros(R, 1, dtype=pdf.dtype, device=pdf.device), torch.cumsum(pdf, -1)], -1)   # R,S-2
    if cdf_eps is not None:
        cdf = cdf + cdf_eps
    nb = wi.shape[1]
    inds = torch.searchsorted(cdf, u.contiguous(), right=True)
    below = (inds - 1).clamp_min(0)
    above = inds.clamp_max(nb)
    c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    b0, b1 = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    den = c1 - c0
    den = torch.where(den < eps, torch.ones_like(den), den)
    return b0 + (u - c0) / den * (b1 - b0)


# --------------------------------------------------------------------------
# the renderer
# --------------------------------------------------------------------------
def run_model(planes, dec, xyz, opts, use_triplane, gather='manual'):
    """renderer.py:266-280 (density_noise not restated: off in every panic3d config)."""
    feat = sample_planes(planes, xyz, opts['box_warp'], use_triplane, gather)
    rgb, sigma = decode(feat, dec['w1'], dec['b1'], dec['w2'], dec['b2'],
                        dec.get('lr_mul', 1.0), dec.get('force_sigmoid', False))
    return rgb, sigma


def render(planes: Tensor, dec: Dict, ro: Tensor, rd: Tensor, opts: Dict,
           u_coarse: Tensor, u_fine: Optional[Tensor], use_triplane: bool = True,
           triplane_crop=None, cull_clouds=None, binarize_clouds=None,
           gather: str = 'manual', depth_bounds: Optional[Tuple[Tensor, Tensor]] = None, return_bounds: bool = False,
           depths: Optional[Tuple[Tensor, Optional[Tensor]]] = None, masks: Optional[Tuple[Tensor, Optional[Tensor]]] = None,
           return_samples: bool = False):
    """ImportanceRenderer.forward, renderer.py:162-264.
    Returns rgb (N,M,32), depth (N,M,1), wsum (N,M,1), xyz (N,M,3).

    `depths` = (coarse (N,M,S,1), fine (N,M,Sf,1) or None) and `masks` = (coarse (N,M*S,1), fine (N,M*Sf,1) or None, bool:
    True where apply_masks forced the density to -1e3) replace the ones render would compute.  Both are constants of the
    reference graph (the fine depths come from no_grad, the masks are in-place overwrites), so injecting another run's
    values - a kernel's fp32 ones into an fp64 run - changes no derivative, only which samples exist and which are masked.
    return_samples appends dict(depths=..., masks=...) of this run, in the form these arguments take."""
    N, M, _ = ro.shape
    S = int(opts['depth_resolution'])
    Sf = int(opts['depth_resolution_importance'])
    bw = opts['box_warp']
    white = bool(opts.get('white_back', False))
    if depths is not None:
        d_c = depths[0]
    elif opts['ray_start'] == 'auto' and opts['ray_end'] == 'auto':
        t0, t1 = ray_limits_box(ro, rd, bw)
        ok = t1 > t0
        if bool(ok.any()):
            t0 = torch.where(ok, t0, t0[ok].min())
            t1 = torch.where(ok, t1, t0[ok].max())   # sic: reference uses ray_start max (renderer.py:170)
        d_c = stratified_depths(u_coarse, t0, t1, opts.get('disparity_space_sampling', False))
    else:
        d_c = stratified_depths(u_coarse, opts['ray_start'], opts['ray_end'],
                                opts.get('disparity_space_sampling', False))
    lo, hi = (None, None) if depth_bounds is None else depth_bounds
    m_c, m_f = (None, None) if masks is None else masks
    flags = (triplane_crop, cull_clouds, binarize_clouds)

    xyz_c = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)
    rgb_c, sig_c = run_model(planes, dec, xyz_c, opts, use_triplane, gather)
    sig_c = apply_masks(sig_c, xyz_c, bw, *flags, mask=m_c)
    rgb_c = rgb_c.reshape(N, M, S, -1)
    sig_c = sig_c.reshape(N, M, S, 1)
    xyz_c = xyz_c.reshape(N, M, S, 3)
    if Sf > 0:
        _, _, w = march(rgb_c, sig_c, d_c, white, lo, hi)
        if depths is not None:
            d_f = depths[1]
        else:
            d_f = importance_depths(d_c.reshape(N * M, S), w.reshape(N * M, S - 1), u_fine).reshape(N, M, Sf, 1).detach()   # no_grad in the reference (renderer.py:332)
        xyz_f = (ro[:, :, None] + d_f * rd[:, :, None]).reshape(N, -1, 3)
        rgb_f, sig_f = run_model(planes, dec, xyz_f, opts, use_triplane, gather)
        sig_f = apply_masks(sig_f, xyz_f, bw, *flags, mask=m_f)
        d_all = torch.cat([d_c, d_f], -2)
        order = torch.sort(d_all, dim=-2, stable=True)[1]
        d_all = torch.gather(d_all, -2, order)
        col = torch.cat([torch.cat([rgb_c, xyz_c], -1),
                         torch.cat([rgb_f.reshape(N, M, Sf, -1), xyz_f.reshape(N, M, Sf, 3)], -1)], -2)
        col = torch.gather(col, -2, order.expand(-1, -1, -1, col.shape[-1]))
        sig = torch.gather(torch.cat([sig_c, sig_f.reshape(N, M, Sf, 1)], -2), -2, order)
    else:
        d_all, col, sig = d_c, torch.cat([rgb_c, xyz_c], -1), sig_c
    out, depth, w = march(col, sig, d_all, white, lo, hi)
    res = (out[..., :-3], depth, w.sum(2), out[..., -3:])
    extra = []
    if return_bounds:          # (min, max) over every depth of this batch: what ray_marcher.py:50 clamps to
        extra.append((d_all.min(), d_all.max()))
    if return_samples:
        extra.append(dict(depths=(d_c, d_f if Sf > 0 else None),
                          masks=(sig_c.reshape(N, -1, 1) == -1e3, sig_f == -1e3 if Sf > 0 else None)))
    return (res, *extra) if extra else res


# --------------------------------------------------------------------------
# deterministic synthetic inputs shared by golden generation, tests and bench
# --------------------------------------------------------------------------
def synth_inputs(seed: int, N: int, R: int, S: int, Sf: int, P: int, C: int = 32,
                 hidden: int = 64, out_dim: int = 33, cameras=None, share_planes: bool = False):
    """numpy-PCG64 seeded inputs (bit-identical on every box with this image)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    n_pl = 1 if share_planes else N
    planes = torch.from_numpy(rng.standard_normal((n_pl, 3, C, P, P), dtype=np.float32))
    if share_planes:
        planes = planes.expand(N, -1, -1, -1, -1)
    dec = dict(w1=torch.from_numpy(rng.standard_normal((hidden, C), dtype=np.float32)),
               b1=torch.from_numpy(0.1 * rng.standard_normal((hidden,), dtype=np.float32)),
               w2=torch.from_numpy(rng.standard_normal((out_dim, hidden), dtype=np.float32)),
               b2=torch.from_numpy(0.1 * rng.standard_normal((out_dim,), dtype=np.float32)),
               lr_mul=1.0, force_sigmoid=False)
    u_c = torch.from_numpy(rng.random((N, R * R, S, 1), dtype=np.float32))
    u_f = torch.from_numpy(rng.random((N * R * R, max(Sf, 1)), dtype=np.float32))[:, :Sf]
    if cameras is None:
        cameras = [(0.0, -180.0 + 30.0 * (i % 12), 1.0, 30.0) for i in range(N)]
    c2w, K = zip(*(camera_params_to_matrix(*c) for c in cameras))
    return planes, dec, torch.stack(c2w), torch.stack(K), u_c, u_f


DEFAULT_OPTS = dict(box_warp=0.7, ray_start=0.5, ray_end=1.5, depth_resolution=96,
                    depth_resolution_importance=96, disparity_space_sampling=False,
                    clamp_mode='softplus', white_back=True, triplane_depth=1)
