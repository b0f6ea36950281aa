"""CPU oracle for multiplane tri-planes (rendering_kwargs['triplane_depth'] = D > 1).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle/``: the product package never imports it.

What it restates (paths relative to ``/root/reference/_train/eg3dc/src/training``):

* ``plane_coords3``      <- volumetric_rendering/renderer.py:26-66 (all three components of project_onto_planes)
* ``sample_multiplane``  <- volumetric_rendering/renderer.py:84-94 (the ``triplane_depth > 1`` branch of
                            sample_from_planes: a trilinear 5-D grid_sample over (C, D, H, W), zero padding,
                            align_corners=False)
* ``render``, ``run_model`` and ``volume``: renderer_oracle.render / run_model and volume_oracle.volume with the plane
  lookup replaced by ``sample_multiplane``.  Everything else of those functions (stratified and importance sampling,
  decoder, masks, marcher, the volume lattice) is unchanged by the reference's multiplane branch.

``sampling(depth)`` is that replacement: inside it, ``renderer_oracle.sample_planes`` - the one place where the renderer
oracle reads the planes - samples (N, 3, C*depth, H, W) multiplane planes.  Pinned against the unmodified reference by
tests/golden/multiplane_*.npz (tests/golden/make_golden_multiplane.py, tests/test_multiplane_cpu.py).
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from oracle import renderer_oracle as orc

Tensor = torch.Tensor


def plane_coords3(xyz: Tensor, use_triplane: bool) -> Tensor:
    """xyz @ inv(plane_axes[p]) for each plane of generate_planes (renderer.py:26-66).  (N,K,3) -> (N,3,K,3): [..., 0] and
    [..., 1] index W and H as in the one-slab case, [..., 2] indexes the slabs."""
    third = [[0, 1, 0], [0, 0, 1], [1, 0, 0]] if use_triplane else [[0, 0, 1], [1, 0, 0], [0, 1, 0]]
    axes = torch.tensor([[[1, 0, 0], [0, 1, 0], [0, 0, 1]], [[1, 0, 0], [0, 0, 1], [0, 1, 0]], third],
                        dtype=xyz.dtype, device=xyz.device)
    return torch.stack([xyz @ torch.linalg.inv(axes[p]) for p in range(3)], dim=1)


def _trilinear_zero_pad(vol: Tensor, gx: Tensor, gy: Tensor, gz: Tensor) -> Tensor:
    """vol (C,D,H,W); gx, gy, gz (K,) normalised coordinates of W, H and D, align_corners=False, zero padding on all three
    axes.  Returns (K,C).  Independent restatement of the 5-D F.grid_sample."""
    C, D, H, W = vol.shape
    fx, fy, fz = ((gx + 1) * W - 1) * 0.5, ((gy + 1) * H - 1) * 0.5, ((gz + 1) * D - 1) * 0.5
    x0f, y0f, z0f = torch.floor(fx), torch.floor(fy), torch.floor(fz)
    wx1, wy1, wz1 = fx - x0f, fy - y0f, fz - z0f
    x0, y0, z0 = x0f.long(), y0f.long(), z0f.long()
    flat = vol.reshape(C, D * H * W)
    out = torch.zeros(gx.shape[0], C, dtype=vol.dtype, device=vol.device)
    for dz, wz in ((0, 1 - wz1), (1, wz1)):
        for dy, wy in ((0, 1 - wy1), (1, wy1)):
            for dx, wx in ((0, 1 - wx1), (1, wx1)):
                xi, yi, zi = x0 + dx, y0 + dy, z0 + dz
                ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H) & (zi >= 0) & (zi < D)
                lin = (zi.clamp(0, D - 1) * H + yi.clamp(0, H - 1)) * W + xi.clamp(0, W - 1)
                out += flat[:, lin].t() * (wx * wy * wz * ok.to(vol.dtype))[:, None]
    return out


def sample_multiplane(planes: Tensor, xyz: Tensor, box_warp: float, use_triplane: bool, depth: int,
                      gather: str = 'manual') -> Tensor:
    """renderer.py:84-94.  planes (N,3,C*depth,H,W): channel c*depth + d is feature c of slab d.  xyz (N,K,3) ->
    (N,3,K,C).  gather='aten' runs the reference's own 5-D F.grid_sample instead of the restatement."""
    N, P, CD, H, W = planes.shape
    C = CD // depth
    vol = planes.reshape(N, P, C, depth, H, W)
    grid = plane_coords3((2.0 / box_warp) * xyz, use_triplane)      # N,3,K,3: (W, H, D) coordinates
    if gather == 'aten':
        o = F.grid_sample(vol.reshape(N * P, C, depth, H, W), grid.reshape(N * P, 1, 1, -1, 3), mode='bilinear',
                          padding_mode='zeros', align_corners=False)
        return o.permute(0, 4, 3, 2, 1).reshape(N, P, -1, C)
    out = torch.empty(N, P, xyz.shape[1], C, dtype=planes.dtype, device=planes.device)
    for n in range(N):
        for p in range(P):
            out[n, p] = _trilinear_zero_pad(vol[n, p], grid[n, p, :, 0], grid[n, p, :, 1], grid[n, p, :, 2])
    return out


@contextlib.contextmanager
def sampling(depth: int):
    """Within the block, renderer_oracle (and volume_oracle, which samples through it) reads planes as multiplane planes of
    `depth` slabs.  Not thread-safe: it rebinds a module attribute for the block's duration."""
    one_slab = orc.sample_planes

    def multiplane(planes, xyz, box_warp, use_triplane, gather='manual'):
        return sample_multiplane(planes, xyz, box_warp, use_triplane, depth, gather)
    orc.sample_planes = multiplane
    try:
        yield
    finally:
        orc.sample_planes = one_slab


def render(planes: Tensor, dec, ro: Tensor, rd: Tensor, opts, *args, **kwargs):
    """renderer_oracle.render for planes of opts['triplane_depth'] slabs (renderer.py:162-264 with :84-94)."""
    with sampling(int(opts['triplane_depth'])):
        return orc.render(planes, dec, ro, rd, opts, *args, **kwargs)


def run_model(planes: Tensor, dec, xyz: Tensor, opts, use_triplane: bool, gather: str = 'manual'):
    """renderer_oracle.run_model for planes of opts['triplane_depth'] slabs (renderer.py:266-280 with :84-94)."""
    with sampling(int(opts['triplane_depth'])):
        return orc.run_model(planes, dec, xyz, opts, use_triplane, gather)


def volume(planes: Tensor, dec, opts, resolution: int, **kwargs):
    """volume_oracle.volume for planes of opts['triplane_depth'] slabs (eg3d_metrics3d.py:114-183)."""
    from oracle import volume_oracle
    with sampling(int(opts['triplane_depth'])):
        return volume_oracle.volume(planes, dec, opts, resolution, **kwargs)
