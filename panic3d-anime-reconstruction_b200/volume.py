"""Dense sigma / colour volume for mesh extraction - the H100 replacement for ``get_eg3d_volume``
(reference ``_util/eg3d_metrics3d.py:94-183``; SURVEY.md section 8f-2).

The reference evaluates resolution^3 = 16.8 M grid points as 168 host-side chunks of 100k: every chunk re-runs the
StyleGAN2 backbone inside ``G.sample_mixed`` (``triplane.py:273-298``), goes through ``ImportanceRenderer.run_model``
and ends with a ``.cpu()`` copy.  Here the tri-planes are synthesised once and one launch of ``p3d_volume_query``
(include/p3d_render.h) generates the reference's ``create_samples`` lattice in-kernel (bit for bit, including its
un-floored float y/x indices), gathers, decodes and writes sigma / rgb / density / coordinates directly in the layout
the reference returns (``reshape(R,R,R,.)`` -> ``flip(dims=(1,))`` -> channels first), so nothing is re-shuffled.

    ``create_samples``, ``sigma2density``     same call surface as the reference helpers (eg3d_metrics3d.py:65-92)
    ``query_volume``                           planes + decoder -> {'coordinates','sigmas','rgbs','densities'}
    ``get_eg3d_volume``                        drop-in for the reference function on a TriPlaneGenerator-like ``G``

No CPU path: tensors must live on a CUDA device (the PyTorch restatement is ``oracle/volume_oracle.py``, tests only).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


def sigma2density(sigma):
    """``1 - exp(-softplus(sigma - 1))``.  Reference eg3d_metrics3d.py:65-69."""
    return 1 - torch.exp(-torch.nn.functional.softplus(sigma - 1))


def create_samples(N=256, voxel_origin=(0, 0, 0), cube_length=2.0):
    """The reference lattice (eg3d_metrics3d.py:70-92) as a (1, N^3, 3) fp32 CPU tensor + (corner, voxel size).

    Point n has z index n % N (integer) but its y and x "indices" are the un-floored fp32 quotients
    (n / N) mod N and ((n / N) / N) mod N, so the lattice is sheared by a fraction of a voxel; each index is then
    scaled by the voxel size and shifted to the cube corner in fp32.  Same values as the reference, bit for bit
    (pinned by tests/test_volume_oracle_golden.py); ``p3d_volume_query`` generates the same points in-kernel."""
    corner = np.asarray(voxel_origin, dtype=np.float64) - cube_length / 2
    step = cube_length / (N - 1)
    n = torch.arange(N ** 3, dtype=torch.int64)
    row = n.to(torch.float32) / N                                   # fp32 quotient, never floored
    index = torch.stack([torch.remainder(row / N, N), torch.remainder(row, N), torch.remainder(n, N).to(torch.float32)], dim=-1)
    shift = torch.tensor([float(corner[2]), float(corner[1]), float(corner[0])], dtype=torch.float32)
    return (index * step + shift).unsqueeze(0), corner, step


def query_volume(planes, decoder, rendering_kwargs, resolution=256, triplane_crop=None, cull_clouds=None,
                 renderer=None, want_rgb=True, want_coordinates=True):
    """planes (N,3,32,H,W) + OSGDecoder -> dict of (N,1|32|3,R,R,R) tensors shaped, ordered and flipped exactly as
    ``get_eg3d_volume`` returns them (``coordinates``, ``sigmas``, ``rgbs``, ``densities``).

    ``renderer`` (an ``ImportanceRenderer``) supplies plane mode / storage / layout cache; a fresh one
    (``use_triplane=True``) is used when omitted.  ``want_rgb`` / ``want_coordinates`` = False skip the 2.1 GB / 0.2 GB
    outputs marching cubes never reads."""
    from .training.volumetric_rendering.renderer import ImportanceRenderer
    if not planes.is_cuda:
        raise RuntimeError('panic3d_b200.volume.query_volume has no CPU path: tensors must be on a CUDA device')
    r = renderer if renderer is not None else ImportanceRenderer(use_triplane=True)
    dev = planes.device
    N, R = planes.shape[0], int(resolution)
    with torch.no_grad(), torch.cuda.device(dev):
        planes_cl = r._planes_cl(planes.detach(), int(rendering_kwargs.get('triplane_depth', 1)))
        opts = dict(rendering_kwargs)
        opts.setdefault('depth_resolution', 2)
        p, wts = r._params(planes_cl, N, 0, opts, decoder, None, None, None, n_points=N * int(resolution) ** 3)
        wt = [t.detach().float().contiguous() for t in wts]
        sig = torch.empty((N, R, R, R, 1), device=dev, dtype=torch.float32)
        dens = torch.empty((N, R, R, R, 1), device=dev, dtype=torch.float32)
        rgb = torch.empty((N, R, R, R, p.out_dim - 1), device=dev, dtype=torch.float32) if want_rgb else None
        xyz = torch.empty((N, R, R, R, 3), device=dev, dtype=torch.float32) if want_coordinates else None
        _lib.check(_lib.lib().p3d_volume_query(
            C.byref(p), planes_cl.data_ptr(), wt[0].data_ptr(), wt[1].data_ptr(), wt[2].data_ptr(), wt[3].data_ptr(), R,
            float(rendering_kwargs['box_warp']) * 1, -1.0 if triplane_crop is None else float(triplane_crop),
            -1.0 if cull_clouds is None else float(cull_clouds), sig.data_ptr(), _lib.ptr(rgb), dens.data_ptr(), _lib.ptr(xyz),
            _lib.stream_ptr(dev)))
    out = {'coordinates': None if xyz is None else xyz.permute(0, 4, 1, 2, 3), 'sigmas': sig.permute(0, 4, 1, 2, 3),
           'rgbs': None if rgb is None else rgb.permute(0, 4, 1, 2, 3), 'densities': dens.permute(0, 4, 1, 2, 3)}
    return _AttrDict(out)


class _AttrDict(dict):
    """Item + attribute access, like the ``addict.Dict`` the reference returns."""
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


def get_eg3d_volume(G, xin, resolution=256, max_batch=100000):
    """Drop-in for ``_util.eg3d_metrics3d.get_eg3d_volume`` (eg3d_metrics3d.py:94-183): same arguments, same returned
    dict.  ``G`` is a ``TriPlaneGenerator``: ``G.f(xin)`` is run once (it resolves ``ws`` from the conditioning, as in
    the reference's warm-up call), the backbone once more for the tri-planes (``triplane.py:283-291``), then ONE
    volume launch replaces the 168-chunk loop; ``max_batch`` is accepted and ignored."""
    del max_batch
    planes = synthesize_planes(G, xin)
    return query_volume(planes, G.decoder, G.rendering_kwargs, resolution=resolution,
                        triplane_crop=xin['triplane_crop'] if 'triplane_crop' in xin else None,
                        cull_clouds=xin['cull_clouds'] if 'cull_clouds' in xin else None,
                        renderer=getattr(G, 'renderer', None))


def synthesize_planes(G, xin):
    """The tri-planes ``get_eg3d_volume`` queries: ``G.f`` once to resolve ``ws``, then the backbone once (no grad)."""
    dev = next(G.parameters()).device if hasattr(G, 'parameters') else torch.device('cuda')
    with torch.no_grad():
        xin_ = _AttrDict({**xin, 'elevations': torch.zeros(1, device=dev), 'azimuths': torch.zeros(1, device=dev)})
        G.f(xin_)
        ws = xin_['ws']
        planes = G.backbone.synthesis(ws, xin['cond'], update_emas=False, noise_mode='const')
        width = G.triplane_width * G.rendering_kwargs.get('triplane_depth', 1)
        return planes.view(len(planes), 3, width, planes.shape[-2], planes.shape[-1])
