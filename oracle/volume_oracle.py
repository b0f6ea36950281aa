"""TEST INFRASTRUCTURE ONLY - CPU restatement of the dense volume query (reference
``_util/eg3d_metrics3d.py:65-183``: ``sigma2density``, ``create_samples``, ``get_eg3d_volume`` minus the backbone).

Pinned against the reference: ``tests/golden/make_golden.py`` executes the reference's own three functions (sliced out
of ``eg3d_metrics3d.py`` so its unrelated imports - pyvista, dnnlib, legacy - are not needed) on a stand-in ``G`` whose
``sample_mixed`` is the reference ``ImportanceRenderer.run_model`` on fixed tri-planes; outputs are committed as
``tests/golden/volume_*.npz`` and ``tests/test_volume_oracle_golden.py`` compares this file with them.
Only ``tests/`` may import this module; the product path is ``panic3d_b200.volume`` -> ``p3d_volume_query``.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import renderer_oracle as orc


def sigma2density(sigma):
    """eg3d_metrics3d.py:65-69."""
    return 1 - torch.exp(-F.softplus(sigma - 1))


def create_samples(N, cube_length):
    """eg3d_metrics3d.py:70-92 with voxel_origin = [0,0,0].  z index = n % N; the y / x indices are the fp32 quotients
    (n/N) % N and ((n/N)/N) % N - the reference never floors them; index * voxel_size + corner, all in fp32."""
    corner = -cube_length / 2
    size = cube_length / (N - 1)
    n = torch.arange(N ** 3, dtype=torch.int64)
    q = n.float() / N
    cols = [(q / N) % N, q % N, (n % N).float()]
    return torch.stack([c * size + corner for c in cols], dim=-1).unsqueeze(0)


def masked_density(samples, sigma, box_warp, triplane_crop=None, cull_clouds=None):
    """eg3d_metrics3d.py:155-162: sigma2density, then the crop and cull overwrites."""
    dens = sigma2density(sigma)
    if triplane_crop is not None:
        dens[orc.crop_mask(samples, triplane_crop, box_warp)] = -1e3
    if cull_clouds is not None:
        dens[orc.cull_mask(dens, cull_clouds)] = -1e3          # sic: the cull test runs on the density (:160-162)
    return dens


def volume(planes, dec, opts, resolution, triplane_crop=None, cull_clouds=None, use_triplane=True):
    """eg3d_metrics3d.py:114-183 for one subject (planes (1,3,C,H,W)); returns the same four tensors, on the planes'
    device and in their dtype (the lattice itself is the fp32 one of ``create_samples``)."""
    R = resolution
    samples = create_samples(R, opts['box_warp'] * 1).to(planes.device, planes.dtype)
    rgb, sigma = orc.run_model(planes, dec, samples, opts, use_triplane)
    dens = masked_density(samples, sigma, opts['box_warp'], triplane_crop, cull_clouds)

    def shape(t, c):
        return t.reshape(1, R, R, R, c).flip(dims=(1,)).permute(0, 4, 1, 2, 3)
    return {'coordinates': shape(samples, 3), 'sigmas': shape(sigma, 1), 'rgbs': shape(rgb, rgb.shape[-1]), 'densities': shape(dens, 1)}


def volume_chunks(planes, dec, opts, resolution, triplane_crop=None, cull_clouds=None, use_triplane=True, chunk=1 << 19,
                  samples=None):
    """``volume`` for one subject in lattice order (sample n, before the reshape and flip), ``chunk`` points at a time, for
    lattices whose whole working set would not fit: yields (n0, samples, rgb, sigma, densities) of points [n0, n0 + chunk),
    on the planes' device and in their dtype.  ``samples`` (1, R^3, 3): the lattice, when the caller already made it."""
    if samples is None:
        samples = create_samples(resolution, opts['box_warp'] * 1)
    for n0 in range(0, samples.shape[1], chunk):
        xyz = samples[:, n0:n0 + chunk].to(planes.device, planes.dtype)
        rgb, sigma = orc.run_model(planes, dec, xyz, opts, use_triplane)
        yield n0, xyz, rgb, sigma, masked_density(xyz, sigma, opts['box_warp'], triplane_crop, cull_clouds)
