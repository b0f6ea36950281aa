"""TEST INFRASTRUCTURE ONLY - CPU restatement of the front-view paste (SURVEY 8f-3; reference
``_train/eg3dc/src/training/triplane.py:555-691``: ``sample_orthofront``, ``get_front_occlusion`` (ray construction),
``get_xyz_discrepancy``, ``paste_front``).

The two extra renders ``paste_front`` asks of ``G.f`` (the occlusion render along +z from the visible surface, and the
optional orthographic front weights) are inputs here: ``occ`` / ``frontw`` are what those calls return.

Pinning.  ``tests/golden/make_golden_paste.py`` runs the reference's OWN ``paste_front`` (imported from
``/root/reference``) on a stand-in ``G`` whose ``f`` returns the given ``occ`` / ``frontw``, and commits its outputs as
``tests/golden/paste_*.npz``; ``tests/test_paste_oracle_golden.py`` compares this file with them.
Third-party arithmetic: ``kornia==0.6.5`` (``_env/Dockerfile``) is NOT installed in this image and is not vendored by
the reference, so ``kornia.filters.sobel`` and ``kornia.morphology.erosion`` are restated below from kornia 0.6.5's
published algorithm (``kornia/filters/sobel.py``: replicate pad, 3x3 Sobel pair divided by its absolute sum 8,
``sqrt(gx^2 + gy^2 + 1e-6)``; ``kornia/morphology/morphology.py``: min over the structuring element anchored at
``(h//2, w//2)``, 'geodesic' border = out-of-image neighbours never lower the minimum) and the generator injects the
same restatement as the ``kornia`` module the reference imports.  For those two functions: **parity unpinned** (no
kornia here to run); everything else in this file is pinned on reference outputs.

Only ``tests/`` (and ``__graft_entry__.smoke()`` / the ``cpu_baseline`` leg of a bench) may import this module; the
product path is ``panic3d_b200.paste`` -> ``p3d_paste_front``.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


# ---------------------------------------------------------------- kornia 0.6.5 restatements (parity unpinned)
def sobel_magnitude(x, eps=1e-6):
    """kornia.filters.sobel(x, normalized=True, eps=1e-6) for x (B,C,H,W): per-channel gradient magnitude."""
    b, c, h, w = x.shape
    kx = torch.tensor([[-1., 0., 1.], [-2., 0., 2.], [-1., 0., 1.]], dtype=x.dtype, device=x.device) / 8
    k = torch.stack([kx, kx.t()])[:, None]                                                # (2,1,3,3): d/dx, d/dy; conv = cross-correlation
    g = F.conv2d(F.pad(x.reshape(b * c, 1, h, w), [1, 1, 1, 1], mode='replicate'), k).view(b, c, 2, h, w)
    return torch.sqrt(g[:, :, 0] * g[:, :, 0] + g[:, :, 1] * g[:, :, 1] + eps)


def erosion_ones(x, e):
    """kornia.morphology.erosion(x, torch.ones(e, e)) (border_type='geodesic', engine 'unfold') for x (B,C,H,W)."""
    o = e // 2
    xp = F.pad(x, [o, e - o - 1, o, e - o - 1], mode='constant', value=1e4)
    win = xp.unfold(2, e, 1).unfold(3, e, 1)                                 # (B,C,H,W,e,e)
    return win.reshape(*x.shape, e * e).min(dim=-1).values


def kornia_shim():
    """A module object with exactly the two kornia entry points triplane.py uses, for the golden generator."""
    import types
    k = types.ModuleType('kornia')
    k.filters = types.ModuleType('kornia.filters')
    k.morphology = types.ModuleType('kornia.morphology')
    k.filters.sobel = lambda t, normalized=True, eps=1e-6: sobel_magnitude(t, eps)
    k.morphology.erosion = lambda t, kernel: erosion_ones(t, int(kernel.shape[0]))
    k.morphology.dilation = lambda t, kernel: -erosion_ones(-t, int(kernel.shape[0]))     # loss_orthocondA only; unused here
    return k


# ---------------------------------------------------------------- reference restatement
def _flip(t):
    """The reference's ``[-1, 1, -1]`` channel factor, on t's device and in t's dtype."""
    return torch.tensor([-1., 1., -1.], dtype=t.dtype, device=t.device)[None, :, None, None]


def orthofront_coords(view_xyz, bw, size):
    """The unnormalised ``grid_sample`` source coordinates (row, column) of ``sample_orthofront``'s lookup in a
    ``size`` x ``size`` image, BEFORE border clipping (aten GridSampler.h, align_corners=False): rows follow world y,
    columns world x.  Tests use them to tell a clipped, a cell-boundary or an interior lookup apart."""
    vij = 1 - (view_xyz[:, [1, 0]] + bw / 2) / bw
    g = vij * 2 - 1
    ix = ((g + 1) * size - 1) / 2
    return ix[:, 0:1], ix[:, 1:2]


def sample_orthofront(front, view_xyz, bw):
    """triplane.py:555-564: look the front image up at the (y, x) world position of every pixel."""
    vij = 1 - (view_xyz[:, [1, 0]] + bw / 2) / bw
    return F.grid_sample(front.permute(0, 1, 3, 2), vij.permute(0, 2, 3, 1) * 2 - 1, padding_mode='border', mode='bilinear',
                         align_corners=False)


def occlusion_rays(image_xyz, ray_start, offset=0.01):
    """triplane.py:565-570 (get_front_occlusion): rays from just in front of the visible surface, along +z."""
    ro = image_xyz * _flip(image_xyz)
    ro[:, 2] -= ray_start - offset
    rd = torch.zeros_like(image_xyz)
    rd[:, 2] = 1
    return ro, rd


def xyz_discrepancy(xyz, ro, rd):
    """triplane.py:601-606: distance of the rendered point from its own ray."""
    p = xyz * _flip(xyz)
    d = p - ro
    return (d - (d * rd).sum(dim=1, keepdim=True) * rd).norm(2, dim=1, keepdim=True)


def paste_front(image, image_xyz, image_weights, front_rgb, occ, ro, rd, box_warp, frontw=None, normalize_images=False,
                thresh_weight=0.95, thresh_edges=0.02, thresh_occ=0.05, thresh_dxyz=0.01, front_weight_erosion=0):
    """triplane.py:608-691 with the two G.f calls replaced by their results (occ, frontw).  Returns the reference's
    dict plus the quantities in front of each threshold (``q_*``) and the source coordinates of every lookup (``src_*``:
    the paste's and the eroded weights' ``grid_sample`` row / column before clipping, the ``nearest`` up-sampling's
    exact ``dst * R / S``) so tests can tell a borderline pixel from an error.  Runs on the inputs' device and dtype."""
    S = front_rgb.shape[-1]
    R = image_xyz.shape[-1]
    with torch.no_grad():                                                      # the masks carry no gradient (:622)
        q_w = F.interpolate(image_weights, S, mode='bilinear')
        wmask = (q_w > thresh_weight).to(q_w.dtype)
        q_s = sobel_magnitude(F.interpolate(image_xyz, S, mode='bilinear')).norm(2, dim=1, keepdim=True)
        smask = (q_s < thresh_edges).to(q_s.dtype)
        fmask = F.interpolate((occ < thresh_occ).to(occ.dtype), S, mode='bilinear')
        q_d_lo = xyz_discrepancy(image_xyz, ro, rd)
        q_d = F.interpolate(q_d_lo, S, mode='nearest')
        dmask = (q_d < thresh_dxyz).to(q_d.dtype)
        if front_weight_erosion >= 1:
            eroded = erosion_ones((frontw > 0.5).to(frontw.dtype), front_weight_erosion)
            fwmask = F.interpolate(sample_orthofront(eroded, F.interpolate(image_xyz, S, mode='bilinear'), box_warp), S, mode='nearest')
            fw_row, fw_col = orthofront_coords(F.interpolate(image_xyz, S, mode='bilinear'), box_warp, eroded.shape[-1])
        else:
            fwmask = torch.ones_like(dmask)
            fw_row = fw_col = None
        mask = wmask * smask * fmask * dmask * fwmask
    up_xyz = F.interpolate(image_xyz, S, mode='bilinear')                      # with gradient when grad_sample (:674-679)
    tocopy = front_rgb * 2 - 1 if normalize_images else front_rgb
    paste = sample_orthofront(tocopy, up_xyz, box_warp)
    out = torch.lerp(image, paste, mask)
    with torch.no_grad():
        src_row, src_col = orthofront_coords(up_xyz, box_warp, S)
    return {'image': out, 'paste': paste, 'mask': mask, 'mask_weights': wmask, 'mask_edges': smask, 'mask_occ': fmask,
            'mask_dxyz': dmask, 'mask_frontweight': fwmask, 'q_weights': q_w, 'q_edges': q_s, 'q_dxyz': q_d, 'q_occ_lo': occ,
            'q_dxyz_lo': q_d_lo, 'src_row': src_row, 'src_col': src_col, 'src_fw_row': fw_row, 'src_fw_col': fw_col,
            'src_nearest': torch.arange(S, dtype=torch.float64, device=image_xyz.device) * R / S}


# ---------------------------------------------------------------- seeded inputs (regenerated, never stored)
def synth_paste_inputs(seed, N, R, S, box_warp=0.7, ray_start=0.5, reach=0.9):
    """Plausible render outputs: a smooth bumpy surface seen from the front with one depth step (so every mask has
    both values), weights with a soft silhouette, rays that agree with the surface except for a band of noise.
    ``reach``: the fraction of the box the surface spans in x and y; above 1 a band of pixels on every side of the
    image looks the front image up outside the box (the lookup clips, as for real background and silhouette pixels)."""
    g = np.random.Generator(np.random.PCG64(seed))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    lin = (np.arange(R, dtype=np.float64) + 0.5) / R
    yy, xx = np.meshgrid(lin, lin, indexing='ij')
    xyz = np.zeros((N, 3, R, R)); wts = np.zeros((N, 1, R, R)); occ = np.zeros((N, 1, R, R)); fw = np.zeros((N, 1, R, R))
    ro = np.zeros((N, 3, R, R)); rd = np.zeros((N, 3, R, R))
    for n in range(N):
        ph = g.uniform(0, 2 * np.pi, 4)
        x = (0.5 - xx) * box_warp * reach + 0.004 * np.sin(9 * yy + ph[0])
        y = (0.5 - yy) * box_warp * reach + 0.004 * np.sin(7 * xx + ph[1])
        z = 0.08 * np.sin(5 * xx + ph[2]) * np.cos(4 * yy + ph[3]) + 0.12 * (xx + 0.3 * yy > 0.8 + 0.1 * n)
        z = z + g.normal(0, 0.004, (R, R)) * (yy > 0.75)                      # a rough band: sobel above threshold
        xyz[n] = np.stack([x, y, z])
        r2 = (xx - 0.5) ** 2 + (yy - 0.5) ** 2
        wts[n, 0] = 1 / (1 + np.exp((r2 - 0.16 - 0.02 * n) * 60)) * (1 - 0.06 * g.uniform(0, 1, (R, R)) * (xx < 0.3))
        occ[n, 0] = g.uniform(0, 0.1, (R, R)) * (np.sin(11 * xx + ph[0]) > -0.3)
        fw[n, 0] = 1 / (1 + np.exp((r2 - 0.12) * 80)) + 0.05 * g.normal(0, 1, (R, R))
        p = xyz[n] * np.array([-1., 1., -1.])[:, None, None]
        d = np.stack([0.05 * np.sin(3 * xx), 0.05 * np.cos(2 * yy), -np.ones_like(xx)])
        d /= np.linalg.norm(d, axis=0, keepdims=True)
        off = g.normal(0, 6e-6, (3, R, R)) * (g.uniform(0, 1, (R, R)) < 0.5)  # half the rays miss their point by ~thresh_dxyz
        ro[n] = p - d * g.uniform(0.4, 1.2, (R, R)) + off
        rd[n] = d
    return {'image': t(g.uniform(-1, 1, (N, 3, S, S))), 'front_rgb': t(g.uniform(0, 1, (N, 3, S, S))),
            'image_xyz': t(xyz), 'image_weights': t(wts), 'occ': t(occ), 'frontw': t(fw), 'ro': t(ro), 'rd': t(rd),
            'box_warp': box_warp, 'ray_start': ray_start}
