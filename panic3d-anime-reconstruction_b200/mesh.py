"""Marching cubes on the device - the H100 replacement for ``marching_cubes`` (reference ``_util/eg3d_metrics3d.py:186-211``;
SURVEY.md section 8f, between the volume query 8f-2 and the writers 8f-4).

The reference copies the density volume and the whole 32-channel colour volume to the host, runs skimage's Lewiner
marching cubes over the 16.7 M cells and looks up every vertex colour in a Python loop.  Here ``p3d_mc_count`` /
``p3d_mc_emit`` (include/p3d_mesh.h) extract the mesh in two passes over the device-resident volume; the rules they follow
(vertex order, face rule with the asymptotic decider, winding, degenerate removal) are in DESIGN.md section 2.

    ``mesh_index``        (D0,D1,D2) CUDA density volume -> device tensors in index space
    ``marching_cubes``    drop-in for the reference function: same arguments, same returned dict of numpy arrays
    ``extract_mesh``      planes + decoder -> the same dict, with colours decoded at the vertex nodes only: the 2.1 GB
                          colour volume is never written
    ``get_eg3d_mesh``     ``get_eg3d_volume`` + ``marching_cubes`` fused on a TriPlaneGenerator-like ``G``

No CPU path: volumes are meshed on a CUDA device (the numpy restatement is ``oracle/mesh_oracle.py``, tests only).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .volume import _AttrDict, query_volume, synthesize_planes


def _device_volume(vol):
    """numpy array (copied to the current CUDA device) or CUDA tensor (zero-copy when contiguous) -> (D0,D1,D2) fp32."""
    if isinstance(vol, np.ndarray):
        if vol.dtype != np.float32:
            raise RuntimeError(f'panic3d_b200.mesh: the volume must be float32, got {vol.dtype}')
        vol = torch.from_numpy(np.ascontiguousarray(vol)).cuda()
    elif torch.is_tensor(vol):
        if not vol.is_cuda:
            raise RuntimeError('panic3d_b200.mesh has no CPU path: the volume must be a numpy array or a CUDA tensor')
        if vol.dtype != torch.float32:
            raise RuntimeError(f'panic3d_b200.mesh: the volume must be float32, got {vol.dtype}')
    else:
        raise RuntimeError(f'panic3d_b200.mesh: the volume must be a numpy array or a CUDA tensor, got {type(vol).__name__}')
    if vol.dim() != 3 or min(vol.shape) < 2:
        raise RuntimeError(f'panic3d_b200.mesh: the volume must be (D0, D1, D2) with every side >= 2, got {tuple(vol.shape)}')
    return vol.contiguous()


def mesh_index(dens, level=0.5, want_normals=True, want_values=True):
    """(D0,D1,D2) fp32 CUDA volume -> dict of device tensors: ``verts`` (V,3) fp32 index-space positions, ``faces`` (F,3)
    int32, ``normals`` (V,3) / ``values`` (V,) fp32 (None when not wanted) and ``floor_node`` (V,) int64, the flat index of
    each vertex's floor node.  Reading the two counts is the only host synchronisation."""
    dens = _device_volume(dens)
    dev = dens.device
    D0, D1, D2 = (int(s) for s in dens.shape)
    L = _lib.lib()
    with torch.cuda.device(dev):
        nbytes = int(L.p3d_mc_workspace_bytes(D0, D1, D2))
        if nbytes == 0:
            raise RuntimeError(f'p3d error: {L.p3d_last_error().decode("utf-8", "replace")}')
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        st = _lib.stream_ptr(dev)
        _lib.check(L.p3d_mc_count(dens.data_ptr(), D0, D1, D2, float(level), ws.data_ptr(), nbytes, counts.data_ptr(), st))
        V, F = (int(x) for x in counts.tolist())
        if V >= 2 ** 31 or F >= 2 ** 31:
            raise RuntimeError(f'panic3d_b200.mesh: {V} vertices / {F} triangles do not fit int32 face indices')
        out = dict(verts=torch.empty((V, 3), dtype=torch.float32, device=dev),
                   faces=torch.empty((F, 3), dtype=torch.int32, device=dev),
                   normals=torch.empty((V, 3), dtype=torch.float32, device=dev) if want_normals else None,
                   values=torch.empty((V,), dtype=torch.float32, device=dev) if want_values else None,
                   floor_node=torch.empty((V,), dtype=torch.int64, device=dev))
        if V:
            _lib.check(L.p3d_mc_emit(dens.data_ptr(), D0, D1, D2, float(level), ws.data_ptr(), nbytes, out['verts'].data_ptr(),
                                     out['faces'].data_ptr(), _lib.ptr(out['normals']), _lib.ptr(out['values']),
                                     out['floor_node'].data_ptr(), st))
    return out


def scale_verts(verts_index, shape_res, boxwarp):
    """The reference's ``mc_vert / shape_res * bw - 0.5*bw`` (eg3d_metrics3d.py:203) on the fp32 index-space vertices, in
    numpy so the arithmetic is the reference's own."""
    return verts_index / shape_res * boxwarp - 0.5 * boxwarp


def host_colors(rgbs, floor_node, shape):
    """``rgbs[:3, a, b, c]`` per vertex, (a, b, c) = the floor node: the reference's colour loop as one gather."""
    a, b, c = np.unravel_index(floor_node, shape)
    return np.ascontiguousarray(np.asarray(rgbs)[:3, a, b, c].T)


def _result(m, shape_res, boxwarp, colors):
    return _AttrDict({'verts': scale_verts(m['verts'].cpu().numpy(), shape_res, boxwarp), 'faces': m['faces'].cpu().numpy(),
                      'normals': m['normals'].cpu().numpy(), 'values': m['values'].cpu().numpy(), 'colors': colors})


def marching_cubes(vol, rgbs, boxwarp, level=0.5):
    """Drop-in for ``_util.eg3d_metrics3d.marching_cubes`` (eg3d_metrics3d.py:186-211): ``vol`` (R,R,R) densities and
    ``rgbs`` (>=3,R,R,R) colours, as numpy arrays (copied to the device; what ``generate.py`` passes) or CUDA tensors
    (zero-copy) -> {'verts','faces','normals','values','colors'} numpy arrays.  ``colors`` is ``rgbs[:3, a, b, c]`` at
    ``(a, b, c) = floor(vertex)``, as the reference's ``mc_vert.astype(int)`` loop."""
    dens = _device_volume(vol)
    shape = tuple(dens.shape)
    if tuple(rgbs.shape[1:]) != shape or rgbs.shape[0] < 3:
        raise RuntimeError(f'panic3d_b200.mesh: rgbs must be (>=3, {shape[0]}, {shape[1]}, {shape[2]}), got {tuple(rgbs.shape)}')
    m = mesh_index(dens, level)
    fl = m['floor_node']
    if torch.is_tensor(rgbs):
        if not rgbs.is_cuda:
            raise RuntimeError('panic3d_b200.mesh has no CPU path: rgbs must be a numpy array or a CUDA tensor')
        a, rest = fl // (shape[1] * shape[2]), fl % (shape[1] * shape[2])
        colors = rgbs[:3, a, rest // shape[2], rest % shape[2]].T.contiguous().cpu().numpy()
    else:
        colors = host_colors(rgbs, fl.cpu().numpy(), shape)
    return _result(m, shape[-1], boxwarp, colors)


def extract_mesh(planes, decoder, rendering_kwargs, resolution=256, triplane_crop=None, cull_clouds=None, level=0.5,
                 renderer=None):
    """planes (1,3,32,H,W) + OSGDecoder -> the ``marching_cubes`` dict of the subject's density volume, all on the device:
    ``query_volume`` without the colour and coordinate outputs, the two marching-cubes passes, the lattice coordinates of
    the vertices' floor nodes and ``p3d_decode_points`` there.  The colours equal ``query_volume(...).rgbs[0, :3]`` at the
    floor nodes bit for bit, without the (1,32,R,R,R) colour volume ever being written."""
    from .training.volumetric_rendering.renderer import ImportanceRenderer
    if not planes.is_cuda:
        raise RuntimeError('panic3d_b200.mesh.extract_mesh has no CPU path: tensors must be on a CUDA device')
    if planes.shape[0] != 1:
        raise RuntimeError(f'panic3d_b200.mesh.extract_mesh meshes one subject, got {planes.shape[0]}')
    r = renderer if renderer is not None else ImportanceRenderer(use_triplane=True)
    dev = planes.device
    R = int(resolution)
    vol = query_volume(planes, decoder, rendering_kwargs, resolution=R, triplane_crop=triplane_crop, cull_clouds=cull_clouds,
                       renderer=r, want_rgb=False, want_coordinates=False)
    m = mesh_index(vol['densities'][0, 0], level)
    V = m['verts'].shape[0]
    with torch.no_grad(), torch.cuda.device(dev):
        coords = torch.empty((1, V, 3), dtype=torch.float32, device=dev)
        if V:
            _lib.check(_lib.lib().p3d_mc_lattice_coords(m['floor_node'].data_ptr(), V, R, float(rendering_kwargs['box_warp']) * 1,
                                                        coords.data_ptr(), _lib.stream_ptr(dev)))
            colors = r.run_model(planes, decoder, coords, None, rendering_kwargs)['rgb'][0, :, :3]
        else:
            colors = torch.empty((0, 3), dtype=torch.float32, device=dev)
    return _result(m, R, rendering_kwargs['box_warp'], colors.contiguous().cpu().numpy())


def get_eg3d_mesh(G, xin, resolution=256, level=0.5):
    """``marching_cubes(get_eg3d_volume(G, xin)...)`` fused (eval ``generate.py:97-103``): ``G.f`` and the backbone run once
    each, as in ``volume.get_eg3d_volume``, then ``extract_mesh``; the colour volume never leaves the device because it is
    never made."""
    planes = synthesize_planes(G, xin)
    return extract_mesh(planes, G.decoder, G.rendering_kwargs, resolution=resolution,
                        triplane_crop=xin['triplane_crop'] if 'triplane_crop' in xin else None,
                        cull_clouds=xin['cull_clouds'] if 'cull_clouds' in xin else None, level=level,
                        renderer=getattr(G, 'renderer', None))
