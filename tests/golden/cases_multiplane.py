"""Multiplane tri-plane cases (rendering_kwargs['triplane_depth'] = D > 1), shared by make_golden_multiplane.py, the CPU
oracle check and tests/test_multiplane_gpu.py.  Inputs are regenerated from a numpy-PCG64 seed; only the reference's
outputs are stored.

Planes are H x W = 24 x 20 (H != W, so a slab stride taken from the wrong side is visible) with 32 features per slab,
i.e. (N, 3, 32*D, 24, 20) as TriPlaneGenerator views its backbone output (triplane.py:200-206)."""
from __future__ import annotations

import copy

import numpy as np
import torch

from oracle import renderer_oracle as orc

H, W = 24, 20
BOX = 0.7

_OPTS = dict(box_warp=BOX, ray_start=0.5, ray_end=1.5, disparity_space_sampling=False, clamp_mode='softplus', white_back=True)

RENDER_CASES = {
    'd2_eg3d48': dict(seed=501, N=2, R=16, D=2, use_triplane=False, opts=dict(_OPTS, depth_resolution=48, depth_resolution_importance=48)),
    'd3_panic48': dict(seed=502, N=2, R=16, D=3, use_triplane=True, opts=dict(_OPTS, depth_resolution=48, depth_resolution_importance=48)),
    'd2_panic96': dict(seed=503, N=1, R=16, D=2, use_triplane=True, opts=dict(_OPTS, depth_resolution=96, depth_resolution_importance=96)),
    'd3_eg3d96_crop_cull': dict(seed=504, N=1, R=16, D=3, use_triplane=False, triplane_crop=0.1, cull_clouds=0.5, sigma_bias=2.5,
                                opts=dict(_OPTS, depth_resolution=96, depth_resolution_importance=96)),
    'd2_ortho48': dict(seed=505, N=2, R=16, D=2, use_triplane=True, ortho=True, cameras=[(0.0, 30.0, 1.0, 30.0), (25.0, -110.0, 1.0, 30.0)],
                       opts=dict(_OPTS, depth_resolution=48, depth_resolution_importance=48)),
}
for _c in RENDER_CASES.values():
    _c['opts']['triplane_depth'] = _c['D']

POINT_CASES = {
    'd2_eg3d': dict(seed=511, N=2, K=600, D=2, use_triplane=False),
    'd3_panic': dict(seed=512, N=2, K=600, D=3, use_triplane=True),
}

# gradients of the reference's own autograd: a render (loss = sum of every output times a seeded upstream gradient) and
# run_model (loss = sum of sigma and rgb times seeded upstream gradients)
GRAD_CASES = {
    'render_d2_eg3d': dict(seed=521, N=1, R=12, D=2, use_triplane=False, opts=dict(_OPTS, depth_resolution=48, depth_resolution_importance=48)),
    'points_d3_panic': dict(seed=522, N=1, K=500, D=3, use_triplane=True),
}
GRAD_CASES['render_d2_eg3d']['opts']['triplane_depth'] = 2


def slab_points(D, use_triplane):
    """Points on slab centres and slab borders of each plane's normal axis, and past the box along each normal (the slabs
    beyond 0 and D - 1 are zero there).  (P, 3)."""
    half = BOX / 2
    normal_axis = [2, 1, 0 if use_triplane else 1]            # plane 0: z, plane 1: y, plane 2: x (panic3d) or y (EG3D)
    vals = [((2 * d + 1) / D - 1) * half for d in range(D)]    # slab centres
    vals += [(2 * d / D - 1) * half for d in range(D + 1)]     # slab borders, including the box faces
    vals += [-half * 1.2, half * 1.2, -half * (1 + 0.9 / D), half * (1 + 0.9 / D), -half * 1.6, half * 1.6]  # past the faces
    base = np.array([0.083, -0.051, 0.127], np.float64)
    pts = []
    for ax in sorted(set(normal_axis)):
        for v in vals:
            q = base.copy()
            q[ax] = v
            pts.append(q)
    return np.array(pts, np.float32)


def point_coords(case):
    """Uniform points over a cube 1.3x the box (some outside along every axis) followed by slab_points."""
    rng = np.random.default_rng(case['seed'] + 1000)
    pts = rng.uniform(-0.45, 0.45, size=(case['N'], case['K'], 3)).astype(np.float32)
    sp = slab_points(case['D'], case['use_triplane'])
    pts = np.concatenate([pts, np.broadcast_to(sp, (case['N'],) + sp.shape)], axis=1)
    return torch.from_numpy(np.ascontiguousarray(pts))


def build_inputs(case):
    """-> planes (N,3,32*D,H,W), dec, c2w, K, u_c, u_f, opts (opts and the cameras only for ray cases)."""
    rng = np.random.default_rng(case['seed'])
    N, D = case['N'], case['D']
    planes = torch.from_numpy(rng.standard_normal((N, 3, 32 * D, H, W), dtype=np.float32))
    dec = dict(w1=torch.from_numpy(rng.standard_normal((64, 32), dtype=np.float32)),
               b1=torch.from_numpy(0.1 * rng.standard_normal((64,), dtype=np.float32)),
               w2=torch.from_numpy(rng.standard_normal((33, 64), dtype=np.float32)),
               b2=torch.from_numpy(0.1 * rng.standard_normal((33,), dtype=np.float32)),
               lr_mul=1.0, force_sigmoid=False)
    dec['b2'][0] += case.get('sigma_bias', 0.0)          # denser fields, so a cull threshold keeps some samples
    opts = copy.deepcopy(case.get('opts', dict(_OPTS, triplane_depth=D)))
    c2w = K = u_c = u_f = None
    if 'R' in case:
        S, Sf, M = opts['depth_resolution'], opts['depth_resolution_importance'], case['R'] ** 2
        u_c = torch.from_numpy(rng.random((N, M, S, 1), dtype=np.float32))
        u_f = torch.from_numpy(rng.random((N * M, Sf), dtype=np.float32))
        cams = case.get('cameras') or [(10.0 * i - 5.0, -150.0 + 70.0 * i, 1.0, 30.0) for i in range(N)]
        c2w, K = zip(*(orc.camera_params_to_matrix(*c) for c in cams))
        c2w, K = torch.stack(c2w), torch.stack(K)
    return planes, dec, c2w, K, u_c, u_f, opts


def upstream(case, shapes):
    """Seeded upstream gradients for the gradient cases, one per output shape."""
    rng = np.random.default_rng(case['seed'] + 2000)
    return [torch.from_numpy(rng.standard_normal(s, dtype=np.float32)) for s in shapes]
