"""Shared helpers for the test-suite (fixture loading, oracle invocation, inputs and stand-ins more than one file uses)."""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from oracle import ops_oracle as oo, renderer_oracle as orc
from tests.golden.cases import build_case_inputs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def load_golden(kind: str, name: str):
    z = np.load(os.path.join(GOLDEN, f'{kind}_{name}.npz'))
    out = {k: (torch.from_numpy(z[k]) if z[k].dtype.kind == 'f' and z[k].ndim > 0 else z[k]) for k in z.files}
    out['case'] = json.loads(str(z['case']))
    return out


def case_rays(case, c2w, K):
    """Rays for a case via the oracle (pinhole or ortho)."""
    R = case['R']
    if case.get('ortho'):
        ros, rds = [], []
        for (elev, azim, dist, _f) in case['cameras']:
            o, d = orc.rays_ortho(elev, azim, dist, case['opts']['box_warp'], R)
            ros.append(o.reshape(1, 3, R * R).permute(0, 2, 1))
            rds.append(d.reshape(1, 3, R * R).permute(0, 2, 1))
        return torch.cat(ros).contiguous(), torch.cat(rds).contiguous()
    return orc.ray_sampler(c2w, K, R)


def oracle_render(case, gather='manual'):
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = case_rays(case, c2w, K)
    return orc.render(planes, dec, ro, rd, opts, u_c, u_f if opts['depth_resolution_importance'] > 0 else None,
                      use_triplane=case.get('use_triplane', True), triplane_crop=case.get('triplane_crop'),
                      cull_clouds=case.get('cull_clouds'), binarize_clouds=case.get('binarize_clouds'), gather=gather)


def profiled(fn):
    """fn() and the number of launches per library profile slot it made (slots: csrc/p3d_common.cuh).  Profiling is
    switched off again even when fn raises."""
    import ctypes as C
    from panic3d_b200 import _lib
    L = _lib.lib()
    L.p3d_profile_enable(1)
    L.p3d_profile_read(None, None, 0, 1)
    try:
        out = fn()
        torch.cuda.synchronize()
        ms, n = (C.c_double * 8)(), (C.c_uint64 * 8)()
        L.p3d_profile_read(ms, n, 8, 1)
    finally:
        L.p3d_profile_enable(0)
    return out, list(n)


def input_checksum(case):
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    return float(planes.double().sum() + u_c.double().sum() + dec['w1'].double().sum())


# ------------------------------------------------------------------------------------------------- render backward cases
def bwd_case(seed, S, Sf, R=15, N=2, opts=None, cameras=None, **kw):
    o = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf)
    o.update(opts or {})
    return dict(seed=seed, N=N, R=R, P=64, opts=o, cameras=cameras, **kw)


# merged intervals per ray = S + Sf - 1
BWD_CASES = {
    'train48': bwd_case(61, 48, 48),                                            # 95: the training setting, three chunks
    # 191, eval flags: the bias puts the cull threshold (sigma = 1 for cull 0.5) inside the samples' sigma range
    'eval96': bwd_case(68, 96, 96, R=5, triplane_crop=0.1, cull_clouds=0.5, force_sigmoid=True, sigma_bias=1.04),
    'ragged31_17': bwd_case(63, 31, 17),                                        # 47: second chunk half full
    'ragged40_26': bwd_case(64, 40, 26),                                        # 65: third chunk has one live lane
    'coarse40': bwd_case(65, 40, 0),                                            # 39: coarse-only path crosses a chunk
    'lrmul_black48': bwd_case(66, 48, 48, lr_mul=0.5, opts=dict(white_back=False)),
}


def bwd_flags(case):
    return dict(triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'), binarize_clouds=case.get('binarize_clouds'))


def bwd_incoming(seed, N, M):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.standard_normal(s).astype(np.float32)) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]


def f32_scalars(kw, act):
    """alpha / gain / clamp cross the C ABI as fp32 (as in the reference plugin: bias_act.h:27-29); give the fp64
    oracle the same rounded scalars so fp64 comparisons can be tight."""
    _, def_alpha, def_gain = oo.ACTS[act]
    out = dict(kw)
    out['alpha'] = float(np.float32(def_alpha if kw.get('alpha') is None else kw['alpha']))
    out['gain'] = float(np.float32(def_gain if kw.get('gain') is None else kw['gain']))
    if kw.get('clamp') is not None:
        out['clamp'] = float(np.float32(kw['clamp']))
    return out


class StandInG:
    """The same stand-in generator the golden script uses: f() returns the fixed results of the two extra renders."""

    def __init__(self, inp, dev):
        self.rendering_kwargs = {'ray_start': inp['ray_start'], 'box_warp': inp['box_warp']}
        self.inp, self.dev, self.seen = inp, dev, {}

    def f(self, xin, return_more=False):
        if xin.get('force_rays') is not None:
            assert xin['paste_params'] is None
            self.seen['occ_ro'], self.seen['occ_rd'] = xin['force_rays']['ray_origins'], xin['force_rays']['ray_directions']
            return {'image_weights': self.inp['occ'].to(self.dev)}
        assert float(xin['fovs'][0]) == -1 and 'paste_params' not in xin
        return {'image_weights': self.inp['frontw'].to(self.dev)}


def synth_image(seed, c, h, w):
    """Smooth gradients + noise + out-of-range values, so every filter type wins on some row and the clamp matters."""
    g = np.random.Generator(np.random.PCG64(seed))
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing='ij')
    img = np.stack([0.5 + 0.6 * np.sin(6 * xx + ch) * np.cos(5 * yy - ch) for ch in range(c)])
    img[:, h // 3: h // 2] += g.normal(0, 0.3, (c, h // 2 - h // 3, w))
    img[:, : h // 8] = np.round(img[:, : h // 8] * 4) / 4                 # flat runs
    return torch.from_numpy(img.astype(np.float32))


class TinyG(torch.nn.Module):
    """Stand-in with the attributes load_eg3dc_model relies on (init_args / init_kwargs via persistence, eg3dc_v0.py:44-50)."""

    def __init__(self, width, depth=2, rendering_kwargs=None):
        super().__init__()
        self.init_args, self.init_kwargs = (width,), {'depth': depth, 'rendering_kwargs': rendering_kwargs}
        self.layers = torch.nn.ModuleList([torch.nn.Linear(width, width) for _ in range(depth)])
        self.register_buffer('w_avg', torch.randn(width))
        self.register_buffer('steps', torch.tensor(7, dtype=torch.int64))
        self.half_w = torch.nn.Parameter(torch.randn(3, 5).half())
        self.rendering_kwargs = rendering_kwargs or {}
        self.neural_rendering_resolution = 64
        self.force_sigmoid = False

    def set_force_sigmoid(self, s):
        self.force_sigmoid = s
