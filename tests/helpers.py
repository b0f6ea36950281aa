"""Shared helpers for the test-suite (fixture loading, oracle invocation)."""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from oracle import renderer_oracle as orc
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
