"""Generate the multiplane golden vectors (triplane_depth > 1) by running the UNMODIFIED reference on the CPU.

    PROJECT_DN=/root/reference python tests/golden/make_golden_multiplane.py

Same recipe as make_golden.py: the reference's ImportanceRenderer is imported as is and its torch.rand_like / torch.rand
jitter is replaced, for the duration of a call, by the uniforms the oracle and the CUDA kernels receive.  Inputs come from
the seeds of tests/golden/cases_multiplane.py; the reference's outputs (and, for GRAD_CASES, the gradients its own
autograd gives the planes and the four decoder tensors) are written as tests/golden/multiplane_*.npz.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.golden.make_golden import ImportanceRenderer, _InjectRand, make_ref_decoder, ref_rays  # noqa: E402
from tests.golden.cases_multiplane import RENDER_CASES, POINT_CASES, GRAD_CASES, build_inputs, point_coords, upstream  # noqa: E402


def _render(case, planes, decoder, ro, rd, u_c, u_f, opts):
    renderer = ImportanceRenderer(use_triplane=case['use_triplane'])
    with _InjectRand([u_c, u_f]):
        return renderer(planes, decoder, ro, rd, opts, triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'))


def run_render_case(name, case):
    planes, dec, c2w, K, u_c, u_f, opts = build_inputs(case)
    ro, rd = ref_rays(dict(case, opts=opts), c2w, K)
    with torch.no_grad():
        rgb, depth, wsum, xyz = _render(case, planes, make_ref_decoder(dec), ro, rd, u_c, u_f, opts)
    np.savez_compressed(os.path.join(HERE, f'multiplane_render_{name}.npz'), rgb=rgb.numpy(), depth=depth.numpy(),
                        wsum=wsum.numpy(), xyz=xyz.numpy(), ro=ro.numpy(), rd=rd.numpy(),
                        input_checksum=np.float64(planes.double().sum() + u_c.double().sum()), case=json.dumps(case))
    print(f'multiplane_render_{name}: rgb {tuple(rgb.shape)} mean {rgb.mean():+.5f} wsum mean {wsum.mean():.5f}')


def run_point_case(name, case):
    planes, dec, _, _, _, _, opts = build_inputs(case)
    pts = point_coords(case)
    renderer = ImportanceRenderer(use_triplane=case['use_triplane'])
    with torch.no_grad():
        out = renderer.run_model(planes, make_ref_decoder(dec), pts, torch.zeros_like(pts), opts)
    np.savez_compressed(os.path.join(HERE, f'multiplane_points_{name}.npz'), rgb=out['rgb'].numpy(), sigma=out['sigma'].numpy(),
                        pts=pts.numpy(), case=json.dumps(case))
    print(f'multiplane_points_{name}: rgb mean {out["rgb"].mean():+.5f} sigma mean {out["sigma"].mean():+.5f}')


def run_grad_case(name, case):
    planes, dec, c2w, K, u_c, u_f, opts = build_inputs(case)
    decoder = make_ref_decoder(dec).requires_grad_(True)
    planes = planes.clone().requires_grad_(True)
    if 'R' in case:
        ro, rd = ref_rays(dict(case, opts=opts), c2w, K)
        outs = _render(case, planes, decoder, ro, rd, u_c, u_f, opts)
        names = ('rgb', 'depth', 'wsum', 'xyz')
    else:
        pts = point_coords(case)
        o = ImportanceRenderer(use_triplane=case['use_triplane']).run_model(planes, decoder, pts, torch.zeros_like(pts), opts)
        outs, names = (o['rgb'], o['sigma']), ('rgb', 'sigma')
    gs = upstream(case, [tuple(t.shape) for t in outs])
    sum(((t * g).sum() for t, g in zip(outs, gs)), torch.zeros(())).backward()
    fc1, fc2 = decoder.net[0], decoder.net[2]
    np.savez_compressed(os.path.join(HERE, f'multiplane_grad_{name}.npz'), d_planes=planes.grad.numpy(),
                        d_w1=fc1.weight.grad.numpy(), d_b1=fc1.bias.grad.numpy(), d_w2=fc2.weight.grad.numpy(),
                        d_b2=fc2.bias.grad.numpy(), **{k: t.detach().numpy() for k, t in zip(names, outs)}, case=json.dumps(case))
    print(f'multiplane_grad_{name}: |d_planes| {planes.grad.abs().sum():.4f}, nonzero {(planes.grad != 0).float().mean():.3f}')


if __name__ == '__main__':
    only = set(sys.argv[1:])
    torch.set_num_threads(os.cpu_count())
    for table, fn in ((RENDER_CASES, run_render_case), (POINT_CASES, run_point_case), (GRAD_CASES, run_grad_case)):
        for name, case in table.items():
            if not only or name in only:
                fn(name, case)
