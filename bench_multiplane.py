"""Multiplane tri-planes (triplane_depth D > 1) on the fp32 SIMT kernels: what 8 taps per plane instead of 4 cost.

    python bench_multiplane.py [--steps 20] [--warmup 5]

Times, with CUDA events around --steps repetitions after --warmup:
  * train_fwd_bwd_D1 / train_fwd_bwd_D2: the training render's forward + backward at config 5's shape (4 views, 64^2
    rays, 48+48 samples, 256^2 planes; planes and decoder require grad, so ImportanceRenderer takes the SIMT autograd path
    for both depths);
  * render96_D2: a 96+96 inference render of one view at 128^2 rays on 256^2 planes with D = 2 (mlp_mode 'auto', which
    runs the SIMT kernels for D > 1).
Prints one JSON line with the milliseconds per call, the card's name and its power limit.  Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in q.split(','))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                       # noqa: BLE001 - report what could not be read, time anyway
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f'unread ({type(e).__name__})')


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_multiplane.py measures on a CUDA device'
    from oracle import renderer_oracle as orc
    from panic3d_b200.training.triplane import OSGDecoder
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    dev = torch.device('cuda:0')
    g = torch.Generator(device=dev).manual_seed(0)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=48, depth_resolution_importance=48)

    def rays(n, res):
        cams = [(0.0, -180.0 + 30.0 * i, 1.0, 30.0) for i in range(n)]
        c2w, K = zip(*(orc.camera_params_to_matrix(*c) for c in cams))
        return RaySampler()(torch.stack(c2w).to(dev), torch.stack(K).to(dev), res)

    res = {}
    ro, rd = rays(4, 64)
    for D in (1, 2):
        planes = torch.randn((4, 3, 32 * D, 256, 256), device=dev, generator=g).requires_grad_(True)
        dec = OSGDecoder(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32}).to(dev)
        r = ImportanceRenderer(use_triplane=True)
        o = dict(opts, triplane_depth=D)

        def step():
            rgb, depth, wsum, xyz = r(planes, dec, ro, rd, o)
            (rgb.mean() + depth.mean() + wsum.mean()).backward()
        res[f'train_fwd_bwd_D{D}_ms'] = round(_time(step, args.steps, args.warmup), 3)
    planes = torch.randn((1, 3, 64, 256, 256), device=dev, generator=g)
    dec = OSGDecoder(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32}).to(dev).requires_grad_(False)
    r = ImportanceRenderer(use_triplane=True)
    ro, rd = rays(1, 128)
    o = dict(orc.DEFAULT_OPTS, triplane_depth=2)
    with torch.no_grad():
        res['render96_D2_128px_ms'] = round(_time(lambda: r(planes, dec, ro, rd, o), args.steps, args.warmup), 3)
    print(json.dumps(dict(res, **_card(), steps=args.steps, warmup=args.warmup)))


if __name__ == '__main__':
    main()
