#!/usr/bin/env python
"""bench_paste.py - the front-view paste (SURVEY.md 8f-3) at the eval size: N views x 128^2 render outputs -> 512^2 images,
thresholds of _scripts/eval/generate.py:59-65.  Not the driver's bench (that is bench.py).  One JSON line per arm:

    python bench_paste.py                      # ours: panic3d_b200.paste.paste_front (p3d_paste_front, one launch)
    python bench_paste.py --impl reference     # the UNMODIFIED reference paste_front of baseline/_ref, eager PyTorch on the same GPU

Both arms run `paste_front(G, x, out, **paste_params)` on the same seeded inputs with the same stand-in `G` whose `f` returns
fixed results for the extra occlusion render (the renders themselves are the renderer's business, measured by bench.py), so
the timed work is the mask / lookup / blend pipeline + the ray construction.  kornia is not installed in this image: the
reference arm imports the two kornia functions it needs from their restatement in oracle/paste_oracle.py (reference-arm
infrastructure, like bench.py's cpu_baseline leg; the product arm never touches oracle/).

Algorithmic HBM bytes per output pixel (fp32): image 12 + front image 12 read, image 12 + paste 12 + mask 4 + five part masks
20 written = 72 B (+ the 128^2 render outputs, 0.3 % of that).  Timing: CUDA events, 5 warm-ups, median of 30, an L2-sized
buffer is written between iterations.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PARAMS = dict(mode='default', thresh_weight=0.95, thresh_edges=0.02, thresh_occ=0.05, offset_occ=0.01, thresh_dxyz=0.000005)


def synth(N, R, S, dev):
    """Smooth front-facing surface, soft silhouette, half the rays slightly off their point (every mask has both values)."""
    g = torch.Generator(device='cpu').manual_seed(0)
    lin = (torch.arange(R, dtype=torch.float32) + 0.5) / R
    yy, xx = torch.meshgrid(lin, lin, indexing='ij')
    xyz = torch.stack([(0.5 - xx) * 0.63, (0.5 - yy) * 0.63, 0.08 * torch.sin(5 * xx) * torch.cos(4 * yy) + 0.12 * (xx + 0.3 * yy > 0.9)])
    xyz = xyz[None].repeat(N, 1, 1, 1) + 0.001 * torch.randn(N, 3, R, R, generator=g)
    r2 = (xx - 0.5) ** 2 + (yy - 0.5) ** 2
    wts = torch.sigmoid((0.17 - r2) * 60)[None, None].repeat(N, 1, 1, 1)
    occ = torch.rand(N, 1, R, R, generator=g) * 0.1
    p = xyz * torch.tensor([-1., 1., -1.])[None, :, None, None]
    rd = torch.zeros(N, 3, R, R); rd[:, 2] = -1
    ro = p - rd * 0.8 + torch.randn(N, 3, R, R, generator=g) * 6e-6 * (torch.rand(N, 1, R, R, generator=g) < 0.5)
    t = dict(image=torch.rand(N, 3, S, S, generator=g) * 2 - 1, front=torch.rand(N, 3, S, S, generator=g), xyz=xyz, wts=wts, occ=occ, ro=ro, rd=rd)
    return {k: v.to(dev).contiguous() for k, v in t.items()}


class StandInG:
    def __init__(self, occ):
        self.rendering_kwargs = {'ray_start': 0.5, 'box_warp': 0.7}
        self.occ = occ

    def f(self, xin, return_more=False):
        return {'image_weights': self.occ}


def timeit(fn, flush, iters=30, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.add_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(2_000_000)           # the host enqueues fn() behind ~1 ms of device idle-spin: device time, not launch latency
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--views', type=int, default=8)
    ap.add_argument('--render', type=int, default=128)
    ap.add_argument('--image', type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_paste.py needs a CUDA device'
    dev = torch.device('cuda:0')
    N, R, S = args.views, args.render, args.image
    d = synth(N, R, S, dev)
    G = StandInG(d['occ'])
    x = {'cond': {'image_ortho_front': d['front']}, 'normalize_images': False, 'paste_params': dict(PARAMS),
         'force_rays': {'ray_origins': d['ro'], 'ray_directions': d['rd']}}
    out = {'image': d['image'], 'image_xyz': d['xyz'], 'image_weights': d['wts']}
    flush = torch.zeros(160 * 1024 * 1024 // 4, device=dev)
    try:
        peak, peak_src = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'], 'measured'
    except Exception:
        peak, peak_src = 3350.0, 'H100 SXM data sheet'
    nbytes = N * S * S * 72 + N * R * R * 4 * (3 + 1 + 1 + 3 + 3)
    line = {'op': 'paste_front', 'impl': args.impl, 'views': N, 'render': R, 'image': S, 'algorithmic_bytes': nbytes, 'hbm_peak_gbs': peak,
            'hbm_peak_source': peak_src}
    if args.impl == 'reference':
        from baseline import ref_env
        ref_env.setup()
        from oracle.paste_oracle import kornia_shim                            # reference arm only: kornia is absent from this image
        k = kornia_shim()
        sys.modules['kornia'], sys.modules['kornia.filters'], sys.modules['kornia.morphology'] = k, k.filters, k.morphology
        import training.triplane as ref_tp
        fn = lambda: ref_tp.paste_front(G, x, out, **PARAMS)
        with torch.no_grad():
            res = fn()
            ms = timeit(fn, flush)
        line.update(ms=ms, kernel='eager PyTorch (~35 launches)')
    else:
        import panic3d_b200.paste as pp
        from panic3d_b200 import _lib
        fn = lambda: pp.paste_front(G, x, out, **PARAMS)
        with torch.no_grad():
            n0 = _lib.launch_count()
            res = fn()
            launches = _lib.launch_count() - n0
            ms = timeit(fn, flush)
            occ_ro, occ_rd = pp.occlusion_rays(d['xyz'], 0.5, 0.01)
            fused = lambda: pp.paste_front_fused(d['image'], d['xyz'], d['wts'], d['front'], d['occ'], d['ro'], d['rd'], 0.7,
                                                 thresh_dxyz=PARAMS['thresh_dxyz'])
            ms_k = timeit(fused, flush)
            lean = lambda: pp.paste_front_fused(d['image'], d['xyz'], d['wts'], d['front'], d['occ'], d['ro'], d['rd'], 0.7,
                                                thresh_dxyz=PARAMS['thresh_dxyz'], want_parts=False)
            ms_lean = timeit(lean, flush)
        line.update(ms=ms, gpu_launches=launches, kernel='k_paste_front', kernel_ms=ms_k, gbs=nbytes / ms_k * 1e-6,
                    frac_of_hbm_peak=nbytes / ms_k * 1e-6 / peak, kernel_ms_without_part_masks=ms_lean,
                    gbs_without_part_masks=(nbytes - N * S * S * 20) / ms_lean * 1e-6)
    line.update(views_per_s=N / ms * 1e3, mask_mean=float(res['mask'].mean()), image_checksum=float(res['image'].double().sum()))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
