#!/usr/bin/env python
"""bench_imageio.py - the image output path (SURVEY.md 8f-4) on the eval sweep's images: 512^2 RGB + 128^2 RGBA (xyza) per view.
One JSON line:  device kernel time + HBM roofline of `p3d_image_to_png_scanlines`, and the wall-clock of saving V views
  * ours: AsyncImageWriter (device quantise + filter, pinned D2H on a side stream, zlib + file write on host threads),
          measured as (a) the time the render loop is blocked (submit only) and (b) until all files are on disk;
  * port: what `I(t).save(fn)` does (reference _util/twodee_v1.py:174-185,732-760: blocking .cpu(), clamp*255 truncate,
          PIL PNG encoder) on the calling thread - `twodee_v1` itself needs torchvision / opencv, absent from this image.
Algorithmic bytes of the kernel: 4 B read per channel value + 1 B written (+ one filter byte per row)."""
from __future__ import annotations

import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument('--views', type=int, default=64)
    ap.add_argument('--threads', type=int, default=8)
    ap.add_argument('--level', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available()
    import numpy as np
    from PIL import Image
    import panic3d_b200.imageio as pio
    dev = torch.device('cuda:0')
    V = args.views
    g = torch.Generator(device='cpu').manual_seed(0)
    lin = torch.linspace(0, 1, 512)
    yy, xx = torch.meshgrid(lin, lin, indexing='ij')
    base = torch.stack([0.5 + 0.5 * torch.sin(9 * xx + c) * torch.cos(7 * yy - c) for c in range(3)])
    imgs = (base[None] + 0.02 * torch.randn(V, 3, 512, 512, generator=g)).to(dev)           # smooth render-like content + sensor-like noise
    xyz = (torch.rand(V, 3, 128, 128, generator=g) * 0.7 - 0.35).to(dev)
    wts = torch.rand(V, 1, 128, 128, generator=g).to(dev)
    try:
        peak = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs']
    except Exception:
        peak = 3350.0                          # H100 SXM data sheet
    # kernel time, 8 views per launch, L2 flushed
    flush = torch.zeros(160 * 1024 * 1024 // 4, device=dev)
    ts = []
    for it in range(25):
        flush.add_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(2_000_000)
        e0.record(); pio.png_scanlines(imgs[:8]); e1.record()
        torch.cuda.synchronize()
        if it >= 5:
            ts.append(e0.elapsed_time(e1))
    ts.sort()
    k_ms = ts[len(ts) // 2]
    nbytes = 8 * 512 * 512 * 3 * 5 + 8 * 512
    out = {'op': 'image_output', 'views': V, 'kernel': 'k_png_scanlines', 'kernel_ms_8_views': k_ms, 'algorithmic_bytes': nbytes,
           'gbs': nbytes / k_ms * 1e-6, 'frac_of_hbm_peak': nbytes / k_ms * 1e-6 / peak, 'threads': args.threads, 'zlib_level': args.level}
    with tempfile.TemporaryDirectory() as d:
        with pio.AsyncImageWriter(threads=args.threads, level=args.level) as w:
            w.save(imgs[:2], [f'{d}/warm{i}.png' for i in range(2)]); w.flush()          # pinned staging allocated
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for v in range(V):
                w.save(imgs[v], f'{d}/rgb{v}.png')
                w.save_xyza(xyz[v:v + 1], wts[v:v + 1], 0.7, f'{d}/xyza{v}.png')
            t1 = time.perf_counter()
            w.flush()
            t2 = time.perf_counter()
        size_ours = sum(os.path.getsize(f'{d}/rgb{v}.png') for v in range(V))
        t3 = time.perf_counter()
        for v in range(V):                                                               # the reference's way, on the calling thread
            a = imgs[v].cpu().float().clamp(0, 1).mul(255).byte().permute(1, 2, 0).numpy()
            Image.fromarray(a).save(f'{d}/ref_rgb{v}.png')
            b = torch.cat([(xyz[v:v + 1] + 0.35) / 0.7, wts[v:v + 1]], dim=1)[0].cpu().float().clamp(0, 1).mul(255).byte().permute(1, 2, 0).numpy()
            Image.fromarray(b).save(f'{d}/ref_xyza{v}.png')
        t4 = time.perf_counter()
        size_ref = sum(os.path.getsize(f'{d}/ref_rgb{v}.png') for v in range(V))
        same = all(np.array_equal(np.asarray(Image.open(f'{d}/rgb{v}.png')), np.asarray(Image.open(f'{d}/ref_rgb{v}.png'))) for v in range(0, V, 7))
    out.update({'ours_render_loop_blocked_ms_per_view': (t1 - t0) / V * 1e3, 'ours_all_on_disk_ms_per_view': (t2 - t0) / V * 1e3,
                'port_blocking_ms_per_view': (t4 - t3) / V * 1e3, 'png_bytes_per_view_ours': size_ours // V, 'png_bytes_per_view_port': size_ref // V,
                'pixels_identical': bool(same), 'host_cores': os.cpu_count()})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
