#!/usr/bin/env python
"""bench_png_device.py - the device PNG encoder (p3d_png_encode_device) against the host zlib path, on eval-shaped views.

Inputs, all generated here from seeds (no file is read):
  * 8 views rendered by bench.py's fused launch (8 views x 128^2 rays x 96+96 samples, 512^2 x 32-ch tri-planes): their
    128^2 RGBA xyza images (xyz and weights, as generate.py saves them) and 512^2 RGB images (the rendered colours,
    bilinearly up-sampled to the eval image size);
  * for context, a flat-background 512^2 RGB image and 512^2 RGB uniform noise.
One JSON line: the card, the render's device time per view (CUDA events, same call), the encoder's device time per view
(CUDA events over many launches after warm-up) and its share of the render's, host core time per view of zlib levels 1, 3
and 6 (p3d_png_encode_host on this thread), the host time per view of the device path (D2H wait + file write, one writer
thread) and of the host path (D2H wait + zlib + file write), and the file sizes of both paths.  The share of the full eval
sweep (super-resolution, paste, mesh) is not measured here; bench_config3.py --save runs that sweep.  Writes only to a
temporary directory."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in q.split(','))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                       # noqa: BLE001 - report what could not be read, time anyway
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f'unread ({type(e).__name__})')


def _events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def render_views(dev):
    """bench.py's flagship render (fused kernel, default settings) on seeded planes; returns its ms per launch and outputs."""
    import bench
    from panic3d_b200 import cameras
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    from panic3d_b200.training.triplane import OSGDecoder
    V, R = bench.VIEWS, bench.R
    torch.manual_seed(1234)
    planes = torch.randn(V, 3, bench.C, bench.P, bench.P, device=dev)
    decoder = OSGDecoder(bench.C, {'decoder_lr_mul': 1, 'decoder_output_dim': 32}).to(dev).requires_grad_(False)
    spin = cameras.cam60[cameras.camsubs['spin12']]
    labels = torch.stack([cameras.camera_params_to_matrix(elev=float(spin[i % 12][0]), azim=float(spin[i % 12][1]), dist=1.0,
                                                          fov=30.0)['camera_label'] for i in range(V)]).to(dev)
    renderer, sampler = ImportanceRenderer(use_triplane=True), RaySampler()
    ro, rd = sampler(labels[:, :16].view(-1, 4, 4), labels[:, 16:25].view(-1, 3, 3), R)
    out = {}

    def step():
        renderer._planes.key = None                                  # distinct tri-planes every step, as bench.py
        with torch.no_grad():
            out['r'] = renderer(planes, decoder, ro, rd, dict(bench.RENDER_OPTS))
    ms = _events(step, 10, 3)
    rgb, depth, wsum, xyz = out['r']
    img = torch.nn.functional.interpolate(rgb[..., :3].permute(0, 2, 1).reshape(V, 3, R, R), size=(512, 512), mode='bilinear',
                                          align_corners=False) * 0.5 + 0.5
    xyz = xyz.permute(0, 2, 1).reshape(V, 3, R, R).contiguous()
    wsum = wsum.permute(0, 2, 1).reshape(V, 1, R, R).contiguous()
    return ms / V, img.contiguous(), xyz, wsum, bench.RENDER_OPTS['box_warp']


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_png_device.py needs a CUDA device')
    import panic3d_b200.imageio as pio
    from panic3d_b200 import _lib
    L = _lib.lib()
    dev = torch.device('cuda:0')
    res = {'op': 'png_encode_device', **_card()}
    render_ms, img, xyz, wsum, bw = render_views(dev)
    res['render_ms_per_view'] = render_ms
    g = torch.Generator(device='cpu').manual_seed(5)
    flat = torch.full((8, 3, 512, 512), 0.9)
    flat[:, :, 200:300, 200:300] = 0.2
    noise = torch.rand(8, 3, 512, 512, generator=g)
    cases = {
        'rgb512': pio.png_scanlines(img),
        'xyza128': pio.png_scanlines(xyz, extra=wsum, scale=[1.0 / bw] * 3 + [1.0], shift=[bw / 2] * 3 + [0.0]),
        'flat512': pio.png_scanlines(flat.to(dev)),
        'noise512': pio.png_scanlines(noise.to(dev)),
    }
    torch.cuda.synchronize()
    for name, (scan, shape) in cases.items():
        H, W, c = shape
        n = scan.shape[0]
        dev_ms = _events(lambda: pio.png_encode_device(scan, shape), args.steps, 5) / n
        files, lens = pio.png_encode_device(scan, shape)
        lens = lens.cpu().tolist()
        host_scan = scan.cpu().numpy()
        r = {'shape': [H, W, c], 'raw_bytes_per_view': int(scan.shape[1]), 'device_ms_per_view': dev_ms,
             'device_share_of_render': dev_ms / render_ms, 'device_bytes_per_view': sum(lens) / n}
        for level in (1, 3, 6):
            cap = L.p3d_png_encode_bound(H, W, c)
            buf = np.empty(cap, np.uint8)
            nb = C.c_size_t(0)
            t0 = time.process_time()
            size = 0
            for i in range(n):
                _lib.check(L.p3d_png_encode_host(host_scan[i].ctypes.data, H, W, c, level, buf.ctypes.data, cap, C.byref(nb)))
                size += nb.value
            r[f'zlib{level}_host_ms_per_view'] = (time.process_time() - t0) / n * 1e3
            r[f'zlib{level}_bytes_per_view'] = size / n
        with tempfile.TemporaryDirectory() as d:
            for enc in ('device', 'host'):
                with pio.AsyncImageWriter(threads=1, level=3, encoder=enc) as w:
                    w._submit(scan, shape, [f'{d}/warm{i}.png' for i in range(n)]); w.flush()    # pinned staging allocated
                    if enc == 'device':
                        files, lens_t = pio.png_encode_device(scan, shape)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for i in range(n):
                        fn = f'{d}/{enc}{i}.png'.encode()
                        if enc == 'device':
                            _lib.check(L.p3d_png_writer_submit_encoded(w._h, files[i].data_ptr(), lens_t[i:].data_ptr(), H, W, c, fn,
                                                                       torch.cuda.current_stream().cuda_stream))
                        else:
                            _lib.check(L.p3d_png_writer_submit(w._h, scan[i].data_ptr(), H, W, c, fn, torch.cuda.current_stream().cuda_stream))
                    w.flush()
                    r[f'{enc}_path_host_ms_per_view'] = (time.perf_counter() - t0) / n * 1e3
        res[name] = r
    res['note'] = ('device_share_of_render is the encoder against the fused render launch alone; the eval sweep share '
                   '(super-resolution, paste, mesh included) is not measured unless bench_config3.py --save is run')
    print(json.dumps(res))


if __name__ == '__main__':
    main()
