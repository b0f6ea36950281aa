#!/usr/bin/env python
"""bench_png_decode.py - the device PNG decoder (`load_images`, p3d_png_decode_device) against the reference's PIL chain
`I(path).resize(512).convert('RGBA').bg('w').convert('RGB').t()`, at the training set's batch: 48 files per step
(12 per sample at batch_gpu = 4).

Inputs, generated here from seeds and written to a temporary directory (nothing in the tree is read or written): 8 views
rendered by bench.py's fused launch (bench_png_device.render_views), bilinearly up-sampled and written by the host
AsyncImageWriter (zlib level 3) as 24 RGB and 24 RGBA 512^2 files (the RGBA alpha is the render's weights, so it holds 0,
255 and values in between); and the same views at 1024^2, resized to 512 (the `resize` arm).

One JSON line per arm: the card, the decode launch sequence's device time per batch and per image (CUDA events over many
launches after warm-up, the staged buffer already pinned), the end-to-end `load_images` wall time per batch (read, inspect,
pack, one H2D copy, decode, status read-back), and the PIL chain's time per image on one host thread and on all host
cores (a process pool).  Whether host decoding limits a training step depends on the step, which is not measured here."""
from __future__ import annotations

import json
import os
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def pil_chain(path, size=512):
    """The reference's chain with PIL and torchvision's to_tensor arithmetic (torchvision is not a dependency here)."""
    from PIL import Image
    im = Image.open(path)
    im = im.resize((size, size), resample=Image.NEAREST).convert('RGBA')
    im = Image.alpha_composite(Image.new('RGBA', im.size, (255, 255, 255, 255)), im).convert('RGB')
    return torch.from_numpy(np.array(im)).permute(2, 0, 1).contiguous().float().div(255)


def _pil_many(paths):
    for p in paths:
        pil_chain(p)
    return len(paths)


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_png_decode.py needs a CUDA device')
    import bench_png_device as bpd
    import panic3d_b200.imageio as pio
    torch.set_num_threads(1)
    dev = torch.device('cuda:0')
    card = bpd._card()
    _, img, xyz, wsum, bw = bpd.render_views(dev)
    V = img.shape[0]
    cores = os.cpu_count() or 1
    with tempfile.TemporaryDirectory() as d:
        arms = {}
        for side in (512, 1024):
            rgb = torch.nn.functional.interpolate(img, size=(side, side), mode='bilinear', align_corners=False)
            alpha = torch.nn.functional.interpolate(wsum, size=(side, side), mode='bilinear', align_corners=False)
            rgba = torch.cat([rgb, alpha], 1).contiguous()
            paths = []
            with pio.AsyncImageWriter(threads=4, level=3) as w:
                for i in range(24):
                    for kind, src in (('rgb', rgb), ('rgba', rgba)):
                        fn = os.path.join(d, f'{kind}{side}_{i}.png')
                        w.save(src[i % V], fn)
                        paths.append(fn)
            arms[f'{side}_to_512'] = paths
        for arm, paths in arms.items():
            n = len(paths)
            res = {'op': 'png_decode_device', 'arm': arm, 'images': n, **card,
                   'file_bytes_per_image': sum(os.path.getsize(p) for p in paths) / n}
            out = pio.load_images(paths, size=512, white_background=True, device=dev)
            for i in (0, 1, n - 1):                                            # the same tensors as the PIL chain
                assert torch.equal(out[i].cpu(), pil_chain(paths[i])), (arm, i)
            st, _ = pio._stage(paths, 512, True, dev)
            for _ in range(args.warmup):
                pio._decode_staged(st)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                pio._decode_staged(st)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            res['device_ms_per_batch'] = ms
            res['device_ms_per_image'] = ms / n
            t0 = time.perf_counter()
            for _ in range(args.steps):
                pio.load_images(paths, size=512, white_background=True, device=dev)
            res['load_images_wall_ms_per_batch'] = (time.perf_counter() - t0) / args.steps * 1e3
            _pil_many(paths[:4])
            t0 = time.perf_counter()
            _pil_many(paths)
            res['pil_1_thread_ms_per_image'] = (time.perf_counter() - t0) / n * 1e3
            with ProcessPoolExecutor(cores) as ex:
                list(ex.map(_pil_many, [paths[k::cores] for k in range(cores)]))              # workers started
                t0 = time.perf_counter()
                list(ex.map(_pil_many, [paths[k::cores] for k in range(cores)]))
                res['pil_all_cores_ms_per_image'] = (time.perf_counter() - t0) / n * 1e3
            res['host_cores'] = cores
            print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
