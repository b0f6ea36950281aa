#!/usr/bin/env python
"""The fp32 training convolutions (panic3d_b200.conv) against cuDNN on every convolution of the 256^2 backbone at batch 4
(channel_base 32768, channel_max 512: conv0 = conv_transpose2d 3/2/0 of each up block, conv1 = conv2d 3/1/1, ToRGB =
conv2d 1x1 to 96 channels), for the three GEMMs of a training step: forward, input gradient and weight gradient.

Arms: ours (3xTF32 on wgmma); cudnn_fp32 (TF32 off, cudnn.benchmark on: the training loop's setting); cudnn_tf32 (TF32 on,
for context only - it is not fp32-accurate).  Device time per call from CUDA events: --warmup calls, then --rounds timed
windows of --reps calls each, median window.  Prints one JSON line per layer and a summary line with the GPU and its
power limit; `faster` lists the layers where ours beat cudnn_fp32 over forward + input gradient + weight gradient."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))


def layers(batch):
    ch = lambda r: min(32768 // r, 512)
    out = [('b4_conv1', False, 512, 512, 4, 3, 1, 1), ('b4_torgb', False, 512, 96, 4, 1, 1, 0)]
    for r in (8, 16, 32, 64, 128, 256):
        out += [(f'b{r}_conv0', True, ch(r // 2), ch(r), r // 2, 3, 2, 0), (f'b{r}_conv1', False, ch(r), ch(r), r, 3, 1, 1),
                (f'b{r}_torgb', False, ch(r), 96, r, 1, 1, 0)]
    return [(name, tr, batch, cin, cout, h, k, s, p) for name, tr, cin, cout, h, k, s, p in out]


def gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--only', default=None, help='comma-separated layer names')
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_conv.py measures on the GPU; no CUDA device found')
    import panic3d_b200.conv as pc
    dev = torch.device('cuda:0')
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = False

    def timeit(fn):
        for _ in range(args.warmup):
            fn()
        ts = []
        for _ in range(args.rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / args.reps)
        return statistics.median(ts)

    only = set(args.only.split(',')) if args.only else None
    faster, rows = [], []
    for name, tr, n, cin, cout, h, k, s, p in layers(args.batch):
        if only and name not in only:
            continue
        g = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(n, cin, h, h, generator=g, device=dev)
        wshape = (cin, cout, k, k) if tr else (cout, cin, k, k)
        w = torch.randn(wshape, generator=g, device=dev) / (cin * k * k) ** 0.5
        prm = pc.make_params(x.shape, w.shape, s, p, tr)
        y = pc.run_forward(prm, x, w)
        dy = torch.randn(y.shape, generator=g, device=dev)
        # the input gradient is the opposite-transpose op on dy (conv2d_gradfix.py:95-104 for its output_padding)
        op = 0 if tr else h - (y.shape[2] - 1) * s - (1 - 2 * p) - (k - 1)
        prm_in = pc.make_params(dy.shape, w.shape, s, p, not tr, op)
        aten = lambda mask: torch.ops.aten.convolution_backward(dy, x, w, None, [s, s], [p, p], [1, 1], tr, [0, 0], 1, mask)
        fwd_t = (lambda: torch.nn.functional.conv_transpose2d(x, w, stride=s, padding=p)) if tr else \
                (lambda: torch.nn.functional.conv2d(x, w, stride=s, padding=p))
        row = {'layer': name, 'shape': {'transpose': tr, 'N': n, 'Cin': cin, 'Cout': cout, 'H': h, 'k': k, 'stride': s, 'padding': p},
               'gflop_per_gemm': pc.flops(prm) / 1e9, 'ms': {}}
        row['ms']['ours'] = {'forward': timeit(lambda: pc.run_forward(prm, x, w)),
                             'input_grad': timeit(lambda: pc.run_forward(prm_in, dy, w)),
                             'weight_grad': timeit(lambda: pc.run_weight_grad(prm, x, dy))}
        for arm, tf32 in (('cudnn_fp32', False), ('cudnn_tf32', True)):
            torch.backends.cudnn.allow_tf32 = tf32
            row['ms'][arm] = {'forward': timeit(fwd_t), 'input_grad': timeit(lambda: aten([True, False, False])),
                              'weight_grad': timeit(lambda: aten([False, True, False]))}
        torch.backends.cudnn.allow_tf32 = False
        tot = {a: sum(v.values()) for a, v in row['ms'].items()}
        row['ms_total'] = tot
        row['tflops_ours'] = 3 * pc.flops(prm) / (tot['ours'] * 1e-3) / 1e12
        row['speedup_vs_fp32'] = tot['cudnn_fp32'] / tot['ours']
        if tot['ours'] < tot['cudnn_fp32']:
            faster.append(name)
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({'summary': True, 'gpu': gpu_info(), 'batch': args.batch, 'faster': faster,
                      'ms_total': {a: sum(r['ms_total'][a] for r in rows) for a in ('ours', 'cudnn_fp32', 'cudnn_tf32')}}))


if __name__ == '__main__':
    main()
