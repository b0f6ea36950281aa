#!/usr/bin/env python
"""bench_ops.py - HBM-roofline measurement of the three StyleGAN ops on the shapes panic3d's path hits
(SURVEY.md section 8a12-a14).  Not the driver's bench (that is bench.py); this produces the per-op numbers quoted in
One JSON line per case:

    {"op": ..., "case": ..., "dtype": ..., "ms": ..., "algorithmic_bytes": ..., "gbs": ..., "frac_of_hbm_peak": ...}

algorithmic bytes = every input element read once + every output element written once (filters/biases ignored).
Timing: CUDA events, >= 5 warm-ups, median of 20; inputs are larger than L2 or an L2-sized buffer is written between
iterations (`flush`).
"""
from __future__ import annotations

import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def hbm_peak():
    try:
        return json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'], 'measured'
    except Exception:
        return 3350.0, 'H100 SXM data sheet'


def timeit(fn, flush_buf, iters=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush_buf is not None:
            flush_buf.add_(1)                      # evict: write a buffer larger than L2
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(2_000_000)               # ~1 ms of GPU idle-spin: the host enqueues fn() behind it, so the
        e0.record()                                # bracket sees device time only, not Python/ctypes launch latency
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument('--only', default='', help='substring filter on "op case"')
    ap.add_argument('--dtypes', default='float16,float32')
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'],
                    help="reference: the UNMODIFIED ops of baseline/_ref with their own JIT CUDA plugins (prebuilt by baseline/install_ref.sh), "
                         "timed on the same GPU for the per-op comparison")
    args = ap.parse_args()
    if args.impl == 'reference':
        from baseline import ref_env
        ref_env.setup()
        from torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu
        assert 'baseline/_ref' in bias_act.__file__.replace(os.sep, '/')
    else:
        import panic3d_b200  # noqa: F401
        from panic3d_b200.torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu
    dev = torch.device('cuda:0')
    peak, src = hbm_peak()
    flush = torch.zeros(192 * 1024 * 1024 // 4, device=dev)          # 192 MB > 50 MB L2
    f4 = upfirdn2d.setup_filter([1, 3, 3, 1], device=dev)
    f12 = upfirdn2d.setup_filter(torch.hann_window(14)[1:-1].numpy(), device=dev)   # 12 taps, separable
    out = []

    def rec(op, case, dtype, x_elems, y_elems, fn):
        if args.only and args.only not in f'{op} {case}':
            return
        esz = torch.finfo(dtype).bits // 8
        ms = timeit(fn, flush)
        byts = (x_elems + y_elems) * esz
        r = {'impl': args.impl, 'op': op, 'case': case, 'dtype': str(dtype).split('.')[-1], 'ms': round(ms, 4), 'algorithmic_bytes': byts,
             'gbs': round(byts / ms / 1e6, 1), 'frac_of_hbm_peak': round(byts / ms / 1e6 / peak, 3), 'peak': f'{peak} GB/s ({src})'}
        out.append(r)
        print(json.dumps(r), flush=True)

    with torch.no_grad():
        for dtype in [getattr(torch, d) for d in args.dtypes.split(',')]:
            # a12: lrelu + clamp 256 on conv outputs up to (N,128,512,512) (networks_stylegan2.py:352); linear+clamp ToRGB
            x = torch.randn(4, 128, 512, 512, device=dev, dtype=dtype)
            b = torch.randn(128, device=dev, dtype=dtype)
            rec('bias_act', 'lrelu clamp256 (4,128,512,512) NCHW', dtype, x.numel(), x.numel(), lambda: bias_act.bias_act(x, b, act='lrelu', clamp=256))
            xcl = x.contiguous(memory_format=torch.channels_last)
            rec('bias_act', 'lrelu clamp256 (4,128,512,512) channels_last', dtype, x.numel(), x.numel(), lambda: bias_act.bias_act(xcl, b, act='lrelu', clamp=256))
            del x, xcl
            x = torch.randn(8, 96, 256, 256, device=dev, dtype=dtype)     # tri-plane ToRGB: linear + clamp
            b = torch.randn(96, device=dev, dtype=dtype)
            rec('bias_act', 'linear clamp256 (8,96,256,256)', dtype, x.numel(), x.numel(), lambda: bias_act.bias_act(x, b, act='linear', clamp=256))
            del x
            # a13: 4x4 [1,3,3,1] at up1/down1 after the transposed conv, up2 for the skip image, down2 in D
            x = torch.randn(4, 128, 513, 513, device=dev, dtype=dtype)
            y = upfirdn2d.upfirdn2d(x, f4, padding=[1, 1, 1, 1], gain=4.0)
            rec('upfirdn2d', 'blur 4x4 up1/down1 (4,128,513,513)', dtype, x.numel(), y.numel(), lambda: upfirdn2d.upfirdn2d(x, f4, padding=[1, 1, 1, 1], gain=4.0))
            del x, y
            x = torch.randn(8, 96, 128, 128, device=dev, dtype=dtype)
            y = upfirdn2d.upsample2d(x, f4, up=2)
            rec('upfirdn2d', 'upsample2d 4x4 up2 (8,96,128,128)', dtype, x.numel(), y.numel(), lambda: upfirdn2d.upsample2d(x, f4, up=2))
            del x, y
            x = torch.randn(4, 128, 512, 512, device=dev, dtype=dtype)
            y = upfirdn2d.downsample2d(x, f4, down=2)
            rec('upfirdn2d', 'downsample2d 4x4 down2 (4,128,512,512)', dtype, x.numel(), y.numel(), lambda: upfirdn2d.downsample2d(x, f4, down=2))
            xcl = x.contiguous(memory_format=torch.channels_last)
            rec('upfirdn2d', 'downsample2d 4x4 down2 (4,128,512,512) channels_last', dtype, x.numel(), y.numel(), lambda: upfirdn2d.downsample2d(xcl, f4, down=2))
            del x, xcl, y
            # a14: StyleGAN3-style layer (not executed by panic3d; measured for completeness)
            x = torch.randn(4, 128, 128, 128, device=dev, dtype=dtype)
            b = torch.randn(128, device=dev, dtype=dtype)
            y = filtered_lrelu.filtered_lrelu(x, f12, f12, b, up=2, down=2, padding=[9, 10, 9, 10], clamp=256)
            rec('filtered_lrelu', 'up2 down2 12-tap (4,128,128,128)', dtype, x.numel(), y.numel(),
                lambda: filtered_lrelu.filtered_lrelu(x, f12, f12, b, up=2, down=2, padding=[9, 10, 9, 10], clamp=256))
            del x, y
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, 'gpurun_out', 'bench_ops.json' if args.impl == 'ours' else 'bench_ops_ref.json'), 'w'), indent=1)


if __name__ == '__main__':
    main()
