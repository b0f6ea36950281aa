#!/usr/bin/env python
"""bench_mesh.py - the eval's geometry stage (generate.py:97-103 -> eg3d_metrics3d.marching_cubes) at the eval size, 256^3.
Not the headline bench (that is bench.py).  One JSON line per arm:

    python bench_mesh.py                      # ours: panic3d_b200.mesh on the device
    python bench_mesh.py --impl reference     # the reference's route: host copies + host marching cubes + colour loop

Workload.  Random tri-planes through a random decoder give a noise surface whose size says nothing about a real subject,
so the marching-cubes timings use a seeded head-sized blob: a density 1 / (1 + exp(d - r)) around a sphere of radius
0.35 R voxels whose radius is modulated by a few seeded low-frequency harmonics (a closed, bumpy surface, ~0.3 M
triangles at 256^3).  The end-to-end ``extract_mesh`` figure uses seeded 512^2 tri-planes with the sigma bias, crop and
cull of tests/golden/cases.py VOLUME_CASES['vol_crop_cull16'], and is labelled with its own V / F.

    ours       mc_ms             p3d_mc_count + CUB scan + p3d_mc_emit on the resident volume (mesh_index)
               marching_cubes_ms the drop-in on CUDA tensors, including the device -> host copies of the result
               extract_ms        extract_mesh: volume query without colours, the two passes, lattice coordinates, decode
                                 of the vertex colours, result copies
    reference  d2h_ms            vol['densities'].cpu() + vol['rgbs'].cpu() (the whole 32-channel colour volume, as
                                 generate.py:99-100 does)
               host_mc_ms        skimage's Lewiner marching cubes when importable, else this project's numpy oracle
                                 (oracle/mesh_oracle.py), named in 'kind'
               colour_loop_ms    the reference's per-vertex list comprehension (eg3d_metrics3d.py:197-200)

Timing: CUDA events, warm-ups, median, for the device arm; a host clock around synchronised work for the reference arm
(its host stages run once: they take seconds).  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        limit = float(out.splitlines()[0])
    except Exception:
        limit = None
    return name, limit


def blob(R, dev, seed=0):
    """Seeded head-sized blob: density 1 / (1 + exp(d - r(theta, phi))) with r = 0.35 R (1 + bumps)."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    coef = (torch.rand(6, generator=g) - 0.5) * 0.16
    lin = torch.arange(R, dtype=torch.float32, device=dev) - (R - 1) / 2
    a, b, c = torch.meshgrid(lin, lin, lin, indexing='ij')
    d = torch.sqrt(a * a + b * b + c * c)
    theta = torch.atan2(b, c)
    phi = torch.acos(torch.clamp(a / torch.clamp(d, min=1e-6), -1, 1))
    bumps = (coef[0] * torch.cos(2 * theta) + coef[1] * torch.sin(3 * theta) + coef[2] * torch.cos(2 * phi)
             + coef[3] * torch.sin(3 * phi) * torch.cos(theta) + coef[4] * torch.cos(4 * phi) + coef[5] * torch.sin(5 * theta) * torch.sin(phi))
    r = 0.35 * R * (1 + bumps)
    return torch.sigmoid(r - d).contiguous()


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(2_000_000)           # enqueue behind device idle-spin: device time, not launch latency
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def planes_case(dev, P):
    from oracle import renderer_oracle as orc
    from tests.golden.cases import VOLUME_CASES
    from panic3d_b200.training.triplane import OSGDecoder
    case = dict(VOLUME_CASES['vol_crop_cull16'], P=P, seed=7)
    o = case['opts']
    planes, dec, _, _, _, _ = orc.synth_inputs(case['seed'], 1, 1, 2, 0, P, cameras=None)
    d = OSGDecoder(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32})
    with torch.no_grad():
        d.net[0].weight.copy_(dec['w1']); d.net[0].bias.copy_(dec['b1'])
        d.net[2].weight.copy_(dec['w2']); d.net[2].bias.copy_(dec['b2'])
        d.net[2].bias[0] += case['sigma_bias']
    return planes.to(dev), d.to(dev).requires_grad_(False), dict(o), case


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--res', type=int, default=256)
    ap.add_argument('--planes', type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_mesh.py needs a CUDA device'
    dev = torch.device('cuda:0')
    R, bw = args.res, 0.7
    name, limit = card()
    dens = blob(R, dev)
    line = {'op': 'marching_cubes', 'impl': args.impl, 'res': R, 'workload': 'seeded head-sized blob, level 0.5',
            'card': name, 'power_limit_w': limit}
    if args.impl == 'reference':
        rgbs = torch.rand((1, 32, R, R, R), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        vol = {'densities': dens[None, None], 'rgbs': rgbs}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        d_np = vol['densities'].cpu().numpy()[0, 0]
        r_np = vol['rgbs'].cpu().numpy()[0, :3]
        t1 = time.perf_counter()
        try:
            import skimage.measure
            kind = 'skimage lewiner'
            mc_vert, mc_face, _, _ = skimage.measure.marching_cubes(d_np, level=0.5, spacing=(1.0, 1.0, 1.0),
                                                                   gradient_direction='descent', step_size=1,
                                                                   allow_degenerate=False, method='lewiner')
        except ImportError:
            from oracle import mesh_oracle as mo
            kind = 'numpy oracle (skimage not importable)'
            m = mo.marching_cubes_index(d_np, 0.5)
            mc_vert, mc_face = m['verts'], m['faces']
        t2 = time.perf_counter()
        mc_color = np.stack([r_np[:3, a, b, c] for a, b, c in mc_vert.astype(int)])
        t3 = time.perf_counter()
        line.update(kind=kind, V=int(len(mc_vert)), F=int(len(mc_face)), bytes_to_host=int(d_np.nbytes + vol['rgbs'].numel() * 4),
                    d2h_ms=(t1 - t0) * 1e3, host_mc_ms=(t2 - t1) * 1e3, colour_loop_ms=(t3 - t2) * 1e3,
                    ms=(t3 - t0) * 1e3, colour_checksum=float(mc_color.astype(np.float64).sum()))
    else:
        import panic3d_b200.mesh as pm
        import panic3d_b200.volume as pv
        from panic3d_b200 import _lib
        rgbs3 = torch.rand((3, R, R, R), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        with torch.no_grad():
            n0 = _lib.launch_count()
            m = pm.mesh_index(dens)
            launches = _lib.launch_count() - n0
            V, F = m['verts'].shape[0], m['faces'].shape[0]
            ws_bytes = int(_lib.lib().p3d_mc_workspace_bytes(R, R, R))
            mc_ms = timeit(lambda: pm.mesh_index(dens))
            mcd_ms = timeit(lambda: pm.marching_cubes(dens, rgbs3, bw))
            planes, dec, opts, case = planes_case(dev, args.planes)
            kw = dict(resolution=R, triplane_crop=case['triplane_crop'], cull_clouds=case['cull_clouds'])
            e = pm.extract_mesh(planes, dec, opts, **kw)
            ex_ms = timeit(lambda: pm.extract_mesh(planes, dec, opts, **kw), iters=10)
            q_ms = timeit(lambda: pv.query_volume(planes, dec, opts, want_rgb=False, want_coordinates=False, **kw), iters=10)
            qrgb_ms = timeit(lambda: pv.query_volume(planes, dec, opts, want_coordinates=False, **kw), iters=10)
        # HBM bytes the two passes need at least: the volume read twice, the packed counts written, scanned (read + write)
        # and read back, the outputs written
        nn = R ** 3
        nbytes = 2 * nn * 4 + 4 * nn * 8 + V * (12 + 12 + 4 + 8) + F * 12
        line.update(kind='p3d_mc_count + CUB scan + p3d_mc_emit', V=V, F=F, gpu_launches=launches, workspace_bytes=ws_bytes,
                    mc_ms=mc_ms, mc_min_bytes=nbytes, mc_gbs=nbytes / mc_ms * 1e-6, marching_cubes_ms=mcd_ms,
                    extract_workload=f'seeded {args.planes}^2 tri-planes, sigma bias {case["sigma_bias"]}, crop {case["triplane_crop"]}, '
                                     f'cull {case["cull_clouds"]}', extract_V=int(len(e['verts'])), extract_F=int(len(e['faces'])),
                    extract_ms=ex_ms, volume_query_no_rgb_ms=q_ms, volume_query_with_rgb_ms=qrgb_ms, ms=mc_ms)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
