#!/usr/bin/env python
"""bench_gather.py - what the tri-plane gather's memory traffic costs the fused renderer (k_render_ws3).

    python bench_gather.py [--rounds K] [--launches L]       GPU: time one fused launch per arm, arms alternated
    python bench_gather.py --model                           CPU: L2 line requests of the coarse pass, per ray order

GPU arms, all on bench.py's workload (8 views of spin12 at elevation 0, 128x128 rays, 96+96 samples, the same seeded
decoder, Philox jitter) with channels-last planes, so that no layout pass runs; the kernel is timed alone (profile slot 5,
CUDA events around each launch), `--launches` launches per arm and round after a warm-up:
  * P512 fp32     the bench's 3x512x512x32 fp32 tri-planes;
  * P512 bf16     the same with bf16 storage: half the bytes per texel line;
  * P8 fp32       8x8 planes: every tap hits one of a few lines, so the instruction stream is that of the P512 arm and
                  almost nothing reaches L2.  P512 - P8 is what the gather's memory traffic costs.

--model replays the coarse-pass tap footprints of the same cameras on the CPU - depths from the Philox uniforms
(oracle/philox.py), points and plane coordinates from oracle/renderer_oracle.py - and counts, per ray order (which rays
form a group) and per row -> load-instruction assignment, the 128 B lines requested, the distinct lines per warp load
instruction (what one instruction asks L2 for) and the distinct lines per 128-row tile."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

R, VIEWS, C = 128, 8, 32
OPTS = dict(box_warp=0.7, ray_start=0.5, ray_end=1.5, depth_resolution=96, depth_resolution_importance=96,
            disparity_space_sampling=False, clamp_mode='softplus', white_back=True)


def spin_views(n):
    from panic3d_b200 import cameras
    spin = cameras.cam60[cameras.camsubs['spin12']]
    return [(float(spin[i % 12][0]), float(spin[i % 12][1])) for i in range(n)]


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except Exception as e:                                   # the timing stands; the card line says what is missing
        return f'nvidia-smi unavailable ({e})'


# ------------------------------------------------------------------------------------------------------ GPU
def run_gpu(args):
    import ctypes as Ct
    import torch
    from panic3d_b200 import _lib, cameras
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    from panic3d_b200.training.triplane import OSGDecoder

    assert torch.cuda.is_available(), 'the GPU arms need a CUDA device (use --model on the CPU)'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    L = _lib.lib()
    torch.manual_seed(1234)
    decoder = OSGDecoder(C, {'decoder_lr_mul': 1, 'decoder_output_dim': 32}).to(dev).requires_grad_(False)
    labels = torch.stack([cameras.camera_params_to_matrix(elev=e, azim=a, dist=1.0, fov=30.0)['camera_label']
                          for e, a in spin_views(VIEWS)]).to(dev)
    ro, rd = RaySampler()(labels[:, :16].view(-1, 4, 4), labels[:, 16:25].view(-1, 3, 3), R)
    ro, rd = ro.float().contiguous(), rd.float().contiguous()
    N, M = ro.shape[:2]

    arms = []
    for label, P, bf16 in (('P512 fp32', 512, False), ('P512 bf16', 512, True), ('P8 fp32', 8, False)):
        g = torch.Generator(device=dev).manual_seed(99)
        cl = torch.randn(N, 3, P, P, C, device=dev, generator=g, dtype=torch.float32)
        cl = cl.to(torch.bfloat16) if bf16 else cl
        r = ImportanceRenderer(use_triplane=True)
        r.planes_bf16, r.mlp_mode = bf16, _lib.P3D_MLP_TC_3XBF16
        planes_cl = r._planes_cl(cl.permute(0, 1, 4, 2, 3))                  # channels-last texels: a zero-copy view
        assert planes_cl.data_ptr() == cl.data_ptr()
        p, wts = r._params(planes_cl, N, M, OPTS, decoder, None, None, None)
        p.seed = 0x5EED
        wt = [t.detach().float().contiguous() for t in wts]
        ws = torch.empty(int(L.p3d_render_workspace_bytes(Ct.byref(p))), dtype=torch.uint8, device=dev)
        out = [torch.empty(s, device=dev) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]

        def launch(p=p, planes_cl=planes_cl, wt=wt, ws=ws, out=out):
            _lib.check(L.p3d_render_forward(Ct.byref(p), planes_cl.data_ptr(), *[t.data_ptr() for t in wt], ro.data_ptr(),
                                            rd.data_ptr(), None, None, ws.data_ptr(), ws.numel(),
                                            *[o.data_ptr() for o in out], _lib.stream_ptr(dev)))
        arms.append(dict(name=label, launch=launch, ms=[], keep=cl))

    slot_ms, slot_n = (Ct.c_double * 8)(), (Ct.c_uint64 * 8)()
    with torch.no_grad():
        for arm in arms:
            for _ in range(3):
                arm['launch']()
        torch.cuda.synchronize()
        L.p3d_profile_enable(1)
        for rnd in range(args.rounds):
            for arm in arms[rnd % len(arms):] + arms[:rnd % len(arms)]:          # rotated: no arm always follows the same one
                arm['launch']()                                                  # untimed: the arm's lines back in L2
                torch.cuda.synchronize()
                L.p3d_profile_read(None, None, 0, 1)
                for _ in range(args.launches):
                    arm['launch']()
                torch.cuda.synchronize()
                L.p3d_profile_read(slot_ms, slot_n, 8, 1)
                assert slot_n[5] == args.launches and slot_n[0] == 0, 'every launch must be one fused kernel (slot 5)'
                arm['ms'].append(slot_ms[5] / args.launches)
        L.p3d_profile_enable(0)
    res = {'card': card(), 'launches_per_round': args.launches, 'rounds': args.rounds, 'arms': {}}
    for arm in arms:
        ms = arm['ms']
        res['arms'][arm['name']] = dict(median_ms=round(statistics.median(ms), 4), min_ms=round(min(ms), 4), max_ms=round(max(ms), 4))
    res['p512_over_p8'] = round(res['arms']['P512 fp32']['median_ms'] / res['arms']['P8 fp32']['median_ms'], 3)
    return res


# ------------------------------------------------------------------------------------------------------ CPU model
def tap_lines(S, P=512, seed=0x5EED, fine=False):
    """Per view: the 128 B line of every coarse tap, (N, M, S, 3 planes, 4 taps) int64, -1 where the kernel predicates the
    plane's loads off (its footprint lies more than one texel outside the plane).  The footprint is clamped into the plane
    the way fused::plane_taps_rec clamps it.  fine: the taps of the fine pass instead, at the depths of the oracle's
    importance sampler fed flat coarse weights (the bench's random planes and decoder put no surface anywhere, and the
    sampler's 0.01 floor spreads the rest)."""
    import numpy as np
    import torch
    from oracle import philox, renderer_oracle as orc
    cams = [orc.camera_params_to_matrix(e, a, 1.0, 30.0) for e, a in spin_views(VIEWS)]
    c2w, K = torch.stack([c[0] for c in cams]), torch.stack([c[1] for c in cams])
    ro, rd = orc.ray_sampler(c2w, K, R)
    N, M = ro.shape[:2]
    u = philox.uniforms(seed, np.arange(N * M * S, dtype=np.uint64), philox.STREAM_COARSE).reshape(N, M, S, 1)
    t = orc.stratified_depths(torch.from_numpy(u), OPTS['ray_start'], OPTS['ray_end'])
    if fine:
        uf = torch.from_numpy(philox.uniforms(seed, np.arange(N * M * S, dtype=np.uint64), philox.STREAM_FINE).reshape(N * M, S))
        z = t.reshape(N * M, S).to(uf.dtype)
        t = orc.importance_depths(z, torch.ones(N * M, S - 1, dtype=z.dtype), uf).reshape(N, M, S, 1).to(t.dtype)
    xyz = (ro[:, :, None] + t * rd[:, :, None]).reshape(N, M * S, 3)
    co = (orc.plane_coords(xyz, True) * (2.0 / OPTS['box_warp'])).numpy().astype(np.float32)        # (N, 3, M*S, 2)
    f = ((co + 1.0) * P - 1.0) * 0.5
    sane = ((f > -2.0) & (f < P + 1.0)).all(-1)
    f0 = np.where(sane[..., None], np.floor(f), -4).astype(np.int64)
    a0 = np.clip(f0, 0, P - 2)
    on = sane & (np.abs(f0 - a0) <= 1).all(-1)                                                        # (N, 3, M*S)
    plane = np.arange(3)[None, :, None]
    lines = np.empty((N, 3, M * S, 4), np.int64)
    for k in range(4):
        dy, dx = k >> 1, k & 1
        lines[..., k] = np.where(on, (plane * P + a0[..., 1] + dy) * P + a0[..., 0] + dx, -1)
    return lines.reshape(N, 3, M, S, 4).transpose(0, 2, 3, 1, 4)


def group_perm(M, GR, order):
    """Ray of row-ray rl of each group of a view, (M / GR, GR).  'linear' is the kernel's order: GR consecutive rays, a
    segment of an image row (ray = row * side + column).  'column' is the alternative: group g takes rows
    [GR (g / side), GR (g / side) + GR) of image column g % side, so that at elevation 0 its rays project onto one line of
    the plane that drops y."""
    import numpy as np
    g = np.arange(M // GR)[:, None]
    rl = np.arange(GR)[None, :]
    if order == 'linear':
        return g * GR + rl
    side = int(round(M ** 0.5))
    return (g // side * GR + rl) * side + g % side


def _distinct(x):
    """Distinct non-negative values along the last axis, summed over the others."""
    import numpy as np
    s = np.sort(x, axis=-1)
    new = np.concatenate([np.ones(s.shape[:-1] + (1,), bool), s[..., 1:] != s[..., :-1]], -1)
    return int((new & (s >= 0)).sum())


def run_model(args):
    import numpy as np
    res = {}
    for S in (96, 48):
        RPT, GR = S // 3, 384 // S
        lines = tap_lines(S)
        M = lines.shape[1]
        for order in ('linear', 'column'):
            perm = group_perm(M, GR, order)
            for rows in ('ray', 'depth'):
                req = ins = til = 0
                for v in range(lines.shape[0]):
                    x = lines[v][perm]                                                     # (G, GR, S, 3, 4)
                    G = x.shape[0]
                    x = x.reshape(G, GR, 3, RPT, 3, 4).transpose(0, 2, 1, 3, 4, 5)         # (G, tile, rl, j, plane, tap)
                    if rows == 'depth':                                                    # 4 rows = 4 rays at one depth index
                        x = x.transpose(0, 1, 3, 2, 4, 5)
                    x = x.reshape(G * 3, 128, 3, 4)                                        # tiles x rows in load order
                    req += int((x >= 0).sum())
                    ins += _distinct(x.reshape(G * 3, 32, 4, 3, 4).transpose(0, 1, 3, 4, 2))
                    til += _distinct(x.reshape(G * 3, 128 * 12))
                res[f'S{S} {order} groups, rows by {rows}'] = dict(lines_requested=req, distinct_per_instruction=ins, distinct_per_tile=til,
                                                                  per_instruction_ratio=round(ins / req, 4), per_tile_ratio=round(til / req, 4))
    for k, v in res.items():
        ref = res[k.split(' ')[0] + ' linear groups, rows by ray']
        v['distinct_per_tile_vs_linear'] = round(v['distinct_per_tile'] / ref['distinct_per_tile'], 4)
        v['distinct_per_instruction_vs_linear'] = round(v['distinct_per_instruction'] / ref['distinct_per_instruction'], 4)
    return res


def l2_model(S=96, P=512, sms=132):
    """What shares L2 while k_render_ws3 runs bench.py's workload (--model).  Groups of GR rays run in waves of `sms`
    groups (CTA b takes groups b, b + sms, ...), so wave w is rays [w sms GR, (w + 1) sms GR) of the call.  Per plane and
    pass: the distinct 128 B texel lines a wave asks for, and how many waves back each of them was last asked for (its
    reuse distance; 'first' = never before in the call).  Then the colour areas: their footprint, how many passes lie
    between a tile's store and its load, and how many of their bytes are live (stored, not yet loaded) at once."""
    import numpy as np
    GR = 384 // S
    res = {'wave_rays': sms * GR}
    for name, fine in (('coarse', False), ('fine', True)):
        lines = tap_lines(S, P, fine=fine)                                                 # (N, M, S, 3, 4)
        N, M = lines.shape[:2]
        wave = (np.arange(N * M) // GR) // sms                                             # wave of each ray of the call
        for p in range(3):
            x = lines[:, :, :, p, :].reshape(N, M, S * 4)
            x = np.where(x >= 0, x + (np.arange(N) * 3 * P * P)[:, None, None], -1).reshape(N * M, S * 4)   # one id per view's line
            keys = x * 4096 + wave[:, None]
            keys = np.unique(keys[x >= 0])
            line, w = keys // 4096, keys % 4096
            per_wave = np.bincount(w)
            same = np.concatenate([[False], line[1:] == line[:-1]])
            dist = np.where(same, w - np.concatenate([[0], w[:-1]]), 0)
            n = len(keys)
            res[f'{name} plane {p}'] = dict(
                distinct_lines_per_wave=int(np.median(per_wave)), mb_per_wave=round(float(np.median(per_wave)) * 128 / 1e6, 2),
                reuse_1_wave=round(float((dist == 1).sum()) / n, 3), reuse_2_7_waves=round(float(((dist >= 2) & (dist < 8)).sum()) / n, 3),
                reuse_8plus_waves=round(float((dist >= 8).sum()) / n, 3), first=round(float((~same).sum()) / n, 3),
                distinct_lines_call_mb=round(len(np.unique(line)) * 128 / 1e6, 1))
    # colour areas of one CTA with n_my groups: tile q of the tile sequence is stored at time q; colours(n) loads group n's
    # six tiles during the pass after F(n) (the decoder signals F(n)'s stores in the next pass's first tile)
    n_my = (N * M // GR + sms - 1) // sms
    passes = [None] * (2 * n_my)
    j_of = {}
    for j in range(2 * n_my):
        k = j - 2
        if j == 0: pd = (0, 0)
        elif n_my == 1: pd = (0, 1)
        elif j == 1: pd = (1, 0)
        elif k < 2 * (n_my - 2): pd = ((k >> 1) + 2, 0) if (k & 1) else (k >> 1, 1)
        else: pd = (n_my - 2 + (k - 2 * (n_my - 2)), 1)
        j_of[pd] = j
    dist_c = [j_of[(n, 1)] + 1 - j_of[(n, 0)] for n in range(n_my)]
    live = []
    for j in range(2 * n_my):                                    # tiles stored and not yet loaded at the end of pass j
        live.append(sum(3 * ((j_of[(n, 0)] <= j < j_of[(n, 1)] + 1) + (j_of[(n, 1)] <= j < j_of[(n, 1)] + 1)) for n in range(n_my)))
    tile_b = 128 * 128
    res['colour areas'] = dict(
        footprint_mb=round(5 * 3 * tile_b * sms / 1e6, 1), bytes_per_call_gb=round(2 * N * M * S * 128 / 1e9, 2),
        store_to_load_passes_coarse=sorted(set(dist_c[2:-2])), store_to_load_passes_fine=[1],
        live_mb_steady=round(float(np.median(live[4:-4])) * tile_b * sms / 1e6, 1), live_mb_max=round(max(live) * tile_b * sms / 1e6, 1))
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--model', action='store_true', help='CPU: count the coarse pass\'s L2 line requests per ray order')
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--launches', type=int, default=50)
    args = ap.parse_args()
    print(json.dumps(dict(run_model(args), l2=l2_model()) if args.model else run_gpu(args)), flush=True)


if __name__ == '__main__':
    main()
