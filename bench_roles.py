#!/usr/bin/env python
"""bench_roles.py - where each role of the fused renderer (k_render_ws3) spends its cycles.

    python bench_roles.py [--launches L] [--lib PATH]

Builds a second copy of the library with -DP3D_WS3_ROLE_CLOCKS into a temporary directory (render_fused_ws3.cu recompiled,
every other object taken from the in-tree build) unless --lib names one, loads it in place of the in-tree library, and runs
bench_gather.py's P512 fp32 arm: bench.py's workload (8 views, 128x128 rays, 96+96 samples) with channels-last planes.
In that build lane 0 of every warp adds clock64() deltas into per-CTA counters: each mbarrier wait by barrier kind and the
phases of each role's work (see RoleClk in csrc/render_fused_ws3.cu).  Printed per role, as a share of the role's cycles
(the sum over its warps of the time from its first to its last instruction): time waiting on each barrier and time in each
phase.  The counters perturb the kernel slightly; its launch time is printed beside them, with the card."""
from __future__ import annotations

import argparse
import ctypes as Ct
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SLOTS = ['total', 'wait a1_full', 'wait a1_empty', 'wait state_free', 'wait fine_ready', 'wait sigc/sigf_ready',
         'wait col_stored', 'wait col_full', 'colours()', 'layer 1', 'hidden', 'layer 2', 'epilogue + store', 'tap table',
         'gather loads + lerp', 'importance']
ROLES = [('gather', 12, ['wait state_free', 'wait fine_ready', 'wait a1_empty', 'tap table', 'gather loads + lerp']),
         # the epilogue includes the state_free wait before a colour area is rewritten, which is also listed on its own
         ('decoder', 8, ['wait a1_full', 'wait state_free', 'layer 1', 'hidden', 'layer 2', 'epilogue + store']),
         # colours() includes its col_stored / col_full waits, which are also listed on their own
         ('ray', 4, ['wait sigc/sigf_ready', 'colours()', 'wait col_stored', 'wait col_full', 'importance'])]
EXCLUSIVE = {'gather': ['wait state_free', 'wait fine_ready', 'wait a1_empty', 'tap table', 'gather loads + lerp'],
             'decoder': ['wait a1_full', 'layer 1', 'hidden', 'layer 2', 'epilogue + store'],
             'ray': ['wait sigc/sigf_ready', 'colours()', 'importance']}


def build_roles_lib(out_dir):
    sys.path.insert(0, os.path.join(ROOT, 'panic3d-anime-reconstruction_b200'))
    import _build
    _build.build()                                              # the in-tree objects the copy links against
    nvcc = _build.find_nvcc()
    src = os.path.join(_build.CSRC, 'render_fused_ws3.cu')
    obj = os.path.join(out_dir, 'render_fused_ws3_roles.o')
    subprocess.run(_build.compile_cmd(nvcc, src, obj, ['-DP3D_WS3_ROLE_CLOCKS']), check=True)
    objs = [_build.object_path(s) for s in _build.sources() if s != src] + [obj]
    lib = os.path.join(out_dir, 'libp3d_roles.so')
    subprocess.run(_build.link_cmd(nvcc, lib, objs), check=True)
    return lib


def run(args, lib_path):
    os.environ['P3D_LIBP3D'] = lib_path                         # read when panic3d_b200._lib is first imported
    import torch
    import bench_gather as bg
    from panic3d_b200 import _lib, cameras
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    from panic3d_b200.training.triplane import OSGDecoder

    assert torch.cuda.is_available(), 'bench_roles.py needs a CUDA device'
    assert _lib.LIB_PATH == lib_path
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    L = _lib.lib()
    clocks = L.p3d_ws3_role_clocks                              # AttributeError: not a -DP3D_WS3_ROLE_CLOCKS build
    clocks.restype, clocks.argtypes = Ct.c_longlong, [Ct.c_void_p, Ct.c_longlong, Ct.c_int]
    torch.manual_seed(1234)
    decoder = OSGDecoder(bg.C, {'decoder_lr_mul': 1, 'decoder_output_dim': 32}).to(dev).requires_grad_(False)
    labels = torch.stack([cameras.camera_params_to_matrix(elev=e, azim=a, dist=1.0, fov=30.0)['camera_label']
                          for e, a in bg.spin_views(bg.VIEWS)]).to(dev)
    ro, rd = RaySampler()(labels[:, :16].view(-1, 4, 4), labels[:, 16:25].view(-1, 3, 3), bg.R)
    ro, rd = ro.float().contiguous(), rd.float().contiguous()
    N, M = ro.shape[:2]
    g = torch.Generator(device=dev).manual_seed(99)
    cl = torch.randn(N, 3, 512, 512, bg.C, device=dev, generator=g, dtype=torch.float32)
    r = ImportanceRenderer(use_triplane=True)
    r.planes_bf16, r.mlp_mode = False, _lib.P3D_MLP_TC_3XBF16
    planes_cl = r._planes_cl(cl.permute(0, 1, 4, 2, 3))
    p, wts = r._params(planes_cl, N, M, bg.OPTS, decoder, None, None, None)
    p.seed = 0x5EED
    wt = [t.detach().float().contiguous() for t in wts]
    ws = torch.empty(int(L.p3d_render_workspace_bytes(Ct.byref(p))), dtype=torch.uint8, device=dev)
    out = [torch.empty(s, device=dev) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]

    def launch():
        _lib.check(L.p3d_render_forward(Ct.byref(p), planes_cl.data_ptr(), *[t.data_ptr() for t in wt], ro.data_ptr(),
                                        rd.data_ptr(), None, None, ws.data_ptr(), ws.numel(),
                                        *[o.data_ptr() for o in out], _lib.stream_ptr(dev)))

    slot_ms, slot_n = (Ct.c_double * 8)(), (Ct.c_uint64 * 8)()
    with torch.no_grad():
        for _ in range(3):
            launch()
        n = clocks(None, 0, 1)                                   # zero the counters after the warm-up
        assert n > 0, f'p3d_ws3_role_clocks failed ({n})'
        L.p3d_profile_enable(1)
        L.p3d_profile_read(None, None, 0, 1)
        for _ in range(args.launches):
            launch()
        torch.cuda.synchronize()
        L.p3d_profile_read(slot_ms, slot_n, 8, 1)
        L.p3d_profile_enable(0)
        buf = (Ct.c_ulonglong * n)()
        assert clocks(buf, n, 1) == n
    ctas = n // (3 * len(SLOTS))
    tot = [[0] * len(SLOTS) for _ in range(3)]
    for c in range(ctas):
        for role in range(3):
            for s in range(len(SLOTS)):
                tot[role][s] += buf[(c * 3 + role) * len(SLOTS) + s]
    res = {'card': bg.card(), 'launches': args.launches, 'ctas': ctas,
           'kernel_ms_per_launch': round(slot_ms[5] / max(1, slot_n[5]), 4), 'roles': {}}
    for role, (name, warps, shown) in enumerate(ROLES):
        total = tot[role][0]
        share = {k: round(100.0 * tot[role][SLOTS.index(k)] / total, 2) for k in shown}
        rest = total - sum(tot[role][SLOTS.index(k)] for k in EXCLUSIVE[name])
        share['composite' if name == 'ray' else 'other'] = round(100.0 * rest / total, 2)
        res['roles'][name] = {'warps': warps, 'cycles_per_warp_per_launch': round(total / warps / ctas / args.launches),
                              'percent': share}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--lib', help='an existing -DP3D_WS3_ROLE_CLOCKS build of libp3d.so (default: build one)')
    args = ap.parse_args()
    if args.lib:
        print(json.dumps(run(args, os.path.abspath(args.lib))), flush=True)
        return
    with tempfile.TemporaryDirectory(prefix='p3d_roles_') as d:
        print(json.dumps(run(args, build_roles_lib(d))), flush=True)


if __name__ == '__main__':
    main()
