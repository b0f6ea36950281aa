#!/usr/bin/env python
"""BASELINE.json configs[2]: the eval script's view sweep (`_scripts/eval/generate.py:108-130`: 4 orthographic + 12
perspective views of one subject through `G.f`, super-resolution head on) on a synthetic-weight TriPlaneGenerator built
with the training configuration's kwargs (`_train/eg3dc/trainers/train_eclustrousC.py:339-343,409-440,479-480`) and the eval
loader's settings (`_train/eg3dc/util/eg3dc_v0.py:24-56`: 96+96 samples, force_sigmoid; `generate.py:53-57`: crop 0.1,
cull 0.5).  `--paste` adds the eval script's `paste_params` (`generate.py:59-65`; SURVEY 8f-3): every view then runs `paste_front`
- the reference's own (its two kornia calls served by the restatement in oracle/paste_oracle.py: kornia is not in this image) in the
reference arm, `panic3d_b200.paste` rebound by `dropin.install_paste()` in ours - including its second render from the visible surface.

Two arms, one process each (module identity is decided at import time), same weights (same seed, same construction order):

    python bench_config3.py --arm reference --out gpurun_out/c3_ref.pt   the UNMODIFIED reference from baseline/_ref on its own GPU
                                                                         path: eager PyTorch renderer + its JIT CUDA plugins
    python bench_config3.py --arm ours      --out gpurun_out/c3_ours.pt  the same reference TriPlaneGenerator / backbone / SR code
                                                                         with panic3d_b200.dropin.install(): our renderer, ray
                                                                         sampler and the three ops underneath it
    python bench_config3.py --compare gpurun_out/c3_ref.pt gpurun_out/c3_ours.pt

Parity pass (deterministic): backbone noise_mode='const', SR noise per the config ('none'), the renderer's jitter injected
identically into both arms (patched torch.rand_like / torch.rand for the reference, `injected_noise` for ours).
Timing pass: the sweep as the eval script runs it (random noise, own jitter), CUDA events around each G.f call."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.abspath(__file__))
REF_TREE = os.path.join(ROOT, 'baseline', '_ref')


def sweep_views():
    """generate.py:108-117: camO front/left/right/back (fov -1 = orthographic) + camP cam60[spin12] (fov 30)."""
    import _databacks.lustrous_renders_v1 as dk
    views = [('camO', 0.0, 0.0, -1.0), ('camO', 0.0, 90.0, -1.0), ('camO', 0.0, -90.0, -1.0), ('camO', 0.0, 180.0, -1.0)]
    for v in dk.camsubs['spin12']:
        e, a = dk.cam60[v]
        views.append(('camP', float(e), float(a), 30.0))
    return views


class InjectRand:
    """Feed pre-drawn uniforms to the reference renderer's torch.rand_like / torch.rand calls, in call order."""

    def __init__(self, torch, queue):
        self.torch, self.queue = torch, list(queue)

    def __enter__(self):
        t = self.torch
        self._rl, self._r = t.rand_like, t.rand
        q = self.queue

        def rand_like(x, *a, **k):
            u = q.pop(0)
            assert u.shape == x.shape, (u.shape, x.shape)
            return u.to(x.device).clone()

        def rand(*size, **k):
            u = q.pop(0)
            return u.to(k.get('device', u.device)).clone()
        t.rand_like, t.rand = rand_like, rand
        return self

    def __exit__(self, *exc):
        self.torch.rand_like, self.torch.rand = self._rl, self._r


def build_generator(args, torch):
    import training.triplane as tp
    res, R = (64, 16) if args.tiny else (512, 128)
    rk = dict(image_resolution=res, disparity_space_sampling=False, clamp_mode='softplus',
              superresolution_module='training.superresolution.SuperresolutionHybrid8XDC', c_gen_conditioning_zero=True,
              gpc_reg_prob=None, c_scale=1.0, superresolution_noise_mode='none', density_reg=0.25, density_reg_p_dist=0.004,
              reg_type='l1', decoder_lr_mul=1.0, sr_antialias=True, white_back=True, triplane_depth=1, use_triplane=True,
              tanh_rgb_output=False, box_warp=0.7, ray_start=0.5, ray_end=1.5, depth_resolution=96, depth_resolution_importance=96,
              avg_camera_radius=1.0, avg_camera_pivot=[0, 0, 0])
    cb, cm = (2048, 32) if args.tiny else (32768, 512)
    torch.manual_seed(0)
    G = tp.TriPlaneGenerator(z_dim=512, c_dim=25, w_dim=512, img_resolution=512, img_channels=3, rendering_kwargs=rk,
                             cond_mode='none', mapping_kwargs=dict(num_layers=2), channel_base=cb, channel_max=cm,
                             fused_modconv_default='inference_only', num_fp16_res=0, sr_num_fp16_res=4,
                             sr_kwargs=dict(channel_base=cb, channel_max=cm, fused_modconv_default='inference_only'),
                             triplane_width=32, backbone_resolution=args.plane)
    G = G.eval().requires_grad_(False)
    G.neural_rendering_resolution = R
    G.set_force_sigmoid(True)                                  # load_eg3dc_model(force_sigmoid=True), generate.py:54
    return G, R


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--arm', choices=['reference', 'ours'])
    ap.add_argument('--out')
    ap.add_argument('--compare', nargs=2)
    ap.add_argument('--plane', type=int, default=256, help='backbone_resolution (256 in the shipped model; BASELINE synthetic: 512)')
    ap.add_argument('--tiny', action='store_true', help='small channels / 16x16 rays (CPU smoke test of the harness)')
    ap.add_argument('--device', default='cuda:0')
    ap.add_argument('--reps', type=int, default=2, help='timed repetitions of the 16-view sweep')
    ap.add_argument('--profile', help='write a per-kernel device-time table of one more sweep (torch.profiler / CUPTI) to this JSON file')
    ap.add_argument('--save', help='ours arm: write every view of the timed sweep as PNGs into this directory through panic3d_b200.imageio.AsyncImageWriter '
                                   '(generate.py:141-148), flush inside the timed region')
    ap.add_argument('--return_more', action='store_true', help='call G.f(x, return_more=True) like generate.py:130 (with --graphs: lean_return_more)')
    ap.add_argument('--graphs', action='store_true', help='ours arm: panic3d_b200.graphs.enable_cuda_graphs(G) - backbone and SR head replayed as CUDA graphs')
    ap.add_argument('--reuse_triplane', action='store_true', help='ours arm: dropin.install_paste(reuse_triplane=True)')
    ap.add_argument('--modconv', action='store_true', help='ours arm: dropin.install_modconv() - the synthesis layers and SR head on the fused modulated-conv kernel')
    ap.add_argument('--paste', action='store_true', help="run the sweep with the eval script's paste_params (generate.py:59-65)")
    args = ap.parse_args()
    import torch
    if args.compare:
        a, b = (torch.load(f) for f in args.compare)
        rep = {'arms': [a['arm'], b['arm']], 'views': len(a['views'])}
        for key in ('image_raw', 'image', 'image_depth', 'image_weights', 'feature_image', 'image_prepaste', 'paste', 'mask', 'mask_weights',
                    'mask_edges', 'mask_occ', 'mask_dxyz'):
            if key in a and key in b:
                d = (a[key].float() - b[key].float()).abs()
                rep[key] = {'max_abs': float(d.max()), 'mean_abs': float(d.mean()), 'frac_within_1e-3': float((d < 1e-3).float().mean()),
                            'shape': list(d.shape)}
        rep['note'] = ('cull_clouds = 0.5 is a hard threshold on sigma (renderer.py:150-153): a sample within rounding of it flips in one arm, '
                       'so isolated rays differ by more than 1e-3 (same criterion as the cull fixtures in tests/test_render_gpu.py); the '
                       '512^2 image goes through the fp16 super-resolution head')
        if 'mask' in a and 'mask' in b:
            # thresh_dxyz = 5e-6 sits at the rounding level of the rendered xyz (|xyz| ~ 0.3, ulp 3e-8; the two renderers agree to ~1e-6):
            # mask_dxyz is decided by noise in EITHER implementation, so the pasted image is compared where the masks agree
            same = ((a['mask'] - b['mask']).abs() < 1e-3)
            d = (a['image'].float() - b['image'].float()).abs()
            rep['paste'] = {'mask_agreement': float(same.float().mean()), 'mask_mean': [float(a['mask'].mean()), float(b['mask'].mean())],
                            'image_max_abs_where_masks_agree': float(d[same.expand_as(d)].max()),
                            'image_mean_abs_where_masks_agree': float(d[same.expand_as(d)].mean())}
            for k in ('mask_weights', 'mask_edges', 'mask_occ', 'mask_dxyz'):
                rep['paste'][k + '_agreement'] = float(((a[k] - b[k]).abs() < 1e-3).float().mean())
        rep['views_per_s'] = {a['arm']: a['views_per_s'], b['arm']: b['views_per_s']}
        rep['speedup'] = b['views_per_s'] / a['views_per_s'] if a['arm'] == 'reference' else a['views_per_s'] / b['views_per_s']
        print(json.dumps(rep))
        return
    sys.path.insert(0, ROOT)
    from baseline import ref_env
    ref_env.setup()
    dev = torch.device(args.device)
    if args.paste and args.arm == 'reference':
        from oracle.paste_oracle import kornia_shim                 # reference arm only: the two kornia calls of ITS paste_front
        k = kornia_shim()
        sys.modules['kornia'], sys.modules['kornia.filters'], sys.modules['kornia.morphology'] = k, k.filters, k.morphology
    if args.arm == 'ours':
        import panic3d_b200.dropin as dropin
        installed = dropin.install()
    import training.triplane as tp
    if args.paste and args.arm == 'ours':
        dropin.install_paste(tp, reuse_triplane=args.reuse_triplane)
    if args.modconv and args.arm == 'ours':
        dropin.install_modconv()
    mod_file = sys.modules[tp.ImportanceRenderer.__module__].__file__
    assert ('baseline/_ref' in mod_file.replace(os.sep, '/')) == (args.arm == 'reference'), mod_file
    G, R = build_generator(args, torch)
    G = G.to(dev)
    graphed = None
    if args.graphs and args.arm == 'ours' and dev.type == 'cuda':
        from panic3d_b200 import graphs
        graphed = graphs.enable_cuda_graphs(G, lean_return_more=args.return_more)
    views = sweep_views()
    ws = None
    S = int(G.rendering_kwargs['depth_resolution'])
    Sf = int(G.rendering_kwargs['depth_resolution_importance'])

    def xin_for(elev, azim, fov):
        one = torch.ones(1, device=dev)
        x = {'elevations': elev * one, 'azimuths': azim * one, 'fovs': fov * one, 'cond': {}, 'seeds': [0],
             'triplane_crop': 0.1, 'cull_clouds': 0.5}
        if ws is not None:
            x['ws'] = ws
        if args.paste:
            x['cond'] = {'image_ortho_front': front}
            x['paste_params'] = {'mode': 'default', 'thresh_weight': 0.95, 'thresh_edges': 0.02, 'thresh_occ': 0.05, 'offset_occ': 0.01,
                                 'thresh_dxyz': 0.000005}
        return x

    res_img = 512                                              # the SR head always outputs img_resolution = 512
    front = torch.rand(1, 3, res_img, res_img, generator=torch.Generator().manual_seed(7)).to(dev)

    outs = {k: [] for k in ('image_raw', 'image', 'image_depth', 'image_weights')}
    pouts = {k: [] for k in ('paste', 'mask', 'mask_weights', 'mask_edges', 'mask_occ', 'mask_dxyz')} if args.paste else {}
    if args.paste:
        outs['image_prepaste'] = []
    syn_fwd = G.backbone.synthesis.forward                      # an nn.Module: patch its forward on the instance
    with torch.no_grad():
        # ---- parity pass
        G.backbone.synthesis.forward = lambda *a, **k: syn_fwd(*a, **dict(k, noise_mode='const'))
        gen = torch.Generator().manual_seed(123)
        for i, (_cm, e, a, f) in enumerate(views):
            u_c = torch.rand(1, R * R, S, 1, generator=gen)
            u_f = torch.rand(R * R, Sf, generator=gen)
            x = xin_for(e, a, f)
            if args.arm == 'reference':
                with InjectRand(torch, [u_c, u_f] * (2 if args.paste else 1)):   # paste_front renders a second time: same jitter again
                    out = G.f(x)
            else:
                G.renderer.injected_noise = (u_c, u_f)
                out = G.f(x)
                G.renderer.injected_noise = None
            ws = x['ws']
            for k in outs:
                outs[k].append(out[k].float().cpu())
            for k in pouts:
                pouts[k].append(out['paste'][k].float().cpu())
        G.backbone.synthesis.forward = syn_fwd
        # ---- timing pass: the sweep as generate.py runs it
        if dev.type == 'cuda':
            for (_cm, e, a, f) in views[:3]:
                G.f(xin_for(e, a, f))
            torch.cuda.synchronize()
            writer = None
            if args.save and args.arm == 'ours':
                import panic3d_b200.imageio as pio
                os.makedirs(args.save, exist_ok=True)
                writer = pio.AsyncImageWriter(threads=8, level=3)
                writer.save(G.f(xin_for(*views[0][1:]))['image'], os.path.join(args.save, 'warm.png')); writer.flush()
            bw = G.rendering_kwargs['box_warp']
            fkw = {'return_more': True} if args.return_more else {}
            t0 = time.perf_counter()
            for rep in range(args.reps):
                for i, (_cm, e, a, f) in enumerate(views):
                    out = G.f(xin_for(e, a, f), **fkw)
                    if writer is not None:
                        writer.save(out['image'], os.path.join(args.save, f'rgb_{rep}_{i:02d}.png'))
                        writer.save_xyza(out['image_xyz'], out['image_weights'], bw, os.path.join(args.save, f'xyza_{rep}_{i:02d}.png'))
            if writer is not None:
                writer.flush()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if writer is not None:
                n_files = len([f_ for f_ in os.listdir(args.save) if f_.endswith('.png')])
                writer.close()
        else:
            t0 = time.perf_counter()
            for (_cm, e, a, f) in views[:2]:
                G.f(xin_for(e, a, f))
            dt = (time.perf_counter() - t0) * len(views) / 2 * args.reps
    vps = args.reps * len(views) / dt
    graph_report = None
    if graphed:
        # self-check: the first views again with the graphs taken out (deterministic pass) must reproduce the graphed outputs
        with torch.no_grad():
            saved = {n: w_ for n, w_ in graphed.items()}
            mods = {'backbone': G.backbone.synthesis, 'superresolution': G.superresolution}
            for n, w_ in saved.items():
                mods[n].forward = w_.fn
            fwd = G.backbone.synthesis.forward
            G.backbone.synthesis.forward = lambda *a, **k: fwd(*a, **dict(k, noise_mode='const'))
            gen = torch.Generator().manual_seed(123)
            worst = 0.0
            for i, (_cm, e, a, f) in enumerate(views[:4]):
                u_c = torch.rand(1, R * R, S, 1, generator=gen)
                u_f = torch.rand(R * R, Sf, generator=gen)
                G.renderer.injected_noise = (u_c, u_f)
                out = G.f(xin_for(e, a, f))
                G.renderer.injected_noise = None
                worst = max(worst, float((out['image'].float().cpu() - outs['image'][i]).abs().max()))
            G.backbone.synthesis.forward = fwd
            for n, w_ in saved.items():
                mods[n].forward = w_
        graph_report = {'eager_vs_graph_max_abs_image': worst,
                        **{n: {'captures': w_.captures, 'replays': w_.hits, 'bypassed': w_.bypassed, 'failed_signatures': len(w_.failed)} for n, w_ in graphed.items()}}
    if args.profile and dev.type == 'cuda':
        try:                                                       # where a view's device time goes (the "next" row: backbone / SR kernels)
            from torch.profiler import profile, ProfilerActivity
            with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
                for (_cm, e, a, f) in views:
                    G.f(xin_for(e, a, f))
                torch.cuda.synchronize()
            rows = sorted(((ev.key, ev.count, getattr(ev, 'device_time_total', getattr(ev, 'cuda_time_total', 0.0))) for ev in prof.key_averages()),
                          key=lambda r: -r[2])
            total = sum(r[2] for r in rows) or 1.0
            json.dump({'arm': args.arm, 'views': len(views), 'device_ms_per_view': total / 1e3 / len(views),
                       'kernels': [{'name': k[:160], 'launches': c, 'ms_per_view': t / 1e3 / len(views), 'share': t / total} for k, c, t in rows[:40]]},
                      open(args.profile, 'w'), indent=1)
        except Exception as e:                                     # profiling is evidence, not part of the measurement
            print('profile failed:', repr(e), file=sys.stderr)
    res = {k: torch.cat(v) for k, v in {**outs, **pouts}.items()}
    res.update(arm=args.arm, views=views, views_per_s=vps, plane=args.plane)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        torch.save(res, args.out)
    line = {'config': 'BASELINE configs[2]: G.f 16-view sweep, SR on, synthetic weights' + (', paste_params on' if args.paste else ''), 'arm': args.arm, 'views_per_s': vps,
            'ms_per_view': 1e3 / vps, 'plane': args.plane, 'rays': R * R, 'samples': [S, Sf],
            'renderer_module': mod_file.replace(ROOT, '.'), 'image_mean': float(res['image'].mean())}
    if args.arm == 'ours':
        from panic3d_b200 import _lib
        line['gpu_launches'] = _lib.launch_count()
    if graph_report:
        line['cuda_graphs'] = graph_report
    if args.save and args.arm == 'ours' and dev.type == 'cuda':
        line['saved_png_files'] = n_files
    if args.return_more:
        line['return_more'] = True
    print(json.dumps(line))


if __name__ == '__main__':
    main()
