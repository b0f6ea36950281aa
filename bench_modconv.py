"""Device time of the fused modulated convolution (panic3d_b200.modconv) against the reference's own layers, per eval layer
shape at N = 1 and for the SR head of one view.

    bash baseline/install_ref.sh            # once, in the build container: the unmodified reference + its CUDA plugins
    python bench_modconv.py [--iters 50] [--rounds 5] [--json out.json]

Two arms on the same GPU, same seeded parameters (oracle.modconv_oracle.init_layer_) and inputs:

    ours       per layer: the kernel route (modconv.synthesis_layer_kernel / torgb_kernel), whatever the eligibility
               rule says; SR head: the reference's own blocks after dropin.install_modconv(), i.e. the eligibility rule
               applied and every other layer on the reference's route
    reference  the UNMODIFIED SynthesisLayer / ToRGBLayer / SynthesisBlock of baseline/_ref, eval mode (fused_modconv),
               eager cuDNN with TF32 allowed and the reference's own bias_act / upfirdn2d CUDA plugins

Every call of both arms is captured once into a CUDA graph (after warm-up: cuDNN's algorithm choice, the plugins' loads),
and `iters` replays are timed with CUDA events: device time of the layer's whole sequence, without the host's Python
and launch overhead.  The arms alternate round by round; the median round is reported.  The SR head is also timed
eagerly (what an uncaptured caller pays).  FLOP/s is shape-computed (modconv.flops).  The card name, power limit and
max SM clock are printed with the results.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--json')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_modconv.py needs a CUDA device')
    from baseline import ref_env
    ref_env.setup()
    import training.networks_stylegan2 as ref
    assert 'baseline/_ref' in ref.__file__.replace(os.sep, '/'), ref.__file__
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.modconv as mc
    from oracle import modconv_oracle as mo
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda')

    def ref_layer(shape):
        return mo.make_layer(*shape, module=ref).to(dev).eval().requires_grad_(False)

    cases = []
    for shape in mo.EVAL_SHAPES:
        name, cin, cout, res, up, kind, dtype, clamp = shape
        ours_l = mo.make_layer(*shape).to(dev).requires_grad_(False)
        ref_l = ref_layer(shape)
        x = torch.randn(1, cin, res // up, res // up, device=dev).to(dtype)
        w = torch.randn(1, 64, device=dev)
        p = mc.make_params(x, ours_l.weight, kind == 'layer', up=up)
        if kind == 'torgb':
            ours = (lambda L=ours_l, x=x, w=w: mc.torgb_kernel(L, x, w))
            refc = (lambda L=ref_l, x=x, w=w: L(x, w, fused_modconv=True))
        else:
            ours = (lambda L=ours_l, x=x, w=w: mc.synthesis_layer_kernel(L, x, w, noise_mode='none'))
            refc = (lambda L=ref_l, x=x, w=w: L(x, w, noise_mode='none', fused_modconv=True))
        cases.append((name, mc.flops(p), ours, refc))

    # the SR head of one view: the reference's own SynthesisBlock x 2, with (ours) and without install_modconv
    import panic3d_b200.dropin as dropin
    dropin.install_modconv(ref)
    installed = (ref.SynthesisLayer.forward, ref.ToRGBLayer.forward)
    original = (ref.SynthesisLayer._p3d_reference_forward, ref.ToRGBLayer._p3d_reference_forward)
    sr_ref = torch.nn.ModuleList([ref.SynthesisBlock(32, 256, w_dim=64, resolution=256, img_channels=3, is_last=False, use_fp16=True, conv_clamp=256),
                                  ref.SynthesisBlock(256, 128, w_dim=64, resolution=512, img_channels=3, is_last=True, use_fp16=True, conv_clamp=256)])
    for i, b in enumerate(sr_ref):
        for j, layer in enumerate([b.conv0, b.conv1, b.torgb]):
            mo.init_layer_(layer, 10 * i + j)
    sr_ref = sr_ref.to(dev).eval().requires_grad_(False)
    xs, imgs, wss = torch.randn(1, 32, 128, 128, device=dev), torch.randn(1, 3, 128, 128, device=dev), torch.randn(1, 6, 64, device=dev)

    def sr_run(forwards):
        def run():
            ref.SynthesisLayer.forward, ref.ToRGBLayer.forward = forwards
            try:
                img, x = imgs.clone(), xs
                for i, b in enumerate(sr_ref):
                    x, img = b(x, img, wss[:, 3 * i:3 * i + 3], noise_mode='none')
                return img
            finally:
                ref.SynthesisLayer.forward, ref.ToRGBLayer.forward = installed
        return run
    sr_ours, sr_refc = sr_run(installed), sr_run(original)
    with torch.no_grad():
        d = float((sr_ours() - sr_refc()).abs().max() / sr_refc().abs().max())
    sr_flops = sum(c[1] for c in cases if c[0].startswith('sr'))
    cases.append(('sr_head_view', sr_flops, sr_ours, sr_refc))

    def graphed(fn):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            fn()
        return gr.replay

    def time_ms(fn, n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / n

    with torch.no_grad():
        arms = [(name, fl, graphed(a), graphed(b)) for name, fl, a, b in cases]
        res = {name: {'ours': [], 'reference': []} for name, *_ in arms}
        eager = {'ours': [], 'reference': []}
        for _ in range(args.rounds):
            for name, _, a, b in arms:
                res[name]['ours'].append(time_ms(a, args.iters))
                res[name]['reference'].append(time_ms(b, args.iters))
            eager['ours'].append(time_ms(sr_ours, args.iters))
            eager['reference'].append(time_ms(sr_refc, args.iters))

    def med(v):
        return sorted(v)[len(v) // 2]
    out = {'card': card(), 'iters': args.iters, 'rounds': args.rounds, 'timing': 'CUDA graph replay (device time)', 'layers': {},
           'sr_head_eager': {k: med(v) for k, v in eager.items()}, 'sr_head_rel_diff_vs_reference': d}
    print(f'card: {out["card"]}')
    print(f'{"layer (graph replay)":20s} {"ours ms":>9s} {"ref ms":>9s} {"speed-up":>8s} {"ours TFLOP/s":>12s} {"ref TFLOP/s":>11s}')
    for name, fl, _, _ in arms:
        o, r = med(res[name]['ours']), med(res[name]['reference'])
        out['layers'][name] = {'ours_ms': o, 'reference_ms': r, 'flops': fl}
        print(f'{name:20s} {o:9.4f} {r:9.4f} {r / o:8.2f} {fl / o / 1e9:12.1f} {fl / r / 1e9:11.1f}')
    eo, er = out['sr_head_eager']['ours'], out['sr_head_eager']['reference']
    print(f'{"sr_head_view eager":20s} {eo:9.4f} {er:9.4f} {er / eo:8.2f}')
    print(f'SR head: max |ours - reference| / max |reference| = {d:.2e}')
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
