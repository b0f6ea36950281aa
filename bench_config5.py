#!/usr/bin/env python
"""BASELINE.json configs[4]: one training iteration's phases on synthetic 512^2 data - the reference's own
TriPlaneGenerator + DualDiscriminator (from baseline/_ref, kwargs of `_train/eg3dc/trainers/train_eclustrousC.py:339-343,
355-377,409-440,479-480`; batch_gpu 4, neural rendering resolution 64, 48+48 samples, fp16 in the SR head and the
discriminator's top resolutions as configured there) run through the four phases of the training loop
(`training/training_loop_v0.py:326-396` -> `training/loss_orthocondA.py`):

    Gmain  run_G (G.mapping + G.f under autograd, :157-180) -> run_D (:182-197) -> softplus(-logits) -> backward      (:549-577)
    Greg   density regularisation: G.sample_mixed(2x1000 points)['sigma'] -> l1 TV loss -> backward                 (:579-600)
    Dmain  softplus(D(G(z))) + softplus(-D(real)) -> backward                                                        (:690-735)
    Dreg   R1: grad of D(real) w.r.t. image and image_raw with create_graph -> penalty -> backward                   (:707-742)

The reference's loss class itself needs the dataset's conditioning dict and kornia (absent from this image), so the
phases are restated here line by line on `cond_mode='none'`; everything below the loss - generator, super-resolution,
discriminator, conv2d_gradfix - is the reference's code.  Two arms, one process each:

    --arm reference   the unmodified modules: eager PyTorch renderer + the reference's JIT plugins (bias_act, upfirdn2d)
    --arm ours        panic3d_b200.dropin.install(): our renderer (forward + backward, run_model backward) and the three ops
    --conv2d          (with --arm ours) also dropin.install_conv2d(): conv2d_gradfix's fp32 calls on the 3xTF32 kernels
                      where conv.measured_faster admits them
    --profile         one more iteration under torch.profiler: the convolutions' share of the step's kernel time

Prints one JSON line with ms per phase (CUDA events, median of --iters) and, with --check, gradient statistics so the two
arms can be compared (same seeds -> same weights and the same latents; the renderer's jitter differs, so losses agree
statistically, not bitwise)."""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys
import types

ROOT = os.path.dirname(os.path.abspath(__file__))
REF_TREE = os.path.join(ROOT, 'baseline', '_ref')


# Kernel names of convolutions: cuDNN's forward / data-gradient / weight-gradient kernels (implicit GEMM, Winograd, FFT) and
# panic3d_b200.conv's.  Anything else (GEMMs of the mapping and FC layers, elementwise ops, the renderer) is not a conv.
CONV_KERNEL = re.compile(r'conv|fprop|dgrad|wgrad|winograd|fft|k_weight_kmajor|k_split_sum', re.I)


def conv_share(phases, modules):
    """One iteration of the phases under torch.profiler (CUDA activity): device time of every kernel, the part in
    convolution kernels (CONV_KERNEL), and the ten largest convolution kernels by time."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for m in modules:
        for p_ in m.parameters():
            p_.grad = None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, fn in phases:
            fn()
        torch.cuda.synchronize()
    per_kernel = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per_kernel[e.name] = per_kernel.get(e.name, 0.0) + e.time_range.elapsed_us() / 1e3
    total = sum(per_kernel.values())
    conv = {k: v for k, v in per_kernel.items() if CONV_KERNEL.search(k)}
    conv_ms = sum(conv.values())
    top = sorted(conv.items(), key=lambda kv: -kv[1])[:10]
    return {'kernel_ms': total, 'conv_ms': conv_ms, 'conv_share': conv_ms / total if total else None,
            'top_conv_kernels': [[k[:120], v] for k, v in top]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--arm', choices=['reference', 'ours'], required=True)
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--tiny', action='store_true', help='small channels (CPU smoke test of the harness)')
    ap.add_argument('--device', default='cuda:0')
    ap.add_argument('--paste', action='store_true',
                    help="training mode 'Agrad' (loss_orthocondA.py:146-150): G.f pastes the front image with grad_sample=True, so Gmain "
                         'back-propagates through paste_front into image_xyz; thresholds are permissive so that a random-weight generator '
                         'yields a non-empty mask')
    ap.add_argument('--conv2d', action='store_true', help='with --arm ours: also install_conv2d() (panic3d_b200.conv)')
    ap.add_argument('--profile', action='store_true',
                    help='after the timed iterations, run the four phases once more under torch.profiler and report the '
                         "convolutions' share of the step's kernel time")
    args = ap.parse_args()
    if args.conv2d and args.arm != 'ours':
        ap.error('--conv2d needs --arm ours')
    sys.path.insert(0, ROOT)
    from baseline import ref_env
    ref_env.setup()
    import numpy as np
    import torch
    dev = torch.device(args.device)
    if args.paste and args.arm == 'reference':
        from oracle.paste_oracle import kornia_shim               # reference arm only: the two kornia calls of ITS paste_front
        k = kornia_shim()
        sys.modules['kornia'], sys.modules['kornia.filters'], sys.modules['kornia.morphology'] = k, k.filters, k.morphology
    if args.arm == 'ours':
        import panic3d_b200.dropin as dropin
        dropin.install()
    import training.triplane as tp
    if args.paste and args.arm == 'ours':
        dropin.install_paste(tp)
    from training.dual_discriminator import DualDiscriminator
    from torch_utils.ops import conv2d_gradfix
    conv2d_gradfix.enabled = True                               # training_loop_v0.py:143
    if args.conv2d:
        dropin.install_conv2d(conv2d_gradfix)
    torch.backends.cuda.matmul.allow_tf32 = False               # :141-142
    torch.backends.cudnn.allow_tf32 = False
    mod_file = sys.modules[tp.ImportanceRenderer.__module__].__file__
    assert ('baseline/_ref' in mod_file.replace(os.sep, '/')) == (args.arm == 'reference'), mod_file

    res = 512
    cb, cm = (2048, 32) if args.tiny else (32768, 512)
    rk = dict(image_resolution=res, disparity_space_sampling=False, clamp_mode='softplus',
              superresolution_module='training.superresolution.SuperresolutionHybrid8XDC', c_gen_conditioning_zero=True,
              gpc_reg_prob=None, c_scale=1.0, superresolution_noise_mode='none', density_reg=0.25, density_reg_p_dist=0.004,
              reg_type='l1', decoder_lr_mul=1.0, sr_antialias=True, white_back=True, triplane_depth=1, use_triplane=True,
              tanh_rgb_output=False, box_warp=0.7, ray_start=0.5, ray_end=1.5, depth_resolution=48, depth_resolution_importance=48,
              avg_camera_radius=1.0, avg_camera_pivot=[0, 0, 0])
    torch.manual_seed(0)
    G = tp.TriPlaneGenerator(z_dim=512, c_dim=25, w_dim=512, img_resolution=res, img_channels=3, rendering_kwargs=rk,
                             cond_mode='none', mapping_kwargs=dict(num_layers=2), channel_base=cb, channel_max=cm,
                             fused_modconv_default='inference_only', num_fp16_res=0, sr_num_fp16_res=4,
                             sr_kwargs=dict(channel_base=cb, channel_max=cm, fused_modconv_default='inference_only'),
                             triplane_width=32, backbone_resolution=256).train().requires_grad_(False).to(dev)
    D = DualDiscriminator(c_dim=25, img_resolution=res, img_channels=3, cond_mode='none', channel_base=cb, channel_max=cm,
                          num_fp16_res=4, conv_clamp=256, block_kwargs=dict(freeze_layers=0), mapping_kwargs=dict(),
                          epilogue_kwargs=dict(mbstd_group_size=4), disc_c_noise=0).train().requires_grad_(False).to(dev)
    import _databacks.lustrous_renders_v1 as dk
    B, R = args.batch, (16 if args.tiny else 64)
    gen = torch.Generator().manual_seed(1)
    gen_z = torch.randn(B, 512, generator=gen).to(dev)
    gen_c = torch.stack([dk.camera_params_to_matrix('eg3d_lustrousB', elev=0.0, azim=-180.0 + 45.0 * i, dist=1.0, fov=30.0)['camera_label']
                         for i in range(B)]).float().to(dev)
    real = {'image': torch.rand(B, 3, res, res, generator=gen).to(dev) * 2 - 1}
    real['image_raw'] = torch.nn.functional.interpolate(real['image'], size=(R, R), mode='bilinear', antialias=True)
    cond = {}
    gain, r1_gamma = 1.0, 1.0
    # training mode 'Agrad': paste_params with grad_sample=True (loss_orthocondA.py:131-150); the thresholds of that mode select nothing
    # on a random-weight generator, so the harness opens them up: mask = (weights > 0.5)
    paste_params = ({'mode': 'default', 'thresh_weight': 0.5, 'thresh_edges': 0.5, 'thresh_occ': 2.0, 'offset_occ': 0.01, 'thresh_dxyz': 10.0,
                     'grad_sample': True} if args.paste else None)
    lin = torch.linspace(0, 1, res)
    yy, xx = torch.meshgrid(lin, lin, indexing='ij')                # a smooth front image: the lookup's gradient is then smooth in xyz,
    front = torch.stack([0.5 + 0.5 * torch.sin(6 * xx + ch) * torch.cos(5 * yy - ch) for ch in range(3)])   # so the arms' different jitter barely moves it
    g_cond = {'image_ortho_front': front[None].repeat(B, 1, 1, 1).to(dev)} if args.paste else cond
    last = {}

    def run_G(update_emas=False):
        ws = G.mapping(gen_z, torch.zeros_like(gen_c), cond, update_emas=update_emas)
        out = G.f({'ws': ws, 'camera_params': gen_c, 'cond': g_cond, 'normalize_images': True, 'neural_rendering_resolution': R,
                   'update_emas': update_emas, 'paste_params': paste_params})
        if paste_params is not None:
            last['mask_mean'] = float(out['paste']['mask'].mean())
        return out, ws

    def run_D(img, c):
        return D(img, c, cond, update_emas=False)

    def phase_Gmain():
        G.requires_grad_(True)
        gen_img, _ = run_G()
        logits = run_D({'image': gen_img['image'], 'image_raw': gen_img['image_raw']}, gen_c)
        torch.nn.functional.softplus(-logits).mean().mul(gain).backward()
        G.requires_grad_(False)

    def phase_Greg():
        G.requires_grad_(True)
        ws = G.mapping(gen_z, torch.zeros_like(gen_c), cond, update_emas=False)
        initial = torch.rand((ws.shape[0], 1000, 3), device=ws.device) * 2 - 1
        perturbed = initial + torch.randn_like(initial) * G.rendering_kwargs['density_reg_p_dist']
        allc = torch.cat([initial, perturbed], dim=1)
        sigma = G.sample_mixed(allc, torch.randn_like(allc), ws, cond, update_emas=False)['sigma']
        tv = torch.nn.functional.l1_loss(sigma[:, :sigma.shape[1] // 2], sigma[:, sigma.shape[1] // 2:]) * G.rendering_kwargs['density_reg']
        tv.mul(gain).backward()
        G.requires_grad_(False)

    def phase_Dmain():
        D.requires_grad_(True)
        with torch.no_grad():
            gen_img, _ = run_G(update_emas=True)
        logits = run_D({'image': gen_img['image'], 'image_raw': gen_img['image_raw']}, gen_c)
        torch.nn.functional.softplus(logits).mean().mul(gain).backward()
        real_logits = run_D({'image': real['image'].detach(), 'image_raw': real['image_raw'].detach()}, gen_c)
        torch.nn.functional.softplus(-real_logits).mean().mul(gain).backward()
        D.requires_grad_(False)

    def phase_Dreg():
        D.requires_grad_(True)
        img = real['image'].detach().requires_grad_(True)
        raw = real['image_raw'].detach().requires_grad_(True)
        logits = run_D({'image': img, 'image_raw': raw}, gen_c)
        with conv2d_gradfix.no_weight_gradients():
            g_img, g_raw = torch.autograd.grad(outputs=[logits.sum()], inputs=[img, raw], create_graph=True, only_inputs=True)
        pen = g_img.square().sum([1, 2, 3]) + g_raw.square().sum([1, 2, 3])
        (pen * (r1_gamma / 2)).mean().mul(gain).backward()
        D.requires_grad_(False)

    phases = [('Gmain', phase_Gmain), ('Greg', phase_Greg), ('Dmain', phase_Dmain), ('Dreg', phase_Dreg)]
    times = {n: [] for n, _ in phases}
    cuda = dev.type == 'cuda'
    for it in range(args.iters + 1):                            # iteration 0 = warm-up (plugin loads, cudnn autotune)
        for name, fn in phases:
            for m in (G, D):
                for p_ in m.parameters():
                    p_.grad = None
            if cuda:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
            fn()
            if cuda:
                e1.record()
                torch.cuda.synchronize()
                if it > 0:
                    times[name].append(e0.elapsed_time(e1))
    prof_line = None
    if args.profile and cuda:
        prof_line = conv_share(phases, (G, D))
    # gradient statistics after a final Gmain + Greg (both arms should agree up to the renderer's jitter)
    for p_ in G.parameters():
        p_.grad = None
    phase_Gmain()
    phase_Greg()
    gstat = {}
    for key, mod in (('backbone', G.backbone), ('decoder', G.decoder), ('superresolution', G.superresolution)):
        gs = [p_.grad.float().norm().item() for p_ in mod.parameters() if p_.grad is not None]
        gstat[key] = {'n_tensors_with_grad': len(gs), 'grad_norm': float(np.sqrt(sum(x * x for x in gs)))}
    line = {'config': 'BASELINE configs[4]: training phases on synthetic 512^2 data (batch %d, R=%d, 48+48)' % (B, R), 'arm': args.arm,
            'conv2d': args.conv2d,
            'ms': {n: (statistics.median(v) if v else None) for n, v in times.items()},
            'ms_total': (sum(statistics.median(v) for v in times.values()) if cuda else None),
            'renderer_module': mod_file.replace(ROOT, '.'), 'grads': gstat}
    if args.paste:
        line['paste'] = {'params': paste_params, 'mask_mean': last.get('mask_mean')}
    if prof_line is not None:
        line['profile'] = prof_line
    if args.arm == 'ours':
        from panic3d_b200 import _lib
        line['gpu_launches'] = _lib.launch_count()
    print(json.dumps(line))


if __name__ == '__main__':
    main()
