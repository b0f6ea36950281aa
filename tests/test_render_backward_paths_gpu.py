"""GPU: the training backward (csrc/render_backward.cu: k_ray_backward + k_sample_backward) at the training size, against a
hand-written fp64 backward on the device, with a bar per element.

Every training step runs these kernels behind _RenderFunction.  The older gradient tests compare with CPU fp32 autograd at
fixture sizes under one normwise bar per tensor.  Here the kernels are called through the C ABI (p3d_render_forward with
mlp_mode fp32 SIMT, then p3d_render_backward), the way _RenderFunction calls them:

  * train       bench.py's training context: 4 views, 64^2 rays, 48+48 samples, 256^2 planes, spin12 cameras; 12288
                sample-backward CTAs, 95 intervals per ray (three 32-lane chunks)
  * train_cull  train + crop 0.1, cull 0.5, sigma bias centred on the cull threshold: partial cull on both passes
  * branches    planes x15, W1 x3, sigma bias +30: >= 5 % of pre-activations above 20 and below -20, >= 5 % of the
                interval arguments smid above 20 (both linear branches of softplus' derivative)
  * binarize    binarize 0.5 + crop: every per-sample sigma gradient is exactly 0, only colours carry gradient
  * contention  9 x 13 planes under 2 x 64^2 rays x 96 samples: texels take thousands of atomic adds, the footprint spills
                over every edge
  * auto_eg3d   'auto' ray limits, EG3D plane order, lr_mul 0.5, black background
  * small       1 view, 8^2 rays, 48+48, median sigma 10: 48 sample-backward CTAs, so the decoder bars are tight
  * softplus    every pre-activation in (5, 20): non-negative features, W1 and sigma row of W2, b1 ~ 5.2, median sigma -1

Each case runs with the upstream gradient of one output at a time (rgb, depth, wsum, xyz), all four together, and bench.py's
loss rgb.mean() + 0.1 depth.mean() + 0.1 wsum.mean() (all upstream gradients positive: no cancellation inflates A).

Reference: oracle/render_backward_oracle.render_backward in fp64 on the device, fed the kernel's fp32 depths (coarse and
fine) and mask decisions read from the forward workspace (constants of the reference graph; with its own, an fp64
searchsorted or a cull decision near its threshold would move whole samples).  tests/test_render_backward_oracle_cpu.py
pins that backward to torch's fp64 autograd of the oracle; test_gpu_fp64_oracle_equals_cpu_oracle pins the device run to
the CPU fp32 oracle.

Bars, per element, from the roundings of the kernel's own operations (u = 2^-24):
    bar_i = (k_i + c) (u A_i + TINY) + 2 |B64_i - Bk_i|
  A      the magnitude adjoint: the same backward with every product and partial sum in absolute value (the suffix sum the
         kernel forms as total - prefix counts as total + prefix), plus floors for errors that are not relative to the
         value (render_backward_oracle._floors: 1 - expf, 1 - sigmoid, the fp32 pre-activations and logits);
  k_i    plane texels: the tap contributions the texel receives (counted from the taps, one fp32 atomic add each);
         decoder tensors: 128 serial fmas per CTA + the number of sample-backward CTAs, each adding once;
  TINY   2^-126 per rounding step: fp32 underflow (a value whose fp64 counterpart lies below the normal range may be 0);
  c      2 L + 192 for L = S + Sf samples per ray: the serial depth inside one element's path - the ray's scans (transmittance
         product and the w P prefix, each <= L), 33 + 64 fmas of the decoder backward, the 33 + 32 fmas of its recomputed
         forward and the handful of elementwise roundings, with margin;
  B64 - Bk  the first-order effect of the forward's rounding: the fp64 backward run on its own fp64 sigma / rgb (B64) and
         on the kernel's fp32 sigma / rgb from the workspace (Bk); factor 2 for the second order.
Texels no sample touches must be exactly 0 (A = 0 there), as must the sigma row of the decoder gradient under binarize.

Forward: outputs within 1e-4 of the fp64 oracle fed the same depths and masks (the SIMT decode's bar), repeated bit for bit.
Backward: a repeat stays within the bar (float atomics change the summation order).  The backward scratch (dsig, omega) is
prefilled with NaN, so a sample k_ray_backward never writes poisons the gradients; NaN fails every ratio.

Negative controls, each missing the kernel by >= 20x its bar: the colour factor 1 instead of 1.002 (bench loss, `small`),
the softplus-derivative threshold 5 instead of 20 (wsum upstream of ones, `softplus`: dsig >= 0 everywhere, so nothing
cancels), no 1/3 plane mean in dx (train, all).

Density regularisation (`test_density_regularisation_phase`): 4 views x (1000 points uniform in [-1, 1]^3 + the same
points perturbed by N(0, 0.004^2)), 256^2 planes, training options, through ImportanceRenderer.run_model under autograd
and loss_orthocondA's L1.  The forward kernel that ran is asserted (mlp_mode and one launch in the decode slot); sigma
within 1e-4 of the fp64 oracle; pairs whose fp64 difference lies within 2e-4 (both forward bars) of 0 may take either sign,
and are counted; gradients against render_backward_oracle.points_backward fed the kernel's signs, bar (k + 192)(u A + TINY).

Run with -s for the worst error / bar of every comparison, the runtime and the peak device memory.
"""
import functools
import math
import time

import pytest
import torch

from oracle import render_backward_oracle as rbo, renderer_oracle as orc
from tests import render_abi as ra
from tests.helpers import BWD_CASES, bwd_flags, bwd_incoming
from tests.render_abi import DEV, FWD_BAR, PARAMS, UPSTREAM, TrainKernel, compare, cull_sigma, dec64, make_decoder, upstream

pytestmark = pytest.mark.gpu
FREE_BYTES = 24 << 30           # the 256^2 cases: kernel buffers (~3 GB) + one view of fp64 oracle intermediates, with margin
CULL_SHARE = 1e-3               # samples whose fp64 cull decision may differ from the kernel's (within its sigma error bound)

TRAIN = dict(N=4, R=64, S=48, Sf=48, H=256, W=256)
CASES = {
    'train': dict(TRAIN),
    'train_cull': dict(TRAIN, flags=dict(triplane_crop=0.1, cull_clouds=0.5), centre_cull=0.5),
    'branches': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, planes_scale=15.0, w1_scale=3.0, sigma_bias=30.0),
    'binarize': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, flags=dict(triplane_crop=0.1, binarize_clouds=0.5)),
    'contention': dict(N=2, R=64, S=48, Sf=48, H=9, W=13),
    'small': dict(N=1, R=8, S=48, Sf=48, H=64, W=64, centre_sigma=10.0),
    'softplus': dict(N=1, R=8, S=48, Sf=48, H=64, W=64, softplus_window=5.2, centre_sigma=-1.0),
    'auto_eg3d': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, opts=dict(ray_start='auto', ray_end='auto', white_back=False),
                      eg3d=True, lr_mul=0.5),
}
SEEDS = ('auto_eg3d', 'binarize', 'branches', 'contention', 'small', 'train', 'train_cull', 'softplus')


def _skip_small_device(case):
    if case['H'] * case['W'] >= 256 * 256:
        ra.skip_unless_free(FREE_BYTES)


# ------------------------------------------------------------------------------------------------- inputs
@functools.lru_cache(maxsize=None)
def _inputs(name):
    case = CASES[name]
    N, R, S, Sf, H, W = (case[k] for k in ('N', 'R', 'S', 'Sf', 'H', 'W'))
    seed = 900 + SEEDS.index(name)
    g = torch.Generator().manual_seed(seed)
    planes = torch.randn(N, 3, 32, H, W, generator=g) * case.get('planes_scale', 1.0)
    _, dec, *_ = orc.synth_inputs(seed, 1, 1, 2, 0, 2)
    dec = dict(dec, lr_mul=case.get('lr_mul', 1.0), w1=dec['w1'] * case.get('w1_scale', 1.0), b2=dec['b2'].clone())
    dec['b2'][0] += case.get('sigma_bias', 0.0)
    if case.get('softplus_window'):
        # non-negative features, W1 and sigma row of W2, every pre-activation just above 5: the derivative's sigmoid branch
        # is 0.1-0.6 % below 1 there, with no cancellation anywhere in the wsum backward
        planes = planes.abs() * 0.2
        dec['w1'] = dec['w1'].abs() * 0.2
        dec['b1'] = dec['b1'] * 0.1 + case['softplus_window']
        dec['w2'] = dec['w2'].clone()
        dec['w2'][0] = dec['w2'][0].abs() * 0.05
    opts = dict(dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf), **case.get('opts', {}))
    ro, rd = ra.rays_at(ra.spin12(N), R)
    M = R * R
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, Sf, generator=g)
    centre = cull_sigma(case['centre_cull']) if case.get('centre_cull') else case.get('centre_sigma')
    if centre is not None:                          # median coarse sigma on `centre`
        d_c = orc.stratified_depths(u_c.to(DEV), opts['ray_start'], opts['ray_end'])
        xyz = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)[:, ::7]
        _, sig = orc.run_model(planes.to(DEV, torch.float64), dec64(dec), xyz, opts, True)
        dec['b2'][0] += centre - sig.median().item()
    return planes, dec, opts, ro, rd, u_c, u_f


# ------------------------------------------------------------------------------------------------- tests
def test_gpu_fp64_oracle_equals_cpu_oracle():
    """The device fp64 run of the render oracle (with injected depths and masks) equals the CPU fp32 oracle on the
    fixture-sized gradient cases, within the fp32 run's rounding; its hand-written gradients equal the CPU fp32 autograd ones
    within 1e-5 of each tensor's largest element."""
    from tests.golden.cases import build_case_inputs
    from tests.helpers import case_rays

    def cases():
        for name in ('train48', 'eval96'):
            case = BWD_CASES[name]
            planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
            ro, rd = case_rays(case, c2w, K)
            up = lambda out: bwd_incoming(case['seed'] + 5, ro.shape[0], ro.shape[1])
            yield name, orc.render, planes, dec, ro, rd, u_c, u_f, opts, bwd_flags(case), 1, up
    ra.pin_device_oracle(cases())


def _case_checks(name, k, b64, bars, cnt, dsig):
    """The property each case exists for, from the kernel's workspace and scratch and the oracle."""
    planes, dec, *_ = _inputs(name)
    if name == 'train':
        # the third 32-lane chunk of k_ray_backward carries gradient: samples ranked >= 64 in their ray get a nonzero
        # dsig on most rays
        R_ = k.N * k.M
        per = torch.cat([dsig[:R_ * k.S].view(R_, k.S), dsig[R_ * k.S:].view(R_, k.Sf)], 1)
        third = ((per != 0) & (k.merged_rank() >= 64)).any(1).double().mean().item()
        print(f'train: {third:.3f} of the rays carry gradient in the third interval chunk')
        assert third > 0.5, third
    if name == 'auto_eg3d':
        t0, t1 = k.v['ray_t0'], k.v['ray_t1']
        distinct = min(torch.unique(t0[n]).numel() for n in range(k.N))
        spread = min((t0[n].max() - t0[n].min()).item() for n in range(k.N))
        xyz = (k.ro[0, :, None] + k.v['depth_c'][0][..., None] * k.rd[0, :, None]).reshape(-1, 3)
        H_, W_ = k.planes_cl.shape[2], k.planes_cl.shape[3]
        moved = (rbo.taps(xyz, H_, W_, k.opts['box_warp'], False)[0][:, 8:] !=
                 rbo.taps(xyz, H_, W_, k.opts['box_warp'], True)[0][:, 8:]).any(1).double().mean().item()
        print(f'auto_eg3d: >= {distinct} distinct per-ray starts per view spanning >= {spread:.3f}, '
              f'{(t1 <= t0).sum().item()} rays miss the box; '
              f'the EG3D order moves plane 2\'s taps for {moved:.3f} of the samples')
        assert distinct >= 64 and spread > 0.01 and moved > 0.5, (distinct, spread, moved)
    if name == 'softplus':
        xyz = (k.ro[0, :, None] + k.v['depth_c'][0][..., None] * k.rd[0, :, None]).reshape(-1, 3)
        pre = rbo._decoder_forward(planes[0].to(DEV, torch.float64), dec64(dec), xyz, k.opts['box_warp'], True)[4]
        inside = ((pre > 5) & (pre < 20)).double().mean().item()
        print(f'softplus: {inside:.4f} of the pre-activations in (5, 20)')
        assert inside > 0.95, inside
    if name == 'contention':
        assert cnt.max().item() >= 1000, cnt.max().item()
        # taps fall on all four edges of every plane
        for edge in (cnt[..., 0, :], cnt[..., -1, :], cnt[..., :, 0], cnt[..., :, -1]):
            assert (edge.sum(-1) > 0).all()
    if name == 'branches':
        xyz = (k.ro[0, :, None] + k.v['depth_c'][0][..., None] * k.rd[0, :, None]).reshape(-1, 3)
        idx, wgt = rbo.taps(xyz, k.planes_cl.shape[2], k.planes_cl.shape[3], k.opts['box_warp'], True)
        flat = planes[0].to(DEV, torch.float64).permute(0, 2, 3, 1).reshape(-1, 32)
        d = dec64(dec)
        pre = rbo.gather(flat, idx, wgt).sum(1) / 3 @ (d['w1'] / math.sqrt(32)).t() + d['b1']
        hi, lo = (pre > 20).double().mean().item(), (pre < -20).double().mean().item()
        t = torch.cat([k.v['depth_c'], k.v['depth_f']], -1)
        sg = torch.gather(torch.cat([k.v['sigma_c'], k.v['sigma_f']], -1), -1, torch.sort(t, dim=-1, stable=True)[1])
        smid = ((sg[..., 1:] + sg[..., :-1]) / 2 - 1)
        sm = (smid > 20).double().mean().item()
        print(f'branches: pre > 20 {hi:.3f}, pre < -20 {lo:.3f}, smid > 20 {sm:.3f}')
        assert hi >= 0.05 and lo >= 0.05 and sm >= 0.05, (hi, lo, sm)
    if name == 'train_cull':
        thresh = cull_sigma(0.5)
        p64, d64 = planes.to(DEV, torch.float64), dec64(dec)
        differ = near = total = 0
        for pas, (dk, sk) in enumerate(((k.v['depth_c'], k.v['sigma_c']), (k.v['depth_f'], k.v['sigma_f']))):
            removed = []
            for n in range(k.N):
                xyz = (k.ro[n, :, None] + dk[n][..., None] * k.rd[n, :, None]).reshape(1, -1, 3)
                _, s64 = orc.run_model(p64[n:n + 1], d64, xyz, k.opts, True)
                crop = orc.crop_mask(xyz, 0.1, k.opts['box_warp'])
                mine = (crop | orc.cull_mask(s64, 0.5))[0, :, 0]
                kern = sk[n].reshape(-1) == -1e3
                bound = rbo.sigma_error_bound(p64[n], d64, xyz[0], k.opts['box_warp'])
                close = (s64[0, :, 0] - thresh).abs() <= bound
                assert not ((mine != kern) & ~close).any(), 'cull decisions differ away from the threshold'
                differ += (mine != kern).sum().item()
                near += (close & ~crop[0, :, 0]).sum().item()
                total += kern.numel()
                removed.append((kern & ~crop[0, :, 0]).sum().item() / max((~crop[0, :, 0]).sum().item(), 1))
            share = sum(removed) / len(removed)
            print(f'train_cull pass {pas}: cull removes {share:.3f} of the uncropped samples')
            assert 0.05 < share < 0.95, share
        print(f'train_cull: {differ} of {total} mask decisions differ, all within the kernel\'s sigma error bound of the '
              f'threshold ({near} samples that close)')
        assert differ / total < CULL_SHARE


@pytest.mark.parametrize('name', sorted(CASES))
def test_backward_matches_fp64_oracle(name):
    case = CASES[name]
    _skip_small_device(case)
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    k = TrainKernel(case, _inputs(name))
    # forward: within the decode bar of the fp64 oracle fed the kernel's depths and masks
    out64 = orc.render(k.planes64, dec64(k.dec), k.ro, k.rd, k.opts, None, None, depths=k.depths(), masks=k.masks(),
                       use_triplane=k.use_triplane, **k.flags)
    for key, a, b in zip(('rgb', 'depth', 'wsum', 'xyz'), k.out, out64):
        err = (a.double() - b).abs().nan_to_num(nan=float('inf')).max().item()
        print(f'{name} forward {key}: max abs err {err:.3e}')
        assert err <= FWD_BAR, (name, key, err)
    del out64
    worst = {}
    for i, kind in enumerate(UPSTREAM):
        grads = upstream(kind, k.N, k.M, 50 + i)
        got, dsig = k.backward(grads)
        assert not torch.isnan(dsig).any(), 'a sample was never written by k_ray_backward'
        b64, bars, cnt = k.bars(grads)
        if i == 0:
            _case_checks(name, k, b64, bars, cnt, dsig)
        taps = ra.per_channel(cnt, 1)
        w = compare(f'{name} [{kind}]', got, b64, bars, taps)
        for key, r in w.items():
            worst[(kind, key)] = r
        assert max(w.values()) <= 1.0, (name, kind, w)
        assert (got['planes'][taps == 0] == 0).all(), 'a texel no sample touches got a gradient'
        if case.get('flags', {}).get('binarize_clouds'):      # no sigma gradient reaches the decoder: its sigma row stays 0
            assert (got['w2'][0] == 0).all() and got['b2'][0].item() == 0, 'binarize: a sigma gradient is not exactly 0'
        if kind == 'depth':
            dead = (k.out[2].reshape(-1) == 0)
            R_ = k.N * k.M
            per_ray = torch.cat([dsig[:R_ * k.S].view(R_, k.S), dsig[R_ * k.S:].view(R_, k.Sf)], 1)
            assert (per_ray[dead] == 0).all(), 'a ray with W = 0 passed a depth gradient'
            print(f'{name}: {dead.sum().item()} rays with W = 0')
        if kind == 'all':
            again, _ = k.backward(grads)
            w2 = compare(f'{name} [repeat]', again, b64, bars)
            assert max(w2.values()) <= 1.0
    for (case_name, kind), (label, kw) in CONTROLS.items():
        if case_name == name:
            grads = upstream(kind, k.N, k.M, 99)
            got, _ = k.backward(grads)
            b64, bars, cnt = k.bars(grads)
            assert max(compare(f'{name} [{kind}]', got, b64, bars, ra.per_channel(cnt, 1)).values()) <= 1.0
            ra.negative_control(label, f'{name} [{kind}]', got, k.oracle(grads, **kw), bars)
    print(f'{name}: worst err / bar {max(worst.values()):.4f} ({max(worst, key=worst.get)}); {time.time() - t0:.1f} s, '
          f'peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB')


# case, upstream -> (label, mutated oracle).  Each must miss the kernel by >= 20x its bar.  `small` is dense (median sigma
# 10, so alpha is far above its 3u floor) and has 48 sample-backward CTAs, so the colour rows of the decoder gradient carry
# the 0.2 % colour factor without cancellation; `softplus` puts every pre-activation just above 5, and its wsum upstream
# makes every dsig non-negative, so dx, d_w1 and d_b1 sum terms of one sign.
CONTROLS = {
    ('small', 'bench'): ('colour factor 1', dict(col_factor=1.0)),
    ('softplus', 'wsum+'): ('softplus derivative threshold 5', dict(sp_thresh=5.0)),
    ('train', 'all'): ('no 1/3 plane mean in dx', dict(plane_mean=1.0)),
}


def test_autograd_route_matches_the_abi_call():
    """ImportanceRenderer under autograd (_RenderFunction) gives the C ABI call's forward bit for bit and its gradients
    within the bars (train_cull: masks and partial cull on the route the training loop takes)."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    name = 'train_cull'
    _skip_small_device(CASES[name])
    k = TrainKernel(CASES[name], _inputs(name))
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    r = ImportanceRenderer(use_triplane=True)
    r.injected_noise = (u_c, u_f)
    d = make_decoder(dec, DEV).requires_grad_(True)
    pg = planes.to(DEV).requires_grad_(True)
    out = r(pg, d, ro, rd, opts, **k.flags)
    for a, b in zip(out, k.out):
        assert torch.equal(a.detach(), b)
    grads = upstream('bench', k.N, k.M, 0)
    got = torch.autograd.grad(sum((o * g).sum() for o, g in zip(out, grads)),
                              [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    b64, bars, _ = k.bars(grads)
    w = compare('autograd route [bench]', dict(zip(PARAMS, got)), b64, bars)
    assert max(w.values()) <= 1.0, w


def test_density_regularisation_phase():
    """The Greg phase on one-slab planes: the forward is the tensor-core 3-pass decode with one launch in the decode slot
    (profile slot 0), and the hand-written points backward the oracle's fp64 autograd gradient."""
    from panic3d_b200 import _lib
    opts, p64, d64, coords, g_sigma, b64, A = ra.density_regularisation(
        orc.run_model, 1, _lib.P3D_MLP_TC_3XBF16, lambda prof: prof[0] == 1, gate_share=0.01, c=192)
    pr = p64.clone().requires_grad_(True)
    dr = {k_: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k_, v in d64.items()}
    ref = torch.autograd.grad((orc.run_model(pr, dr, coords, opts, True)[1] * g_sigma[..., None]).sum(),
                              [pr] + [dr[k_] for k_ in ('w1', 'b1', 'w2', 'b2')])
    for key, rf in zip(PARAMS, ref):       # relative to A: d_b2[0] is a sum of +-1/n that cancels to 0 exactly
        assert (b64[key] - rf).abs().max().item() <= 1e-10 * A[key].max().item(), key
