"""GPU: multiplane tri-planes (triplane_depth D > 1) on the training path at the training size - the TRI instances of
k_sample_decode and k_sample_backward (csrc/render_v1.cu, csrc/render_backward.cu) and the trilinear taps of
csrc/render_device.cuh - against a hand-written fp64 backward on the device, with a bar per element.

The kernels are called through the C ABI the way _RenderFunction calls them (p3d_render_forward in fp32 SIMT mode with
plane_depth = D, then p3d_render_backward): planes in the (N,3,D,H,W,C) layout, injected uniforms, NaN-filled outputs, a
0xFF workspace, NaN-prefilled backward scratch, and every forward twice, bit-identical.  Cases (each asserts from the data
the property it exists for):

  * train_d2       bench_multiplane.py's training shape: 4 views, spin12 cameras, 64^2 rays, 48+48, 256^2 planes, D = 2,
                   panic3d order; the third 32-lane interval chunk carries gradient on most rays
  * train_d3_cull  the same with D = 3, crop 0.1 + cull 0.5, sigma centred on the cull threshold: partial cull on both
                   passes; mask decisions differ from fp64 only within sigma_error_bound(depth=3), counted
  * slabs_d4       2 views, D = 4, 96 x 64 planes: every slab of every plane receives taps; >= 1 % of the samples lie in
                   the zero-padding bands below slab 0 and above slab D - 1 (one of the two slab taps outside); samples
                   more than half a slab past the box along a normal read nothing from that plane
  * contention_d2  2 views x 64^2 rays x 96 samples on 13 x 9 x 2 planes: >= 1000 contributions on some texel, taps on
                   all six faces of every plane's slab stack
  * auto_eg3d_d2   'auto' limits, EG3D order, lr_mul 0.5, black background: plane 2's normal (y in EG3D, x in panic3d)
                   moves its slab taps for most samples
  * strided_d2     planes as a view (64-channel texels sliced to 32, one padding row per slab stack, so stride_plane >
                   D H stride_row): forward bit-identical to the contiguous copy, gradient within the bar of it
  * bf16_d2        bf16 storage through the C ABI (k_sample_backward<true, true>), against the oracle on the rounded planes;
                   every sample's sigma is within the decode bound of the rounded planes' and most are not of the unrounded

Each runs with the upstream gradient of rgb, depth, wsum and xyz alone, all four, and bench.py's loss.

Reference: render_backward_oracle.render_backward(depth=D) in fp64 on the device, fed the kernel's depths and mask
decisions (tests/test_multiplane_cpu.py pins it to torch's fp64 autograd of multiplane_oracle.render;
test_gpu_fp64_oracle_equals_cpu_oracle pins the device run to the CPU fp32 oracle on the multiplane fixtures).  Bars as in
tests/test_render_backward_paths_gpu.py, bar_i = (k_i + c)(u A_i + 2^-126) + 2 |B64_i - Bk_i|, with k_i the trilinear
tap contributions a texel receives (texel_counts(depth=D)) and c = 2 L + 192 + 13: the one-slab constant plus the 12 extra
gather fmas of the recomputed forward (24 taps instead of 12) and the extra rounding of the weight (wx wy) wz.  Texels no
tap reaches must be exactly 0.

Also: view separation (train_d2: every view rendered and back-propagated alone under autograd with the batch's depth
bounds), the density-regularisation phase at D = 2 (_PointsFunction, k_sample_backward in point mode) and the 96+96
inference render at 128^2 rays on 256^2 planes (fp32 and bf16 storage).

Negative controls on slabs_d4, each missing the kernel by >= 20x its bar: the oracle reading channel d C + c instead of
c D + d, the slab coordinate with align_corners=True, plane 2's normal from the other plane order, dx without the 1/3
plane mean.

Run with -s for every worst error / bar, the runtime and the peak device memory.
"""
import functools
import time

import pytest
import torch

from oracle import multiplane_oracle as mo, render_backward_oracle as rbo, renderer_oracle as orc
from tests import render_abi as ra
from tests.render_abi import DEV, FWD_BAR, PARAMS, UPSTREAM, TrainKernel, compare, cull_sigma, dec64, make_decoder, upstream

pytestmark = pytest.mark.gpu
FREE_BYTES = 24 << 30           # the 256^2 cases: kernel buffers + one view of fp64 oracle intermediates, with margin
CULL_SHARE = 1e-3
C_TRI = 13                      # extra serial steps of the trilinear gather over the bilinear one (see the docstring)

TRAIN = dict(N=4, R=64, S=48, Sf=48, H=256, W=256)
CASES = {
    'train_d2': dict(TRAIN, D=2),
    'train_d3_cull': dict(TRAIN, D=3, flags=dict(triplane_crop=0.1, cull_clouds=0.5), centre_cull=0.5),
    # one spin12-like view and one from above, so that samples leave the box along every plane's normal
    'slabs_d4': dict(N=2, R=32, S=48, Sf=48, H=96, W=64, D=4, views=((0.0, 30.0), (75.0, 0.0))),
    'contention_d2': dict(N=2, R=64, S=48, Sf=48, H=13, W=9, D=2),     # H >= W in every case (run_mutations.py multiplane)
    'auto_eg3d_d2': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, D=2, opts=dict(ray_start='auto', ray_end='auto', white_back=False),
                         eg3d=True, lr_mul=0.5),
    'strided_d2': dict(N=2, R=32, S=48, Sf=48, H=64, W=48, D=2, strided=True),
    'bf16_d2': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, D=2, bf16=True),
}
SEEDS = sorted(CASES)


@functools.lru_cache(maxsize=None)
def _inputs(name):
    """planes (N,3,32*D,H,W) fp32 (channel c*D + d is feature c of slab d), dec, opts, ro, rd, u_c, u_f."""
    case = CASES[name]
    N, R, S, Sf, H, W, D = (case[k] for k in ('N', 'R', 'S', 'Sf', 'H', 'W', 'D'))
    seed = 1700 + SEEDS.index(name)
    g = torch.Generator().manual_seed(seed)
    planes = torch.randn(N, 3, 32 * D, H, W, generator=g)
    _, dec, *_ = orc.synth_inputs(seed, 1, 1, 2, 0, 2)
    dec = dict(dec, lr_mul=case.get('lr_mul', 1.0), b2=dec['b2'].clone())
    opts = dict(dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf, triplane_depth=D),
                **case.get('opts', {}))
    ro, rd = ra.rays_at(case['views'] if 'views' in case else ra.spin12(N), R)
    M = R * R
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, Sf, generator=g)
    if case.get('centre_cull'):                     # median coarse sigma on the cull threshold
        d_c = orc.stratified_depths(u_c.to(DEV), opts['ray_start'], opts['ray_end'])
        xyz = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)[:, ::7]
        _, sig = mo.run_model(planes.to(DEV, torch.float64), dec64(dec), xyz, opts, True)
        dec['b2'][0] += cull_sigma(case['centre_cull']) - sig.median().item()
    return planes, dec, opts, ro, rd, u_c, u_f


def _normal_fz(xyz, D, box_warp, use_triplane):
    """(3,K) fp32 slab coordinate fz of every plane (dev::plane_normal, dev::slab_footprint): slab d is centred on fz = d."""
    s = (2.0 / box_warp) * xyz
    gz = torch.stack([s[:, 2], s[:, 1], s[:, 0 if use_triplane else 1]])
    return ((gz + 1) * D - 1) * 0.5


# ------------------------------------------------------------------------------------------------- tests
def test_gpu_fp64_oracle_equals_cpu_oracle():
    """The device fp64 multiplane render oracle, fed the CPU fp32 run's depths and masks, equals the CPU fp32 oracle on the
    multiplane fixture cases within the fp32 run's rounding; its hand-written gradient equals the fp32 autograd one."""
    from tests.golden.cases_multiplane import RENDER_CASES, build_inputs

    def cases():
        for name in ('d2_eg3d48', 'd3_eg3d96_crop_cull'):
            case = RENDER_CASES[name]
            planes, dec, c2w, K, u_c, u_f, opts = build_inputs(case)
            ro, rd = orc.ray_sampler(c2w, K, case['R'])
            kw = dict(triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'),
                      use_triplane=case['use_triplane'])
            gen = torch.Generator().manual_seed(case['seed'])
            up = lambda out: [torch.randn(t.shape, generator=gen) for t in out]
            yield name, mo.render, planes, dec, ro, rd, u_c, u_f, opts, kw, case['D'], up
    ra.pin_device_oracle(cases())


def _case_checks(name, k, cnt, dsig):
    """The property each case exists for, from the kernel's workspace and scratch and the oracle."""
    planes, dec, *_ = _inputs(name)
    bw, D = k.opts['box_warp'], k.D
    if name == 'train_d2':
        R_ = k.N * k.M
        per = torch.cat([dsig[:R_ * k.S].view(R_, k.S), dsig[R_ * k.S:].view(R_, k.Sf)], 1)
        third = ((per != 0) & (k.merged_rank() >= 64)).any(1).double().mean().item()
        print(f'train_d2: {third:.3f} of the rays carry gradient in the third interval chunk')
        assert third > 0.5, third
    if name == 'train_d3_cull':
        thresh = cull_sigma(0.5)
        d64 = dec64(dec)
        differ = near = total = 0
        for pas, (dk, sk) in enumerate(((k.v['depth_c'], k.v['sigma_c']), (k.v['depth_f'], k.v['sigma_f']))):
            removed = []
            for n in range(k.N):
                xyz = (k.ro[n, :, None] + dk[n][..., None] * k.rd[n, :, None]).reshape(-1, 3)
                s64 = rbo._decoder_forward(k.planes64[n], d64, xyz, bw, True, D)[6][:, 0]      # the kernel's taps, fp64
                crop = orc.crop_mask(xyz[None], 0.1, bw)[0, :, 0]
                mine = crop | orc.cull_mask(s64[None, :, None], 0.5)[0, :, 0]
                kern = sk[n].reshape(-1) == -1e3
                close = (s64 - thresh).abs() <= rbo.sigma_error_bound(k.planes64[n], d64, xyz, bw, True, D)
                assert not ((mine != kern) & ~close).any(), 'cull decisions differ away from the threshold'
                differ += (mine != kern).sum().item()
                near += (close & ~crop).sum().item()
                total += kern.numel()
                removed.append((kern & ~crop).sum().item() / max((~crop).sum().item(), 1))
            share = sum(removed) / len(removed)
            print(f'train_d3_cull pass {pas}: cull removes {share:.3f} of the uncropped samples')
            assert 0.05 < share < 0.95, share
        print(f'train_d3_cull: {differ} of {total} mask decisions differ, all within the kernel\'s sigma error bound of the '
              f'threshold ({near} samples that close)')
        assert differ / total < CULL_SHARE
    if name == 'slabs_d4':
        assert (cnt.sum((-1, -2)) > 0).all(), 'a slab of a plane received no tap'
        xyz = torch.cat([k.samples(n) for n in range(k.N)])
        fz = _normal_fz(xyz, D, bw, True)
        idx3 = rbo.taps(xyz, k.H, k.W, bw, True, D)[0].view(-1, 3, 8)
        idx2 = rbo.taps(xyz, k.H, k.W, bw, True)[0].view(-1, 3, 4)
        K = xyz.shape[0] // k.N
        feat = torch.cat([mo.sample_multiplane(k.planes64[n:n + 1], xyz[None, n * K:(n + 1) * K], bw, True, D)[0]
                          for n in range(k.N)], 1)                                                  # (3,NK,C)
        for p in range(3):
            # one of the two slab taps outside: z0 = -1 or z0 + 1 = D
            below = ((fz[p] > -1) & (fz[p] < 0)).double().mean().item()
            above = ((fz[p] > D - 1) & (fz[p] < D)).double().mean().item()
            past = ((fz[p] < -1) | (fz[p] >= D)) & (idx2[:, p] >= 0).any(1)
            print(f'slabs_d4 plane {p}: {below:.3f} of the samples in the band below slab 0, {above:.3f} above slab {D - 1}; '
                  f'{past.sum().item()} inside the plane but past the box along its normal')
            assert below >= 0.01 and above >= 0.01, (p, below, above)
            assert past.any() and (idx3[past, p] < 0).all() and (feat[p, past] == 0).all(), p
    if name == 'contention_d2':
        print(f'contention_d2: up to {cnt.max().item()} contributions per texel')
        assert cnt.max().item() >= 1000, cnt.max().item()
        for face in (cnt[:, :, 0], cnt[:, :, -1], cnt[..., 0, :], cnt[..., -1, :], cnt[..., :, 0], cnt[..., :, -1]):
            assert (face.sum((-1, -2)) > 0).all(), 'a face of a slab stack received no tap'
    if name == 'auto_eg3d_d2':
        # plane 2's eight taps (texels and weights) with its EG3D normal (y) against the panic3d one (x)
        xyz = k.samples(0)
        own = rbo.taps(xyz, k.H, k.W, bw, False, D)
        other = rbo.taps(xyz, k.H, k.W, bw, False, D, normal_triplane=True)
        moved = ((own[0][:, 16:] != other[0][:, 16:]) | (own[1][:, 16:] != other[1][:, 16:])).any(1).double().mean().item()
        print(f'auto_eg3d_d2: the EG3D normal moves plane 2\'s slab taps for {moved:.3f} of the samples')
        assert moved > 0.5, moved


@pytest.mark.parametrize('name', sorted(CASES))
def test_backward_matches_fp64_oracle(name):
    case = CASES[name]
    if case['H'] * case['W'] >= 256 * 256:
        ra.skip_unless_free(FREE_BYTES)
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    k = TrainKernel(case, _inputs(name))
    dec = k.dec
    out64 = mo.render(k.planes64, dec64(dec), k.ro, k.rd, k.opts, None, None, depths=k.depths(), masks=k.masks(),
                      use_triplane=k.use_triplane, **k.flags)
    for key, a, b in zip(('rgb', 'depth', 'wsum', 'xyz'), k.out, out64):
        err = (a.double() - b).abs().nan_to_num(nan=float('inf')).max().item()
        print(f'{name} forward {key}: max abs err {err:.3e}')
        assert err <= FWD_BAR, (name, key, err)
    del out64
    if case.get('bf16'):
        # the kernel read bf16 texels: its per-sample sigma is within the SIMT decode's error bound of the fp64 decode of the
        # rounded planes, and away from that of the unrounded ones
        xyz, d64 = k.samples(0), dec64(dec)
        sk = torch.cat([k.v['sigma_c'][0].reshape(-1), k.v['sigma_f'][0].reshape(-1)]).double()
        share = []
        for pl in (k.planes64[0], _inputs(name)[0][0].to(DEV, torch.float64)):
            s64 = rbo._decoder_forward(pl, d64, xyz, k.opts['box_warp'], k.use_triplane, k.D)[6][:, 0]
            bound = rbo.sigma_error_bound(pl, d64, xyz, k.opts['box_warp'], k.use_triplane, k.D)
            share.append(((sk - s64).abs() <= bound).double().mean().item())
        print(f'{name}: sigma within the decode bound of the rounded planes for {share[0]:.4f} of the samples, of the '
              f'unrounded ones for {share[1]:.4f}')
        assert share[0] == 1.0 and share[1] < 0.5, share
    if case.get('strided'):
        ref = TrainKernel(case, _inputs(name), strided=False)
        for a, b in zip(k.out, ref.out):
            assert torch.equal(a, b), 'the strided planes render differently from their contiguous copy'
    worst = {}
    for i, kind in enumerate(UPSTREAM):
        grads = upstream(kind, k.N, k.M, 50 + i)
        got, dsig = k.backward(grads)
        assert not torch.isnan(dsig).any(), 'a sample was never written by k_ray_backward'
        b64, bars, cnt = k.bars(grads, C_TRI)
        if i == 0:
            _case_checks(name, k, cnt, dsig)
        taps = ra.per_channel(cnt, k.D)
        w = compare(f'{name} [{kind}]', got, b64, bars, taps)
        worst.update({(kind, key): r for key, r in w.items()})
        assert max(w.values()) <= 1.0, (name, kind, w)
        assert (got['planes'][taps == 0] == 0).all(), 'a texel no tap reaches got a gradient'
        if kind == 'all':
            again, _ = k.backward(grads)
            assert max(compare(f'{name} [repeat]', again, b64, bars).values()) <= 1.0
            if case.get('strided'):
                contiguous, _ = ref.backward(grads)
                w2 = compare(f'{name} [contiguous copy]', got, {q: contiguous[q].double() for q in PARAMS}, bars)
                assert max(w2.values()) <= 1.0, w2
            if name == 'train_d2':
                _views_alone(name, k, grads, b64, bars, cnt)
        if (name, kind) in CONTROLS:
            _negative_controls(name, k, grads, got, bars)
    print(f'{name}: worst err / bar {max(worst.values()):.4f} ({max(worst, key=worst.get)}); {time.time() - t0:.1f} s, '
          f'peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB')


def _views_alone(name, k, grads, b64, bars, cnt):
    """Each view rendered and back-propagated alone through ImportanceRenderer under autograd, with the batch's depth-clamp
    bounds injected: its forward equals the batch's bit for bit, its plane gradient the batch oracle's slice within the bar,
    exactly 0 where the view's taps do not reach."""
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    b2 = torch.empty(2, device=DEV)
    _lib.check(_lib.lib().p3d_render_depth_bounds(k.ws.data_ptr(), b2.data_ptr(), _lib.stream_ptr(DEV)))
    torch.cuda.synchronize()
    r = ImportanceRenderer(use_triplane=k.use_triplane)
    r.depth_bounds_reduce = lambda t: t.copy_(b2)
    d = make_decoder(dec, DEV).requires_grad_(True)
    M = k.M
    for i in range(k.N):
        r.injected_noise = (u_c[i:i + 1], u_f[i * M:(i + 1) * M])
        pv = planes[i:i + 1].to(DEV).requires_grad_(True)
        out = r(pv, d, ro[i:i + 1], rd[i:i + 1], opts, **k.flags)
        for o, f in zip(out, k.out):
            assert torch.equal(o.detach(), f[i:i + 1]), 'a view alone renders differently from the batch'
        g = torch.autograd.grad(sum((o * gg[i:i + 1]).sum() for o, gg in zip(out, grads)), [pv])[0]
        err, r_ = ra.ratio(g, b64['planes'][i:i + 1], bars['planes'][i:i + 1])
        print(f'view {i} alone d_planes: max abs err {err:.3e}, worst err / bar {r_:.4f}')
        assert r_ <= 1.0, (i, r_)
        assert (g[ra.per_channel(cnt[i:i + 1], k.D) == 0] == 0).all()


# upstream -> mutated oracles.  Each must miss the kernel by >= 20x its bar.
CONTROLS = {('slabs_d4', 'all')}


def _negative_controls(name, k, grads, got, bars):
    N, D, H, W = k.N, k.D, k.H, k.W
    swapped = k.planes64.reshape(N, 3, D, 32, H, W).transpose(2, 3).reshape(N, 3, 32 * D, H, W)   # [c*D + d] = [d*32 + c]
    real_taps = rbo.taps
    controls = {
        'slab order d*C + c': lambda: dict(k.oracle(grads, planes=swapped)),
        'slab coordinate with align_corners=True': lambda: k.oracle(grads),
        "plane 2's normal from the other plane order": lambda: k.oracle(grads),
        'dx without the 1/3 plane mean': lambda: k.oracle(grads, plane_mean=1.0),
    }
    patches = {'slab coordinate with align_corners=True': dict(slab_align_corners=True),
               "plane 2's normal from the other plane order": dict(normal_triplane=not k.use_triplane)}
    for label, run in controls.items():
        rbo.taps = functools.partial(real_taps, **patches.get(label, {}))
        try:
            mut = run()
        finally:
            rbo.taps = real_taps
        if label == 'slab order d*C + c':        # back to the planes' own indexing
            mut['planes'] = mut['planes'].reshape(N, 3, 32, D, H, W).transpose(2, 3).reshape(N, 3, 32 * D, H, W)
        ra.negative_control(label, name, got, mut, bars)


# ------------------------------------------------------------------------------------------------- density regularisation
def test_density_regularisation_phase_d2():
    """The Greg phase on D = 2 planes (_PointsFunction: the TRI point decode in fp32 SIMT mode, no fused launch, then
    k_sample_backward in point mode).  90 % of the pairs read no texel at D = 2 (the slab axis adds a third bound); of
    the ~400 others, two 0.004-apart points differ by under 2e-4 in sigma for a few: gate share 3 %."""
    from panic3d_b200 import _lib
    ra.skip_unless_free(FREE_BYTES)
    ra.density_regularisation(mo.run_model, 2, _lib.P3D_MLP_FP32_SIMT, lambda prof: prof[0] >= 1 and prof[5] == 0,
                              gate_share=0.03, c=192 + C_TRI)


# ------------------------------------------------------------------------------------------------- inference
@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
def test_inference_render_at_the_eval_shape(bf16):
    """A 96+96 render of 2 views at 128^2 rays on 256^2 D = 2 planes through ImportanceRenderer with mlp_mode 'auto': the
    SIMT kernels run and the fused slot does not; within 1e-4 of the fp64 oracle (on the bf16-rounded planes for bf16
    storage) fed the depths and masks of the device fp32 oracle."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from tests.helpers import profiled
    ra.skip_unless_free(FREE_BYTES)
    t0 = time.time()
    N, R, H, D = 2, 128, 256, 2
    g = torch.Generator().manual_seed(1800 + bf16)
    planes = torch.randn(N, 3, 32 * D, H, H, generator=g)
    _, dec, *_ = orc.synth_inputs(1800, 1, 1, 2, 0, 2)
    opts = dict(orc.DEFAULT_OPTS, triplane_depth=D)
    S, Sf = opts['depth_resolution'], opts['depth_resolution_importance']
    ro, rd = ra.rays_at(ra.spin12(N), R)
    u_c, u_f = torch.rand(N, R * R, S, 1, generator=g), torch.rand(N * R * R, Sf, generator=g)
    r = ImportanceRenderer(use_triplane=True)
    r.injected_noise = (u_c, u_f)
    r.planes_bf16 = bf16
    with torch.no_grad():
        out, n = profiled(lambda: r(planes.to(DEV), make_decoder(dec, DEV), ro, rd, opts))
    assert n[0] >= 1 and n[5] == 0, n
    ref = (planes.bfloat16().float() if bf16 else planes).to(DEV)
    dev_dec = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in dec.items()}
    _, smp = mo.render(ref, dev_dec, ro, rd, opts, u_c.to(DEV), u_f.to(DEV), use_triplane=True, return_samples=True)
    out64 = mo.render(ref.double(), dec64(dec), ro, rd, opts, None, None, use_triplane=True, depths=smp['depths'],
                      masks=smp['masks'])
    for key, a, b in zip(('rgb', 'depth', 'wsum', 'xyz'), out, out64):
        err = (a.double() - b).abs().nan_to_num(nan=float('inf')).max().item()
        print(f'eval render D=2 {"bf16" if bf16 else "fp32"} {key}: max abs err {err:.3e}')
        assert err <= FWD_BAR, (key, err)
    print(f'eval render: {time.time() - t0:.1f} s')
