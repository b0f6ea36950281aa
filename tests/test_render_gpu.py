"""GPU parity: the CUDA renderer (through the ctypes C-ABI) vs (a) outputs of the unmodified
reference (tests/golden/*.npz) and (b) the CPU oracle, on identical planes / decoder / rays / jitter.
Tolerance: north_star's 1e-3 max-abs (fp32); the fp32 SIMT kernels are expected ~1e-5."""
import json

import numpy as np
import pytest
import torch

from oracle import renderer_oracle as orc
from tests.golden.cases import RENDER_CASES, POINT_CASES, build_case_inputs
from tests.helpers import load_golden, oracle_render

pytestmark = pytest.mark.gpu
TOL = 1e-3          # the bar
TIGHT = 1e-4        # what the fp32 path should really reach (no cull discontinuity)


def _dev():
    return torch.device('cuda:0')


def make_decoder(dec, dev):
    from panic3d_b200.training.triplane import OSGDecoder
    d = OSGDecoder(dec['w1'].shape[1], {'decoder_lr_mul': dec['lr_mul'], 'decoder_output_dim': dec['w2'].shape[0] - 1})
    with torch.no_grad():
        d.net[0].weight.copy_(dec['w1']); d.net[0].bias.copy_(dec['b1'])
        d.net[2].weight.copy_(dec['w2']); d.net[2].bias.copy_(dec['b2'])
    d.set_force_sigmoid(bool(dec['force_sigmoid']))
    return d.to(dev).requires_grad_(False)


def gpu_rays(case, c2w, K, dev):
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    from panic3d_b200 import cameras
    R = case['R']
    if case.get('ortho'):
        ros, rds = [], []
        for (e, a, d, _f) in case['cameras']:
            r = cameras.get_rays_ortho(e, a, d, case['opts']['box_warp'], R, device=dev)
            ros.append(r['ray_origins'].reshape(1, 3, R * R).permute(0, 2, 1))
            rds.append(r['ray_directions'].reshape(1, 3, R * R).permute(0, 2, 1))
        return torch.cat(ros).contiguous(), torch.cat(rds).contiguous()
    return RaySampler()(c2w.to(dev), K.to(dev), R)


def gpu_render(case, mlp_mode=0, planes_layout='nchw'):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = gpu_rays(case, c2w, K, dev)
    r = ImportanceRenderer(use_triplane=case.get('use_triplane', True))
    r.mlp_mode = mlp_mode
    r.injected_noise = (u_c, u_f)
    pl = planes.to(dev)
    if planes_layout == 'channels_last':     # (N,96,H,W) torch.channels_last, viewed as (N,3,32,H,W)
        N, P, Cc, H, W = pl.shape
        pl = pl.reshape(N, P * Cc, H, W).contiguous(memory_format=torch.channels_last).view(N, P, Cc, H, W)
        assert pl.stride(2) == 1
    with torch.no_grad():
        out = r(pl, make_decoder(dec, dev), ro, rd, opts, triplane_crop=case.get('triplane_crop'),
                cull_clouds=case.get('cull_clouds'), binarize_clouds=case.get('binarize_clouds'))
    torch.cuda.synchronize()
    return [t.cpu() for t in out], (ro.cpu(), rd.cpu())


def _strided(case, outs):
    """Big cases store every `store_stride`-th ray of the reference output (tests/golden/make_golden.py)."""
    st = int(case.get('store_stride', 1))
    return [o[:, ::st] for o in outs] if st > 1 else list(outs)


@pytest.mark.parametrize('name', sorted(RENDER_CASES))
def test_render_matches_reference_fixture(name):
    g = load_golden('render', name)
    outs, _ = gpu_render(g['case'])
    rgb, depth, wsum, xyz = _strided(g['case'], outs)
    has_cull = bool(g['case'].get('cull_clouds') or g['case'].get('binarize_clouds'))
    for got, key in ((rgb, 'rgb'), (depth, 'depth'), (wsum, 'wsum'), (xyz, 'xyz')):
        err = (got - g[key]).abs()
        if has_cull:
            # the reference's cull mask is a hard threshold on sigma (renderer.py:150-153): a sample whose
            # alpha sits within rounding of the threshold may flip; such flips are isolated, so require
            # 99.9% of outputs within TIGHT and everything within 2e-2
            assert (err < TIGHT).float().mean().item() > 0.999, f'{name}:{key}'
            assert err.max().item() < 2e-2, f'{name}:{key} max {err.max().item()}'
        else:
            assert err.max().item() < TIGHT, f'{name}:{key} max abs err {err.max().item()} (bar {TOL})'


@pytest.mark.parametrize('name', ['small_plain', 'small_ortho', 'small_batch3'])
def test_rays_match_oracle(name):
    from tests.helpers import case_rays
    case = RENDER_CASES[name]
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = gpu_rays(case, c2w, K, _dev())
    o_ro, o_rd = case_rays(case, c2w, K)
    assert (ro.cpu() - o_ro).abs().max().item() < 1e-6
    assert (rd.cpu() - o_rd).abs().max().item() < 1e-6


def test_channels_last_planes_are_zero_copy_and_equal():
    case = RENDER_CASES['small_batch3']
    a, _ = gpu_render(case, planes_layout='nchw')
    b, _ = gpu_render(case, planes_layout='channels_last')
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize('name', sorted(POINT_CASES))
def test_run_model_matches_reference_fixture(name):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    g = load_golden('points', name)
    case = g['case']
    dev = _dev()
    planes, dec, *_r, opts = build_case_inputs(case)
    r = ImportanceRenderer(use_triplane=case.get('use_triplane', True))
    with torch.no_grad():
        out = r.run_model(planes.to(dev), make_decoder(dec, dev), g['pts'].to(dev), None, opts)
    assert (out['rgb'].cpu() - g['rgb']).abs().max().item() < TIGHT
    assert (out['sigma'].cpu() - g['sigma']).abs().max().item() < TIGHT
    assert out['sigma'].shape == (planes.shape[0], case['K'], 1)


def test_run_model_out_of_box_and_nan_points():
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = POINT_CASES['pts_small']
    dev = _dev()
    planes, dec, *_r, opts = build_case_inputs(case)
    pts = torch.tensor([[[0.0, 0.0, 0.0], [10.0, -10.0, 3.0], [1e30, 0.0, 0.0], [0.3499, 0.3499, -0.3499]]]).expand(2, -1, -1).contiguous()
    r = ImportanceRenderer(use_triplane=True)
    with torch.no_grad():
        out = r.run_model(planes.to(dev), make_decoder(dec, dev), pts.to(dev), None, opts)
    rgb, sigma = orc.run_model(planes, dec, pts, opts, True)
    assert (out['rgb'].cpu() - rgb).abs().max().item() < TIGHT
    assert (out['sigma'].cpu() - sigma).abs().max().item() < TIGHT


def test_philox_jitter_is_statistically_equivalent():
    """Without injected noise the kernels draw Philox uniforms; the render must agree with the
    injected-noise render to within Monte-Carlo noise and be reproducible under torch.manual_seed."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = RENDER_CASES['mid_train48']
    dev = _dev()
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = gpu_rays(case, c2w, K, dev)
    r = ImportanceRenderer(use_triplane=True)
    d = make_decoder(dec, dev)
    outs = []
    for seed in (1, 1, 2):
        torch.manual_seed(seed)
        with torch.no_grad():
            outs.append(r(planes.to(dev), d, ro, rd, opts)[0].cpu())
    assert torch.equal(outs[0], outs[1])
    assert not torch.equal(outs[0], outs[2])
    ref = load_golden('render', 'mid_train48')['rgb']
    assert (outs[0] - ref).abs().mean().item() < 0.05
    assert abs(outs[0].mean().item() - ref.mean().item()) < 0.01


def test_full_size_properties():
    """BASELINE configs[1] sizes (N=2 here to bound memory/time): size-independent properties."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    from panic3d_b200.training.triplane import OSGDecoder
    from panic3d_b200 import cameras
    dev = _dev()
    torch.manual_seed(0)
    N, R, P = 2, 128, 512
    planes = torch.randn(N, 3, 32, P, P, device=dev)
    dec = OSGDecoder(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32}).to(dev).requires_grad_(False)
    lab = torch.stack([cameras.camera_params_to_matrix(elev=0, azim=a, dist=1, fov=30)['camera_label'] for a in (0, 30)]).to(dev)
    ro, rd = RaySampler()(lab[:, :16].view(-1, 4, 4), lab[:, 16:].view(-1, 3, 3), R)
    opts = dict(orc.DEFAULT_OPTS)
    r = ImportanceRenderer(use_triplane=True)
    u_c = torch.rand(N, R * R, 96, 1, device=dev)
    u_f = torch.rand(N * R * R, 96, device=dev)
    r.injected_noise = (u_c, u_f)
    with torch.no_grad():
        rgb, depth, wsum, xyz = r(planes, dec, ro, rd, opts)
        # (1) batch independence: each view rendered alone equals its slice of the batch (depth clamp aside)
        r.injected_noise = (u_c[1:], u_f[R * R:])
        rgb1, depth1, wsum1, xyz1 = r(planes[1:], dec, ro[1:], rd[1:], opts)
    assert torch.equal(rgb[1:], rgb1) and torch.equal(wsum[1:], wsum1) and torch.equal(xyz[1:], xyz1)
    # (2) ranges: weights in [0,1], white background => rgb = 2*(sum w c + 1 - sum w) - 1 in [-1, 1+eps]
    assert wsum.min().item() >= 0 and wsum.max().item() <= 1 + 1e-5
    assert rgb.min().item() >= -1 - 3e-3 and rgb.max().item() <= 1 + 3e-3
    # (3) depth clamped to the sampled range
    assert depth.min().item() >= 0.5 and depth.max().item() <= 1.5 + 1.0 / 95 + 1e-6
    # (4) xyz consistency: composite of positions == o*wsum + d*sum(w t) with white back, i.e.
    #     (xyz+1)/2 - (1-wsum) = ro*wsum + rd*(depth*wsum) wherever depth was not clamped
    lhs = (xyz + 1) / 2 - (1 - wsum)
    rhs = ro * wsum + rd * (depth * wsum)
    ok = (wsum.squeeze(-1) > 1e-3)
    assert (lhs - rhs)[ok].abs().max().item() < 1e-4
    # (5) rays that miss the box entirely are pure background
    miss = (wsum.squeeze(-1) == 0)
    if miss.any():
        assert (rgb[miss] - 1).abs().max().item() < 1e-6


# ---------------------------------------------------------------------------------------------
# fused tensor-core renderer (mlp_mode 1 = 3-pass split bf16 tensor cores, 2 = single-pass bf16)
# ---------------------------------------------------------------------------------------------
FUSED_CASES = ['config1', 'mid_train48', 'mid_eval96', 'fused48_ortho', 'fused48_auto_limits', 'fused48_disparity',
               'fused48_black_eg3dplanes', 'fused48_shared_planes', 'fused48_binarize', 'fused96_lrmul_black', 'headline96']


@pytest.mark.parametrize('name', FUSED_CASES)
def test_fused_tc_3xbf16_matches_reference_fixture(name):
    """The benchmarked kernel (k_render_ws3, mlp_mode 1) against outputs of the unmodified reference: BASELINE configs[0],
    the option matrix (ortho rays, 'auto' limits, disparity, EG3D plane order, black background, shared planes, binarize,
    lr_mul) at 48+48 / 96+96, and `headline96` = the benchmarked configuration itself (128^2 rays, 96+96, 512^2 planes)."""
    g = load_golden('render', name)
    outs, _ = gpu_render(g['case'], mlp_mode=1)
    rgb, depth, wsum, xyz = _strided(g['case'], outs)
    has_cull = bool(g['case'].get('cull_clouds') or g['case'].get('binarize_clouds'))
    for got, key in ((rgb, 'rgb'), (depth, 'depth'), (wsum, 'wsum'), (xyz, 'xyz')):
        err = (got - g[key]).abs()
        if has_cull:
            assert (err < TOL).float().mean().item() > 0.999, f'{name}:{key}'
            assert err.max().item() < 2e-2, f'{name}:{key} max {err.max().item()}'
        else:
            assert err.max().item() < TOL, f'{name}:{key} max abs err {err.max().item()}'
        print(f'{name}:{key} fused 3xbf16 max abs err {err.max().item():.3e}')


def test_fused_headline_config_matches_live_oracle_and_is_the_default_path():
    """BASELINE configs[1] geometry (128x128 rays, 96+96 samples, 512^2 planes; N=2) through the DEFAULT renderer settings
    (mlp_mode 'auto' -> the fused tensor-core kernel) against the CPU oracle run live on the box, every ray, strict tolerance."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from panic3d_b200 import _lib
    case = RENDER_CASES['headline96']
    ref = oracle_render(case)
    dev = _dev()
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = gpu_rays(case, c2w, K, dev)
    r = ImportanceRenderer(use_triplane=True)
    assert r.mlp_mode == 'auto'
    r.injected_noise = (u_c, u_f)
    _lib.lib().p3d_profile_enable(1)
    _lib.lib().p3d_profile_read(None, None, 0, 1)
    with torch.no_grad():
        out = r(planes.to(dev), make_decoder(dec, dev), ro, rd, opts)
    torch.cuda.synchronize()
    import ctypes as C
    ms = (C.c_double * 8)(); n = (C.c_uint64 * 8)()
    _lib.lib().p3d_profile_read(ms, n, 8, 1)
    _lib.lib().p3d_profile_enable(0)
    assert n[5] == 1 and n[0] == 0, 'the default path must be the fused kernel (profile slot 5), not the SIMT kernels'
    for got, want, key in zip(out, ref, ('rgb', 'depth', 'wsum', 'xyz')):
        err = (got.cpu() - want).abs().max().item()
        print(f'headline96 vs live oracle: {key} max abs err {err:.3e}')
        assert err < TOL, (key, err)


@pytest.mark.parametrize('name', ['config1'])
def test_fused_tc_bf16_fast_mode_is_close(name):
    g = load_golden('render', name)
    (rgb, depth, wsum, xyz), _ = gpu_render(g['case'], mlp_mode=2)
    assert (rgb - g['rgb']).abs().max().item() < 5e-2
    assert (rgb - g['rgb']).abs().mean().item() < 5e-3
    assert (wsum - g['wsum']).abs().max().item() < 5e-2


def test_fused_rejects_unsupported_sampling_loudly():
    with pytest.raises(RuntimeError, match='fused'):
        gpu_render(RENDER_CASES['small_plain'], mlp_mode=1)       # 12+12 samples: no fused kernel -> error, no fallback


def test_deferred_depth_clamp_makes_shards_equal_the_batch():
    """The multi-GPU protocol on one GPU: views rendered one at a time with the batch-wide depth bounds injected
    through `depth_bounds_reduce` reproduce the batch render exactly (incl. composite depth, ray_marcher.py:50)."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = RENDER_CASES['small_batch3']
    dev = _dev()
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = gpu_rays(case, c2w, K, dev)
    d = make_decoder(dec, dev)
    M = ro.shape[1]
    r = ImportanceRenderer(use_triplane=True)
    seen = {}
    r.depth_bounds_reduce = lambda b2: seen.__setitem__('b', b2.clone())
    r.injected_noise = (u_c, u_f)
    with torch.no_grad():
        full = r(planes.to(dev), d, ro, rd, opts)
        parts = []
        r.depth_bounds_reduce = lambda b2: b2.copy_(seen['b'])
        for i in range(3):
            r.injected_noise = (u_c[i:i + 1], u_f[i * M:(i + 1) * M])
            parts.append(r(planes[i:i + 1].to(dev), d, ro[i:i + 1], rd[i:i + 1], opts))
    g = load_golden('render', 'small_batch3')
    for k, key in enumerate(('rgb', 'depth', 'wsum', 'xyz')):
        cat = torch.cat([p[k] for p in parts])
        assert torch.equal(cat, full[k]), key
        assert (cat.cpu() - g[key]).abs().max().item() < TIGHT


# ---------------------------------------------------------------------------------------------
# backward (training path): gradients w.r.t. tri-planes and decoder tensors vs torch.autograd on the oracle
# ---------------------------------------------------------------------------------------------
GRAD_CASES = ['small_plain', 'small_eval_flags_dense', 'small_black_eg3dplanes', 'small_batch3', 'small_lrmul_uneven', 'small_ortho']


@pytest.mark.parametrize('name', GRAD_CASES)
def test_renderer_backward_matches_oracle_autograd(name):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from tests.helpers import case_rays
    case = RENDER_CASES[name]
    dev = _dev()
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = case_rays(case, c2w, K)
    rng = np.random.default_rng(case['seed'] + 5)
    N, M = ro.shape[0], ro.shape[1]
    gw = [torch.from_numpy(rng.standard_normal(s).astype(np.float32)) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
    flags = dict(triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'), binarize_clouds=case.get('binarize_clouds'))

    # oracle (CPU autograd)
    pl = planes.clone().requires_grad_(True)
    dref = {k: (v.clone().requires_grad_(True) if isinstance(v, torch.Tensor) else v) for k, v in dec.items()}
    out = orc.render(pl, dref, ro, rd, opts, u_c, u_f if opts['depth_resolution_importance'] > 0 else None,
                     use_triplane=case.get('use_triplane', True), **flags)
    loss = sum((o * g_).sum() for o, g_ in zip(out, gw))
    ref = torch.autograd.grad(loss, [pl, dref['w1'], dref['b1'], dref['w2'], dref['b2']])

    # CUDA
    r = ImportanceRenderer(use_triplane=case.get('use_triplane', True))
    r.injected_noise = (u_c, u_f)
    d = make_decoder(dec, dev).requires_grad_(True)
    pg = planes.to(dev).requires_grad_(True)
    got_out = r(pg, d, ro.to(dev), rd.to(dev), opts, **flags)
    for o, o_ref in zip(got_out, out):
        assert (o.detach().cpu() - o_ref.detach()).abs().max().item() < TIGHT
    loss_g = sum((o * g_.to(dev)).sum() for o, g_ in zip(got_out, gw))
    got = torch.autograd.grad(loss_g, [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    for g_, r_, nm in zip(got, ref, ('planes', 'w1', 'b1', 'w2', 'b2')):
        assert g_.shape == r_.shape, nm
        err = (g_.cpu() - r_).abs().max().item()
        scale = max(1e-3, r_.abs().max().item())
        assert err < 2e-3 * scale, f'{name}:{nm} max abs err {err} (scale {scale})'


@pytest.mark.parametrize('name', sorted(POINT_CASES))
def test_run_model_backward_matches_oracle_autograd(name):
    """ImportanceRenderer.run_model under autograd (renderer.py:266-280): gradients w.r.t. tri-planes and decoder tensors
    for random incoming (g_rgb, g_sigma) against torch.autograd on the CPU oracle."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    g = load_golden('points', name)
    case = g['case']
    dev = _dev()
    planes, dec, *_r, opts = build_case_inputs(case)
    pts = g['pts']
    rng = np.random.default_rng(case['seed'] + 7)
    N, K = pts.shape[0], pts.shape[1]
    gw = [torch.from_numpy(rng.standard_normal(sh).astype(np.float32)) for sh in ((N, K, 32), (N, K, 1))]
    pl = planes.clone().requires_grad_(True)
    dref = {k: (v.clone().requires_grad_(True) if isinstance(v, torch.Tensor) else v) for k, v in dec.items()}
    rgb_o, sig_o = orc.run_model(pl, dref, pts, opts, case.get('use_triplane', True))
    ref = torch.autograd.grad((rgb_o * gw[0]).sum() + (sig_o * gw[1]).sum(), [pl, dref['w1'], dref['b1'], dref['w2'], dref['b2']])
    r = ImportanceRenderer(use_triplane=case.get('use_triplane', True))
    d = make_decoder(dec, dev).requires_grad_(True)
    pg = planes.to(dev).requires_grad_(True)
    out = r.run_model(pg, d, pts.to(dev), None, opts)
    assert out['rgb'].requires_grad and out['sigma'].requires_grad
    assert (out['rgb'].detach().cpu() - g['rgb']).abs().max().item() < TIGHT
    assert (out['sigma'].detach().cpu() - g['sigma']).abs().max().item() < TIGHT
    got = torch.autograd.grad((out['rgb'] * gw[0].to(dev)).sum() + (out['sigma'] * gw[1].to(dev)).sum(),
                              [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    for g_, r_, nm in zip(got, ref, ('planes', 'w1', 'b1', 'w2', 'b2')):
        assert g_.shape == r_.shape, nm
        err = (g_.cpu() - r_).abs().max().item()
        scale = max(1e-3, r_.abs().max().item())
        assert err < 2e-3 * scale, f'{name}:{nm} max abs err {err} (scale {scale})'


def test_density_regularisation_graph_of_the_training_loop():
    """The Greg phase of loss_orthocondA.py:579-600 on the renderer level: sigma of 2K points (K random + K perturbed)
    through run_model, TV loss = l1(sigma[:K], sigma[K:]) * density_reg, backward into the tri-planes (i.e. the backbone)
    and the decoder - against the same graph on the CPU oracle."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = POINT_CASES['pts_small']
    dev = _dev()
    planes, dec, *_r, opts = build_case_inputs(case)
    gen = torch.Generator().manual_seed(5)
    N, K = planes.shape[0], 1000
    initial = torch.rand((N, K, 3), generator=gen) * 2 - 1
    perturbed = initial + torch.randn((N, K, 3), generator=gen) * 0.004          # density_reg_p_dist
    coords = torch.cat([initial, perturbed], dim=1) * (opts['box_warp'] / 2)

    def tv(sigma):
        return torch.nn.functional.l1_loss(sigma[:, :K], sigma[:, K:]) * 0.25     # density_reg

    pl = planes.clone().requires_grad_(True)
    dref = {k: (v.clone().requires_grad_(True) if isinstance(v, torch.Tensor) else v) for k, v in dec.items()}
    _, sig_o = orc.run_model(pl, dref, coords, opts, True)
    ref = torch.autograd.grad(tv(sig_o), [pl, dref['w1'], dref['b1'], dref['w2'], dref['b2']])
    r = ImportanceRenderer(use_triplane=True)
    d = make_decoder(dec, dev).requires_grad_(True)
    pg = planes.to(dev).requires_grad_(True)
    loss = tv(r.run_model(pg, d, coords.to(dev), torch.rand_like(coords).to(dev), opts)['sigma'])
    assert abs(loss.item() - tv(sig_o).item()) < 1e-5
    loss.mul(1.0).backward()
    for g_, r_, nm in zip((pg.grad, d.net[0].weight.grad, d.net[0].bias.grad, d.net[2].weight.grad, d.net[2].bias.grad), ref,
                          ('planes', 'w1', 'b1', 'w2', 'b2')):
        err = (g_.cpu() - r_).abs().max().item()
        scale = max(1e-6, r_.abs().max().item())
        assert err < 2e-3 * scale, f'{nm} max abs err {err} (scale {scale})'


def test_renderer_backward_is_once_differentiable():
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = RENDER_CASES['small_plain']
    dev = _dev()
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = gpu_rays(case, c2w, K, dev)
    r = ImportanceRenderer(use_triplane=True)
    r.injected_noise = (u_c, u_f)
    pg = planes.to(dev).requires_grad_(True)
    out = r(pg, make_decoder(dec, dev), ro, rd, opts)
    (gp,) = torch.autograd.grad(out[0].sum(), [pg], create_graph=True)
    with pytest.raises(RuntimeError):
        gp.sum().backward()


def test_renderer_no_grad_path_unchanged_and_grad_path_equal():
    """The autograd path (fp32 SIMT kernels + saved scratch) returns the same forward values as the inference path."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = RENDER_CASES['small_plain']
    dev = _dev()
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = gpu_rays(case, c2w, K, dev)
    r = ImportanceRenderer(use_triplane=True)
    r.injected_noise = (u_c, u_f)
    d = make_decoder(dec, dev)
    with torch.no_grad():
        a = r(planes.to(dev), d, ro, rd, opts)
    b = r(planes.to(dev).requires_grad_(True), d, ro, rd, opts)
    assert all(t.requires_grad for t in b)
    for x, y in zip(a, b):
        assert torch.equal(x, y.detach())


# ---------------------------------------------------------------------------------------------
# edge cases: empty and ragged inputs, unusual sample counts, error behaviour
# ---------------------------------------------------------------------------------------------
def _tiny(dev, N=1, M=5, P=8, seed=0):
    from panic3d_b200.training.triplane import OSGDecoder
    g = torch.Generator().manual_seed(seed)
    planes = torch.randn(N, 3, 32, P, P, generator=g)
    dec = OSGDecoder(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32}).requires_grad_(False)
    ro = torch.tensor([0.0, 0.0, 1.0]).expand(N, M, 3).contiguous()
    rd = torch.nn.functional.normalize(torch.randn(N, M, 3, generator=g) * 0.1 + torch.tensor([0.0, 0.0, -1.0]), dim=-1)
    return planes, dec, ro, rd


def test_empty_batch_and_single_ray():
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    r = ImportanceRenderer(use_triplane=True)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=8, depth_resolution_importance=8)
    planes, dec, ro, rd = _tiny(dev, N=1, M=1)
    with torch.no_grad():
        out = r(planes.to(dev), dec.to(dev), ro.to(dev), rd.to(dev), opts)
        assert [tuple(o.shape) for o in out] == [(1, 1, 32), (1, 1, 1), (1, 1, 1), (1, 1, 3)]
        assert all(torch.isfinite(o).all() for o in out)
        # zero views: empty outputs, no launch, no error
        out0 = r(planes[:0].to(dev), dec.to(dev), ro[:0].to(dev), rd[:0].to(dev), opts)
        assert [tuple(o.shape) for o in out0] == [(0, 1, 32), (0, 1, 1), (0, 1, 1), (0, 1, 3)]
        pts = r.run_model(planes.to(dev), dec.to(dev), torch.zeros(1, 0, 3, device=dev), None, opts)
        assert tuple(pts['rgb'].shape) == (1, 0, 32) and tuple(pts['sigma'].shape) == (1, 0, 1)


@pytest.mark.parametrize('S,Sf,M', [(4, 3, 7), (5, 0, 33), (31, 17, 130), (64, 64, 3), (200, 56, 2)])
def test_ragged_sample_counts_match_oracle(S, Sf, M):
    """Ray counts that are not multiples of any tile size and odd sample counts (v1 path) against the oracle."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    planes, dec_m, ro, rd = _tiny(dev, N=2, M=M, P=16, seed=S * 100 + Sf)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf)
    g = torch.Generator().manual_seed(1)
    u_c, u_f = torch.rand(2, M, S, 1, generator=g), torch.rand(2 * M, max(Sf, 1), generator=g)[:, :Sf]
    r = ImportanceRenderer(use_triplane=True)
    r.injected_noise = (u_c, u_f)
    with torch.no_grad():
        out = r(planes.to(dev), dec_m.to(dev), ro.to(dev), rd.to(dev), opts)
    dec = {k: v.detach().cpu() for k, v in dict(w1=dec_m.net[0].weight, b1=dec_m.net[0].bias, w2=dec_m.net[2].weight, b2=dec_m.net[2].bias).items()}
    ref = orc.render(planes, dec, ro, rd, opts, u_c, u_f if Sf > 0 else None, use_triplane=True)
    for o, o_ref in zip(out, ref):
        assert (o.cpu() - o_ref).abs().max().item() < TIGHT


def test_fused_handles_ray_counts_that_leave_partial_groups():
    """M = 12 rays (3 fused groups of 4 at S=96) and N = 3 views: odd number of groups per CTA, tail tiles."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    planes, dec_m, ro, rd = _tiny(dev, N=3, M=12, P=16, seed=5)
    opts = dict(orc.DEFAULT_OPTS)
    g = torch.Generator().manual_seed(2)
    u_c, u_f = torch.rand(3, 12, 96, 1, generator=g), torch.rand(36, 96, generator=g)
    outs = []
    for mode in (0, 1):
        r = ImportanceRenderer(use_triplane=True)
        r.mlp_mode = mode
        r.injected_noise = (u_c, u_f)
        with torch.no_grad():
            outs.append(r(planes.to(dev), dec_m.to(dev), ro.to(dev), rd.to(dev), opts))
    for a_, b_ in zip(*outs):
        assert (a_ - b_).abs().max().item() < 1e-4


def test_bad_inputs_raise():
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    planes, dec, ro, rd = _tiny(dev)
    r = ImportanceRenderer(use_triplane=True)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=8, depth_resolution_importance=8)
    with torch.no_grad():
        with pytest.raises(NotImplementedError):
            r(planes.to(dev), dec.to(dev), ro.to(dev), rd.to(dev), dict(opts, triplane_depth=2))
        with pytest.raises(NotImplementedError):
            r(planes.to(dev), dec.to(dev), ro.to(dev), rd.to(dev), dict(opts, density_noise=0.1))
        with pytest.raises(RuntimeError):
            r(planes.to(dev), dec.to(dev), ro.to(dev), rd.to(dev), dict(opts, depth_resolution=1))          # < 2 coarse samples
        with pytest.raises(RuntimeError, match='unsupported'):
            r(planes[:, :, :16].to(dev), dec.to(dev), ro.to(dev), rd.to(dev), opts)                       # 16-channel planes
        with pytest.raises(ValueError):
            r(planes[:, :2].to(dev), dec.to(dev), ro.to(dev), rd.to(dev), opts)                           # two planes


@pytest.mark.parametrize('name,mlp_mode', [('small_batch3', 0), ('mid_train48', 0), ('mid_train48', 1)])
def test_host_entry_point_pipelines_views_and_equals_device_path(name, mlp_mode):
    """p3d_render_forward_host (host buffers in, host buffers out; per-view H2D / render / D2H pipeline with the
    batch-wide depth clamp applied at the end) equals the device-resident call bit for bit, and the fixture."""
    import ctypes as Ct
    from panic3d_b200 import _lib
    case = RENDER_CASES[name]
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    N, R, S, Sf = planes.shape[0], case['R'], opts['depth_resolution'], opts['depth_resolution_importance']
    ref, _ = gpu_render(case, mlp_mode=mlp_mode)
    p = _lib.RenderParams()
    p.n_views, p.n_rays, p.n_coarse, p.n_fine = N, R * R, S, Sf
    p.channels, p.plane_h, p.plane_w, p.hidden, p.out_dim = planes.shape[2], planes.shape[3], planes.shape[4], 64, 33
    p.box_warp = opts['box_warp']
    p.ray_mode, p.ray_start, p.ray_end = 0, float(opts['ray_start']), float(opts['ray_end'])
    p.white_back, p.plane_mode = int(bool(opts.get('white_back'))), 1
    d = make_decoder(dec, 'cpu')
    fc1, fc2 = d.net[0], d.net[2]
    p.w1_gain, p.b1_gain, p.w2_gain, p.b2_gain = float(fc1.weight_gain), float(fc1.bias_gain), float(fc2.weight_gain), float(fc2.bias_gain)
    p.mlp_mode = mlp_mode
    h = [t.detach().float().contiguous() for t in (planes, fc1.weight, fc1.bias, fc2.weight, fc2.bias, c2w.reshape(N, 16), K.reshape(N, 9), u_c, u_f)]
    outs = [torch.empty(s, dtype=torch.float32) for s in ((N, R * R, 32), (N, R * R, 1), (N, R * R, 1), (N, R * R, 3))]
    L = _lib.lib()
    for _ in range(2):                                        # second call reuses the arena / events
        _lib.check(L.p3d_render_forward_host(Ct.byref(p), *[t.data_ptr() for t in h[:7]], R, h[7].data_ptr(), h[8].data_ptr(),
                                             outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), outs[3].data_ptr()))
    L.p3d_host_arena_release()
    g = load_golden('render', name)
    for got, want, key in zip(outs, ref, ('rgb', 'depth', 'wsum', 'xyz')):
        assert torch.equal(got, want), key
        assert (got - g[key]).abs().max().item() < (TIGHT if mlp_mode == 0 else 1e-3), key


def test_fused_renderer_is_bit_reproducible():
    """Two runs of the warp-specialised kernel on the same inputs agree bit for bit (the colour reduction publishes
    one partial per warp, so no result depends on the order of shared-memory atomics)."""
    a, _ = gpu_render(RENDER_CASES['mid_eval96'], mlp_mode=1)
    b, _ = gpu_render(RENDER_CASES['mid_eval96'], mlp_mode=1)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize('shape', [(5, 32, 20, 12), (3, 32, 64, 64), (2, 32, 7, 9), (6, 32, 128, 130)])
@pytest.mark.parametrize('bf16', [False, True])
def test_planes_to_channels_last_layout_pass(shape, bf16):
    """p3d_planes_to_channels_last == permute(0,2,3,1) (+ bf16 rounding): vector fast path (HW % 4 == 0, incl. a partial
    last 128-pixel tile) and the generic 32x32 transpose (odd HW)."""
    from panic3d_b200 import _lib
    dev = _dev()
    n, c, h, w = shape
    x = torch.randn(n, c, h, w, device=dev)
    out = torch.empty((n, h, w, c), device=dev, dtype=torch.bfloat16 if bf16 else torch.float32)
    _lib.check(_lib.lib().p3d_planes_to_channels_last(x.data_ptr(), out.data_ptr(), n, c, h, w, 1 if bf16 else 0, _lib.stream_ptr(dev)))
    ref = x.permute(0, 2, 3, 1).contiguous()
    assert torch.equal(out, ref.to(torch.bfloat16) if bf16 else ref)
