"""GPU: multiplane tri-planes (rendering_kwargs['triplane_depth'] = D > 1) through ImportanceRenderer and the C ABI.

The fp32 SIMT kernels gather trilinearly over the D slabs of each plane (k_sample_decode / k_sample_backward, TRI
instances).  Checked here against the reference's own outputs (tests/golden/multiplane_*.npz) and against the CPU
oracle run live: renders, bf16 storage, points on slab centres and borders and past the box along each normal, run_model,
the volume query, the gradients of renders and of run_model, determinism, plane_depth 1 == 0, the kernel choice of
mlp_mode 'auto', and mesh extraction.  Every plane here is 24 x 20 texels (H > W)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import multiplane_oracle as mo, renderer_oracle as orc
from tests.golden.cases_multiplane import RENDER_CASES, POINT_CASES, build_inputs, point_coords, upstream
from tests.helpers import profiled
from tests.render_abi import decode_points_call, render_forward

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    import panic3d_b200  # noqa: F401
    return torch.device('cuda:0')


def _decoder(dec, dev, grad=False):
    from panic3d_b200.training.triplane import OSGDecoder
    d = OSGDecoder(32, {'decoder_lr_mul': dec.get('lr_mul', 1.0), 'decoder_output_dim': 32}).to(dev)
    with torch.no_grad():
        d.net[0].weight.copy_(dec['w1']); d.net[0].bias.copy_(dec['b1'])
        d.net[2].weight.copy_(dec['w2']); d.net[2].bias.copy_(dec['b2'])
    return d.requires_grad_(grad)


def _golden(name):
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', f'multiplane_{name}.npz'))


def _err(a, b):
    return float((a.detach().double().cpu() - torch.as_tensor(np.asarray(b)).double()).abs().max())


def _render(case, dev, planes=None, bf16=False, mlp_mode='auto'):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    p_, dec, _, _, u_c, u_f, opts = build_inputs(case)
    planes = p_ if planes is None else planes
    z = _golden(f'render_{case["name"]}') if 'name' in case else None
    r = ImportanceRenderer(use_triplane=case['use_triplane'])
    r.injected_noise = (u_c, u_f)
    r.planes_bf16 = bf16
    r.mlp_mode = mlp_mode
    ro, rd = torch.from_numpy(z['ro']).to(dev), torch.from_numpy(z['rd']).to(dev)
    with torch.no_grad():
        out, n = profiled(lambda: r(planes.to(dev), _decoder(dec, dev), ro, rd, opts, triplane_crop=case.get('triplane_crop'),
                                    cull_clouds=case.get('cull_clouds')))
    return out, n, z


@pytest.mark.parametrize('name', sorted(RENDER_CASES))
def test_render_matches_reference_and_oracle(name):
    dev = _dev()
    case = dict(RENDER_CASES[name], name=name)
    out, n, z = _render(case, dev)
    assert n[0] >= 1 and n[5] == 0, "mlp_mode 'auto' must render multiplane planes with the SIMT kernels"
    planes, dec, _, _, u_c, u_f, opts = build_inputs(case)
    ref = mo.render(planes, dec, torch.from_numpy(z['ro']), torch.from_numpy(z['rd']), opts, u_c, u_f,
                     use_triplane=case['use_triplane'], triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'))
    for key, got, want in zip(('rgb', 'depth', 'wsum', 'xyz'), out, ref):
        assert _err(got, z[key]) < 1e-3, (key, 'reference', _err(got, z[key]))
        assert _err(got, want) < 1e-4, (key, 'oracle', _err(got, want))


@pytest.mark.parametrize('name', ['d2_eg3d48', 'd3_panic48'])
def test_render_bf16_storage_matches_oracle_on_rounded_planes(name):
    dev = _dev()
    case = dict(RENDER_CASES[name], name=name)
    out, n, z = _render(case, dev, bf16=True)
    assert n[0] >= 1 and n[5] == 0
    planes, dec, _, _, u_c, u_f, opts = build_inputs(case)
    ref = mo.render(planes.bfloat16().float(), dec, torch.from_numpy(z['ro']), torch.from_numpy(z['rd']), opts, u_c, u_f,
                     use_triplane=case['use_triplane'])
    for key, got, want in zip(('rgb', 'depth', 'wsum', 'xyz'), out, ref):
        assert _err(got, want) < 1e-4, (key, _err(got, want))
    assert _err(out[0], z['rgb']) > 1e-6, 'bf16 storage must have rounded the planes'


@pytest.mark.parametrize('name', sorted(POINT_CASES))
def test_run_model_on_slab_centres_borders_and_past_the_box(name):
    """run_model on uniform points and on the slab points of cases_multiplane.slab_points (the last rows)."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    case = POINT_CASES[name]
    z = _golden(f'points_{name}')
    planes, dec, _, _, _, _, opts = build_inputs(case)
    pts = point_coords(case)
    r = ImportanceRenderer(use_triplane=case['use_triplane'])
    with torch.no_grad():
        out, n = profiled(lambda: r.run_model(planes.to(dev), _decoder(dec, dev), pts.to(dev), None, opts))
    assert n[0] >= 1, 'run_model on multiplane planes must run the SIMT decode'
    rgb, sigma = mo.run_model(planes, dec, pts, opts, case['use_triplane'])
    assert _err(out['rgb'], z['rgb']) < 1e-3 and _err(out['sigma'], z['sigma']) < 1e-3
    assert _err(out['rgb'], rgb) < 1e-4 and _err(out['sigma'], sigma) < 1e-4
    # 1.6 half-boxes out along an axis a point is past every slab of the plane whose normal that axis is, and outside the
    # two other planes: its features are exactly zero
    K = case['K']
    slab = pts[:, K:]
    feat = mo.sample_multiplane(planes, slab, opts['box_warp'], case['use_triplane'], case['D'])
    far = (slab.abs() > 0.35 * 1.5).any(-1)
    assert bool(far.any()) and float(feat[:, :, far[0]].abs().sum(-1).min()) == 0.0
    assert _err(out['sigma'][:, K:], sigma[:, K:]) < 1e-4


def test_volume_query_on_an_odd_lattice_with_crop_and_cull():
    from panic3d_b200.volume import query_volume
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    case = dict(POINT_CASES['d2_eg3d'], N=1)
    planes, dec, _, _, _, _, opts = build_inputs(dict(case, sigma_bias=1.5))
    r = ImportanceRenderer(use_triplane=False)
    _, n = profiled(lambda: query_volume(planes.to(dev), _decoder(dec, dev), opts, resolution=97, triplane_crop=0.1, cull_clouds=0.35,
                                         renderer=r))
    assert n[0] >= 1
    got = query_volume(planes.to(dev), _decoder(dec, dev), opts, resolution=97, triplane_crop=0.1, cull_clouds=0.35, renderer=r)
    want = mo.volume(planes.to(dev), {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in dec.items()}, opts, 97,
                     triplane_crop=0.1, cull_clouds=0.35, use_triplane=False)
    assert float((got['sigmas'] - want['sigmas']).abs().max()) < 1e-4
    assert float((got['rgbs'] - want['rgbs']).abs().max()) < 1e-4
    assert torch.equal(got['coordinates'], want['coordinates'])
    dg, dw = got['densities'], want['densities']
    same = (dg == -1e3) == (dw == -1e3)
    assert float(same.float().mean()) > 0.999 and 0.05 < float((dw == -1e3).float().mean()) < 0.95
    both = (dg != -1e3) & (dw != -1e3)
    assert float((dg - dw)[both].abs().max()) < 1e-4


# ----------------------------------------------------------------------------------------------------------- gradients
def _oracle_render_grads(planes, dec, ro, rd, opts, u_c, u_f, use_triplane, gs):
    """Autograd of the fp64 oracle on the device, with the fp32 oracle's sample depths and masks (constants of the
    reference graph)."""
    _, samples = mo.render(planes, dec, ro, rd, opts, u_c, u_f, use_triplane=use_triplane, return_samples=True)
    dev = torch.device('cuda:0')
    p64 = planes.to(dev, torch.float64).requires_grad_(True)
    d64 = {k: (v.to(dev, torch.float64).requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
    depths = tuple(None if t is None else t.to(dev, torch.float64) for t in samples['depths'])
    masks = tuple(None if t is None else t.to(dev) for t in samples['masks'])
    outs = mo.render(p64, d64, ro.to(dev, torch.float64), rd.to(dev, torch.float64), opts, None, None, use_triplane=use_triplane,
                      depths=depths, masks=masks)
    sum(((o * g.to(dev, torch.float64)).sum() for o, g in zip(outs, gs) if g is not None), torch.zeros((), device=dev, dtype=torch.float64)).backward()
    return p64.grad, [d64[k].grad for k in ('w1', 'b1', 'w2', 'b2')]


def _check_grads(gp, gw, rp, rw):
    # relative to each tensor's largest entry, with a floor of 1e-3 of the largest over all five: a gradient that vanishes
    # analytically (d_b2 of a TV loss, which no constant shift of sigma changes) leaves only rounding to compare
    floor = 1e-3 * max(float(w.abs().max()) for w in [rp] + rw)
    for got, want in zip([gp] + gw, [rp] + rw):
        rel = float((got.double() - want).abs().max()) / max(float(want.abs().max()), floor)
        assert rel < 2e-3, rel
    assert bool((gp[rp == 0] == 0).all()), 'texels no tap touched must receive exactly 0'
    assert float((rp != 0).float().mean()) > 0.1


@pytest.mark.parametrize('which', ['rgb', 'depth', 'wsum', 'xyz', 'all'])
def test_render_gradients_match_oracle_autograd(which):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    case = dict(RENDER_CASES['d2_eg3d48'], N=1)
    planes, dec, c2w, K, u_c, u_f, opts = build_inputs(case)
    ro, rd = orc.ray_sampler(c2w, K, case['R'])
    M = ro.shape[1]
    shapes = {'rgb': (1, M, 32), 'depth': (1, M, 1), 'wsum': (1, M, 1), 'xyz': (1, M, 3)}
    gs = upstream(case, list(shapes.values()))
    gs = [g if which in ('all', k) else None for k, g in zip(shapes, gs)]
    r = ImportanceRenderer(use_triplane=False)
    r.injected_noise = (u_c, u_f)
    pg = planes.to(dev).requires_grad_(True)
    d = _decoder(dec, dev, grad=True)
    (out, n) = profiled(lambda: r(pg, d, ro.to(dev), rd.to(dev), opts))
    sum(((o * g.to(dev)).sum() for o, g in zip(out, gs) if g is not None), torch.zeros((), device=dev)).backward()
    assert pg.grad.shape == planes.shape
    rp, rw = _oracle_render_grads(planes, dec, ro, rd, opts, u_c, u_f, False, gs)
    assert float((rp == 0).float().mean()) > 0.01, 'the rays must leave some texels untouched'
    _check_grads(pg.grad, [d.net[0].weight.grad, d.net[0].bias.grad, d.net[2].weight.grad, d.net[2].bias.grad], rp, rw)


def test_run_model_gradients_of_a_tv_loss_match_oracle_autograd():
    """The density-regularisation phase: a TV-style loss on run_model's sigma over a small jittered lattice."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    case = dict(POINT_CASES['d3_panic'], N=1)
    planes, dec, _, _, _, _, opts = build_inputs(case)
    G = 14
    lin = torch.linspace(-0.4, 0.4, G)
    pts = torch.stack(torch.meshgrid(lin, lin, lin, indexing='ij'), -1).reshape(1, -1, 3)
    pts = pts + 0.01 * torch.from_numpy(np.random.default_rng(7).standard_normal(pts.shape).astype(np.float32))

    def tv(sigma):
        s = sigma.reshape(G, G, G)
        return ((s[1:] - s[:-1]) ** 2).mean() + ((s[:, 1:] - s[:, :-1]) ** 2).mean() + ((s[:, :, 1:] - s[:, :, :-1]) ** 2).mean()

    r = ImportanceRenderer(use_triplane=True)
    pg = planes.to(dev).requires_grad_(True)
    d = _decoder(dec, dev, grad=True)
    tv(r.run_model(pg, d, pts.to(dev), None, opts)['sigma']).backward()
    p64 = planes.to(dev, torch.float64).requires_grad_(True)
    d64 = {k: (v.to(dev, torch.float64).requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
    tv(mo.run_model(p64, d64, pts.to(dev, torch.float64), opts, True)[1]).backward()
    _check_grads(pg.grad, [d.net[0].weight.grad, d.net[0].bias.grad, d.net[2].weight.grad, d.net[2].bias.grad],
                 p64.grad, [d64[k].grad for k in ('w1', 'b1', 'w2', 'b2')])


# ----------------------------------------------------------------------------------------------- C ABI and kernel choice
def _abi_inputs(dev, D, N=1, M=384):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = dict(RENDER_CASES['d2_eg3d48'], D=D, N=N)
    planes, dec, c2w, K, _, _, opts = build_inputs(case)
    opts['triplane_depth'] = D
    r = ImportanceRenderer(use_triplane=False)
    planes_cl = r._planes_cl(planes.to(dev), D)
    p, wts = r._params(planes_cl, N, M, opts, _decoder(dec, dev), None, None, None)
    ro, rd = orc.ray_sampler(c2w, K, 16)
    ro = torch.cat([ro, ro[:, :M - 256]], 1).to(dev).contiguous()
    rd = torch.cat([rd, rd.flip(1)[:, :M - 256]], 1).to(dev).contiguous()
    return p, planes_cl, [t.detach().float().contiguous() for t in wts], ro, rd


def _abi_render(p, planes_cl, wt, ro, rd):
    from panic3d_b200 import _lib
    dev = planes_cl.device
    N, M = p.n_views, p.n_rays
    out = [torch.empty(sh, device=dev) for sh in ((N, M, 32), (N, M), (N, M), (N, M, 3))]
    ws = torch.empty(int(_lib.lib().p3d_render_workspace_bytes(C.byref(p))), dtype=torch.uint8, device=dev)
    render_forward(p, planes_cl, wt, ro, rd, None, None, ws, out)
    pts = ro[:, :200] + 0.9 * rd[:, :200]
    rgb, sig = torch.empty((N, 200, 32), device=dev), torch.empty((N, 200), device=dev)
    decode_points_call(p, planes_cl, wt, pts.contiguous(), rgb, sig)
    torch.cuda.synchronize()
    return out + [rgb, sig]


def test_repeated_forward_is_bit_identical():
    dev = _dev()
    p, planes_cl, wt, ro, rd = _abi_inputs(dev, 3)
    p.mlp_mode, p.seed = 0, 1234
    a, b = _abi_render(p, planes_cl, wt, ro, rd), _abi_render(p, planes_cl, wt, ro, rd)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_plane_depth_one_equals_zero_bit_for_bit():
    dev = _dev()
    p, planes_cl, wt, ro, rd = _abi_inputs(dev, 1)
    p.mlp_mode, p.seed = 0, 99
    assert p.plane_depth == 0
    a = _abi_render(p, planes_cl, wt, ro, rd)
    p.plane_depth = 1
    b = _abi_render(p, planes_cl, wt, ro, rd)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_auto_runs_simt_and_explicit_tensor_core_raises():
    from panic3d_b200.volume import query_volume
    dev = _dev()
    case = dict(RENDER_CASES['d2_eg3d48'], name='d2_eg3d48')
    _, n, _ = _render(case, dev)
    assert n[0] >= 1 and n[5] == 0
    for mode in (1, 2):
        with pytest.raises(RuntimeError, match='tensor-core'):
            _render(case, dev, mlp_mode=mode)
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    planes, dec, _, _, _, _, opts = build_inputs(POINT_CASES['d2_eg3d'])
    r = ImportanceRenderer(use_triplane=False)
    r.mlp_mode = 1
    with torch.no_grad(), pytest.raises(RuntimeError, match='tensor-core'):
        r.run_model(planes.to(dev), _decoder(dec, dev), point_coords(POINT_CASES['d2_eg3d']).to(dev), None, opts)
    with pytest.raises(RuntimeError, match='tensor-core'):
        query_volume(planes.to(dev), _decoder(dec, dev), opts, resolution=9, renderer=r)


def test_extract_mesh_on_two_slab_planes():
    from panic3d_b200.mesh import extract_mesh
    from panic3d_b200.volume import query_volume
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    planes, dec, _, _, _, _, opts = build_inputs(dict(POINT_CASES['d2_eg3d'], N=1, sigma_bias=1.0))
    r = ImportanceRenderer(use_triplane=False)
    m = extract_mesh(planes.to(dev), _decoder(dec, dev), opts, resolution=48, renderer=r)
    vol = query_volume(planes.to(dev), _decoder(dec, dev), opts, resolution=48, renderer=r)
    d = vol['densities'][0, 0]
    assert bool((d > 0.5).any()) and bool((d < 0.5).any()), 'the field must cross the level'
    assert len(m['faces']) > 0 and np.isfinite(m['verts']).all() and m['colors'].shape == (len(m['verts']), 3)


def test_multiplane_input_checks():
    """triplane_depth must split the plane channels into slabs of the 32 features the kernels take."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = _dev()
    case = dict(RENDER_CASES['d2_eg3d48'], D=1, N=1)
    planes, dec, c2w, K, _, _, opts = build_inputs(case)
    ro, rd = orc.ray_sampler(c2w, K, 4)
    r = ImportanceRenderer(use_triplane=True)
    opts = dict(opts, depth_resolution=8, depth_resolution_importance=8, triplane_depth=1)
    args = lambda pl: (pl.to(dev), _decoder(dec, dev), ro.to(dev), rd.to(dev))
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match='features per slab'):
            r(*args(planes), dict(opts, triplane_depth=2))                       # 32 channels in 2 slabs: 16 features per slab
        with pytest.raises(ValueError, match='triplane_depth'):
            r(*args(planes), dict(opts, triplane_depth=3))                       # 32 channels do not split into 3 slabs
        pts = torch.zeros(1, 4, 3, device=dev)
        with pytest.raises(NotImplementedError, match='features per slab'):
            r.run_model(*args(planes)[:2], pts, None, dict(opts, triplane_depth=2))
        pg = planes.to(dev).requires_grad_(True)
        with torch.enable_grad(), pytest.raises(NotImplementedError, match='features per slab'):
            r(pg, _decoder(dec, dev), ro.to(dev), rd.to(dev), dict(opts, triplane_depth=2))     # the autograd path
    planes2 = torch.cat([planes, planes], 2)                                       # 64 channels in 2 slabs: renders
    with torch.no_grad():
        rgb = r(*args(planes2), dict(opts, triplane_depth=2))[0]
    assert bool(torch.isfinite(rgb).all())
