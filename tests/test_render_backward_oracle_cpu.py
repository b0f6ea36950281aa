"""CPU: the render oracle's injected depths and masks, and the hand-written backward the GPU gradient tests build their bars
from (oracle/render_backward_oracle.py)."""
import numpy as np
import pytest
import torch

from oracle import render_backward_oracle as rbo, renderer_oracle as orc

CASES = {
    'crop_cull': dict(opts=dict(), flags=dict(triplane_crop=0.1, cull_clouds=0.5)),
    'binarize': dict(opts=dict(), flags=dict(triplane_crop=0.1, binarize_clouds=0.5)),
    'auto_eg3d_black': dict(opts=dict(ray_start='auto', ray_end='auto', white_back=False), flags=dict(), eg3d=True, lr_mul=0.5),
    'coarse_only': dict(opts=dict(depth_resolution_importance=0), flags=dict(), force_sigmoid=True),
}


def _inputs(name, seed=7, N=2, R=6, S=12, Sf=12, P=16):
    case = CASES[name]
    opts = dict(dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf), **case['opts'])
    Sf = opts['depth_resolution_importance']
    planes, dec, c2w, K, u_c, u_f = orc.synth_inputs(seed, N, R, S, Sf, P)
    dec = dict(dec, lr_mul=case.get('lr_mul', 1.0), force_sigmoid=case.get('force_sigmoid', False))
    dec['b2'] = dec['b2'].clone()
    dec['b2'][0] += 1.0                        # sigma around the cull threshold (sigma ~1 for cull 0.5)
    ro, rd = orc.ray_sampler(c2w, K, R)
    rng = np.random.default_rng(seed + 1)
    grads = [torch.from_numpy(rng.standard_normal(s)) for s in ((N, R * R, 32), (N, R * R, 1), (N, R * R, 1), (N, R * R, 3))]
    return planes, dec, ro, rd, opts, u_c, (u_f if Sf else None), case, grads


@pytest.mark.parametrize('name', sorted(CASES))
def test_render_reproduces_itself_from_its_own_depths_and_masks(name):
    planes, dec, ro, rd, opts, u_c, u_f, case, _ = _inputs(name)
    kw = dict(use_triplane=not case.get('eg3d'), **case['flags'])
    out, smp = orc.render(planes, dec, ro, rd, opts, u_c, u_f, return_samples=True, **kw)
    again = orc.render(planes, dec, ro, rd, opts, None, None, depths=smp['depths'], masks=smp['masks'], **kw)
    for a, b in zip(out, again):
        assert torch.equal(a, b)
    if case['flags']:
        m = torch.cat([smp['masks'][0].reshape(-1)] + ([] if smp['masks'][1] is None else [smp['masks'][1].reshape(-1)]))
        assert 0 < m.float().mean() < 1, 'the masks both keep and remove samples'


@pytest.mark.parametrize('name', sorted(CASES))
def test_hand_written_backward_equals_fp64_autograd(name):
    """The signed twin of the magnitude adjoint is the gradient: render_backward equals torch autograd of the fp64 render
    fed the fp32 run's depths and masks, to 1e-10 of each tensor's largest element; the magnitude run bounds it."""
    planes, dec, ro, rd, opts, u_c, u_f, case, grads = _inputs(name)
    kw = dict(use_triplane=not case.get('eg3d'), **case['flags'])
    _, smp = orc.render(planes, dec, ro, rd, opts, u_c, u_f, return_samples=True, **kw)
    p64 = planes.double().requires_grad_(True)
    d64 = {k: (v.double().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
    out = orc.render(p64, d64, ro, rd, opts, None, None, depths=smp['depths'], masks=smp['masks'], **kw)
    loss = sum((o * g).sum() for o, g in zip(out, grads))
    ref = torch.autograd.grad(loss, [p64] + [d64[k] for k in ('w1', 'b1', 'w2', 'b2')])
    dec64 = {k: (v.double() if torch.is_tensor(v) else v) for k, v in dec.items()}
    got = rbo.render_backward(planes.double(), dec64, ro, rd, opts, smp['depths'], smp['masks'], grads, **kw)
    A = rbo.render_backward(planes.double(), dec64, ro, rd, opts, smp['depths'], smp['masks'], grads, mag=True, c=1e30, **kw)
    for key, r in zip(('planes', 'w1', 'b1', 'w2', 'b2'), ref):
        err = (got[key] - r).abs().max().item()
        assert err <= 1e-10 * r.abs().max().item(), (name, key, err)
        assert (r.abs() <= A[key] * (1 + 1e-12) + 1e-300).all(), (name, key)
    if case['flags'].get('binarize_clouds'):
        # only colours carry gradient: the sigma row of the last layer gets none
        assert got['w2'][0].abs().max().item() == 0 and got['b2'][0].item() == 0


def test_texel_counts_match_the_taps():
    planes, dec, ro, rd, opts, u_c, u_f, case, _ = _inputs('crop_cull')
    _, smp = orc.render(planes, dec, ro, rd, opts, u_c, u_f, return_samples=True)
    cnt = rbo.texel_counts(ro, rd, smp['depths'], 16, 16, opts['box_warp'])
    n_samples = ro.shape[1] * (opts['depth_resolution'] + opts['depth_resolution_importance'])
    assert cnt.shape == (2, 3, 16, 16) and 0 < cnt.sum(dim=(1, 2, 3)).max().item() <= 12 * n_samples


def test_points_backward_equals_fp64_autograd():
    """render_backward_oracle.points_backward (the density-regularisation backward) is the gradient of run_model's sigma."""
    planes, dec, *_ = _inputs('crop_cull')
    g = torch.Generator().manual_seed(3)
    xyz = (torch.rand(2, 300, 3, generator=g) * 2 - 1) * 0.4
    g_sigma = torch.randn(2, 300, generator=g, dtype=torch.float64)
    p64 = planes.double().requires_grad_(True)
    d64 = {k: (v.double().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
    ref = torch.autograd.grad((orc.run_model(p64, d64, xyz, orc.DEFAULT_OPTS, True)[1] * g_sigma[..., None]).sum(),
                              [p64] + [d64[k] for k in ('w1', 'b1', 'w2', 'b2')])
    dd = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in d64.items()}
    got = rbo.points_backward(planes.double(), dd, xyz, g_sigma, orc.DEFAULT_OPTS['box_warp'])
    A = rbo.points_backward(planes.double(), dd, xyz, g_sigma, orc.DEFAULT_OPTS['box_warp'], mag=True, c=1e30)
    for key, r in zip(('planes', 'w1', 'b1', 'w2', 'b2'), ref):
        assert (got[key] - r).abs().max().item() <= 1e-10 * r.abs().max().item(), key
        assert (r.abs() <= A[key] * (1 + 1e-12) + 1e-300).all(), key
    bound = rbo.sigma_error_bound(planes[0].double(), dd, xyz[0], orc.DEFAULT_OPTS['box_warp'])
    _, s32 = orc.run_model(planes[:1], dec, xyz[:1], orc.DEFAULT_OPTS, True)
    _, s64 = orc.run_model(planes[:1].double(), dd, xyz[:1], orc.DEFAULT_OPTS, True)
    assert ((s32.double() - s64)[0, :, 0].abs() <= bound).all(), 'the fp32 oracle is within the fp32 decode bound'
