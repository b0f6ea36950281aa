"""GPU: the training-path backward (k_ray_backward + k_sample_backward) at sample counts that need several 32-lane chunks
per ray, against torch.autograd on the CPU oracle.

k_ray_backward walks a ray's merged intervals in warp-wide chunks and carries the transmittance product (`carry`) and the
prefix sum of w_i dL/dw_i (`pcarry`) from one chunk to the next.  The fixture-backed gradient cases of test_render_gpu.py
have at most 31 intervals, so those carries are never used there; the cases below have 39 to 191 intervals, including
counts that end one lane into a chunk.  Every case also has a ray count that is not a multiple of 4 (the `ray >= R` tail
of k_ray_backward) and R * S not a multiple of 128 (a partial last CTA of k_sample_backward)."""
import numpy as np
import pytest
import torch

from oracle import renderer_oracle as orc
from tests.golden.cases import build_case_inputs
from tests.helpers import BWD_CASES, bwd_case, bwd_flags, bwd_incoming, case_rays
from tests.render_abi import make_decoder

pytestmark = pytest.mark.gpu
TIGHT = 1e-4        # forward outputs of the fp32 SIMT path vs the oracle
GRAD_REL = 2e-3     # gradients: max abs error < GRAD_REL * max(1e-3, max |reference|)


PARAMS = ('planes', 'w1', 'b1', 'w2', 'b2')


def _loss(outs, gw):
    return sum((o * g_.to(o.device)).sum() for o, g_ in zip(outs, gw))


def _grad_err(got, ref):
    """max |got - ref| and the bar it has to stay under."""
    err = (got.cpu() - ref).abs().max().item()
    return err, GRAD_REL * max(1e-3, ref.abs().max().item())


def _cull_census(case, planes, dec, ro, rd, u_c, u_f, opts):
    """Per pass (coarse, fine): the share of the samples the crop keeps that cull then removes, and the smallest distance of
    their sigma from the cull threshold.  Same steps as orc.render up to the masks of the fine pass."""
    N, M = ro.shape[0], ro.shape[1]
    S, bw = opts['depth_resolution'], opts['box_warp']
    crop, cull = case['triplane_crop'], case['cull_clouds']
    thresh = 1.0 + float(np.log(np.expm1(-np.log1p(-cull))))       # cull_mask(sigma, cull) <=> sigma < thresh
    d_c = orc.stratified_depths(u_c, opts['ray_start'], opts['ray_end'])
    xyz_c = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)
    rgb_c, sig_c = orc.run_model(planes, dec, xyz_c, opts, True)
    masked_c = orc.apply_masks(sig_c, xyz_c, bw, crop, cull, None)
    _, _, w = orc.march(rgb_c.reshape(N, M, S, -1), masked_c.reshape(N, M, S, 1), d_c, bool(opts['white_back']))
    d_f = orc.importance_depths(d_c.reshape(N * M, S), w.reshape(N * M, S - 1), u_f).reshape(N, M, -1, 1)
    xyz_f = (ro[:, :, None] + d_f * rd[:, :, None]).reshape(N, -1, 3)
    _, sig_f = orc.run_model(planes, dec, xyz_f, opts, True)
    census = []
    for sig, xyz in ((sig_c, xyz_c), (sig_f, xyz_f)):
        s = sig[~orc.crop_mask(xyz, crop, bw)]
        census.append((orc.cull_mask(s, cull).float().mean().item(), (s - thresh).abs().min().item()))
    return census


@pytest.mark.parametrize('name', sorted(BWD_CASES))
def test_multi_chunk_backward_matches_oracle_autograd(name):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = BWD_CASES[name]
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = case_rays(case, c2w, K)
    N, M = ro.shape[0], ro.shape[1]
    S, Sf = opts['depth_resolution'], opts['depth_resolution_importance']
    assert S + Sf - 1 > 32 and (N * M) % 4 != 0 and (N * M * S) % 128 != 0 and (Sf == 0 or (N * M * Sf) % 128 != 0)
    if case.get('cull_clouds'):
        # cull must remove some of the samples the crop keeps (constant sigma, no gradient) but not all of them, and no sigma
        # may sit within rounding of the threshold, where kernel and oracle could disagree on the mask
        for frac, margin in _cull_census(case, planes, dec, ro, rd, u_c, u_f, opts):
            print(f'{name}: cull removes {frac:.3f} of the uncropped samples; closest sigma {margin:.2e} from the threshold')
            assert 0.05 < frac < 0.95 and margin > 1e-4, (frac, margin)
    gw = bwd_incoming(case['seed'] + 5, N, M)

    pl = planes.clone().requires_grad_(True)
    dref = {k: (v.clone().requires_grad_(True) if isinstance(v, torch.Tensor) else v) for k, v in dec.items()}
    out = orc.render(pl, dref, ro, rd, opts, u_c, u_f if Sf > 0 else None, use_triplane=True, **bwd_flags(case))
    ref = torch.autograd.grad(_loss(out, gw), [pl, dref['w1'], dref['b1'], dref['w2'], dref['b2']])

    dev = torch.device('cuda:0')
    r = ImportanceRenderer(use_triplane=True)
    r.injected_noise = (u_c, u_f)
    d = make_decoder(dec, dev).requires_grad_(True)
    pg = planes.to(dev).requires_grad_(True)
    got_out = r(pg, d, ro.to(dev), rd.to(dev), opts, **bwd_flags(case))
    for o, o_ref, key in zip(got_out, out, ('rgb', 'depth', 'wsum', 'xyz')):
        err = (o.detach().cpu() - o_ref.detach()).abs().max().item()
        assert err < TIGHT, f'{name}:{key} forward max abs err {err}'
    got = torch.autograd.grad(_loss(got_out, gw), [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    for g_, r_, nm in zip(got, ref, PARAMS):
        assert g_.shape == r_.shape, nm
        err, bar = _grad_err(g_, r_)
        print(f'{name}:{nm} grad max abs err {err:.3e} (bar {bar:.3e}, ratio {err / bar:.3f})')
        assert err < bar, f'{name}:{nm} max abs err {err} (bar {bar})'


def test_sharded_backward_sums_to_the_batch_backward():
    """Data-parallel training on one GPU: each view rendered alone under autograd, with the batch's depth-clamp bounds
    injected through `depth_bounds_reduce`, reproduces the batch forward bit for bit; its plane gradient matches the batch's
    gradient of that view, and the per-view decoder gradients sum to the batch's, within the gradient bar (the scatter
    into the gradients is a float atomic add, so the summation order differs).  The backward's depth gradient is gated on
    the rank-local bounds in the workspace while the forward clamps to the reduced ones; a ray's unclamped depth is a
    convex combination of its own interval midpoints, so it lies inside both and the gate agrees."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = bwd_case(67, 48, 48, N=3, cameras=[(0.0, -180.0, 1.0, 30.0), (0.0, 90.0, 1.0, 30.0), (60.0, -45.0, 1.2, 45.0)])
    planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
    ro, rd = case_rays(case, c2w, K)
    N, M = ro.shape[0], ro.shape[1]
    gw = bwd_incoming(case['seed'] + 5, N, M)
    dev = torch.device('cuda:0')
    r = ImportanceRenderer(use_triplane=True)
    d = make_decoder(dec, dev).requires_grad_(True)
    params = [d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias]
    seen = {}
    r.depth_bounds_reduce = lambda b2: seen.__setitem__('b', b2.clone())
    r.injected_noise = (u_c, u_f)
    pg = planes.to(dev).requires_grad_(True)
    full_out = r(pg, d, ro.to(dev), rd.to(dev), opts)
    full = torch.autograd.grad(_loss(full_out, gw), [pg] + params)

    # each view's own bounds differ from the batch's, so this is the case where the two gates could disagree
    local = []
    r.depth_bounds_reduce = lambda b2: local.append(b2.cpu())
    for i in range(N):
        r.injected_noise = (u_c[i:i + 1], u_f[i * M:(i + 1) * M])
        with torch.no_grad():
            r(planes[i:i + 1].to(dev), d, ro[i:i + 1].to(dev), rd[i:i + 1].to(dev), opts)
    assert any(not torch.equal(b, seen['b'].cpu()) for b in local)

    r.depth_bounds_reduce = lambda b2: b2.copy_(seen['b'])
    plane_grads, dec_sum = [], [torch.zeros_like(p) for p in params]
    for i in range(N):
        r.injected_noise = (u_c[i:i + 1], u_f[i * M:(i + 1) * M])
        pv = planes[i:i + 1].to(dev).requires_grad_(True)
        out = r(pv, d, ro[i:i + 1].to(dev), rd[i:i + 1].to(dev), opts)
        for o, f in zip(out, full_out):
            assert torch.equal(o.detach(), f.detach()[i:i + 1])
        g = torch.autograd.grad(_loss(out, [x[i:i + 1] for x in gw]), [pv] + params)
        plane_grads.append(g[0])
        dec_sum = [a + b for a, b in zip(dec_sum, g[1:])]
    for got, want, nm in zip([torch.cat(plane_grads)] + dec_sum, full, PARAMS):
        err, bar = _grad_err(got, want.cpu())
        print(f'sharded:{nm} grad max abs err {err:.3e} (bar {bar:.3e})')
        assert err < bar, f'sharded:{nm} max abs err {err} (bar {bar})'
