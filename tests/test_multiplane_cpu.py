"""CPU: multiplane tri-planes (triplane_depth > 1).  The oracle against the reference's own outputs and gradients
(tests/golden/multiplane_*.npz, written by make_golden_multiplane.py), and the C ABI's host-side answers for
plane_depth > 1: no tensor-core kernel, no host-buffer entry point, short plane strides refused."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import multiplane_oracle as mo, renderer_oracle as orc
from tests.golden.cases_multiplane import RENDER_CASES, POINT_CASES, GRAD_CASES, build_inputs, point_coords, upstream, H, W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _load(name):
    return np.load(os.path.join(GOLDEN, f'multiplane_{name}.npz'))


def _maxerr(a, b):
    return float((torch.as_tensor(np.asarray(a)) - torch.as_tensor(np.asarray(b))).abs().max())


@pytest.mark.parametrize('name', sorted(RENDER_CASES))
def test_oracle_render_matches_reference(name):
    case = RENDER_CASES[name]
    z = _load(f'render_{name}')
    assert json.loads(str(z['case'])) == json.loads(json.dumps(case))
    planes, dec, _, _, u_c, u_f, opts = build_inputs(case)
    assert float(planes.double().sum() + u_c.double().sum()) == float(z['input_checksum'])
    ro, rd = torch.from_numpy(z['ro']), torch.from_numpy(z['rd'])
    out = mo.render(planes, dec, ro, rd, opts, u_c, u_f, use_triplane=case['use_triplane'],
                     triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'))
    for key, got in zip(('rgb', 'depth', 'wsum', 'xyz'), out):
        assert _maxerr(got, z[key]) < 2e-5, (key, _maxerr(got, z[key]))
    assert float(z['wsum'].max()) > 0.05, 'the case must composite something'


@pytest.mark.parametrize('name', sorted(POINT_CASES))
def test_oracle_run_model_matches_reference(name):
    case = POINT_CASES[name]
    z = _load(f'points_{name}')
    planes, dec, _, _, _, _, opts = build_inputs(case)
    pts = point_coords(case)
    assert np.array_equal(pts.numpy(), z['pts'])
    rgb, sigma = mo.run_model(planes, dec, pts, opts, case['use_triplane'])
    assert _maxerr(rgb, z['rgb']) < 2e-5 and _maxerr(sigma, z['sigma']) < 2e-5
    # the aten gather (5-D grid_sample) agrees with the manual one
    rgb_a, sigma_a = mo.run_model(planes, dec, pts, opts, case['use_triplane'], gather='aten')
    assert _maxerr(rgb_a, z['rgb']) < 2e-5 and _maxerr(sigma_a, z['sigma']) < 2e-5


@pytest.mark.parametrize('name', sorted(GRAD_CASES))
def test_oracle_autograd_matches_reference_gradients(name):
    case = GRAD_CASES[name]
    z = _load(f'grad_{name}')
    planes, dec, _, _, u_c, u_f, opts = build_inputs(case)
    planes = planes.clone().requires_grad_(True)
    dec = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
    if 'R' in case:
        ro, rd = orc.ray_sampler(*build_inputs(case)[2:4], case['R'])
        outs = mo.render(planes, dec, ro, rd, opts, u_c, u_f, use_triplane=case['use_triplane'])
    else:
        outs = mo.run_model(planes, dec, point_coords(case), opts, case['use_triplane'])
    gs = upstream(case, [tuple(t.shape) for t in outs])
    sum(((t * g).sum() for t, g in zip(outs, gs)), torch.zeros(())).backward()
    for key, got in (('d_planes', planes.grad), ('d_w1', dec['w1'].grad), ('d_b1', dec['b1'].grad), ('d_w2', dec['w2'].grad),
                     ('d_b2', dec['b2'].grad)):
        want = torch.from_numpy(z[key])
        rel = float((got - want).abs().max() / want.abs().max())
        assert rel < 2e-5, (key, rel)
        if key == 'd_planes':
            assert torch.equal(got == 0, want == 0), 'the same texels must be untouched'


def test_slab_points_cover_centres_borders_and_outside():
    from tests.golden.cases_multiplane import slab_points, BOX
    for D in (2, 3):
        for use_triplane in (False, True):
            sp = torch.from_numpy(slab_points(D, use_triplane)).double()
            n = mo.plane_coords3(sp[None] * (2.0 / BOX), use_triplane)[0, ..., 2]    # (3, P) normal coordinate per plane
            fz = ((n + 1) * D - 1) / 2
            for p in range(3):
                on_plane = fz[p]
                assert any(abs(v - d) < 1e-6 for v in on_plane.tolist() for d in range(D)), 'slab centres'
                assert (on_plane < -0.5).any() and (on_plane > D - 0.5).any(), 'points past both faces along the normal'


def test_plane_coords3_normals():
    """The third component of project_onto_planes: z, y, y for EG3D planes and z, y, x for use_triplane."""
    xyz = torch.tensor([[[0.1, 0.2, 0.3]]])
    for use_triplane, normals, firsts in ((False, [0.3, 0.2, 0.2], [(0.1, 0.2), (0.1, 0.3), (0.3, 0.1)]),
                                          (True, [0.3, 0.2, 0.1], [(0.1, 0.2), (0.1, 0.3), (0.2, 0.3)])):
        c = mo.plane_coords3(xyz, use_triplane)[0, :, 0]
        assert torch.allclose(c[:, 2], torch.tensor(normals))
        assert torch.allclose(c[:, :2], torch.tensor(firsts))
        assert torch.allclose(c[:, :2], orc.plane_coords(xyz, use_triplane)[0, :, 0])


# ---------------------------------------------------------------------------------------------------------------- C ABI
def _params(D=2, mlp_mode=0, stride_plane=None, stride_view=None):
    from panic3d_b200 import _lib
    p = _lib.RenderParams()
    p.n_views, p.n_rays, p.n_coarse, p.n_fine = 1, 384, 48, 48
    p.channels, p.plane_h, p.plane_w, p.hidden, p.out_dim = 32, H, W, 64, 33
    p.stride_col, p.stride_row = 32, 32 * W
    p.stride_plane = 32 * W * H * max(D, 1) if stride_plane is None else stride_plane
    p.stride_view = 3 * p.stride_plane if stride_view is None else stride_view
    p.box_warp, p.ray_start, p.ray_end = 0.7, 0.5, 1.5
    p.w1_gain = p.b1_gain = p.w2_gain = p.b2_gain = 1.0
    p.mlp_mode, p.plane_depth = mlp_mode, D
    return p


def test_params_struct_keeps_its_size():
    from panic3d_b200 import _lib
    assert C.sizeof(_lib.RenderParams) == 184
    assert _lib.RenderParams.plane_depth.offset == 180


def test_supported_queries_refuse_multiplane():
    from panic3d_b200 import _lib
    L = _lib.lib()
    for D, want in ((0, 1), (1, 1), (2, 0), (3, 0)):
        p = _params(D, mlp_mode=_lib.P3D_MLP_TC_3XBF16)
        assert L.p3d_render_fused_supported(C.byref(p)) == want, D
        assert L.p3d_decode_tc_supported(C.byref(p), 4096) == want, D


def test_explicit_tensor_core_request_and_host_entry_point_refuse_multiplane():
    from panic3d_b200 import _lib
    L = _lib.lib()
    P3D_EUNSUPPORTED = -4
    for mode in (_lib.P3D_MLP_TC_3XBF16, _lib.P3D_MLP_TC_BF16):
        p = _params(2, mlp_mode=mode)
        p.n_views = 0                                  # refused before anything touches a device
        assert L.p3d_render_forward(C.byref(p), *([None] * 9), None, 0, *([None] * 5)) == P3D_EUNSUPPORTED
        assert b'tensor-core' in L.p3d_last_error()
        assert L.p3d_decode_points(C.byref(p), *([None] * 6), 0, None, None, None) == P3D_EUNSUPPORTED
        assert L.p3d_volume_query(C.byref(p), *([None] * 5), 8, 0.7, -1.0, -1.0, *([None] * 5)) == P3D_EUNSUPPORTED
    p = _params(2)
    p.n_rays = 16 * 16
    buf = (C.c_float * 16)()
    assert L.p3d_render_forward_host(C.byref(p), *([C.cast(buf, C.c_void_p)] * 7), 16, None, None, *([C.cast(buf, C.c_void_p)] * 4)) == P3D_EUNSUPPORTED
    assert b'plane_depth' in L.p3d_last_error()


def test_short_plane_strides_are_refused():
    from panic3d_b200 import _lib
    L = _lib.lib()
    P3D_EINVAL = -1
    args = lambda p: (C.byref(p), *([None] * 6), 0, None, None, None)
    assert L.p3d_decode_points(*args(_params(2))) == 0                                   # zero points: accepted, nothing runs
    assert L.p3d_decode_points(*args(_params(2, stride_plane=32 * W * (2 * H - 1)))) == P3D_EINVAL
    assert b'stride_plane' in L.p3d_last_error()
    assert L.p3d_decode_points(*args(_params(3, stride_plane=32 * W * H * 3, stride_view=32 * W * H * 8))) == P3D_EINVAL
    assert b'stride_view' in L.p3d_last_error()
    assert L.p3d_decode_points(*args(_params(3, stride_view=0))) == 0                    # one tri-plane shared by every view
    assert L.p3d_decode_points(*args(_params(1, stride_plane=32 * W * H))) == 0          # one slab: today's addressing
    assert L.p3d_decode_points(*args(_params(-1))) == P3D_EINVAL


def test_channels_not_divisible_by_depth_raise():
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    r = ImportanceRenderer()
    planes = torch.zeros(1, 3, 64, 4, 4)
    with pytest.raises(ValueError, match='triplane_depth'):
        r._planes_cl(planes, 3)
    with pytest.raises(ValueError, match='triplane_depth'):
        r._shape_probe(planes, dict(triplane_depth=3))
    assert tuple(r._shape_probe(planes, dict(triplane_depth=2)).shape) == (1, 3, 2, 4, 4, 32)
    assert tuple(r._shape_probe(planes, dict(triplane_depth=1)).shape) == (1, 3, 4, 4, 64)


def test_multiplane_texel_layout_and_gradient_indexing_round_trip():
    """_multiplane_texels puts feature c of slab d (input channel c*D + d) at [..., d, h, w, c]; _planes_grad maps such a
    buffer back to the input's (N,3,C*D,H,W) indexing."""
    from panic3d_b200.training.volumetric_rendering.renderer import _multiplane_texels, _planes_grad
    planes = torch.randn(2, 3, 32 * 3, 5, 4)
    t = _multiplane_texels(planes, 3)
    assert t.shape == (2, 3, 3, 5, 4, 32) and t.is_contiguous()
    assert torch.equal(t[1, 2, 1, 3, 2, 7], planes[1, 2, 7 * 3 + 1, 3, 2])
    assert torch.equal(_planes_grad(t, torch.float32), planes)


# ------------------------------------------------------------------------------ the hand-written backward's multiplane taps
BWD_FLAGS = {'crop_cull': dict(triplane_crop=0.1, cull_clouds=0.5), 'binarize': dict(triplane_crop=0.1, binarize_clouds=0.5)}


def _bwd_inputs(D, use_triplane, seed=7, N=2, R=6, S=12, Sf=12, P=16):
    """renderer_oracle.synth_inputs' decoder and rays, with planes of D slabs ((N, 3, 32*D, P, P); the same planes as
    tests/test_render_backward_oracle_cpu.py at D = 1)."""
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf, triplane_depth=D)
    planes, dec, c2w, K, u_c, u_f = orc.synth_inputs(seed, N, R, S, Sf, P)
    if D > 1:
        planes = torch.from_numpy(np.random.default_rng(seed + 100).standard_normal((N, 3, 32 * D, P, P), dtype=np.float32))
    dec = dict(dec, b2=dec['b2'].clone())
    dec['b2'][0] += 1.0                        # sigma around the cull threshold
    ro, rd = orc.ray_sampler(c2w, K, R)
    rng = np.random.default_rng(seed + 1)
    grads = [torch.from_numpy(rng.standard_normal(s)) for s in ((N, R * R, 32), (N, R * R, 1), (N, R * R, 1), (N, R * R, 3))]
    return planes, dec, ro, rd, opts, u_c, u_f, grads


def _oracle(D):
    """The render oracle for planes of D slabs: at D = 1 the reference's one-slab lookup, not a 5-D grid_sample over one slab."""
    return mo if D > 1 else orc


def _dec64(dec, grad=False):
    return {k: (v.double().requires_grad_(grad) if torch.is_tensor(v) else v) for k, v in dec.items()}


@pytest.mark.parametrize('flags', sorted(BWD_FLAGS))
@pytest.mark.parametrize('use_triplane', [True, False])
@pytest.mark.parametrize('D', [1, 2, 3])
def test_hand_written_backward_with_slabs_equals_fp64_autograd(D, use_triplane, flags):
    """render_backward(depth=D) equals torch's fp64 autograd of multiplane_oracle.render fed the fp32 run's depths and
    masks, to 1e-10 of each tensor's largest element, and its magnitude run bounds it."""
    from oracle import render_backward_oracle as rbo
    planes, dec, ro, rd, opts, u_c, u_f, grads = _bwd_inputs(D, use_triplane)
    kw = dict(use_triplane=use_triplane, **BWD_FLAGS[flags])
    _, smp = _oracle(D).render(planes, dec, ro, rd, opts, u_c, u_f, return_samples=True, **kw)
    m = torch.cat([smp['masks'][0].reshape(-1), smp['masks'][1].reshape(-1)])
    assert 0 < m.float().mean() < 1, 'the masks both keep and remove samples'
    p64, d64 = planes.double().requires_grad_(True), _dec64(dec, True)
    out = _oracle(D).render(p64, d64, ro, rd, opts, None, None, depths=smp['depths'], masks=smp['masks'], **kw)
    ref = torch.autograd.grad(sum((o * g).sum() for o, g in zip(out, grads)), [p64] + [d64[k] for k in ('w1', 'b1', 'w2', 'b2')])
    got = rbo.render_backward(planes.double(), _dec64(dec), ro, rd, opts, smp['depths'], smp['masks'], grads, depth=D, **kw)
    A = rbo.render_backward(planes.double(), _dec64(dec), ro, rd, opts, smp['depths'], smp['masks'], grads, mag=True, c=1e30,
                            depth=D, **kw)
    for key, r in zip(('planes', 'w1', 'b1', 'w2', 'b2'), ref):
        assert got[key].shape == r.shape, key
        err = (got[key] - r).abs().max().item()
        assert err <= 1e-10 * r.abs().max().item(), (key, err)
        assert (r.abs() <= A[key] * (1 + 1e-12) + 1e-300).all(), key
    assert (ref[0] != 0).any() and (ref[0] == 0).any()


@pytest.mark.parametrize('use_triplane', [True, False])
@pytest.mark.parametrize('D', [1, 2, 3])
def test_points_backward_with_slabs_equals_fp64_autograd(D, use_triplane):
    """points_backward(depth=D) is the gradient of multiplane_oracle.run_model's sigma, on points that include slab centres,
    slab borders and points past the box along each normal; sigma_error_bound(depth=D) bounds the fp32 oracle's sigma."""
    from oracle import render_backward_oracle as rbo
    from tests.golden.cases_multiplane import slab_points
    planes, dec, *_ = _bwd_inputs(D, use_triplane)
    g = torch.Generator().manual_seed(3)
    xyz = torch.cat([(torch.rand(2, 300, 3, generator=g) * 2 - 1) * 0.4,
                     torch.from_numpy(slab_points(max(D, 2), use_triplane)).expand(2, -1, -1)], 1).contiguous()
    g_sigma = torch.randn(2, xyz.shape[1], generator=g, dtype=torch.float64)
    opts = dict(orc.DEFAULT_OPTS, triplane_depth=D)
    p64, d64 = planes.double().requires_grad_(True), _dec64(dec, True)
    ref = torch.autograd.grad((_oracle(D).run_model(p64, d64, xyz, opts, use_triplane)[1] * g_sigma[..., None]).sum(),
                              [p64] + [d64[k] for k in ('w1', 'b1', 'w2', 'b2')])
    bw = opts['box_warp']
    got = rbo.points_backward(planes.double(), _dec64(dec), xyz, g_sigma, bw, use_triplane, depth=D)
    A = rbo.points_backward(planes.double(), _dec64(dec), xyz, g_sigma, bw, use_triplane, mag=True, c=1e30, depth=D)
    for key, r in zip(('planes', 'w1', 'b1', 'w2', 'b2'), ref):
        assert (got[key] - r).abs().max().item() <= 1e-10 * r.abs().max().item(), key
        assert (r.abs() <= A[key] * (1 + 1e-12) + 1e-300).all(), key
    bound = rbo.sigma_error_bound(planes[0].double(), _dec64(dec), xyz[0], bw, use_triplane, depth=D)
    s32 = _oracle(D).run_model(planes[:1], dec, xyz[:1], opts, use_triplane)[1]
    s64 = _oracle(D).run_model(planes[:1].double(), _dec64(dec), xyz[:1], opts, use_triplane)[1]
    assert ((s32.double() - s64)[0, :, 0].abs() <= bound).all(), 'the fp32 oracle is within the fp32 decode bound'


@pytest.mark.parametrize('gather', ['manual', 'aten'])
@pytest.mark.parametrize('use_triplane', [True, False])
@pytest.mark.parametrize('D', [2, 3])
def test_taps_weighted_sum_equals_sample_multiplane(D, use_triplane, gather):
    """The 24 taps of render_backward_oracle.taps, summed with their weights over the texels of render_backward_oracle.texels,
    are sample_multiplane's features; texel_counts counts exactly the in-bounds taps."""
    from oracle import render_backward_oracle as rbo
    from tests.golden.cases_multiplane import slab_points
    planes, _, ro, rd, opts, u_c, _, _ = _bwd_inputs(D, use_triplane)
    g = torch.Generator().manual_seed(11)
    xyz = torch.cat([(torch.rand(1, 500, 3, generator=g) * 2 - 1) * 0.45,
                     torch.from_numpy(slab_points(D, use_triplane))[None]], 1)
    idx, wgt = rbo.taps(xyz[0], 16, 16, opts['box_warp'], use_triplane, D)
    assert idx.shape == (xyz.shape[1], 24) and int(idx.max()) < 3 * D * 16 * 16
    p64 = planes[:1].double()
    got = rbo.gather(rbo.texels(p64[0], D), idx, wgt)                                     # (K,3,C)
    # the manual gather takes the same fp32 footprint (fp64 sums); aten's grid_sample wants one dtype, so it runs in fp64
    # from the fp32 points and differs by the footprint's fp32 rounding
    xyz_g = xyz if gather == 'manual' else xyz.double()
    want = mo.sample_multiplane(p64, xyz_g, opts['box_warp'], use_triplane, D, gather)[0]  # (3,K,C)
    assert (got - want.permute(1, 0, 2)).abs().max().item() <= (1e-12 if gather == 'manual' else 1e-5)
    # every slab is reached
    z = (idx[idx >= 0] // (16 * 16)) % D
    assert set(z.tolist()) == set(range(D))
    d_c = orc.stratified_depths(u_c, opts['ray_start'], opts['ray_end'])
    cnt = rbo.texel_counts(ro, rd, (d_c, None), 16, 16, opts['box_warp'], use_triplane, D)
    assert cnt.shape == (2, 3, D, 16, 16)
    for n in range(2):
        xyz_n = (ro[n, :, None] + d_c[n, ..., 0, None] * rd[n, :, None]).reshape(-1, 3)
        assert cnt[n].sum().item() == (rbo.taps(xyz_n, 16, 16, opts['box_warp'], use_triplane, D)[0] >= 0).sum().item()


def test_oracle_sampling_is_scoped():
    """multiplane_oracle.sampling replaces the renderer oracle's plane lookup for its block only, also when it raises."""
    one_slab = orc.sample_planes
    with mo.sampling(2):
        assert orc.sample_planes is not one_slab
    assert orc.sample_planes is one_slab
    with pytest.raises(KeyError):
        with mo.sampling(2):
            raise KeyError
    assert orc.sample_planes is one_slab
