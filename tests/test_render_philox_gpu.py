"""GPU: renders that draw their own jitter, against the CPU oracle fed the same uniforms.

Production renders inject nothing: the default `ImportanceRenderer` path, every training step (`_RenderFunction`),
`bench.py` and the host entry point pass NULL uniform pointers, so the kernels draw Philox4x32-10 uniforms in-kernel
(`philox_uniform`, csrc/p3d_common.cuh).  `oracle.philox` restates that rule (coarse sample s of global ray r: index
r*S + s, stream 0; fine sample f: index r*Sf + f, stream 1; the host path's per-view seed), so every ray of a production
render can be checked at the bars of the injected-noise tests instead of statistically.  No test here sets
`injected_noise`.

Each case draws its seed the way the renderer does (`oracle.philox.drawn_seed` after `torch.manual_seed(k)`) or passes
it through the C ABI, renders, and compares every output of every ray with `orc.render` on `render_uniforms` of that
seed.  Negative controls show the comparison can see a wrong stream: the oracle fed the uniforms of a wrong rule
(seed ^ 1, the two streams swapped, fine index r*S + f, every host view on the base seed) must miss the kernel by more
than CONTROL times the bar on some output."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import philox as ph, renderer_oracle as orc
from tests.golden.cases import RENDER_CASES, build_case_inputs
from tests.helpers import case_rays, profiled
from tests.render_abi import make_decoder

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
TIGHT = 1e-4        # fp32 SIMT kernels (they reach ~1e-6)
TOL = 1e-3          # fused tensor-core renderer
GRAD_REL = 2e-3     # gradients: max abs error < GRAD_REL * max(1e-3, max |reference|)
CONTROL = 20        # a wrong uniform rule must miss the kernel by more than CONTROL x the bar
PROF_SAMPLE_DECODE, PROF_FUSED = 0, 5          # profile slots (csrc/p3d_common.cuh)
KEYS = ('rgb', 'depth', 'wsum', 'xyz')


def _case(seed, S, Sf, R=15, N=2, P=64, **kw):
    return dict(seed=seed, N=N, R=R, P=P, opts=dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf),
                cameras=None, **kw)


def _flags(case):
    return dict(triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'), binarize_clouds=case.get('binarize_clouds'))


def _inputs(case):
    planes, dec, c2w, K, _u_c, _u_f, opts = build_case_inputs(case)      # the fixture uniforms are not used
    ro, rd = case_rays(case, c2w, K)
    return planes, dec, ro, rd, opts


def _renderer(mlp_mode):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    r = ImportanceRenderer(use_triplane=True)
    r.mlp_mode = mlp_mode
    assert r.injected_noise is None
    return r


def _render(planes, dec, ro, rd, opts, flags, mlp_mode, k):
    """A production render (no injected noise) as the first RNG draw after torch.manual_seed(k).  -> outputs (CPU),
    launches per profile slot."""
    r = _renderer(mlp_mode)
    d = make_decoder(dec, DEV)              # before the seed: building a module draws from the CPU generator
    x, o, v = planes.to(DEV), ro.to(DEV), rd.to(DEV)
    torch.manual_seed(k)
    with torch.no_grad():
        out, prof = profiled(lambda: r(x, d, o, v, opts, **flags))
    return [t.cpu() for t in out], prof


def _oracle(planes, dec, ro, rd, opts, flags, uniforms, **kw):
    u_c, u_f = uniforms
    return orc.render(planes, dec, ro, rd, opts, u_c, u_f if opts['depth_resolution_importance'] > 0 else None,
                      use_triplane=True, **flags, **kw)


def _max_err(a, b):
    """max |a - b|; a NaN anywhere counts as an infinite error (max() would otherwise drop it)."""
    e = (a.detach().cpu().double() - b.detach().cpu().double()).abs().max().item()
    return math.inf if math.isnan(e) else e


def _check(tag, got, want, bar):
    worst = 0.0
    for a, b, key in zip(got, want, KEYS):
        assert a.shape == b.shape, (tag, key)
        err = _max_err(a, b)
        worst = max(worst, err / bar)
        assert err < bar, f'{tag}:{key} max abs err {err:.3e} (bar {bar:.0e})'
    print(f'PHILOX {tag}: worst error {worst:.4f} of the bar {bar:.0e}')


def _wrong_rules(seed, N, M, S, Sf, fine_index_on_S=False):
    """Uniforms of rules a kernel could wrongly implement, in render_uniforms' shapes."""
    def arr(x, shape):
        return torch.from_numpy(x.reshape(shape))
    idx_c, idx_f = np.arange(N * M * S, dtype=np.uint64), np.arange(N * M * Sf, dtype=np.uint64)
    rules = {
        'seed ^ 1': ph.render_uniforms(seed ^ 1, N, M, S, Sf),
        'streams swapped': (arr(ph.uniforms(seed, idx_c, ph.STREAM_FINE), (N, M, S, 1)),
                            arr(ph.uniforms(seed, idx_f, ph.STREAM_COARSE), (N * M, Sf))),
    }
    if fine_index_on_S:
        assert S != Sf
        rf = np.arange(N * M, dtype=np.uint64)[:, None] * np.uint64(S) + np.arange(Sf, dtype=np.uint64)[None]
        rules['fine index r*S + f'] = (ph.render_uniforms(seed, N, M, S, 0)[0], arr(ph.uniforms(seed, rf, ph.STREAM_FINE), (N * M, Sf)))
    return rules


def _controls(tag, got, oracle_of, rules, bar):
    for name, uniforms in rules.items():
        dist = max(_max_err(a, b) for a, b in zip(got, oracle_of(uniforms)))
        print(f'PHILOX {tag}: control "{name}" misses by {dist / bar:.0f} x the bar')
        assert dist > CONTROL * bar, (tag, name, dist)


# ---------------------------------------------------------------------------------------------
# fp32 SIMT kernels (k_sample_decode coarse stream, k_ray_importance fine stream with rng_base = ray * Sf)
# ---------------------------------------------------------------------------------------------
SIMT_CASES = {                          # N = 2 (ray indices cross a view), 2 x 15^2 = 450 rays (not a multiple of 4)
    'train48': _case(81, 48, 48),                                           # the training setting
    'uneven64_32': _case(82, 64, 32),                                       # S != Sf: only the SIMT kernels take it
    'eval96_crop': _case(83, 96, 96, triplane_crop=0.1, force_sigmoid=True),
    'coarse40': _case(84, 40, 0),
}


@pytest.mark.parametrize('name', sorted(SIMT_CASES))
def test_simt_render_draws_the_restated_uniforms(name):
    case = SIMT_CASES[name]
    planes, dec, ro, rd, opts = _inputs(case)
    N, M = ro.shape[:2]
    S, Sf = opts['depth_resolution'], opts['depth_resolution_importance']
    assert N >= 2 and (N * M) % 4 != 0
    k = case['seed']
    got, prof = _render(planes, dec, ro, rd, opts, _flags(case), 0, k)
    assert prof[PROF_FUSED] == 0 and prof[PROF_SAMPLE_DECODE] >= 1, prof
    seed = ph.drawn_seed(k)
    oracle_of = lambda u: _oracle(planes, dec, ro, rd, opts, _flags(case), u)
    _check(f'simt {name}', got, oracle_of(ph.render_uniforms(seed, N, M, S, Sf)), TIGHT)
    _controls(f'simt {name}', got, oracle_of, _wrong_rules(seed, N, M, S, Sf, fine_index_on_S=0 < Sf != S), TIGHT)


# ---------------------------------------------------------------------------------------------
# the fused renderer (k_render_ws3) through the default mlp_mode 'auto'
# ---------------------------------------------------------------------------------------------
FUSED_CASES = {                         # 2 x 16^2 rays: whole groups of 384 / S rays in each view
    'fused48': _case(85, 48, 48, R=16),
    # 96 samples resolve 64^2 planes so finely that another draw of uniforms moves the render by < 1e-2; 512^2 planes and
    # denser sigma make the jitter visible at CONTROL x the bar
    'fused96': _case(86, 96, 96, R=16, P=512, sigma_bias=2.0),
}


def _fused(planes, dec, ro, rd, opts, k):
    got, prof = _render(planes, dec, ro, rd, opts, {}, 'auto', k)
    assert prof[PROF_FUSED] == 1 and prof[PROF_SAMPLE_DECODE] == 0, 'mlp_mode auto must render with the fused kernel'
    return got


@pytest.mark.parametrize('name', sorted(FUSED_CASES))
def test_fused_render_draws_the_restated_uniforms(name):
    case = FUSED_CASES[name]
    planes, dec, ro, rd, opts = _inputs(case)
    N, M = ro.shape[:2]
    S, Sf = opts['depth_resolution'], opts['depth_resolution_importance']
    k = case['seed']
    got = _fused(planes, dec, ro, rd, opts, k)
    seed = ph.drawn_seed(k)
    oracle_of = lambda u: _oracle(planes, dec, ro, rd, opts, {}, u)
    _check(f'fused {name}', got, oracle_of(ph.render_uniforms(seed, N, M, S, Sf)), TOL)
    _controls(f'fused {name}', got, oracle_of, _wrong_rules(seed, N, M, S, Sf), TOL)


@pytest.mark.parametrize('name', sorted(FUSED_CASES))
def test_fused_and_simt_draw_the_same_uniforms(name):
    """Under the same torch seed the fused and the SIMT kernels must draw identical uniforms, so their renders agree to
    the fused kernel's bar."""
    case = FUSED_CASES[name]
    planes, dec, ro, rd, opts = _inputs(case)
    k = case['seed'] + 1
    fused = _fused(planes, dec, ro, rd, opts, k)
    simt, prof = _render(planes, dec, ro, rd, opts, {}, 0, k)
    assert prof[PROF_FUSED] == 0 and prof[PROF_SAMPLE_DECODE] >= 1, prof
    _check(f'fused vs simt {name}', fused, simt, TOL)


def test_fused_headline_config_draws_the_restated_uniforms():
    """The benchmarked configuration (2 views x 128^2 rays, 96+96 samples, 512^2 planes) under its own noise source."""
    case = RENDER_CASES['headline96']
    planes, dec, ro, rd, opts = _inputs(case)
    N, M = ro.shape[:2]
    assert (N, M, opts['depth_resolution'], opts['depth_resolution_importance'], planes.shape[-1]) == (2, 128 * 128, 96, 96, 512)
    k = 1234
    got = _fused(planes, dec, ro, rd, opts, k)
    want = _oracle(planes, dec, ro, rd, opts, {}, ph.render_uniforms(ph.drawn_seed(k), N, M, 96, 96))
    _check('fused headline96', got, want, TOL)


def test_fused_late_laps_draw_their_own_rays():
    """n_groups = 4 * n_sm + r at 48+48: every CTA runs 4 or 5 ray groups of its persistent loop, and a group of a late
    lap (grp = blockIdx.x + n * gridDim.x) must draw the uniforms of its own global rays."""
    from tests.render_abi import box_rays, planes_and_decoder
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    S, k, N = 48, 4, 2
    GR = 384 // S
    groups = k * n_sm + 18
    M = groups * GR // N
    assert groups % N == 0 and 18 < n_sm and (groups + n_sm - 1) // n_sm == k + 1
    planes, dec = planes_and_decoder(460, N, 64, 64)
    ro, rd = box_rays(460, N, M)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=S)
    got = _fused(planes, dec, ro, rd, opts, 461)
    want = _oracle(planes, dec, ro, rd, opts, {}, ph.render_uniforms(ph.drawn_seed(461), N, M, S, S))
    _check(f'fused {groups} groups on {n_sm} SMs', got, want, TOL)


# ---------------------------------------------------------------------------------------------
# the training path: _RenderFunction = SIMT forward + p3d_render_backward, no injected noise
# ---------------------------------------------------------------------------------------------
def test_training_step_draws_the_restated_uniforms_forward_and_backward():
    case = _case(87, 48, 48)
    planes, dec, ro, rd, opts = _inputs(case)
    N, M = ro.shape[:2]
    rng = np.random.default_rng(case['seed'] + 5)
    gw = [torch.from_numpy(rng.standard_normal(s).astype(np.float32)) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
    k = case['seed']

    r = _renderer('auto')
    d = make_decoder(dec, DEV).requires_grad_(True)
    pg = planes.to(DEV).requires_grad_(True)
    torch.manual_seed(k)
    got_out, prof = profiled(lambda: r(pg, d, ro.to(DEV), rd.to(DEV), opts))
    assert prof[PROF_FUSED] == 0 and prof[PROF_SAMPLE_DECODE] >= 1, 'the autograd path renders with the SIMT kernels'
    assert all(o.requires_grad for o in got_out)
    got = torch.autograd.grad(sum((o * g_.to(DEV)).sum() for o, g_ in zip(got_out, gw)),
                              [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])

    seed = ph.drawn_seed(k)
    pl = planes.clone().requires_grad_(True)
    dref = {kk: (v.clone().requires_grad_(True) if isinstance(v, torch.Tensor) else v) for kk, v in dec.items()}
    out = _oracle(pl, dref, ro, rd, opts, {}, ph.render_uniforms(seed, N, M, 48, 48))
    ref = torch.autograd.grad(sum((o * g_).sum() for o, g_ in zip(out, gw)), [pl, dref['w1'], dref['b1'], dref['w2'], dref['b2']])

    _check('training forward', got_out, out, TIGHT)
    worst = 0.0
    for g_, r_, nm in zip(got, ref, ('planes', 'w1', 'b1', 'w2', 'b2')):
        assert g_.shape == r_.shape, nm
        err, bar = _max_err(g_, r_), GRAD_REL * max(1e-3, r_.abs().max().item())
        worst = max(worst, err / bar)
        assert err < bar, f'training grad {nm}: max abs err {err:.3e} (bar {bar:.3e})'
    print(f'PHILOX training gradients: worst error {worst:.4f} of the bar')
    with torch.no_grad():
        _controls('training forward', [o.detach() for o in got_out],
                  lambda u: _oracle(planes, dec, ro, rd, opts, {}, u), _wrong_rules(seed, N, M, 48, 48), TIGHT)


# ---------------------------------------------------------------------------------------------
# the host entry point: one view per launch, seed + v * 0x9E3779B97F4A7C15 per view, batch-wide depth clamp
# ---------------------------------------------------------------------------------------------
def test_host_entry_point_draws_a_stream_per_view():
    from panic3d_b200 import _lib
    case = _case(88, 48, 48, N=3)
    planes, dec, c2w, K, _u_c, _u_f, opts = build_case_inputs(case)
    ro, rd = case_rays(case, c2w, K)
    N, R, S, Sf = 3, case['R'], 48, 48
    M = R * R
    seed = 0xFFFFFFFF00000001            # upper key word set: a seed torch never draws (its top bit is always clear)
    p = _lib.RenderParams()
    p.n_views, p.n_rays, p.n_coarse, p.n_fine = N, M, S, Sf
    p.channels, p.plane_h, p.plane_w, p.hidden, p.out_dim = planes.shape[2], planes.shape[3], planes.shape[4], 64, 33
    p.box_warp = opts['box_warp']
    p.ray_mode, p.ray_start, p.ray_end = _lib.P3D_RAYS_NUMERIC, float(opts['ray_start']), float(opts['ray_end'])
    p.white_back, p.plane_mode = int(bool(opts['white_back'])), _lib.P3D_PLANES_PANIC3D
    fc1, fc2 = make_decoder(dec, 'cpu').net[::2]
    p.w1_gain, p.b1_gain, p.w2_gain, p.b2_gain = float(fc1.weight_gain), float(fc1.bias_gain), float(fc2.weight_gain), float(fc2.bias_gain)
    p.mlp_mode = _lib.P3D_MLP_FP32_SIMT
    p.seed = seed
    h = [t.detach().float().contiguous() for t in (planes, fc1.weight, fc1.bias, fc2.weight, fc2.bias, c2w.reshape(N, 16), K.reshape(N, 9))]
    got = [torch.empty(s, dtype=torch.float32) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
    L = _lib.lib()
    try:
        _, prof = profiled(lambda: _lib.check(L.p3d_render_forward_host(C.byref(p), *[t.data_ptr() for t in h], R, None, None,
                                                                      *[o.data_ptr() for o in got])))
    finally:
        L.p3d_host_arena_release()
    assert prof[PROF_FUSED] == 0 and prof[PROF_SAMPLE_DECODE] >= N, prof

    def oracle_of(view_seed):
        """Each view alone with its own uniforms (ray indices from 0), then the batch-wide depth clamp."""
        outs, lo, hi = [], [], []
        unbounded = (torch.tensor(-math.inf), torch.tensor(math.inf))
        for v in range(N):
            o, (a, b) = _oracle(planes[v:v + 1], dec, ro[v:v + 1], rd[v:v + 1], opts, {},
                                ph.render_uniforms(view_seed(v), 1, M, S, Sf), depth_bounds=unbounded, return_bounds=True)
            outs.append(o); lo.append(a); hi.append(b)
        cat = [torch.cat([o[i] for o in outs]) for i in range(4)]
        cat[1] = torch.clamp(cat[1], torch.stack(lo).min(), torch.stack(hi).max())
        return cat

    assert ph.host_view_seed(seed, 2) < seed                   # view 2's seed wraps modulo 2^64
    _check('host entry point', got, oracle_of(lambda v: ph.host_view_seed(seed, v)), TIGHT)
    _controls('host entry point', got, oracle_of, {'every view on the base seed': lambda v: seed}, TIGHT)


# ---------------------------------------------------------------------------------------------
# the seed contract of ImportanceRenderer: one draw from torch's CPU generator per render
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('grad', [False, True])
def test_each_render_draws_one_seed_from_the_torch_generator(grad):
    case = FUSED_CASES['fused48']
    planes, dec, ro, rd, opts = _inputs(case)
    r = _renderer('auto')
    d = make_decoder(dec, DEV).requires_grad_(grad)
    x, o, v = planes.to(DEV), ro.to(DEV), rd.to(DEV)

    def render(k):
        torch.manual_seed(k)
        with torch.set_grad_enabled(grad):
            out = [t.detach().cpu() for t in r(x, d, o, v, opts)]
        return out, int(torch.empty((), dtype=torch.int64).random_().item())

    a, after_a = render(7)
    b, _ = render(7)
    c, _ = render(8)
    for t, u, key in zip(a, b, KEYS):
        assert torch.equal(t, u), f'{key}: same torch seed, different render'
    assert not torch.equal(a[0], c[0]) and not torch.equal(a[2], c[2])
    torch.manual_seed(7)
    first, second = (int(torch.empty((), dtype=torch.int64).random_().item()) for _ in range(2))
    assert first == ph.drawn_seed(7) and after_a == second, 'a render must consume exactly one draw'
