"""GPU: the fused renderer (k_render_ws3, csrc/render_fused_ws3.cu) at the bench size, against the fp64 oracle with a bar
per ray and output component.

k_render_ws3 is the default kernel of ImportanceRenderer, smoke() and bench.py.  The other GPU files compare it with one
flat bar; here every call goes through the C ABI (p3d_render_forward, mlp_mode 1 or 2) with injected uniforms, NaN-filled
outputs and a NaN-filled workspace (its rgb_c / rgb_f buffers are the kernel's colour areas, so a colour tile read before
its bulk store lands, or from the wrong slice, turns into NaN).  Every call is made twice: exactly one launch in profile
slot 5 each, bit-identical results, no NaN anywhere (checked after the values, which a kernel reading memory it never
wrote can get wrong while still repeating itself).

Cases (each asserts the property it exists for):
  headline      2 views, 128^2 rays, 96+96, 512^2 planes: 62-63 groups per CTA on 132 SMs
  bench8        bench.py's batch, 8 views: 248-249 groups per CTA (the colour areas and col_full parities wrap many times);
                bars on every BENCH_STRIDE-th ray, NaN and repeat checks on every ray
  train48       4 views, 64^2, 48+48, 256^2: bench.py's training context
  eval_flags96  crop 0.1, cull 0.5, force_sigmoid, sigma bias centred on the cull: 20-50 % of the uncropped samples culled
  binarize48    binarize 0.5 + crop
  auto_eg3d     'auto' limits, EG3D plane order, black background, lr_mul 0.5, cameras at distance 2: some rays miss the
                box and take the batch-bound fallback
  ortho, disparity, shared_planes
  bf16_cl       bf16 (N,96,H,W) channels_last planes consumed zero-copy, against the oracle on the bf16-rounded planes
  n_my_1/2/3    fewer groups than SMs, then exactly 2 and 3 groups on the deepest CTA
  all_miss48/96 'auto' limits, every ray of the call misses the box: bounds[4] == 0 and the coarse depths descend (t0 = -1,
                t1 = -2); sigma bias -4 keeps every ray's importance pdf positive, so every ray is compared
  all_miss_negpdf48  all_miss48 without that bias: every ray's pdf is non-positive somewhere (see below)
  descending96  numeric ray_start 1.5 > ray_end 0.5: descending coarse depths
  single_pass   mlp_mode 2 against its own bars, and >= 10x mode 1's error
  saturated48, dense48  the negative controls' cases (CONTROL_CASES)
The descending cases are also checked against the fp32 SIMT kernel (mlp_mode 0) at its 1e-4 bar.

Reference: oracle/renderer_oracle.py in float64 on the device, a view and CHUNK rays at a time (its depth clamp is applied
with the batch's bounds afterwards).  test_gpu_fp64_oracle_equals_cpu_oracle pins that run to the CPU fp32 oracle on the
config1 and mid_eval96 fixtures.

Bars.  The kernel's error is bounded per sample and propagated to first order through the oracle:
  * per sample: the decoder's sigma and colour bars (tests/render_abi.py: three_pass_bars for mode 1,
    single_pass_bars for mode 2; test_three_pass_bars_hold_on_the_decode checks the first on p3d_decode_points at the
    oracle's own sample positions), plus the point's fp32 rounding (ray_point, the grid transform: 4 v (|o| + |t d| + box)
    per coordinate, v = 2^-24) times the one-sided finite-difference slopes of sigma and colour;
  * per depth: coarse 16 v (|t| + |t0| + |t1|); fine 8 v (|t| + |t1 - t0|) for the lerp, and (2 S + 40) v on every cdf
    entry (fp32 weights, their sum, the division and the scans);
  * per interval alpha = 1 - ex2.approx(-log2(e) softplus(smid) dt): 2^-22 (1 - alpha) + v alpha + (1 - alpha) (dt (4
    2^-22 softplus + 2 2^-22 + sigmoid(smid) v (|s_a| + |s_b| + 2)) + 6 v softplus dt), in both marches.
  The oracle's render is restated as a graph of these perturbations (zero-valued leaves: `render_abi.render_graph`, built by
  `render_abi.ray_oracle` with this kernel's rounding model `render_abi.FUSED_MODE1` / `FUSED_MODE2`): the coarse
  sigma / colour / depth perturbations move the coarse weights, the importance depths (kept differentiable) and, through
  each fine sample's slope along its ray, the fine sigma and colour.  For each output component o_k of a ray (32 rgb,
  depth, wsum, 3 xyz), one vector-Jacobian product per component over a chunk of rays (rays are independent) gives
      bar_k = 2 (sum over leaves |do_k / d leaf| beta_leaf) + floor_k
  floor_k covers the roundings of the sums that form the output ((L + 8) v relative on each weight and on every partial
  sum; L = S + Sf).  The factor 2 covers second-order terms: every leaf's relative size is <= ~1e-4, so products of two
  perturbations are below 1e-4 of the first-order sum.
  The merge of two samples whose depths are within rounding of each other may order them either way; the outputs change by
  less than the slopes times the depth bar, since both samples sit at the same point.
Masks: a cull, binarize or crop decision is a jump.  A ray is excluded when one of its samples' fp64 sigma lies within its
sigma bar (plus the rounding of the host's sigma_cull) of the threshold, or its |x| / |z| within the position bar of the
crop bound; the excluded rays are counted and bounded (EXCLUDE_SHARE).  Rays whose W is 0 in either run (every sample
masked) compare their depth with the batch's largest depth.

Negative controls: the oracle with the colour map s - 0.001 instead of 1.002 s - 0.001 (on saturated48, whose colours sit
near 1, where the gain matters most and the decoder's colour error, scaled by s (1 - s), least), with the importance pdf
floor 0.005 and with omega = w_i instead of (w_{i-1} + w_i) / 2 (both on dense48, whose weight sits on a few intervals).
Each must miss the kernel by >= 20x the bar somewhere.

Descending coarse depths make negative weights.  Where the importance pdf they give is non-positive, the cdf is not
monotone and the reference's own fine depths depend on the probe order of its searchsorted; such rays are counted and not
compared.  Only all_miss_negpdf48 has any (all of them; it keeps the determinism, NaN and limit checks); every other case
asserts that it has none.

Run with -s for the worst error / bar of every case and output, the excluded rays, runtime and peak device memory.
"""
import ctypes as C
import functools
import time

import pytest
import torch

from oracle import renderer_oracle as orc
from tests import render_abi as ra
from tests.render_abi import (BW, DEV, OUTPUTS, U32, Worst, cull_sigma, dec64, decode_points, make_decoder, n_sm,
                              three_pass_bars)

pytestmark = pytest.mark.gpu
PROF_FUSED = 5                    # profile slot of k_render_ws3 (csrc/p3d_common.cuh)
CHUNK = 1024                      # rays per oracle call
BENCH_STRIDE = 16
SIMT_BAR = 1e-4                   # the SIMT kernel against the oracle (tests/test_render_gpu.py)
EXCLUDE_SHARE = {1: 0.01, 2: 0.05}
# The mask cases exclude far more rays: a fine sample's band is its sigma slope along the ray times the bound of how far its
# depth may move, which is loose (see DESIGN.md section 2).  Measured on an H100: eval_flags96 92 %, binarize48 25 %.
EXCLUDE_SHARE_MASKS = {'eval_flags96': 0.95, 'binarize48': 0.35}
PIN = 2e-6                        # fp64 device oracle vs the CPU fp32 one: the fp32 run's rounding (measured 7.6e-7)
FREE_BYTES = 12 << 30             # the 512^2 cases: measured peak 8.1 GB (bench8), with margin
OUT_COLS = dict(rgb=slice(0, 32), depth=slice(32, 33), wsum=slice(33, 34), xyz=slice(34, 37))
AUTO = dict(ray_start='auto', ray_end='auto')

CASES = {
    'headline': dict(N=2, R=128, S=96, P=512, per_cta=(62, 63)),
    'bench8': dict(N=8, R=128, S=96, P=512, per_cta=(248, 249), stride=BENCH_STRIDE),
    'train48': dict(N=4, R=64, S=48, P=256),
    'eval_flags96': dict(N=1, R=64, S=96, P=256, flags=dict(triplane_crop=0.1, cull_clouds=0.5), force_sigmoid=True,
                         centre_cull=0.5, quantile=0.35),
    'binarize48': dict(N=2, R=32, S=48, P=64, flags=dict(triplane_crop=0.1, binarize_clouds=0.5), centre_cull=0.5),
    'auto_eg3d': dict(N=2, R=32, S=48, P=64, opts=dict(AUTO, white_back=False), eg3d=True, lr_mul=0.5, dist=2.0),
    'ortho': dict(N=1, R=64, S=96, P=128, rays='ortho'),
    'disparity': dict(N=2, R=32, S=48, P=64, opts=dict(disparity_space_sampling=True)),
    'shared_planes': dict(N=3, R=32, S=96, P=64, shared=True),
    'bf16_cl': dict(N=2, R=64, S=96, P=128, bf16=True),
    'n_my_1': dict(N=1, R=8, S=96, P=64, groups=lambda sms: 16),
    'n_my_2': dict(N=1, R=64, S=96, P=64, groups=lambda sms: sms + 5),
    'n_my_3': dict(N=1, R=64, S=48, P=64, groups=lambda sms: 2 * sms + 7),
    'all_miss48': dict(N=2, R=32, S=48, P=64, rays='miss', opts=dict(AUTO), sigma_bias=-4.0),
    'all_miss96': dict(N=1, R=32, S=96, P=64, rays='miss', opts=dict(AUTO), sigma_bias=-4.0),
    'all_miss_negpdf48': dict(N=2, R=32, S=48, P=64, rays='miss', opts=dict(AUTO), seed_as='all_miss48'),
    'descending96': dict(N=2, R=32, S=96, P=64, opts=dict(ray_start=1.5, ray_end=0.5)),
    'single_pass': dict(N=1, R=64, S=96, P=128, mode=2),
    # negative-control cases: colours saturated near 1 (the colour map's gain is all that separates s - 0.001 from the
    # kernel, and the decoder's colour error is scaled by s (1 - s)), and a dense case (weight on a few intervals, so
    # omega's neighbour and the pdf floor move the outputs far more than the bars)
    'saturated48': dict(N=1, R=32, S=48, P=64, colour_bias=8.0),
    'dense48': dict(N=1, R=32, S=48, P=64, sigma_bias=8.0),
}
# input seed of a case: 1300 + its index here (cases added later go at the end, so no other case's inputs change)
SEEDS = sorted(['headline', 'bench8', 'train48', 'eval_flags96', 'binarize48', 'auto_eg3d', 'ortho', 'disparity', 'shared_planes',
                'bf16_cl', 'n_my_1', 'n_my_2', 'n_my_3', 'all_miss48', 'all_miss96', 'descending96', 'single_pass']) + ['saturated48', 'dense48']
DESCENDING = ('all_miss48', 'all_miss96', 'all_miss_negpdf48', 'descending96')
# the one case whose importance pdf is non-positive on every ray (see _chunk): checked for determinism, no NaN and its
# limits, not against the oracle
NEGATIVE_PDF = ('all_miss_negpdf48',)


def _per_cta(n_groups, sms):
    """render_fused_ws3.cu: grid = min(n_groups, n_sm), CTA b runs ceil((n_groups - b) / grid) groups."""
    grid = min(n_groups, sms)
    return [(n_groups - b + grid - 1) // grid for b in range(grid)]


# ------------------------------------------------------------------------------------------------- inputs
def _rays(case, N, R):
    kind = case.get('rays', 'spin')
    if kind == 'ortho':
        ro, rd = zip(*(orc.rays_ortho(20.0, -135.0 + 40 * n, 1.0, BW, R) for n in range(N)))
        f = lambda t: torch.cat(t).permute(0, 2, 3, 1).reshape(N, R * R, 3)
        return f(ro).to(DEV).contiguous(), f(rd).to(DEV).contiguous()
    if kind == 'miss':
        # origins at x in [0.4, 0.6], beyond the box's half side 0.35, directions with no x component: every ray misses the
        # box, yet the points at t in [-2, -1] ('auto' limits of a miss) project inside the (y, z) plane for many samples
        g = torch.Generator().manual_seed(7)
        a, b = torch.rand(N, R * R, generator=g), torch.rand(N, R * R, generator=g)
        ro = torch.stack([0.4 + 0.2 * a, 0.4 * b - 0.2, torch.full_like(a, 1.0)], -1)
        rd = torch.nn.functional.normalize(torch.stack([torch.zeros_like(a), 0.3 * (b - 0.5), torch.ones_like(a)], -1), dim=-1)
        return ro.to(DEV).contiguous(), rd.to(DEV).contiguous()
    return ra.rays_at(ra.spin12(N), R, case.get('dist', 1.0))


@functools.lru_cache(maxsize=None)
def _inputs(name):
    case = CASES[name]
    N, R, S, P = (case[k] for k in ('N', 'R', 'S', 'P'))
    seed = 1300 + SEEDS.index(case.get('seed_as', name))
    g = torch.Generator().manual_seed(seed)
    planes = torch.randn(1 if case.get('shared') else N, 3, 32, P, P, generator=g)
    if case.get('shared'):
        planes = planes.expand(N, -1, -1, -1, -1)
    if case.get('bf16'):
        planes = planes.bfloat16().float()
    _, dec, *_ = orc.synth_inputs(seed, 1, 1, 2, 0, 2)
    dec = dict(dec, lr_mul=case.get('lr_mul', 1.0), force_sigmoid=case.get('force_sigmoid', False), b2=dec['b2'].clone())
    dec['b2'][0] += case.get('sigma_bias', 0.0)
    dec['b2'][1:] += case.get('colour_bias', 0.0)
    opts = dict(dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=S), **case.get('opts', {}))
    ro, rd = _rays(case, N, R)
    if case.get('groups'):
        M = case['groups'](n_sm()) * (384 // S)
        assert M <= R * R
        ro, rd = ro[:, :M].contiguous(), rd[:, :M].contiguous()
    M = ro.shape[1]
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, S, generator=g)
    if case.get('centre_cull'):                     # median coarse sigma on the cull threshold
        d_c = orc.stratified_depths(u_c.to(DEV), opts['ray_start'], opts['ray_end'])
        xyz = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)[:, ::7]
        _, sig = orc.run_model(planes.to(DEV, torch.float64), dec64(dec), xyz, opts, not case.get('eg3d'))
        dec['b2'][0] += cull_sigma(case['centre_cull']) - sig.quantile(case.get('quantile', 0.5)).item()
    return planes, dec, opts, ro, rd, u_c.to(DEV).contiguous(), u_f.to(DEV).contiguous()


# ------------------------------------------------------------------------------------------------- the kernel, through the C ABI
def _kernel(name, mode=None, checks_later=False):
    """p3d_render_forward twice into NaN-filled outputs and workspace: one launch in slot 5 each, bit-identical, no NaN.
    Returns (rgb, depth, wsum, xyz), the workspace bounds words; with checks_later, the checks of the two runs are left to
    the caller (ra.repeats), which makes them after comparing the values."""
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = CASES[name]
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    mode = case.get('mode', 1) if mode is None else mode
    N, M = ro.shape[:2]
    r = ImportanceRenderer(use_triplane=not case.get('eg3d'))
    r.planes_bf16 = bool(case.get('bf16'))
    r.mlp_mode = mode
    decoder = make_decoder(dec, DEV)
    with torch.no_grad(), torch.cuda.device(DEV):
        if case.get('bf16'):               # a (N,96,H,W) channels_last backbone output, consumed zero-copy
            n, p_, c, h, w = planes.shape
            x = planes.to(DEV, torch.bfloat16).reshape(n, p_ * c, h, w).contiguous(memory_format=torch.channels_last)
            cl = r._planes_cl(x.view(n, p_, c, h, w))
            assert cl.data_ptr() == x.data_ptr(), 'bf16 channels_last planes were copied'
        else:
            cl = r._planes_cl(planes.to(DEV))
        fl = case.get('flags', {})
        p, wts = r._params(cl, N, M, opts, decoder, fl.get('triplane_crop'), fl.get('cull_clouds'), fl.get('binarize_clouds'))
        assert p.mlp_mode == mode
        p.defer_depth_clamp = 0
        wt = [t.detach().float().contiguous() for t in wts]
        ws = torch.empty(int(_lib.lib().p3d_render_workspace_bytes(C.byref(p))), dtype=torch.uint8, device=DEV)
        out = [torch.empty(s, device=DEV) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
        first, second = ra.twice(lambda: ra.render_forward(p, cl, wt, ro, rd, u_c, u_f, ws, out),
                                 out + [ws[:64].view(torch.int32)], PROF_FUSED if mode != 0 else None, [ws], checks_later=True)
        if checks_later:
            return first[:4], first[4], second[:4]
        ra.repeats(first[:4], second[:4], OUTPUTS, nan=True)
        return first[:4], first[4]


# ------------------------------------------------------------------------------------------------- oracle and bars
def _limits(name):
    """Per-ray coarse limits (N,M,1) fp64 as oracle.render forms them."""
    case = CASES[name]
    _, _, opts, ro, rd, *_ = _inputs(name)
    if opts['ray_start'] == 'auto':
        t0, t1 = orc.ray_limits_box(ro.double(), rd.double(), BW)
        ok = t1 > t0
        if bool(ok.any()):
            t0 = torch.where(ok, t0, t0[ok].min())
            t1 = torch.where(ok, t1, t0[ok].max())
        return t0, t1
    full = lambda v: torch.full(ro.shape[:2] + (1,), float(v), device=DEV, dtype=torch.float64)
    return full(opts['ray_start']), full(opts['ray_end'])


def _chunk(name, v, sl, mode, with_bars=True, controls=False):
    """The oracle's outputs (m, 37) for rays `sl` of view v, and (with_bars) their bars (m, 37), the rays to exclude (m,)
    and the mutated oracles' outputs (controls): ra.ray_oracle with the fused kernel's rounding model."""
    case = CASES[name]
    planes, dec, opts, ro_all, rd_all, u_c_all, u_f_all = _inputs(name)
    M = ro_all.shape[1]
    ro, rd = ro_all[v, sl].double(), rd_all[v, sl].double()
    m = ro.shape[0]
    u_c = u_c_all[v, sl].double()
    u_f = u_f_all[v * M:(v + 1) * M][sl].double()
    t0, t1 = (t[v, sl] for t in _limits(name))
    if opts['ray_start'] == 'auto':
        d_c = orc.stratified_depths(u_c[None], t0[None], t1[None])[0]
    else:
        d_c = orc.stratified_depths(u_c[None], opts['ray_start'], opts['ray_end'], opts.get('disparity_space_sampling', False))[0]
    tri = not case.get('eg3d')
    if mode == 2:
        assert tri and not dec['force_sigmoid']
    p64 = planes[v:v + 1].to(DEV, torch.float64)
    res, ctx = ra.ray_oracle(ra.FUSED_MODE1 if mode == 1 else ra.FUSED_MODE2, p64, dec64(dec), opts, case.get('flags', {}), tri,
                             ro, rd, d_c, t0, t1, u_f, case['S'], with_bars=with_bars)
    if controls:
        c0, f0, w, zero, white, samples = (ctx[k] for k in ('c0', 'f0', 'w', 'zero', 'white', 'samples'))
        # the colour map without its gain: s - 0.001 instead of 1.002 s - 0.001
        dec_s = dec64(dict(dec, force_sigmoid=True))
        rgb_s = lambda smp: orc.run_model(p64, dec_s, smp['xyz'].reshape(1, -1, 3), opts, tri)[0].reshape(m, -1, 32) - 0.001
        c0s, f0s = dict(c0, rgb=rgb_s(c0)), dict(f0, rgb=rgb_s(f0))
        res['ctl_colour_map'] = ra.render_graph(ro, rd, d_c, u_f, c0s, f0s, white, zero)[0]
        # the pdf floor moves the fine depths: decode at the moved depths
        floor5 = functools.partial(orc.importance_depths, floor=0.005)
        f5 = samples(floor5(d_c[..., 0], w, u_f)[..., None])
        res['ctl_pdf_floor'] = ra.render_graph(ro, rd, d_c, u_f, c0, f5, white, zero, importance=floor5)[0]
        res['ctl_omega'] = ra.render_graph(ro, rd, d_c, u_f, c0, f0, white, zero, left=True)[0]
    return res


def _rays_of(name):
    case = CASES[name]
    M = _inputs(name)[3].shape[1]
    idx = torch.arange(0, M, case.get('stride', 1), device=DEV)
    return [(v, idx[i:i + CHUNK]) for v in range(case['N']) for i in range(0, idx.numel(), CHUNK)]


def _flat(out, v, sl):
    rgb, depth, wsum, xyz = out
    return torch.cat([rgb[v, sl], depth[v, sl], wsum[v, sl], xyz[v, sl]], -1)


def _compare(name, out, mode, controls=()):
    """The kernel's outputs against the oracle's, ray by ray.  Returns the worst abs errors, ratios and control ratios."""
    res_all = [(v, sl, _chunk(name, v, sl, mode, controls=bool(controls))) for v, sl in _rays_of(name)]
    t_hi = max(r['t_max'].item() for *_, r in res_all)
    worst = {key: Worst() for key in OUTPUTS}
    n_near = n_total = n_ill = 0
    ctl = {c: 0.0 for c in controls}
    cull = [0, 0]
    for v, sl, r in res_all:
        got = _flat(out, v, sl)
        want, bar = r['o'].clone(), r['bar'].clone()
        dead = (want[:, 33] == 0) | (got[:, 33] == 0)
        want[dead, 32] = t_hi                                  # nan_to_num(inf) then the clamp to the batch's largest depth
        bar[dead, 32] = 64 * U32 * abs(t_hi)
        keep = ~r['near'] & ~r['illdef']
        n_ill += r['illdef'].sum().item()
        if keep.any():
            for key, cols in OUT_COLS.items():
                worst[key].add(got[keep][:, cols], want[keep][:, cols], bar[keep][:, cols])
        n_near += r['near'].sum().item()
        n_total += r['near'].numel()
        for c in controls:
            err = (got.double() - r[c]).abs()[keep]
            cols = slice(0, 32) if c != 'ctl_pdf_floor' else slice(0, 37)
            if err.shape[0]:
                ctl[c] = max(ctl[c], (err[:, cols] / bar[keep][:, cols]).max().item())
        if r['cull_share']:
            cull[0] += r['cull_share'][0]
            cull[1] += r['cull_share'][1]
    for key in OUTPUTS:
        print(f'{name} mode {mode} {key}: max abs err {worst[key].err:.3e}, worst err / bar {worst[key].ratio:.4f}')
    print(f'{name}: {n_near} of {n_total} rays excluded (a sample within its bar of a mask threshold), {n_ill} with a '
          f'non-positive importance pdf')
    if name in NEGATIVE_PDF:
        assert n_ill == n_total, (name, n_ill, n_total)
    else:
        assert n_ill == 0, (name, n_ill)
    return worst, n_near / max(n_total, 1), ctl, cull


# ------------------------------------------------------------------------------------------------- tests
def test_gpu_fp64_oracle_equals_cpu_oracle():
    """oracle.render in fp64 on the device equals the CPU fp32 oracle that the reference fixtures pin (config1,
    mid_eval96) within the fp32 run's rounding.  The device run takes the CPU run's depths and mask decisions (as
    test_render_backward_paths_gpu does): a cull decision within fp32 rounding of its threshold would otherwise move a whole
    sample, and how the CPU's fp32 sums round depends on the host's thread count."""
    from tests.golden.cases import RENDER_CASES, build_case_inputs
    from tests.helpers import case_rays
    for fixture in ('config1', 'mid_eval96'):
        case = RENDER_CASES[fixture]
        planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
        ro, rd = case_rays(case, c2w, K)
        fl = {k: case[k] for k in ('triplane_crop', 'cull_clouds', 'binarize_clouds') if case.get(k)}
        cpu, smp = orc.render(planes, dec, ro, rd, opts, u_c, u_f, return_samples=True, **fl)
        to = lambda t: None if t is None else t.to(DEV)
        gpu = orc.render(planes.to(DEV, torch.float64), dec64(dec), ro.to(DEV), rd.to(DEV), opts, None, None,
                         depths=tuple(to(t) for t in smp['depths']), masks=tuple(to(t) for t in smp['masks']), **fl)
        for key, a, b in zip(OUTPUTS, gpu, cpu):
            assert a.dtype == torch.float64
            err = (a.cpu() - b.double()).abs().max().item()
            print(f'pin {fixture} {key}: {err:.2e}')
            assert err <= PIN, (fixture, key, err)


@pytest.mark.parametrize('name', list(CASES))
def test_render_graph_is_the_oracle(name):
    """_chunk's zero-leaf graph gives oracle.render's fp64 outputs, with every case's masks, limits, plane order and
    background, so the bars are derivatives of the oracle the kernel is compared with.  'auto' cases pass render the
    whole batch (its fallback limits are reduced over the batch); the others the first 256 rays of view 0.  depth is
    compared where W > 0 (render clamps the others to its batch's largest depth)."""
    case = CASES[name]
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    N, M = ro.shape[:2]
    n = M if opts['ray_start'] == 'auto' else min(256, M)
    views = range(N) if opts['ray_start'] == 'auto' else range(1)
    fl = case.get('flags', {})
    want = orc.render(planes[:len(views)].to(DEV, torch.float64), dec64(dec), ro[:len(views), :n].double(), rd[:len(views), :n].double(),
                      opts, u_c[:len(views), :n].double(), u_f.view(N, M, -1)[:len(views), :n].reshape(len(views) * n, -1).double(),
                      use_triplane=not case.get('eg3d'), **fl)
    worst = dict.fromkeys(OUTPUTS, 0.0)
    for v in views:
        for i in range(0, n, CHUNK):
            sl = torch.arange(i, min(i + CHUNK, n), device=DEV)
            got = _chunk(name, v, sl, 1, with_bars=False)['o']
            ref = _flat(want, v, sl)
            live = ref[:, 33] > 0
            for key, a_, b_ in zip(OUTPUTS, ref.split([32, 1, 1, 3], -1), got.split([32, 1, 1, 3], -1)):
                if key == 'depth':
                    a_, b_ = a_[live], b_[live]
                worst[key] = max(worst[key], (a_ - b_).abs().max().item() if a_.numel() else 0.0)
    print(f'{name} graph vs render: ' + ', '.join(f'{k} {e:.1e}' for k, e in worst.items()))
    assert max(worst.values()) <= 1e-12, (name, worst)


def test_three_pass_bars_hold_on_the_decode():
    """The per-sample mode 1 bar (three_pass_bars) holds on p3d_decode_points (the same decoder code, fused_common.cuh) at
    the oracle's own coarse and fine sample positions of train48's first view."""
    name = 'train48'
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    n = 1024
    p64, d64 = planes[:1].to(DEV, torch.float64), dec64(dec)
    _, smp = orc.render(p64, d64, ro[:1, :n].double(), rd[:1, :n].double(), opts, u_c[:1, :n].double(), u_f[:n].double(),
                        return_samples=True)
    pts = [(ro[:1, :n, None].double() + d * rd[:1, :n, None].double()).reshape(1, -1, 3) for d in smp['depths']]
    xyz = torch.cat(pts, 1).float()
    x64 = xyz.double()
    rgb, sig = orc.run_model(p64, d64, x64, opts, True)
    b_rgb, b_sig = three_pass_bars(p64, d64, x64)
    k_rgb, k_sig = decode_points(planes[:1].to(DEV), dec, xyz, 1)
    for key, k, w, b in (('rgb', k_rgb, rgb, b_rgb), ('sigma', k_sig, sig, b_sig)):
        err = (k.double() - w).abs().nan_to_num(nan=float('inf'))
        print(f'decode at the render samples {key}: max abs err {err.max().item():.3e}, worst err / bar {(err / b).max().item():.4f}, '
              f'median bar {b.median().item():.2e}')
        assert (err / b).max().item() <= 1.0, key


CONTROLS = {'ctl_colour_map': 'colour map s - 0.001 instead of 1.002 s - 0.001', 'ctl_pdf_floor': 'importance pdf floor 0.005',
            'ctl_omega': 'omega = w_i'}
# control -> the case it must miss the kernel by >= 20x the bar on (every control is computed and printed on each)
CONTROL_CASES = {'ctl_colour_map': 'saturated48', 'ctl_pdf_floor': 'dense48', 'ctl_omega': 'dense48'}
CONTROL_MIN = 20.0


def _case_checks(name, out, bounds):
    case = CASES[name]
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    N, M = ro.shape[:2]
    S = case['S']
    groups = N * M // (384 // S)
    per = _per_cta(groups, n_sm())
    if case.get('per_cta'):
        assert (min(per), max(per)) == case['per_cta'], (name, min(per), max(per))
    if name == 'n_my_1':
        assert groups < n_sm() and max(per) == 1
    if name == 'n_my_2':
        assert max(per) == 2, per
    if name == 'n_my_3':
        assert max(per) == 3, per
    if name in ('all_miss48', 'all_miss96', 'all_miss_negpdf48'):
        assert bounds[4].item() == 0, 'a ray hit the box'
        t0, t1 = _limits(name)
        assert (t1 < t0).all(), 'coarse depths do not descend'
    if name == 'descending96':
        assert opts['ray_start'] > opts['ray_end']
    if name == 'saturated48':
        assert (out[0] > 0.99).double().mean().item() > 0.9, 'colours are not saturated'
    if name == 'auto_eg3d':
        t0, t1 = orc.ray_limits_box(ro.double(), rd.double(), BW)
        miss = (t1 <= t0).double().mean().item()
        print(f'auto_eg3d: {miss:.3f} of the rays miss the box')
        assert 0.01 < miss < 0.9, miss
    print(f'{name}: {groups} groups, {min(per)}-{max(per)} per CTA')


@pytest.mark.parametrize('name', [n for n in CASES if n != 'single_pass'])
def test_fused_matches_fp64_oracle(name):
    case = CASES[name]
    if case['P'] >= 512:
        free, _ = torch.cuda.mem_get_info()
        if free < FREE_BYTES:
            pytest.skip(f'needs {FREE_BYTES >> 30} GB of free device memory')
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    # the values first: a kernel that reads memory it never wrote may still repeat itself
    out, bounds, again = _kernel(name, checks_later=True)
    _case_checks(name, out, bounds)
    controls = tuple(CONTROLS) if name in CONTROL_CASES.values() else ()
    worst, share, ctl, cull = _compare(name, out, 1, controls)
    if cull[1]:
        print(f'{name}: cull removes {cull[0] / cull[1]:.3f} of the uncropped coarse samples')
        if name == 'eval_flags96':
            assert 0.2 <= cull[0] / cull[1] <= 0.5, cull
    for c, r in ctl.items():
        print(f'negative control "{CONTROLS[c]}" on {name}: worst err / bar {r:.1f}')
    print(f'{name}: {time.time() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB')
    assert share <= EXCLUDE_SHARE_MASKS.get(name, EXCLUDE_SHARE[1]), share
    assert max(w.ratio for w in worst.values()) <= 1.0, (name, {k: w.ratio for k, w in worst.items()})
    ra.repeats(out, again, OUTPUTS, nan=True)
    for c, r in ctl.items():
        if CONTROL_CASES[c] == name:
            assert r >= CONTROL_MIN, (CONTROLS[c], r)
    if name in DESCENDING:                 # the SIMT kernel sorts after mapping: the same outputs at its own bar
        simt, _ = _kernel(name, mode=0)
        for key, a, b in zip(OUTPUTS, simt, out):
            err = (a - b).abs().max().item()
            print(f'{name} SIMT vs fused {key}: {err:.3e}')
        for v, sl in _rays_of(name):
            r = _chunk(name, v, sl, 1, with_bars=False)
            if name in NEGATIVE_PDF:
                continue
            err = (_flat(simt, v, sl).double() - r['o']).abs().max().item()
            assert err <= SIMT_BAR, (name, 'SIMT', err)


def test_single_pass_matches_fp64_oracle():
    """mlp_mode 2 within its propagated bars, and >= 10x further from the oracle than mode 1."""
    name = 'single_pass'
    two, _ = _kernel(name, mode=2)
    one, _ = _kernel(name, mode=1)
    w2, share2, *_ = _compare(name, two, 2)
    w1, share1, *_ = _compare(name, one, 1)
    assert share2 <= EXCLUDE_SHARE[2] and share1 <= EXCLUDE_SHARE[1]
    assert max(w.ratio for w in w2.values()) <= 1.0 and max(w.ratio for w in w1.values()) <= 1.0
    for key in ('rgb', 'wsum'):
        assert w2[key].err >= 10 * w1[key].err, ('single pass is not reaching the kernel', key, w2[key].err, w1[key].err)
