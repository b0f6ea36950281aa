"""GPU: the fp32 SIMT renderer (render_forward_v1, csrc/render_v1.cu) at the training size and across the sample counts it
accepts, against the fp64 oracle drawing its own coarse and fine depths, with a bar per ray and output component.

render_forward_v1 (k_ray_limits, the coarse k_sample_decode, k_ray_importance, the fine k_sample_decode, k_ray_composite,
k_depth_finalize) is the forward of every training step (ImportanceRenderer.forward under autograd renders in
P3D_MLP_FP32_SIMT) and renders every configuration the fused kernel rejects.  Every call goes through the C ABI
(p3d_render_forward, mlp_mode 0) into NaN-filled outputs and a NaN-filled workspace, twice: per run 2 launches in profile
slot 0 (1 without a fine pass), 1 in slot 1 (0 without), 1 in slot 2 and none in slot 5 (the fused kernel); both runs
bit-identical, no NaN in the outputs, the coarse and fine depths or the sample values.  Uniforms are injected, except in
ragged_m, which draws them in the kernel (Philox) and hands the oracle the restated ones (oracle/philox.py).

Cases (each asserts from its data the property it exists for):
  train         4 views, 64^2 rays, 48+48, 256^2 planes, spin12 cameras: the forward of every training step
  train_cull    train with crop 0.1 and cull 0.5, sigma centred on the cull: rays with a sample within its bar of a mask
                threshold are excluded and counted; some rays have every sample masked (W = 0, depth NaN before
                k_depth_finalize)
  eval96        2 views, 128^2 rays, 96+96, 512^2 planes in mode 0: the parity kernel bench.py times
  s256_sf256    S + Sf = 512: the last chunk of importance_ray's my[8] holds live bins (nb = 253) and all 16 om[] chunks of
                composite_weights are live (L = 512)
  s4_sf508      sort_pow2 = 512 and a single pdf bin
  s33_sf33, s97_sf257  Sf just above a power of two: 31 / 255 +inf pads sort last and never reach the composite
  s4_sf1, s2_sf0, s192_sf192  the smallest sizes (one fine sample; no importance pass) and gen_videos' doubled sampling
  ragged_m      3 views of 61 rays: R % 4 == 3, so the last warp of the last block of the per-ray kernels idles
  auto_axis     'auto' limits, ortho cameras at elevation 0 and azimuth 0 / 90 / 180 (direction components +0 and -0),
                origins exactly on a box face (0 * inf = NaN limits: the reference, and since this file the kernel, render
                such a ray with the batch's fallback limits), origins inside the box, a ray through a box edge; the kernel's
                limits equal math_utils.get_ray_limits_box's on the same fp32 rays bit for bit
  auto_nohit    auto_axis's face-lying rays alone: every limit pair is NaN or a miss, the batch has no fallback, and each
                NaN ray takes the miss limits (-1, -2) (the kernel's one deviation from the reference, which renders NaN:
                NaN depths would break the rank merge); forward and backward
  disparity, descending  disparity sampling; numeric ray_start 1.5 > ray_end 0.5
  bf16          bf16 channels_last planes, against the oracle on the rounded planes
  dense         the negative controls' case (sigma bias 8: the weight sits on a few intervals)

Reference: oracle/renderer_oracle.py in float64 on the device, a view and CHUNK rays at a time, with its own coarse and fine
depths; bars from tests/render_abi.ray_oracle with the SIMT rounding model render_abi.SIMT (per-sample decoder bar
simt_bars, expf / log1pf alpha, simt_cdf on the importance cdf).  test_simt_bars_hold_on_the_decode checks the per-sample
bar on p3d_decode_points in mode 0.  The importance depths are also pinned directly: per ray, the kernel's sorted fine depths
lie within the largest of that ray's fine-depth bars of the oracle's sorted ones.

Negative controls (CONTROLS): the oracle's importance sampler without the 0.01 pdf floor, with bin edges at the coarse depths
t[below] / t[above] instead of the interval midpoints, and with the max-pool of the weights shifted by one bin.  Each must
miss the kernel by >= 20x its bar.

test_backward_at_the_envelope_edge runs p3d_render_backward after this forward at (256, 256) and (200, 200) (more than
48 KB of shared memory per k_ray_backward CTA: the opt-in path), (4, 1) and (2, 0), against render_backward_oracle with the
per-element bars of render_abi, for one upstream of all four outputs and bench.py's loss; and after auto_nohit's forward.

Run with -s for the worst error / bar of every comparison, the excluded rays, every control's miss, runtime and peak memory.
"""
import ctypes as C
import functools
import time
import zlib

import pytest
import torch
import torch.nn.functional as F

from oracle import philox as ph, renderer_oracle as orc
from tests import render_abi as ra
from tests.helpers import profiled
from tests.render_abi import BW, DEV, OUTPUTS, U32, Worst, cull_sigma, dec64, make_decoder

pytestmark = pytest.mark.gpu
CHUNK = 1024                      # rays per oracle call
PROF = (0, 1, 2, 5)               # profile slots: sample decode, importance, composite, fused (csrc/p3d_common.cuh)
PHILOX_SEED = 0x5eed5eed12345678
EXCLUDE_SHARE = 0.01
# the cull case excludes far more rays: a fine sample's band is its sigma slope along the ray times the bound of how far its
# depth may move, which is loose.  Measured on an H100: 45 %
EXCLUDE_SHARE_MASKS = {'train_cull': 0.6}
FREE_BYTES = 12 << 30
OUT_COLS = dict(rgb=slice(0, 32), depth=slice(32, 33), wsum=slice(33, 34), xyz=slice(34, 37))
AUTO = dict(ray_start='auto', ray_end='auto')

# small cases first: a mutation run stops at the first failing test
CASES = {
    's2_sf0': dict(N=2, R=8, S=2, Sf=0, P=64),
    's4_sf1': dict(N=2, R=8, S=4, Sf=1, P=64),
    's33_sf33': dict(N=2, R=8, S=33, Sf=33, P=64),
    's4_sf508': dict(N=1, R=8, S=4, Sf=508, P=64),
    's97_sf257': dict(N=1, R=8, S=97, Sf=257, P=64),
    's256_sf256': dict(N=1, R=8, S=256, Sf=256, P=64),
    's192_sf192': dict(N=1, R=16, S=192, Sf=192, P=128),
    'ragged_m': dict(N=3, R=8, M=61, S=48, Sf=48, P=64, philox=True),
    'auto_axis': dict(N=3, R=8, S=48, Sf=48, P=64, rays='axis', opts=AUTO),
    # rays 0-7 of auto_axis's first view: every ray starts on a box face, none hits the box, so there is no fallback;
    # sigma bias -4 as in descending (the miss limits make the coarse depths descend)
    'auto_nohit': dict(N=1, R=8, M=8, S=48, Sf=48, P=64, rays='axis', opts=AUTO, sigma_bias=-4.0),
    'disparity': dict(N=2, R=16, S=48, Sf=48, P=64, opts=dict(disparity_space_sampling=True)),
    # sigma bias -4 keeps the pdf of the negative weights that descending depths make positive (see ray_oracle's illdef)
    'descending': dict(N=2, R=16, S=48, Sf=48, P=64, opts=dict(ray_start=1.5, ray_end=0.5), sigma_bias=-4.0),
    'bf16': dict(N=2, R=16, S=48, Sf=48, P=128, bf16=True),
    'dense': dict(N=1, R=16, S=48, Sf=48, P=64, sigma_bias=8.0),
    'train': dict(N=4, R=64, S=48, Sf=48, P=256),
    'train_cull': dict(N=4, R=64, S=48, Sf=48, P=256, flags=dict(triplane_crop=0.1, cull_clouds=0.5), centre_cull=0.5),
    'eval96': dict(N=2, R=128, S=96, Sf=96, P=512),
}
BACKWARD = {'s256_sf256_bwd': dict(S=256, Sf=256), 's200_sf200_bwd': dict(S=200, Sf=200), 's4_sf1_bwd': dict(S=4, Sf=1),
            's2_sf0_bwd': dict(S=2, Sf=0), 'auto_nohit_bwd': dict(S=48, Sf=48, inputs='auto_nohit')}


def _seed(name):
    return 1500 + zlib.crc32(name.encode()) % 1000


# ------------------------------------------------------------------------------------------------- inputs
def _axis_rays(R):
    """Ortho rays at elevation 0, azimuth 0 / 90 / 180, direction components within 1e-6 of 0 made exactly +-0 (the
    sign rays_ortho's rounding gives them).  In each view rays 0-3 start exactly on the faces of the two axes the rays run
    across (the fp32 half side the kernel and math_utils use), rays 4-7 are the same with those direction zeros negated,
    ray 8 starts inside the box and ray 9 passes through the box edge x = z = h at y = 0.1."""
    h = torch.tensor(BW / 2, dtype=torch.float32).item()
    ros, rds = [], []
    for az in (0.0, 90.0, 180.0):
        o, d = (t[0].permute(1, 2, 0).reshape(-1, 3).clone() for t in orc.rays_ortho(0.0, az, 1.0, BW, R))
        zero = d.abs() < 1e-6
        d = torch.where(zero, torch.copysign(torch.zeros_like(d), d), d)
        o = torch.where(o.abs() < 1e-6, torch.zeros_like(o), o)
        a, b = [i for i in range(3) if bool(zero[:, i].all())]
        for k, (ax, v) in enumerate(((a, h), (a, -h), (b, h), (b, -h))):
            o[k, ax] = v
            o[4 + k, ax] = v
            d[4 + k, [a, b]] = -d[4 + k, [a, b]]
        o[8] = torch.tensor([0.05, -0.1, 0.02])
        e = F.normalize(torch.tensor([[-1.0, 0.0, -1.0]]), dim=-1)[0]
        d[9] = e
        o[9] = torch.tensor([h, 0.1, h]) - 0.6 * e
        ros.append(o)
        rds.append(d)
    return torch.stack(ros).to(DEV).contiguous(), torch.stack(rds).to(DEV).contiguous()


@functools.lru_cache(maxsize=None)
def _inputs(name):
    case = CASES[name]
    N, R, S, Sf, P = (case[k] for k in ('N', 'R', 'S', 'Sf', 'P'))
    seed = _seed(name)
    g = torch.Generator().manual_seed(seed)
    planes = torch.randn(N, 3, 32, P, P, generator=g)
    if case.get('bf16'):
        planes = planes.bfloat16().float()
    _, dec, *_ = orc.synth_inputs(seed, 1, 1, 2, 0, 2)
    dec = dict(dec, b2=dec['b2'].clone())
    dec['b2'][0] += case.get('sigma_bias', 0.0)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf, **case.get('opts', {}))
    ro, rd = [t[:N].contiguous() for t in _axis_rays(R)] if case.get('rays') == 'axis' else ra.rays_at(ra.spin12(N), R)
    if case.get('M'):
        ro, rd = ro[:, :case['M']].contiguous(), rd[:, :case['M']].contiguous()
    M = ro.shape[1]
    if case.get('philox'):
        u_c, u_f = ph.render_uniforms(PHILOX_SEED, N, M, S, Sf)
    else:
        u_c, u_f = torch.rand(N, M, S, 1, generator=g), torch.rand(N * M, Sf, generator=g)
    if case.get('centre_cull'):                     # median coarse sigma on the cull threshold
        d_c = orc.stratified_depths(u_c.to(DEV), opts['ray_start'], opts['ray_end'])
        xyz = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)[:, ::7]
        _, sig = orc.run_model(planes.to(DEV, torch.float64), dec64(dec), xyz, opts, True)
        dec['b2'][0] += cull_sigma(case['centre_cull']) - sig.median().item()
    return planes, dec, opts, ro, rd, u_c.to(DEV).contiguous(), u_f.to(DEV).contiguous()


# ------------------------------------------------------------------------------------------------- the kernel, through the C ABI
@functools.lru_cache(maxsize=1)
def _kernel(name):
    """p3d_render_forward in mode 0 twice into NaN-filled outputs and a NaN-filled workspace: its launches per profile
    slot each time, both runs bit-identical.  Returns (rgb, depth, wsum, xyz) and the workspace views."""
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = CASES[name]
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    N, M = ro.shape[:2]
    S, Sf = case['S'], case['Sf']
    r = ImportanceRenderer(use_triplane=True)
    r.planes_bf16 = bool(case.get('bf16'))
    r.mlp_mode = _lib.P3D_MLP_FP32_SIMT
    decoder = make_decoder(dec, DEV)
    with torch.no_grad(), torch.cuda.device(DEV):
        if case.get('bf16'):               # a (N,96,H,W) channels_last backbone output, consumed zero-copy
            n, p_, c, hh, ww = planes.shape
            x = planes.to(DEV, torch.bfloat16).reshape(n, p_ * c, hh, ww).contiguous(memory_format=torch.channels_last)
            cl = r._planes_cl(x.view(n, p_, c, hh, ww))
            assert cl.dtype == torch.bfloat16 and cl.data_ptr() == x.data_ptr()
        else:
            cl = r._planes_cl(planes.to(DEV))
        fl = case.get('flags', {})
        p, wts = r._params(cl, N, M, opts, decoder, fl.get('triplane_crop'), fl.get('cull_clouds'), fl.get('binarize_clouds'))
        assert p.mlp_mode == _lib.P3D_MLP_FP32_SIMT and (p.n_coarse, p.n_fine) == (S, Sf)
        p.defer_depth_clamp = 0
        if case.get('philox'):
            p.seed, u_c, u_f = PHILOX_SEED, None, None
        wt = [t.detach().float().contiguous() for t in wts]
        nbytes = int(_lib.lib().p3d_render_workspace_bytes(C.byref(p)))
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=DEV)
        out = [torch.empty(s, device=DEV) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
        want = [2 if Sf else 1, 1 if Sf else 0, 1, 0]
        runs = []
        for _ in range(2):
            for t in out:
                t.fill_(float('nan'))
            ws.fill_(0xFF)                 # every float of the workspace NaN
            torch.cuda.synchronize()
            _, prof = profiled(lambda: ra.render_forward(p, cl, wt, ro, rd, u_c, u_f, ws, out))
            assert [prof[s] for s in PROF] == want, (name, [prof[s] for s in PROF], want)
            runs.append([t.clone() for t in out] + [ws.clone()])
        ra.repeats(runs[0][:4], runs[1][:4], OUTPUTS, nan=True)
        assert torch.equal(runs[0][4], runs[1][4]), 'two runs differ in the workspace'
        v, total = ra.workspace_views(runs[0][4], N, M, S, Sf)
        assert total == nbytes, (total, nbytes)
        for k in ('depth_c', 'sigma_c', 'rgb_c', 'depth_f', 'sigma_f', 'rgb_f'):
            assert not torch.isnan(v[k]).any(), f'{k} has NaN (an element never written)'
        return runs[0][:4], v


# ------------------------------------------------------------------------------------------------- oracle and bars
def _limits(name, f32=False):
    """Per-ray coarse limits (N,M,1) as the renderer forms them; 'auto': math_utils.get_ray_limits_box on the fp32 rays
    (what k_ray_limits computes, bit for bit) with the batch's fallback for rays that miss (or have a NaN limit);
    f32: the raw fp32 limits, before the fallback.  In a batch where no ray hits the box, a NaN limit takes the miss
    limits (-1, -2): the kernel's deviation from the reference, which renders NaN there (coarse_sample_depth,
    render_device.cuh)."""
    from panic3d_b200.training.volumetric_rendering import math_utils
    _, _, opts, ro, rd, *_ = _inputs(name)
    if opts['ray_start'] == 'auto':
        t0, t1 = math_utils.get_ray_limits_box(ro.cpu(), rd.cpu(), BW)
        if f32:
            return t0, t1
        ok = t1 > t0
        if bool(ok.any()):
            t0, t1 = torch.where(ok, t0, t0[ok].min()), torch.where(ok, t1, t0[ok].max())
        else:
            nan = torch.isnan(t0) | torch.isnan(t1)
            t0, t1 = torch.where(nan, -1.0, t0), torch.where(nan, -2.0, t1)
        return t0.to(DEV, torch.float64), t1.to(DEV, torch.float64)
    full = lambda v: torch.full(ro.shape[:2] + (1,), float(v), device=DEV, dtype=torch.float64)
    return full(opts['ray_start']), full(opts['ray_end'])


def _importance(floor=0.01, edges='mid', shift=0):
    """orc.importance_depths restated with one change for the negative controls: the pdf floor, the bin edges ('mid':
    interval midpoints; 'depth': the coarse depths t[below] / t[above]) or the max-pooled weights shifted by `shift`
    bins (the last value repeated)."""
    def draw(z, w, u, cdf_eps=None, eps=1e-5):
        R, S = z.shape
        wp = F.max_pool1d(w[:, None, :], 2, 1, padding=1)
        if shift:
            wp = torch.cat([wp[..., shift:], wp[..., -1:].expand(-1, -1, shift)], -1)
        wp = F.avg_pool1d(wp, 2, 1)[:, 0] + floor
        bins = 0.5 * (z[:, :-1] + z[:, 1:]) if edges == 'mid' else z[:, :-1]
        wi = wp[:, 1:-1] + eps
        pdf = wi / wi.sum(-1, keepdim=True)
        cdf = torch.cat([torch.zeros(R, 1, dtype=pdf.dtype, device=pdf.device), torch.cumsum(pdf, -1)], -1)
        if cdf_eps is not None:
            cdf = cdf + cdf_eps
        nb = wi.shape[1]
        inds = torch.searchsorted(cdf, u.contiguous(), right=True)
        below, above = (inds - 1).clamp_min(0), inds.clamp_max(nb)
        c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
        b0, b1 = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
        den = c1 - c0
        den = torch.where(den < eps, torch.ones_like(den), den)
        return b0 + (u - c0) / den * (b1 - b0)
    return draw


CONTROLS = {'no_pdf_floor': ('importance pdf without the 0.01 floor', _importance(floor=0.0)),
            'edges_at_depths': ('bin edges at t[below] / t[above], not the interval midpoints', _importance(edges='depth')),
            'pool_shifted': ('max-pooled weights shifted by one bin', _importance(shift=1))}
CONTROL_CASE = 'dense'
CONTROL_MIN = 20.0


def _chunk(name, v, sl, controls=False, with_bars=True):
    """ra.ray_oracle for rays `sl` of view v with the SIMT rounding model, the fine-depth bars included; with controls,
    the mutated oracles' outputs (m,37) and fine depths."""
    case = CASES[name]
    planes, dec, opts, ro_all, rd_all, u_c_all, u_f_all = _inputs(name)
    M = ro_all.shape[1]
    ro, rd = ro_all[v, sl].double(), rd_all[v, sl].double()
    u_c = u_c_all[v, sl].double()
    u_f = u_f_all[v * M:(v + 1) * M][sl].double()
    t0, t1 = (t[v, sl] for t in _limits(name))
    if opts['ray_start'] == 'auto':
        d_c = orc.stratified_depths(u_c[None], t0[None], t1[None])[0]
    else:
        d_c = orc.stratified_depths(u_c[None], opts['ray_start'], opts['ray_end'], opts.get('disparity_space_sampling', False))[0]
    p64 = planes[v:v + 1].to(DEV, torch.float64)
    res, ctx = ra.ray_oracle(ra.SIMT, p64, dec64(dec), opts, case.get('flags', {}), True, ro, rd, d_c, t0, t1, u_f, case['Sf'],
                             with_bars=with_bars, fine_bars=True)
    if controls:
        for c, (_, draw) in CONTROLS.items():
            t_f = draw(d_c[..., 0], ctx['w'], u_f)[..., None]
            f = ctx['samples'](t_f)
            res[c] = ra.render_graph(ro, rd, d_c, u_f, ctx['c0'], f, ctx['white'], ctx['zero'], importance=draw)[0]
            res[c + '_t_f'] = t_f[..., 0]
    return res


def _rays_of(name):
    M = _inputs(name)[3].shape[1]
    idx = torch.arange(M, device=DEV)
    return [(v, idx[i:i + CHUNK]) for v in range(CASES[name]['N']) for i in range(0, M, CHUNK)]


def _flat(out, v, sl):
    rgb, depth, wsum, xyz = out
    return torch.cat([rgb[v, sl], depth[v, sl], wsum[v, sl], xyz[v, sl]], -1)


def _compare(name, out, ws, controls=False):
    """The kernel's outputs and fine depths against the oracle's, ray by ray.  Returns the worst errors of the outputs
    and the fine depths, the share of excluded rays, the controls' worst miss / bar and the cull share."""
    Sf = CASES[name]['Sf']
    res_all = [(v, sl, _chunk(name, v, sl, controls)) for v, sl in _rays_of(name)]
    t_hi = max(r['t_max'].item() for *_, r in res_all)
    worst = {key: Worst() for key in OUTPUTS + ('fine depths',)}
    n_near = n_total = n_ill = n_dead = 0
    ctl = dict.fromkeys(CONTROLS if controls else (), 0.0)
    ctl_t = dict(ctl)
    cull = [0, 0]
    for v, sl, r in res_all:
        got = _flat(out, v, sl)
        want, bar = r['o'].clone(), r['bar'].clone()
        dead = (want[:, 33] == 0) | (got[:, 33] == 0)
        want[dead, 32] = t_hi                                  # nan_to_num(inf) then the clamp to the batch's largest depth
        bar[dead, 32] = 64 * U32 * abs(t_hi)
        keep = ~r['near'] & ~r['illdef']
        n_dead += (dead & keep).sum().item()
        n_ill += r['illdef'].sum().item()
        if keep.any():
            for key, cols in OUT_COLS.items():
                worst[key].add(got[keep][:, cols], want[keep][:, cols], bar[keep][:, cols])
        if Sf and keep.any():
            # the importance depths: sorted per ray, within the ray's largest fine-depth bar
            t_k = torch.sort(ws['depth_f'][v, sl], -1)[0]
            t_o = torch.sort(r['t_f'][..., 0], -1)[0]
            fbar = r['fine_move'].max(1, keepdim=True).values.expand_as(t_o)
            worst['fine depths'].add(t_k[keep], t_o[keep], fbar[keep])
            for c in ctl:
                ctl_t[c] = max(ctl_t[c], ((t_k.double() - torch.sort(r[c + '_t_f'], -1)[0]).abs() / fbar)[keep].max().item())
        n_near += r['near'].sum().item()
        n_total += r['near'].numel()
        for c in ctl:
            err = (got.double() - r[c]).abs()[keep]
            if err.shape[0]:
                ctl[c] = max(ctl[c], (err / bar[keep]).max().item())
        if r['cull_share']:
            cull[0] += r['cull_share'][0]
            cull[1] += r['cull_share'][1]
    for key, w in worst.items():
        print(f'{name} {key}: max abs err {w.err:.3e}, worst err / bar {w.ratio:.4f}')
    print(f'{name}: {n_near} of {n_total} rays excluded (a sample within its bar of a mask threshold), {n_ill} with a '
          f'non-positive importance pdf, {n_dead} compared rays with W = 0')
    assert n_ill == 0, (name, n_ill)
    if name == 'train_cull':              # k_depth_finalize's NaN -> inf is compared on some ray
        assert n_dead > 0
    for c in ctl:
        print(f'negative control "{CONTROLS[c][0]}" on {name}: worst err / bar {ctl[c]:.1f} (outputs), {ctl_t[c]:.1f} (fine depths)')
    return worst, n_near / max(n_total, 1), ctl, cull


# ------------------------------------------------------------------------------------------------- tests
def test_simt_bars_hold_on_the_decode():
    """The per-sample SIMT bar (render_abi.simt_bars plus the grid transform's rounding of the exact fp32 points,
    render_abi.decoded with ray_point=False) holds on p3d_decode_points in mode 0 (k_sample_decode's decoder) at the
    oracle's own coarse and fine sample positions of train's first view.  The ratio against simt_bars alone is printed."""
    name = 'train'
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    n = 1024
    p64, d64 = planes[:1].to(DEV, torch.float64), dec64(dec)
    _, smp = orc.render(p64, d64, ro[:1, :n].double(), rd[:1, :n].double(), opts, u_c[:1, :n].double(), u_f[:n].double(),
                        return_samples=True)
    xyz = torch.cat([(ro[:1, :n, None].double() + d * rd[:1, :n, None].double()).reshape(1, -1, 3) for d in smp['depths']], 1).float()
    x64 = xyz.double()
    sig, rgb, _, _, b_sig, b_rgb = ra.decoded(ra.SIMT, p64, d64, opts, True, x64, torch.zeros_like(x64), ray_point=False)
    a_rgb, a_sig = ra.simt_bars(p64, d64, x64)
    k_rgb, k_sig = ra.decode_points(planes[:1].to(DEV), dec, xyz, 0)
    for key, k, w, b, b_alone in (('rgb', k_rgb, rgb, b_rgb, a_rgb), ('sigma', k_sig, sig, b_sig, a_sig)):
        err = (k.double() - w).abs().nan_to_num(nan=float('inf'))
        print(f'SIMT decode at the render samples {key}: max abs err {err.max().item():.3e}, worst err / bar '
              f'{(err / b).max().item():.4f} (simt_bars alone: {(err / b_alone).max().item():.4f}), median bar '
              f'{b.median().item():.2e}')
        assert (err / b).max().item() <= 1.0, key


@pytest.mark.parametrize('name', list(CASES))
def test_ray_oracle_is_the_oracle(name, monkeypatch):
    """_chunk's zero-leaf graph (ray_oracle with_bars=False) gives oracle.render's fp64 outputs for every case: Sf = 0,
    Sf != S, disparity, descending depths, masks, and 'auto' limits with the batch's fallback.  For 'auto', render's
    fp64 restatement of the limits is replaced by the reference's own fp32 math_utils.get_ray_limits_box on the same rays
    (what _limits and the kernel use); render then applies the fallback itself.  auto_nohit has no fallback: there the
    reference renders NaN (asserted), and the kernel's miss limits (-1, -2) for NaN rays are given to render instead.
    'auto' cases pass render the whole batch, the others the first 256 rays of view 0.  depth is compared where W > 0
    (render clamps the others to its batch's largest depth)."""
    from panic3d_b200.training.volumetric_rendering import math_utils
    case = CASES[name]
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    N, M = ro.shape[:2]
    auto = opts['ray_start'] == 'auto'
    n = M if auto else min(256, M)
    views = range(N) if auto else range(1)
    fl = case.get('flags', {})
    args = (planes[:len(views)].to(DEV, torch.float64), dec64(dec), ro[:len(views), :n].double(), rd[:len(views), :n].double(),
            opts, u_c[:len(views), :n].double(), u_f.view(N, M, case['Sf'])[:len(views), :n].reshape(len(views) * n, -1).double())

    def limits32(o, d, bw, miss_for_nan=False):
        t0, t1 = (t.to(o) for t in math_utils.get_ray_limits_box(o.float().cpu(), d.float().cpu(), bw))
        if miss_for_nan:
            nan = torch.isnan(t0) | torch.isnan(t1)
            t0, t1 = torch.where(nan, -1.0, t0), torch.where(nan, -2.0, t1)
        return t0, t1
    if auto:
        monkeypatch.setattr(orc, 'ray_limits_box', limits32)
        if name == 'auto_nohit':
            ref = orc.render(*args, **fl)
            assert all(torch.isnan(t).all() for t in (ref[0], ref[3])), 'the reference no longer renders NaN here'
            monkeypatch.setattr(orc, 'ray_limits_box', functools.partial(limits32, miss_for_nan=True))
    want = orc.render(*args, **fl)
    worst = dict.fromkeys(OUTPUTS, 0.0)
    for v in views:
        for i in range(0, n, CHUNK):
            sl = torch.arange(i, min(i + CHUNK, n), device=DEV)
            got = _chunk(name, v, sl, with_bars=False)['o']
            ref = _flat(want, v, sl)
            live = ref[:, 33] > 0
            for key, a_, b_ in zip(OUTPUTS, ref.split([32, 1, 1, 3], -1), got.split([32, 1, 1, 3], -1)):
                if key == 'depth':
                    a_, b_ = a_[live], b_[live]
                err = (a_ - b_).abs().nan_to_num(nan=float('inf'))
                worst[key] = max(worst[key], err.max().item() if err.numel() else 0.0)
    print(f'{name} graph vs render: ' + ', '.join(f'{k} {e:.1e}' for k, e in worst.items()))
    assert max(worst.values()) <= 1e-12, (name, worst)


def _case_checks(name, out, ws):
    case = CASES[name]
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    N, M = ro.shape[:2]
    S, Sf = case['S'], case['Sf']
    p2 = 1
    while p2 < Sf:
        p2 <<= 1
    if Sf:
        t_f = ws['depth_f']
        # sorted ascending and finite: no +inf pad of the bitonic sort reached the fine depths (or the composite)
        assert torch.isfinite(t_f).all() and (t_f[..., 1:] >= t_f[..., :-1]).all(), 'fine depths not sorted or not finite'
    if name == 'train_cull':
        assert (out[2] == 0).any(), 'no ray with every sample masked (W = 0: k_depth_finalize\'s NaN -> inf)'
    if name == 's256_sf256':
        nb, L = S - 3, S + Sf
        assert 7 * 32 < nb <= 8 * 32, nb                     # my[7] holds live bins
        assert L == 16 * 32 and 4 * 4 * L * 4 == 32 << 10       # all 16 om[] chunks live, 32 KB of composite smem
    if name == 's4_sf508':
        assert p2 == 512 and S - 3 == 1
    if name in ('s33_sf33', 's97_sf257'):
        assert p2 - Sf >= {'s33_sf33': 31, 's97_sf257': 255}[name], (p2, Sf)
    if name == 's2_sf0':
        assert Sf == 0
    if name == 's192_sf192':
        assert S == Sf == 2 * 96
    if name == 'ragged_m':
        assert M % 4 and (N * M) % 4 == 3, (N, M)
    if name == 'descending':
        assert opts['ray_start'] > opts['ray_end'] and (ws['depth_c'][..., 0] > ws['depth_c'][..., -1]).all()
    if name == 'auto_axis':
        t0, t1 = _limits(name, f32=True)
        k0, k1 = ws['ray_t0'].cpu(), ws['ray_t1'].cpu()
        for key, a, b in (('t0', k0, t0[..., 0]), ('t1', k1, t1[..., 0])):
            same = (a == b) | (torch.isnan(a) & torch.isnan(b))
            assert same.all(), (key, a[~same][:8], b[~same][:8])
        d = rd.cpu()
        nan = torch.isnan(t0[..., 0]) | torch.isnan(t1[..., 0])
        inside = (t0[..., 0] < 0) & (t1[..., 0] > 0)
        print(f'auto_axis: {int(nan.sum())} rays with a NaN limit (0 * inf), {int(inside.sum())} starting inside the box, '
              f'{int(((d == 0) & ~torch.signbit(d)).sum())} +0 and {int(((d == 0) & torch.signbit(d)).sum())} -0 direction components')
        assert nan.sum() >= 8 * N and inside.sum() >= N
        assert ((d == 0) & torch.signbit(d)).any() and ((d == 0) & ~torch.signbit(d)).any()
        assert (t1 > t0).any()                                   # the fallback exists
    if name == 'auto_nohit':
        t0, t1 = _limits(name, f32=True)
        nan = torch.isnan(t0) | torch.isnan(t1)
        assert nan.all() and not (t1 > t0).any(), 'a ray has finite limits or hits the box'
        k0, k1 = _limits(name)
        assert (k0 == -1).all() and (k1 == -2).all()
        assert (ws['depth_c'][..., 0] > ws['depth_c'][..., -1]).all(), 'coarse depths are not the miss limits\' descending ones'


@pytest.mark.parametrize('name', [n for n in CASES if n != CONTROL_CASE])
def test_simt_matches_fp64_oracle(name):
    if CASES[name]['P'] >= 512:
        ra.skip_unless_free(FREE_BYTES)
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    out, ws = _kernel(name)
    _case_checks(name, out, ws)
    worst, share, _, cull = _compare(name, out, ws)
    if cull[1]:
        print(f'{name}: cull removes {cull[0] / cull[1]:.3f} of the uncropped coarse samples')
        assert 0.2 <= cull[0] / cull[1] <= 0.8, cull
    print(f'{name}: {time.time() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB')
    assert share <= EXCLUDE_SHARE_MASKS.get(name, EXCLUDE_SHARE), share
    assert max(w.ratio for w in worst.values()) <= 1.0, (name, {k: w.ratio for k, w in worst.items()})


@functools.lru_cache(maxsize=1)
def _control_compare():
    return _compare(CONTROL_CASE, *_kernel(CONTROL_CASE), controls=True)


@pytest.mark.parametrize('control', list(CONTROLS))
def test_negative_control(control):
    """The oracle with one importance-sampling change misses the kernel by >= 20x its bar on `dense`, while the true
    oracle holds there."""
    worst, share, ctl, _ = _control_compare()
    assert share <= EXCLUDE_SHARE
    assert max(w.ratio for w in worst.values()) <= 1.0, {k: w.ratio for k, w in worst.items()}
    assert ctl[control] >= CONTROL_MIN, (CONTROLS[control][0], ctl[control])


@pytest.mark.parametrize('name', list(BACKWARD))
def test_backward_at_the_envelope_edge(name):
    """p3d_render_backward after the SIMT forward at the edge of the sample counts it accepts, against the fp64
    render_backward_oracle on the kernel's depths and masks, per-element bars (render_abi.TrainKernel.bars)."""
    case = BACKWARD[name]
    S, Sf = case['S'], case['Sf']
    if name in ('s256_sf256_bwd', 's200_sf200_bwd'):
        # k_ray_backward: 4 warps x 8 floats per merged sample; above 48 KB it opts in with cudaFuncSetAttribute
        assert 128 * (S + Sf) > 49152
    t0 = time.time()
    if case.get('inputs'):                 # a forward case's inputs
        inputs = _inputs(case['inputs'])
    else:
        N, R = 1, 8
        seed = _seed(name)
        g = torch.Generator().manual_seed(seed)
        planes = torch.randn(N, 3, 32, 64, 64, generator=g)
        _, dec, *_ = orc.synth_inputs(seed, 1, 1, 2, 0, 2)
        opts = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf)
        ro, rd = ra.rays_at(ra.spin12(N), R)
        M = ro.shape[1]
        inputs = (planes, dec, opts, ro, rd, torch.rand(N, M, S, 1, generator=g), torch.rand(N * M, Sf, generator=g))
    k = ra.TrainKernel(case, inputs)
    if name == 'auto_nohit_bwd':           # the forward's miss limits for NaN rays: finite, descending coarse depths
        assert torch.isfinite(k.v['depth_c']).all() and (k.v['depth_c'][..., 0] > k.v['depth_c'][..., -1]).all()
    worst = 0.0
    for i, kind in enumerate(('all', 'bench')):
        grads = ra.upstream(kind, k.N, k.M, 70 + i)
        got, dsig = k.backward(grads)
        assert not torch.isnan(dsig).any(), 'a sample was never written by k_ray_backward'
        b64, bars, cnt = k.bars(grads)
        taps = ra.per_channel(cnt, 1)
        w = ra.compare(f'{name} [{kind}]', got, b64, bars, taps)
        worst = max(worst, max(w.values()))
        assert (got['planes'][taps == 0] == 0).all(), 'a texel no sample touches got a gradient'
    print(f'{name}: worst err / bar {worst:.4f}; {time.time() - t0:.1f} s')
    assert worst <= 1.0, (name, worst)
