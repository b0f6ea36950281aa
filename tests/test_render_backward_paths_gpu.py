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
import ctypes as C
import functools
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import render_backward_oracle as rbo, renderer_oracle as orc
from tests.test_render_gpu import make_decoder

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
TINY = 2.0 ** -126              # fp32 underflow: a step whose fp64 value is below the normal range may come out 0 in fp32
FWD_BAR = 1e-4                  # fp32 SIMT forward vs the fp64 oracle (tests/test_render_backward_gpu.py TIGHT)
KT = 128                        # samples per k_sample_backward CTA (render_backward.cu kT)
FREE_BYTES = 24 << 30           # the 256^2 cases: kernel buffers (~3 GB) + one view of fp64 oracle intermediates, with margin
CULL_SHARE = 1e-3               # samples whose fp64 cull decision may differ from the kernel's (within its sigma error bound)
UPSTREAM = ('rgb', 'depth', 'wsum', 'xyz', 'all', 'bench')
PARAMS = ('planes', 'w1', 'b1', 'w2', 'b2')

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


def _big(case):
    return case['H'] * case['W'] >= 256 * 256


def _skip_small_device(case):
    free, _ = torch.cuda.mem_get_info()
    if _big(case) and free < FREE_BYTES:
        pytest.skip(f'needs {FREE_BYTES >> 30} GB of free device memory, {free >> 30} GB free')


def _cull_sigma(cull):
    """sigma below which cull_mask removes a sample: 1 - exp(-softplus(sigma - 1)) < cull."""
    return 1.0 + math.log(math.expm1(-math.log1p(-cull)))


# ------------------------------------------------------------------------------------------------- inputs
def _rays(N, R):
    """bench.py's training rays: spin12 cameras (dist 1, fov 30) through RaySampler."""
    from panic3d_b200 import cameras
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    spin = cameras.cam60[cameras.camsubs['spin12']]
    lab = torch.stack([cameras.camera_params_to_matrix(elev=float(spin[i][0]), azim=float(spin[i][1]), dist=1.0, fov=30.0)
                       ['camera_label'] for i in range(N)]).to(DEV)
    ro, rd = RaySampler()(lab[:, :16].view(-1, 4, 4), lab[:, 16:25].view(-1, 3, 3), R)
    return ro.float().contiguous(), rd.float().contiguous()


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
    ro, rd = _rays(N, R)
    M = R * R
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, Sf, generator=g)
    centre = _cull_sigma(case['centre_cull']) if case.get('centre_cull') else case.get('centre_sigma')
    if centre is not None:                          # median coarse sigma on `centre`
        d_c = orc.stratified_depths(u_c.to(DEV), opts['ray_start'], opts['ray_end'])
        xyz = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)[:, ::7]
        _, sig = orc.run_model(planes.to(DEV, torch.float64), _dec64(dec), xyz, opts, True)
        dec['b2'][0] += centre - sig.median().item()
    return planes, dec, opts, ro, rd, u_c, u_f


def _dec64(dec):
    return {k: (v.to(DEV, torch.float64) if torch.is_tensor(v) else v) for k, v in dec.items()}


def _upstream(kind, N, M, seed):
    g = torch.Generator().manual_seed(seed)
    shapes = ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))
    if kind == 'wsum+':
        return [t.to(DEV) for t in (torch.zeros(shapes[0]), torch.zeros(shapes[1]), torch.ones(shapes[2]), torch.zeros(shapes[3]))]
    if kind == 'bench':
        out = [torch.full(shapes[0], 1.0 / (N * M * 32)), torch.full(shapes[1], 0.1 / (N * M)),
               torch.full(shapes[2], 0.1 / (N * M)), torch.zeros(shapes[3])]
    else:
        out = [torch.randn(s, generator=g) for s in shapes]
        keep = {'rgb': 0, 'depth': 1, 'wsum': 2, 'xyz': 3}.get(kind)
        if keep is not None:
            out = [t if i == keep else torch.zeros_like(t) for i, t in enumerate(out)]
    return [t.to(DEV) for t in out]


# ------------------------------------------------------------------------------------------------- the kernels, through the C ABI
def _workspace_views(ws, N, M, S, Sf):
    """workspace_layout (c_api.cu:92) restated: bounds, depth_c, sigma_c, rgb_c, depth_f, sigma_f, rgb_f, ray_t0, ray_t1,
    each 256-byte aligned.  Returns the views and the total."""
    R = N * M
    sizes = [64, R * S * 4, R * S * 4, R * S * 32 * 4, R * Sf * 4, R * Sf * 4, R * Sf * 32 * 4, R * 4, R * 4]
    offs, off = [], 0
    for b in sizes:
        offs.append(off)
        off += (b + 255) // 256 * 256
    f = lambda i, n: ws[offs[i]:offs[i] + n * 4].view(torch.float32)
    v = dict(depth_c=f(1, R * S).view(N, M, S), sigma_c=f(2, R * S).view(N, M, S), rgb_c=f(3, R * S * 32).view(N, M, S, 32),
             depth_f=f(4, R * Sf).view(N, M, Sf), sigma_f=f(5, R * Sf).view(N, M, Sf),
             rgb_f=f(6, R * Sf * 32).view(N, M, Sf, 32), ray_t0=f(7, R).view(N, M), ray_t1=f(8, R).view(N, M))
    return v, off


class Kernel:
    """One forward (kept with its workspace) and any number of backwards of the training path."""

    def __init__(self, name):
        from panic3d_b200 import _lib
        from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
        case = CASES[name]
        planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
        self.case_name, self.case, self.opts, self.ro, self.rd = name, case, opts, ro, rd
        N, _, Cc, H, W = planes.shape
        M = ro.shape[1]
        self.N, self.M, self.S, self.Sf = N, M, case['S'], case['Sf']
        self.flags = case.get('flags', {})
        r = ImportanceRenderer(use_triplane=not case.get('eg3d'))
        self.decoder = make_decoder(dec, DEV)
        probe = torch.empty((N, 3, H, W, Cc), device='meta')
        p, wts = r._params(probe, N, M, opts, self.decoder, self.flags.get('triplane_crop'), self.flags.get('cull_clouds'),
                           self.flags.get('binarize_clouds'))
        self.planes_cl = planes.to(DEV).permute(0, 1, 3, 4, 2).contiguous()
        p.stride_view, p.stride_plane, p.stride_row, p.stride_col, _ = self.planes_cl.stride()
        p.planes_bf16, p.mlp_mode, p.defer_depth_clamp = 0, _lib.P3D_MLP_FP32_SIMT, 0
        self.p, self.wt = p, [t.detach().float().contiguous() for t in wts]
        self.u_c, self.u_f = u_c.to(DEV).contiguous(), u_f.to(DEV).contiguous()
        L = _lib.lib()
        nbytes = int(L.p3d_render_workspace_bytes(C.byref(p)))
        runs = []
        for _ in range(2):
            ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
            out = [torch.full(s, float('nan'), device=DEV) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
            _lib.check(L.p3d_render_forward(C.byref(p), self.planes_cl.data_ptr(), *[t.data_ptr() for t in self.wt],
                                            ro.data_ptr(), rd.data_ptr(), self.u_c.data_ptr(), self.u_f.data_ptr(),
                                            ws.data_ptr(), ws.numel(), *[o.data_ptr() for o in out], _lib.stream_ptr(DEV)))
            torch.cuda.synchronize()
            runs.append((ws, out))
        for a, b in zip(runs[0][1], runs[1][1]):
            assert torch.equal(a, b), 'two forwards differ'
        self.ws, self.out = runs[0]
        self.v, total = _workspace_views(self.ws, N, M, self.S, self.Sf)
        assert total == nbytes, (total, nbytes)
        for k in ('depth_c', 'sigma_c', 'rgb_c', 'depth_f', 'sigma_f', 'rgb_f'):
            assert torch.equal(self.v[k], _workspace_views(runs[1][0], N, M, self.S, self.Sf)[0][k]), k
            assert not torch.isnan(self.v[k]).any(), k

    def backward(self, grads):
        from panic3d_b200 import _lib
        L, p = _lib.lib(), self.p
        scratch = torch.empty(int(L.p3d_render_backward_scratch_bytes(C.byref(p))), dtype=torch.uint8, device=DEV)
        scratch.view(torch.float32)[:scratch.numel() // 4].fill_(float('nan'))
        d_planes = torch.zeros_like(self.planes_cl)
        d_w = [torch.zeros_like(t) for t in self.wt]
        g = [t.float().contiguous() for t in grads]
        _lib.check(L.p3d_render_backward(C.byref(p), self.planes_cl.data_ptr(), *[t.data_ptr() for t in self.wt],
                                         self.ro.data_ptr(), self.rd.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                                         self.out[1].data_ptr(), *[t.data_ptr() for t in g], scratch.data_ptr(), scratch.numel(),
                                         d_planes.data_ptr(), *[t.data_ptr() for t in d_w], _lib.stream_ptr(DEV)))
        torch.cuda.synchronize()
        R = self.N * self.M
        sc = scratch.view(torch.float32)
        dsig = sc[:R * (self.S + self.Sf)]
        grads_out = dict(zip(PARAMS, [d_planes.permute(0, 1, 4, 2, 3)] + d_w))
        return grads_out, dsig

    # the kernel's constants, in the form the oracle takes them
    def depths(self):
        return self.v['depth_c'][..., None], (self.v['depth_f'][..., None] if self.Sf else None)

    def masks(self):
        N = self.N
        return (self.v['sigma_c'].reshape(N, -1, 1) == -1e3, self.v['sigma_f'].reshape(N, -1, 1) == -1e3 if self.Sf else None)

    def fwd_values(self):
        return [(self.v['sigma_c'][n], self.v['rgb_c'][n], self.v['sigma_f'][n], self.v['rgb_f'][n]) for n in range(self.N)]


# ------------------------------------------------------------------------------------------------- oracle and bars
def _oracle(k, grads, **kw):
    planes, dec, *_ = _inputs(k.case_name)
    return rbo.render_backward(planes.to(DEV, torch.float64), _dec64(dec), k.ro, k.rd, k.opts, k.depths(), k.masks(), grads,
                               use_triplane=not k.case.get('eg3d'), dead=k.out[2][..., 0] == 0, **k.flags, **kw)


def _bars(k, grads):
    """(B64, bar) per parameter: bar = (k_i + c) u A + 2 |B64 - Bk|."""
    L = k.S + k.Sf
    c = 2 * L + 192
    b64 = _oracle(k, grads)
    bk = _oracle(k, grads, fwd=k.fwd_values())
    A = _oracle(k, grads, mag=True, c=c)
    n_cta = -(-k.N * k.M * k.S // KT) + (-(-k.N * k.M * k.Sf // KT) if k.Sf else 0)
    H, W = k.planes_cl.shape[2], k.planes_cl.shape[3]
    cnt = rbo.texel_counts(k.ro, k.rd, k.depths(), H, W, k.opts['box_warp'], not k.case.get('eg3d'))
    bars = {}
    for key in PARAMS:
        kk = cnt[:, :, None].double() if key == 'planes' else float(KT + n_cta)
        bars[key] = (kk + c) * (U * A[key] + TINY) + 2 * (b64[key] - bk[key]).abs()
        bars[key + '_fwd'] = 2 * (b64[key] - bk[key]).abs()
    return b64, bars, cnt


def _ratio(got, want, bar):
    err = (got.double() - want).abs().nan_to_num(nan=float('inf'))
    r = err / bar
    r = torch.where(err == 0, torch.zeros_like(r), r)           # 0 / 0: an exact zero where the bar is zero
    return err.max().item(), r.max().item()


def _compare(tag, got, want, bars, cnt=None):
    worst = {}
    for key in PARAMS:
        err, ratio = _ratio(got[key], want[key], bars[key])
        print(f'{tag} d_{key}: max abs err {err:.3e}, worst err / bar {ratio:.4f}')
        worst[key] = ratio
        if ratio > 1 and key == 'planes' and cnt is not None:
            err = (got[key].double() - want[key]).abs()
            e = torch.where(err == 0, torch.zeros_like(err), err / bars[key]).nan_to_num(nan=float('inf'))
            i = int(e.argmax())
            n, p, ch, y, x = np.unravel_index(i, e.shape)
            print(f'  worst texel {(n, p, ch, y, x)}: got {got[key][n, p, ch, y, x].item():.6e} want '
                  f'{want[key][n, p, ch, y, x].item():.6e} bar {bars[key][n, p, ch, y, x].item():.3e} (forward part '
                  f'{bars[key + "_fwd"][n, p, ch, y, x].item():.3e}) taps {cnt[n, p, y, x].item()}')
    return worst


# ------------------------------------------------------------------------------------------------- tests
def test_gpu_fp64_oracle_equals_cpu_oracle():
    """The device fp64 run of the render oracle (with injected depths and masks) equals the CPU fp32 oracle on the
    fixture-sized gradient cases, within the fp32 run's rounding; its hand-written gradients equal the CPU fp32 autograd ones
    within 1e-5 of each tensor's largest element."""
    from tests.golden.cases import build_case_inputs
    from tests.helpers import case_rays
    from tests.test_render_backward_gpu import BWD_CASES, _flags, _incoming, _loss
    for name in ('train48', 'eval96'):
        case = BWD_CASES[name]
        planes, dec, c2w, K, u_c, u_f, opts = build_case_inputs(case)
        ro, rd = case_rays(case, c2w, K)
        fl = _flags(case)
        pl = planes.clone().requires_grad_(True)
        dref = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
        out, smp = orc.render(pl, dref, ro, rd, opts, u_c, u_f, return_samples=True, **fl)
        gw = _incoming(case['seed'] + 5, ro.shape[0], ro.shape[1])
        ref = torch.autograd.grad(_loss(out, gw), [pl] + [dref[k] for k in ('w1', 'b1', 'w2', 'b2')])
        to = lambda t: None if t is None else t.to(DEV)
        dep, msk = tuple(map(to, smp['depths'])), tuple(map(to, smp['masks']))
        out64 = orc.render(planes.to(DEV, torch.float64), _dec64(dec), ro.to(DEV), rd.to(DEV), opts, None, None,
                           depths=dep, masks=msk, **fl)
        for a, b in zip(out64, out):
            assert a.dtype == torch.float64
            assert (a.cpu() - b.detach().double()).abs().max().item() <= 2e-6, name
        g64 = rbo.render_backward(planes.to(DEV, torch.float64), _dec64(dec), ro.to(DEV), rd.to(DEV), opts, dep, msk,
                                  [g.to(DEV, torch.float64) for g in gw], **fl)
        for key, r in zip(PARAMS, ref):
            err = (g64[key].cpu() - r.double()).abs().max().item()
            print(f'pin {name} d_{key}: {err:.2e} of max {r.abs().max().item():.2e}')
            assert err <= 1e-5 * r.abs().max().item(), (name, key, err)


def _merged_rank(k):
    """Rank of every sample (coarse then fine, (N*M, L)) in its ray's merged order."""
    t = torch.cat([k.v['depth_c'], k.v['depth_f']], -1).reshape(k.N * k.M, -1)
    order = torch.sort(t, dim=-1, stable=True)[1]
    return torch.empty_like(order).scatter_(1, order, torch.arange(t.shape[1], device=DEV).expand_as(order).contiguous())


def _case_checks(name, k, b64, bars, cnt, dsig):
    """The property each case exists for, from the kernel's workspace and scratch and the oracle."""
    planes, dec, *_ = _inputs(name)
    if name == 'train':
        # the third 32-lane chunk of k_ray_backward carries gradient: samples ranked >= 64 in their ray get a nonzero
        # dsig on most rays
        R_ = k.N * k.M
        per = torch.cat([dsig[:R_ * k.S].view(R_, k.S), dsig[R_ * k.S:].view(R_, k.Sf)], 1)
        third = ((per != 0) & (_merged_rank(k) >= 64)).any(1).double().mean().item()
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
        pre = rbo._decoder_forward(planes[0].to(DEV, torch.float64), _dec64(dec), xyz, k.opts['box_warp'], True)[4]
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
        d = _dec64(dec)
        pre = rbo.gather(flat, idx, wgt).sum(1) / 3 @ (d['w1'] / math.sqrt(32)).t() + d['b1']
        hi, lo = (pre > 20).double().mean().item(), (pre < -20).double().mean().item()
        t = torch.cat([k.v['depth_c'], k.v['depth_f']], -1)
        sg = torch.gather(torch.cat([k.v['sigma_c'], k.v['sigma_f']], -1), -1, torch.sort(t, dim=-1, stable=True)[1])
        smid = ((sg[..., 1:] + sg[..., :-1]) / 2 - 1)
        sm = (smid > 20).double().mean().item()
        print(f'branches: pre > 20 {hi:.3f}, pre < -20 {lo:.3f}, smid > 20 {sm:.3f}')
        assert hi >= 0.05 and lo >= 0.05 and sm >= 0.05, (hi, lo, sm)
    if name == 'train_cull':
        thresh = _cull_sigma(0.5)
        p64, d64 = planes.to(DEV, torch.float64), _dec64(dec)
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
    k = Kernel(name)
    # forward: within the decode bar of the fp64 oracle fed the kernel's depths and masks
    planes, dec, *_ = _inputs(name)
    out64 = orc.render(planes.to(DEV, torch.float64), _dec64(dec), k.ro, k.rd, k.opts, None, None, depths=k.depths(),
                       masks=k.masks(), use_triplane=not case.get('eg3d'), **k.flags)
    for key, a, b in zip(('rgb', 'depth', 'wsum', 'xyz'), k.out, out64):
        err = (a.double() - b).abs().nan_to_num(nan=float('inf')).max().item()
        print(f'{name} forward {key}: max abs err {err:.3e}')
        assert err <= FWD_BAR, (name, key, err)
    del out64
    worst = {}
    for i, kind in enumerate(UPSTREAM):
        grads = _upstream(kind, k.N, k.M, 50 + i)
        got, dsig = k.backward(grads)
        assert not torch.isnan(dsig).any(), 'a sample was never written by k_ray_backward'
        b64, bars, cnt = _bars(k, grads)
        if i == 0:
            _case_checks(name, k, b64, bars, cnt, dsig)
        w = _compare(f'{name} [{kind}]', got, b64, bars, cnt)
        for key, r in w.items():
            worst[(kind, key)] = r
        assert max(w.values()) <= 1.0, (name, kind, w)
        untouched = (cnt == 0)[:, :, None].expand_as(got['planes'])
        assert (got['planes'][untouched] == 0).all(), 'a texel no sample touches got a gradient'
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
            w2 = _compare(f'{name} [repeat]', again, b64, bars)
            assert max(w2.values()) <= 1.0
    for (case_name, kind), ctl in CONTROLS.items():
        if case_name == name:
            _negative_control(name, kind, k, ctl)
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


def _negative_control(name, kind, k, ctl):
    label, kw = ctl
    grads = _upstream(kind, k.N, k.M, 99)
    got, _ = k.backward(grads)
    b64, bars, cnt = _bars(k, grads)
    assert max(_compare(f'{name} [{kind}]', got, b64, bars, cnt).values()) <= 1.0
    mut = _oracle(k, grads, **kw)
    for key in PARAMS:
        d = (got[key].double() - mut[key]).abs()
        i = int(d.argmax())
        print(f'  control {key}: max |got - mutant| {d.max().item():.3e} where bar {bars[key].reshape(-1)[i].item():.3e} '
              f'(forward part {bars[key + "_fwd"].reshape(-1)[i].item():.3e}), |grad| {mut[key].reshape(-1)[i].abs().item():.3e}')
    worst = max(_ratio(got[key], mut[key], bars[key])[1] for key in PARAMS)
    print(f'negative control "{label}" on {name} [{kind}]: worst err / bar {worst:.1f}')
    assert worst >= 20, (label, worst)


def test_autograd_route_matches_the_abi_call():
    """ImportanceRenderer under autograd (_RenderFunction) gives the C ABI call's forward bit for bit and its gradients
    within the bars (train_cull: masks and partial cull on the route the training loop takes)."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    name = 'train_cull'
    _skip_small_device(CASES[name])
    k = Kernel(name)
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    r = ImportanceRenderer(use_triplane=True)
    r.injected_noise = (u_c, u_f)
    d = make_decoder(dec, DEV).requires_grad_(True)
    pg = planes.to(DEV).requires_grad_(True)
    out = r(pg, d, ro, rd, opts, **k.flags)
    for a, b in zip(out, k.out):
        assert torch.equal(a.detach(), b)
    grads = _upstream('bench', k.N, k.M, 0)
    got = torch.autograd.grad(sum((o * g).sum() for o, g in zip(out, grads)),
                              [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    b64, bars, _ = _bars(k, grads)
    w = _compare('autograd route [bench]', dict(zip(PARAMS, got)), b64, bars)
    assert max(w.values()) <= 1.0, w


# ------------------------------------------------------------------------------------------------- density regularisation
GREG_POINTS, GREG_DIST = 1000, 0.004          # loss_orthocondA.py:592-593 (density_reg_p_dist)
GREG_GATE_SHARE = 0.01


def test_density_regularisation_phase():
    """The Greg phase (loss_orthocondA.py:579-600): 4 views x (1000 points uniform in [-1, 1]^3 + the same points plus
    N(0, 0.004^2)) through run_model under autograd (_PointsFunction) on 256^2 planes with the training options, then the
    L1 between the two halves' sigma.  Asserts which forward kernel ran, the forward against the fp64 oracle, the pairs
    whose sign is within rounding of 0 (counted), and the plane and decoder gradients per element."""
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from tests.helpers import profiled
    t0 = time.time()
    N, H = 4, 256
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=48, depth_resolution_importance=48)
    g = torch.Generator().manual_seed(1234)
    planes = torch.randn(N, 3, 32, H, H, generator=g)
    _, dec, *_ = orc.synth_inputs(1234, 1, 1, 2, 0, 2)
    x = torch.rand(N, GREG_POINTS, 3, generator=g) * 2 - 1
    coords = torch.cat([x, x + torch.randn(x.shape, generator=g) * GREG_DIST], 1).to(DEV)
    r = ImportanceRenderer(use_triplane=True)
    d = make_decoder(dec, DEV).requires_grad_(True)
    pg = planes.to(DEV).requires_grad_(True)
    # the forward's mode is chosen as for a ray render with M = 0 rays (renderer.py run_model under autograd)
    probe = torch.empty((N, 3, H, H, 32), device='meta')
    p, _ = r._params(probe, N, 0, dict(opts), d, None, None, None)
    print(f'Greg: forward mlp_mode {p.mlp_mode} (0 fp32 SIMT, 1 tensor-core 3-pass)')
    assert p.mlp_mode == _lib.P3D_MLP_TC_3XBF16, p.mlp_mode
    out, prof = profiled(lambda: r.run_model(pg, d, coords, None, opts))
    assert prof[0] == 1, prof                                          # one decode launch (profile slot 0)
    sigma = out['sigma']
    p64, d64 = planes.to(DEV, torch.float64), _dec64(dec)
    _, s64 = orc.run_model(p64, d64, coords, opts, True)
    err = (sigma.detach().double() - s64).abs().nan_to_num(nan=float('inf')).max().item()
    print(f'Greg: forward sigma max abs err {err:.3e}')
    assert err <= FWD_BAR, err
    diff_k = (sigma[:, :GREG_POINTS] - sigma[:, GREG_POINTS:]).detach()
    diff64 = s64[:, :GREG_POINTS] - s64[:, GREG_POINTS:]
    # a point with two coordinates outside the box reads no texel, so a pair of such points has exactly equal sigma in both
    # runs (sign 0, no gradient); the sign of every other pair is gated when its fp64 difference is within 2e-4 of 0
    blank = (diff64 == 0) & (diff_k == 0)
    gated = (diff64.abs() <= 2 * FWD_BAR) & ~blank
    flipped = torch.sign(diff_k.double()) != torch.sign(diff64)
    assert not (flipped & ~gated).any(), 'an L1 sign differs away from 0'
    print(f'Greg: {blank.sum().item()} of {blank.numel()} pairs read no texel (difference exactly 0 in both); of the rest '
          f'{gated.sum().item()} lie within 2e-4 of 0 (sign gated), {flipped.sum().item()} signs differ from the fp64 ones')
    assert gated.sum().item() <= GREG_GATE_SHARE * (~blank).sum().item()
    loss = F.l1_loss(sigma[:, :GREG_POINTS], sigma[:, GREG_POINTS:])
    got = torch.autograd.grad(loss, [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    # the upstream gradient is the kernel's sign: the oracle differentiates the same loss at the same sign pattern
    sgn = torch.sign(diff_k[..., 0].double()) / diff_k.numel()
    g_sigma = torch.cat([sgn, -sgn], 1)
    c = 192
    b64 = rbo.points_backward(p64, d64, coords, g_sigma, opts['box_warp'])
    A = rbo.points_backward(p64, d64, coords, g_sigma, opts['box_warp'], mag=True, c=c)
    # the hand-written points backward is the gradient (fp64 autograd of the oracle)
    pr = p64.clone().requires_grad_(True)
    dr = {k_: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k_, v in d64.items()}
    ref = torch.autograd.grad((orc.run_model(pr, dr, coords, opts, True)[1] * g_sigma[..., None]).sum(),
                              [pr] + [dr[k_] for k_ in ('w1', 'b1', 'w2', 'b2')])
    for key, rf in zip(PARAMS, ref):       # relative to A: d_b2[0] is a sum of +-1/n that cancels to 0 exactly
        assert (b64[key] - rf).abs().max().item() <= 1e-10 * A[key].max().item(), key
    # tap contributions per texel: texel_counts with origins at the points, zero directions and unit depths
    cnt = rbo.texel_counts(coords, torch.zeros_like(coords), (torch.ones(N, 2 * GREG_POINTS, 1, 1, device=DEV), None), H, H,
                           opts['box_warp'])
    n_cta = -(-N * 2 * GREG_POINTS // KT)
    worst = 0.0
    for key, gk in zip(PARAMS, got):
        kk = cnt[:, :, None].double() if key == 'planes' else float(KT + n_cta)
        bar = (kk + c) * (U * A[key] + TINY)
        e, ratio = _ratio(gk, b64[key], bar)
        print(f'Greg d_{key}: max abs err {e:.3e}, worst err / bar {ratio:.4f}')
        worst = max(worst, ratio)
    assert worst <= 1.0, worst
    untouched = (cnt == 0)[:, :, None].expand_as(got[0])
    assert (got[0][untouched] == 0).all()
    print(f'Greg: {time.time() - t0:.1f} s')
