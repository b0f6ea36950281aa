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
import ctypes as C
import functools
import time

import pytest
import torch

from oracle import multiplane_oracle as mo, render_backward_oracle as rbo, renderer_oracle as orc
from tests.test_render_backward_paths_gpu import (DEV, FWD_BAR, KT, PARAMS, TINY, U, UPSTREAM, _cull_sigma, _dec64, _rays,
                                                  _ratio, _upstream, _workspace_views)
from tests.test_render_gpu import make_decoder

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


def _skip_small_device(big):
    free, _ = torch.cuda.mem_get_info()
    if big and free < FREE_BYTES:
        pytest.skip(f'needs {FREE_BYTES >> 30} GB of free device memory, {free >> 30} GB free')


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
    ro, rd = _rays_at(case['views'], R) if 'views' in case else _rays(N, R)
    M = R * R
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, Sf, generator=g)
    if case.get('centre_cull'):                     # median coarse sigma on the cull threshold
        d_c = orc.stratified_depths(u_c.to(DEV), opts['ray_start'], opts['ray_end'])
        xyz = (ro[:, :, None] + d_c * rd[:, :, None]).reshape(N, -1, 3)[:, ::7]
        _, sig = mo.run_model(planes.to(DEV, torch.float64), _dec64(dec), xyz, opts, True)
        dec['b2'][0] += _cull_sigma(case['centre_cull']) - sig.median().item()
    return planes, dec, opts, ro, rd, u_c, u_f


def _rays_at(views, R):
    """_rays for cameras at (elevation, azimuth) in degrees, distance 1, fov 30."""
    from panic3d_b200 import cameras
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    lab = torch.stack([cameras.camera_params_to_matrix(elev=e, azim=a, dist=1.0, fov=30.0)['camera_label']
                       for e, a in views]).to(DEV)
    ro, rd = RaySampler()(lab[:, :16].view(-1, 4, 4), lab[:, 16:25].view(-1, 3, 3), R)
    return ro.float().contiguous(), rd.float().contiguous()


def _texels_cl(planes, D):
    """(N,3,C*D,H,W) -> (N,3,D,H,W,C) contiguous, restated: feature c of slab d is input channel c*D + d."""
    N, P, CD, H, W = planes.shape
    return planes.reshape(N, P, CD // D, D, H, W).permute(0, 1, 3, 4, 5, 2).contiguous()


def _from_texels(t):
    """(N,3,D,H,W,C) -> the input planes' (N,3,C*D,H,W) indexing."""
    N, P, D, H, W, Cc = t.shape
    return t.permute(0, 1, 5, 2, 3, 4).reshape(N, P, Cc * D, H, W)


class Kernel:
    """One forward (kept with its workspace) and any number of backwards, through the C ABI."""

    def __init__(self, name, strided=None):
        from panic3d_b200 import _lib
        from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
        case = CASES[name]
        planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
        strided = case.get('strided', False) if strided is None else strided
        bf16 = case.get('bf16', False)
        N, _, CD, H, W = planes.shape
        D = case['D']
        M = ro.shape[1]
        self.case_name, self.case, self.opts, self.ro, self.rd, self.D = name, case, opts, ro, rd, D
        self.N, self.M, self.S, self.Sf, self.H, self.W = N, M, case['S'], case['Sf'], H, W
        self.flags = case.get('flags', {})
        self.use_triplane = not case.get('eg3d')
        self.planes_ref = planes.bfloat16().float() if bf16 else planes       # what the kernel reads
        self.planes64 = self.planes_ref.to(DEV, torch.float64)
        r = ImportanceRenderer(use_triplane=self.use_triplane)
        self.decoder = make_decoder(dec, DEV)
        probe = torch.empty((N, 3, D, H, W, 32), device='meta')
        p, wts = r._params(probe, N, M, opts, self.decoder, self.flags.get('triplane_crop'), self.flags.get('cull_clouds'),
                           self.flags.get('binarize_clouds'))
        assert p.plane_depth == D
        cl = _texels_cl(planes.to(DEV), D)
        if strided:
            # 64-channel texels sliced to their first 32, and one padding row after each plane's slab stack; NaN wherever
            # the kernel must not read
            buf = torch.full((N, 3, D * H + 1, W, 64), float('nan'), device=DEV)
            buf[:, :, :D * H, :, :32] = cl.reshape(N, 3, D * H, W, 32)
            cl = buf[:, :, :D * H, :, :32]
            p.stride_view, p.stride_plane, p.stride_row, p.stride_col, _ = cl.stride()
            assert p.stride_plane > D * H * p.stride_row and p.stride_col == 64
        else:
            cl = cl.to(torch.bfloat16) if bf16 else cl
            p.stride_view, p.stride_plane, _, p.stride_row, p.stride_col, _ = cl.stride()
        self.planes_cl = cl
        p.planes_bf16, p.mlp_mode, p.defer_depth_clamp = (1 if bf16 else 0), _lib.P3D_MLP_FP32_SIMT, 0
        self.p, self.wt = p, [t.detach().float().contiguous() for t in wts]
        self.u_c, self.u_f = u_c.to(DEV).contiguous(), u_f.to(DEV).contiguous()
        L = _lib.lib()
        nbytes = int(L.p3d_render_workspace_bytes(C.byref(p)))
        runs = []
        for _ in range(2):
            ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
            out = [torch.full(s, float('nan'), device=DEV) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
            _lib.check(L.p3d_render_forward(C.byref(p), cl.data_ptr(), *[t.data_ptr() for t in self.wt],
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
        d_planes = torch.zeros((self.N, 3, self.D, self.H, self.W, 32), device=DEV)       # contiguous by the ABI
        d_w = [torch.zeros_like(t) for t in self.wt]
        g = [t.float().contiguous() for t in grads]
        _lib.check(L.p3d_render_backward(C.byref(p), self.planes_cl.data_ptr(), *[t.data_ptr() for t in self.wt],
                                         self.ro.data_ptr(), self.rd.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                                         self.out[1].data_ptr(), *[t.data_ptr() for t in g], scratch.data_ptr(), scratch.numel(),
                                         d_planes.data_ptr(), *[t.data_ptr() for t in d_w], _lib.stream_ptr(DEV)))
        torch.cuda.synchronize()
        dsig = scratch.view(torch.float32)[:self.N * self.M * (self.S + self.Sf)]
        return dict(zip(PARAMS, [_from_texels(d_planes)] + d_w)), dsig

    def depths(self):
        return self.v['depth_c'][..., None], self.v['depth_f'][..., None]

    def masks(self):
        return self.v['sigma_c'].reshape(self.N, -1, 1) == -1e3, self.v['sigma_f'].reshape(self.N, -1, 1) == -1e3

    def fwd_values(self):
        return [(self.v['sigma_c'][n], self.v['rgb_c'][n], self.v['sigma_f'][n], self.v['rgb_f'][n]) for n in range(self.N)]

    def samples(self, n):
        """Positions (K,3) of view n's samples, coarse then fine, as the kernel makes them."""
        return torch.cat([(self.ro[n, :, None] + d[n][..., None] * self.rd[n, :, None]).reshape(-1, 3)
                          for d in (self.v['depth_c'], self.v['depth_f'])])


# ------------------------------------------------------------------------------------------------- oracle and bars
def _oracle(k, grads, planes=None, **kw):
    _, dec, *_ = _inputs(k.case_name)
    return rbo.render_backward(k.planes64 if planes is None else planes, _dec64(dec), k.ro, k.rd, k.opts, k.depths(),
                               k.masks(), grads, use_triplane=k.use_triplane, dead=k.out[2][..., 0] == 0, depth=k.D,
                               **k.flags, **kw)


def _per_channel(cnt):
    """(N,3,D,H,W) tap counts -> (N,3,32*D,H,W), the planes' indexing."""
    N, P, D, H, W = cnt.shape
    return cnt[:, :, None].expand(N, P, 32, D, H, W).reshape(N, P, 32 * D, H, W)


def _bars(k, grads):
    """(B64, bars, tap counts (N,3,D,H,W)): bar = (k_i + c)(u A + TINY) + 2 |B64 - Bk|."""
    c = 2 * (k.S + k.Sf) + 192 + C_TRI
    b64 = _oracle(k, grads)
    bk = _oracle(k, grads, fwd=k.fwd_values())
    A = _oracle(k, grads, mag=True, c=c)
    n_cta = -(-k.N * k.M * k.S // KT) + -(-k.N * k.M * k.Sf // KT)
    cnt = rbo.texel_counts(k.ro, k.rd, k.depths(), k.H, k.W, k.opts['box_warp'], k.use_triplane, k.D)
    bars = {}
    for key in PARAMS:
        kk = _per_channel(cnt).double() if key == 'planes' else float(KT + n_cta)
        bars[key] = (kk + c) * (U * A[key] + TINY) + 2 * (b64[key] - bk[key]).abs()
    return b64, bars, cnt


def _compare(tag, got, want, bars):
    worst = {}
    for key in PARAMS:
        err, ratio = _ratio(got[key], want[key], bars[key])
        print(f'{tag} d_{key}: max abs err {err:.3e}, worst err / bar {ratio:.4f}')
        worst[key] = ratio
    return worst


def _normal_fz(xyz, D, box_warp, use_triplane):
    """(3,K) fp32 slab coordinate fz of every plane (dev::plane_normal, trilinear_footprint): slab d is centred on fz = d."""
    s = (2.0 / box_warp) * xyz
    gz = torch.stack([s[:, 2], s[:, 1], s[:, 0 if use_triplane else 1]])
    return ((gz + 1) * D - 1) * 0.5


# ------------------------------------------------------------------------------------------------- tests
def test_gpu_fp64_oracle_equals_cpu_oracle():
    """The device fp64 multiplane render oracle, fed the CPU fp32 run's depths and masks, equals the CPU fp32 oracle on the
    multiplane fixture cases within the fp32 run's rounding; its hand-written gradient equals the fp32 autograd one."""
    from tests.golden.cases_multiplane import RENDER_CASES, build_inputs
    for name in ('d2_eg3d48', 'd3_eg3d96_crop_cull'):
        case = RENDER_CASES[name]
        planes, dec, c2w, K, u_c, u_f, opts = build_inputs(case)
        ro, rd = orc.ray_sampler(c2w, K, case['R'])
        fl = dict(triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'))
        pl = planes.clone().requires_grad_(True)
        dref = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
        out, smp = mo.render(pl, dref, ro, rd, opts, u_c, u_f, use_triplane=case['use_triplane'], return_samples=True, **fl)
        gen = torch.Generator().manual_seed(case['seed'])
        gw = [torch.randn(t.shape, generator=gen) for t in out]
        ref = torch.autograd.grad(sum((o * g).sum() for o, g in zip(out, gw)), [pl] + [dref[k] for k in ('w1', 'b1', 'w2', 'b2')])
        to = lambda t: None if t is None else t.to(DEV)
        dep, msk = tuple(map(to, smp['depths'])), tuple(map(to, smp['masks']))
        out64 = mo.render(planes.to(DEV, torch.float64), _dec64(dec), ro.to(DEV), rd.to(DEV), opts, None, None,
                          use_triplane=case['use_triplane'], depths=dep, masks=msk, **fl)
        for a, b in zip(out64, out):
            assert a.dtype == torch.float64
            assert (a.cpu() - b.detach().double()).abs().max().item() <= 2e-6, name
        g64 = rbo.render_backward(planes.to(DEV, torch.float64), _dec64(dec), ro.to(DEV), rd.to(DEV), opts, dep, msk,
                                  [g.to(DEV, torch.float64) for g in gw], use_triplane=case['use_triplane'], depth=case['D'], **fl)
        for key, r in zip(PARAMS, ref):
            err = (g64[key].cpu() - r.double()).abs().max().item()
            print(f'pin {name} d_{key}: {err:.2e} of max {r.abs().max().item():.2e}')
            assert err <= 1e-5 * r.abs().max().item(), (name, key, err)


def _merged_rank(k):
    t = torch.cat([k.v['depth_c'], k.v['depth_f']], -1).reshape(k.N * k.M, -1)
    order = torch.sort(t, dim=-1, stable=True)[1]
    return torch.empty_like(order).scatter_(1, order, torch.arange(t.shape[1], device=DEV).expand_as(order).contiguous())


def _case_checks(name, k, cnt, dsig):
    """The property each case exists for, from the kernel's workspace and scratch and the oracle."""
    planes, dec, *_ = _inputs(name)
    bw, D = k.opts['box_warp'], k.D
    if name == 'train_d2':
        R_ = k.N * k.M
        per = torch.cat([dsig[:R_ * k.S].view(R_, k.S), dsig[R_ * k.S:].view(R_, k.Sf)], 1)
        third = ((per != 0) & (_merged_rank(k) >= 64)).any(1).double().mean().item()
        print(f'train_d2: {third:.3f} of the rays carry gradient in the third interval chunk')
        assert third > 0.5, third
    if name == 'train_d3_cull':
        thresh = _cull_sigma(0.5)
        d64 = _dec64(dec)
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
    _skip_small_device(case['H'] * case['W'] >= 256 * 256)
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    k = Kernel(name)
    _, dec, *_ = _inputs(name)
    out64 = mo.render(k.planes64, _dec64(dec), k.ro, k.rd, k.opts, None, None, depths=k.depths(), masks=k.masks(),
                      use_triplane=k.use_triplane, **k.flags)
    for key, a, b in zip(('rgb', 'depth', 'wsum', 'xyz'), k.out, out64):
        err = (a.double() - b).abs().nan_to_num(nan=float('inf')).max().item()
        print(f'{name} forward {key}: max abs err {err:.3e}')
        assert err <= FWD_BAR, (name, key, err)
    del out64
    if case.get('bf16'):
        # the kernel read bf16 texels: its per-sample sigma is within the SIMT decode's error bound of the fp64 decode of the
        # rounded planes, and away from that of the unrounded ones
        xyz, d64 = k.samples(0), _dec64(dec)
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
        ref = Kernel(name, strided=False)
        for a, b in zip(k.out, ref.out):
            assert torch.equal(a, b), 'the strided planes render differently from their contiguous copy'
    worst = {}
    for i, kind in enumerate(UPSTREAM):
        grads = _upstream(kind, k.N, k.M, 50 + i)
        got, dsig = k.backward(grads)
        assert not torch.isnan(dsig).any(), 'a sample was never written by k_ray_backward'
        b64, bars, cnt = _bars(k, grads)
        if i == 0:
            _case_checks(name, k, cnt, dsig)
        w = _compare(f'{name} [{kind}]', got, b64, bars)
        worst.update({(kind, key): r for key, r in w.items()})
        assert max(w.values()) <= 1.0, (name, kind, w)
        assert (got['planes'][_per_channel(cnt) == 0] == 0).all(), 'a texel no tap reaches got a gradient'
        if kind == 'all':
            again, _ = k.backward(grads)
            assert max(_compare(f'{name} [repeat]', again, b64, bars).values()) <= 1.0
            if case.get('strided'):
                contiguous, _ = ref.backward(grads)
                w2 = _compare(f'{name} [contiguous copy]', got, {q: contiguous[q].double() for q in PARAMS}, bars)
                assert max(w2.values()) <= 1.0, w2
            if name == 'train_d2':
                _views_alone(k, grads, b64, bars, cnt)
        if (name, kind) in CONTROLS:
            _negative_controls(k, grads, got, bars)
    print(f'{name}: worst err / bar {max(worst.values()):.4f} ({max(worst, key=worst.get)}); {time.time() - t0:.1f} s, '
          f'peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB')


def _views_alone(k, grads, b64, bars, cnt):
    """Each view rendered and back-propagated alone through ImportanceRenderer under autograd, with the batch's depth-clamp
    bounds injected: its forward equals the batch's bit for bit, its plane gradient the batch oracle's slice within the bar,
    exactly 0 where the view's taps do not reach."""
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(k.case_name)
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
        err, ratio = _ratio(g, b64['planes'][i:i + 1], bars['planes'][i:i + 1])
        print(f'view {i} alone d_planes: max abs err {err:.3e}, worst err / bar {ratio:.4f}')
        assert ratio <= 1.0, (i, ratio)
        assert (g[_per_channel(cnt[i:i + 1]) == 0] == 0).all()


# upstream -> mutated oracles.  Each must miss the kernel by >= 20x its bar.
CONTROLS = {('slabs_d4', 'all')}


def _negative_controls(k, grads, got, bars):
    N, D, H, W = k.N, k.D, k.H, k.W
    swapped = k.planes64.reshape(N, 3, D, 32, H, W).transpose(2, 3).reshape(N, 3, 32 * D, H, W)   # [c*D + d] = [d*32 + c]
    real_taps = rbo.taps
    controls = {
        'slab order d*C + c': lambda: dict(_oracle(k, grads, planes=swapped)),
        'slab coordinate with align_corners=True': lambda: _oracle(k, grads),
        "plane 2's normal from the other plane order": lambda: _oracle(k, grads),
        'dx without the 1/3 plane mean': lambda: _oracle(k, grads, plane_mean=1.0),
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
        worst = max(_ratio(got[key], mut[key], bars[key])[1] for key in PARAMS)
        print(f'negative control "{label}" on {k.case_name}: worst err / bar {worst:.1f}')
        assert worst >= 20, (label, worst)


# ------------------------------------------------------------------------------------------------- density regularisation
GREG_POINTS, GREG_DIST = 1000, 0.004
# 90 % of the pairs read no texel at D = 2 (the slab axis adds a third bound); of the ~400 others, two 0.004-apart points
# differ by under 2e-4 in sigma for a few
GREG_GATE_SHARE = 0.03


def test_density_regularisation_phase_d2():
    """The Greg phase on D = 2 planes: 4 views x (1000 points uniform in [-1, 1]^3 + the same points plus N(0, 0.004^2))
    through run_model under autograd (_PointsFunction: the TRI point decode, then k_sample_backward in point mode) on 256^2
    planes, then the L1 between the two halves' sigma."""
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from tests.helpers import profiled
    _skip_small_device(True)
    t0 = time.time()
    N, H, D = 4, 256, 2
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=48, depth_resolution_importance=48, triplane_depth=D)
    g = torch.Generator().manual_seed(1234)
    planes = torch.randn(N, 3, 32 * D, H, H, generator=g)
    _, dec, *_ = orc.synth_inputs(1234, 1, 1, 2, 0, 2)
    x = torch.rand(N, GREG_POINTS, 3, generator=g) * 2 - 1
    coords = torch.cat([x, x + torch.randn(x.shape, generator=g) * GREG_DIST], 1).to(DEV)
    r = ImportanceRenderer(use_triplane=True)
    d = make_decoder(dec, DEV).requires_grad_(True)
    pg = planes.to(DEV).requires_grad_(True)
    p, _ = r._params(r._shape_probe(pg, opts), N, 0, dict(opts), d, None, None, None)
    assert p.plane_depth == D and p.mlp_mode == _lib.P3D_MLP_FP32_SIMT, (p.plane_depth, p.mlp_mode)
    out, prof = profiled(lambda: r.run_model(pg, d, coords, None, opts))
    assert prof[0] >= 1 and prof[5] == 0, prof
    sigma = out['sigma']
    p64, d64 = planes.to(DEV, torch.float64), _dec64(dec)
    _, s64 = mo.run_model(p64, d64, coords, opts, True)
    err = (sigma.detach().double() - s64).abs().nan_to_num(nan=float('inf')).max().item()
    print(f'Greg D=2: forward sigma max abs err {err:.3e}')
    assert err <= FWD_BAR, err
    diff_k = (sigma[:, :GREG_POINTS] - sigma[:, GREG_POINTS:]).detach()
    diff64 = s64[:, :GREG_POINTS] - s64[:, GREG_POINTS:]
    blank = (diff64 == 0) & (diff_k == 0)
    gated = (diff64.abs() <= 2 * FWD_BAR) & ~blank
    flipped = torch.sign(diff_k.double()) != torch.sign(diff64)
    assert not (flipped & ~gated).any(), 'an L1 sign differs away from 0'
    print(f'Greg D=2: {blank.sum().item()} of {blank.numel()} pairs read no texel; of the rest {gated.sum().item()} lie '
          f'within 2e-4 of 0 (sign gated), {flipped.sum().item()} signs differ from the fp64 ones')
    assert gated.sum().item() <= GREG_GATE_SHARE * (~blank).sum().item()
    loss = torch.nn.functional.l1_loss(sigma[:, :GREG_POINTS], sigma[:, GREG_POINTS:])
    got = torch.autograd.grad(loss, [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    sgn = torch.sign(diff_k[..., 0].double()) / diff_k.numel()
    g_sigma = torch.cat([sgn, -sgn], 1)
    c = 192 + C_TRI
    b64 = rbo.points_backward(p64, d64, coords, g_sigma, opts['box_warp'], depth=D)
    A = rbo.points_backward(p64, d64, coords, g_sigma, opts['box_warp'], mag=True, c=c, depth=D)
    cnt = rbo.texel_counts(coords, torch.zeros_like(coords), (torch.ones(N, 2 * GREG_POINTS, 1, 1, device=DEV), None), H, H,
                           opts['box_warp'], True, D)
    n_cta = -(-N * 2 * GREG_POINTS // KT)
    worst = 0.0
    for key, gk in zip(PARAMS, got):
        kk = _per_channel(cnt).double() if key == 'planes' else float(KT + n_cta)
        e, ratio = _ratio(gk, b64[key], (kk + c) * (U * A[key] + TINY))
        print(f'Greg D=2 d_{key}: max abs err {e:.3e}, worst err / bar {ratio:.4f}')
        worst = max(worst, ratio)
    assert worst <= 1.0, worst
    assert (got[0][_per_channel(cnt) == 0] == 0).all()
    print(f'Greg D=2: {time.time() - t0:.1f} s')


# ------------------------------------------------------------------------------------------------- inference
@pytest.mark.parametrize('bf16', [False, True], ids=['fp32', 'bf16'])
def test_inference_render_at_the_eval_shape(bf16):
    """A 96+96 render of 2 views at 128^2 rays on 256^2 D = 2 planes through ImportanceRenderer with mlp_mode 'auto': the
    SIMT kernels run and the fused slot does not; within 1e-4 of the fp64 oracle (on the bf16-rounded planes for bf16
    storage) fed the depths and masks of the device fp32 oracle."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from tests.helpers import profiled
    _skip_small_device(True)
    t0 = time.time()
    N, R, H, D = 2, 128, 256, 2
    g = torch.Generator().manual_seed(1800 + bf16)
    planes = torch.randn(N, 3, 32 * D, H, H, generator=g)
    _, dec, *_ = orc.synth_inputs(1800, 1, 1, 2, 0, 2)
    opts = dict(orc.DEFAULT_OPTS, triplane_depth=D)
    S, Sf = opts['depth_resolution'], opts['depth_resolution_importance']
    ro, rd = _rays(N, R)
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
    out64 = mo.render(ref.double(), _dec64(dec), ro, rd, opts, None, None, use_triplane=True, depths=smp['depths'],
                      masks=smp['masks'])
    for key, a, b in zip(('rgb', 'depth', 'wsum', 'xyz'), out, out64):
        err = (a.double() - b).abs().nan_to_num(nan=float('inf')).max().item()
        print(f'eval render D=2 {"bf16" if bf16 else "fp32"} {key}: max abs err {err:.3e}')
        assert err <= FWD_BAR, (key, err)
    print(f'eval render: {time.time() - t0:.1f} s')
