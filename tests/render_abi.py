"""The renderer's GPU tests' harness: inputs, the C ABI calls made the way the package makes them, the decoder's error bars
and the training path's kernel, oracle, bars and shared tests, each written once.

The package is imported inside the functions that need it, so the test files that import this module still collect
without the library.
"""
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import render_backward_oracle as rbo, renderer_oracle as orc
from tests.helpers import profiled

DEV = 'cuda:0'
U = U32 = 2.0 ** -24            # unit roundoff of fp32
TINY = 2.0 ** -126              # fp32 underflow: a step whose fp64 value is below the normal range may come out 0 in fp32
U_BF16 = 2.0 ** -8              # unit roundoff of bf16 (8 significant bits, round to nearest)
LOG2E, LN2 = 1.0 / math.log(2.0), math.log(2.0)
MUFU_EX2, MUFU_LG2, MUFU_RCP = 2.0 ** -22, 2.0 ** -22, 2.0 ** -23
ULP2 = 2.0 ** -22               # expf and log1pf: 2 ulp (CUDA C++ Programming Guide, single-precision maximum ulp errors)
BW = orc.DEFAULT_OPTS['box_warp']
BAR = 1e-4                      # the tensor-core 3-pass decode (mlp_mode 1) vs the fp64 oracle
FWD_BAR = 1e-4                  # fp32 SIMT forward vs the fp64 oracle (tests/test_render_backward_gpu.py TIGHT)
KT = 128                        # samples per k_sample_backward CTA (render_backward.cu kT)
PARAMS = ('planes', 'w1', 'b1', 'w2', 'b2')
UPSTREAM = ('rgb', 'depth', 'wsum', 'xyz', 'all', 'bench')
OUTPUTS = ('rgb', 'depth', 'wsum', 'xyz')
PROF_SAMPLE_DECODE = 0          # profile slot (csrc/p3d_common.cuh)


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def skip_unless_free(nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f'needs {nbytes >> 30} GB of free device memory, {free >> 30} GB free')


def dec64(dec):
    return {k: (v.to(DEV, torch.float64) if torch.is_tensor(v) else v) for k, v in dec.items()}


def make_decoder(dec, dev):
    from panic3d_b200.training.triplane import OSGDecoder
    d = OSGDecoder(dec['w1'].shape[1], {'decoder_lr_mul': dec['lr_mul'], 'decoder_output_dim': dec['w2'].shape[0] - 1})
    with torch.no_grad():
        d.net[0].weight.copy_(dec['w1']); d.net[0].bias.copy_(dec['b1'])
        d.net[2].weight.copy_(dec['w2']); d.net[2].bias.copy_(dec['b2'])
    d.set_force_sigmoid(bool(dec['force_sigmoid']))
    return d.to(dev).requires_grad_(False)


def cull_sigma(cull):
    """sigma below which cull_mask removes a sample: 1 - exp(-softplus(sigma - 1)) < cull."""
    return 1.0 + math.log(math.expm1(-math.log1p(-cull)))


def ratio(got, want, bar):
    """Worst |got - want| and worst |got - want| / bar; NaN counts as infinitely wrong, 0 / 0 as exact."""
    err = (got.double() - want).abs().nan_to_num(nan=float('inf'))
    r = err / bar
    r = torch.where(err == 0, torch.zeros_like(r), r)
    return err.max().item(), r.max().item()


class Worst:
    """Worst |got - want| and worst |got - want| / bar of one output over pieces; NaN counts as infinitely wrong."""

    def __init__(self):
        self.err = self.ratio = 0.0

    def add(self, got, want, bar):
        err = (got.double() - want).abs().nan_to_num(nan=float('inf'))
        self.err = max(self.err, err.max().item())
        self.ratio = max(self.ratio, (err / bar).max().item())


# ------------------------------------------------------------------------------------------------- inputs
def spin12(n):
    """(elevation, azimuth) of bench.py's first n spin12 cameras."""
    from panic3d_b200 import cameras
    return cameras.cam60[cameras.camsubs['spin12']][:n]


def rays_at(views, R, dist=1.0):
    """RaySampler's R x R rays of cameras at (elevation, azimuth) in degrees, distance `dist`, fov 30."""
    from panic3d_b200 import cameras
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    lab = torch.stack([cameras.camera_params_to_matrix(elev=e, azim=a, dist=dist, fov=30.0)['camera_label']
                       for e, a in views]).to(DEV)
    ro, rd = RaySampler()(lab[:, :16].view(-1, 4, 4), lab[:, 16:25].view(-1, 3, 3), R)
    return ro.float().contiguous(), rd.float().contiguous()


def planes_and_decoder(seed, n, h, w):
    rng = np.random.default_rng(seed)
    planes = torch.from_numpy(rng.standard_normal((n, 3, 32, h, w), dtype=np.float32))
    _, dec, *_ = orc.synth_inputs(seed, 1, 1, 2, 0, 2)
    return planes, dec


def box_rays(seed, n, m):
    """Origins on the unit sphere aimed at random points of the box: with t in [0.5, 1.5] the samples cross the box and
    leave it on the far side."""
    g = torch.Generator().manual_seed(seed)
    o = F.normalize(torch.randn(n, m, 3, generator=g), dim=-1)
    target = (torch.rand(n, m, 3, generator=g) * 2 - 1) * 0.3
    return o.contiguous(), F.normalize(target - o, dim=-1).contiguous()


def upstream(kind, N, M, seed):
    """Upstream gradients (rgb, depth, wsum, xyz): one output's alone, all four, bench.py's loss, or a wsum of ones."""
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


# ------------------------------------------------------------------------------------------------- the C ABI
def workspace_views(ws, N, M, S, Sf):
    """workspace_layout (c_api.cu:103) restated: bounds, depth_c, sigma_c, rgb_c, depth_f, sigma_f, rgb_f, ray_t0, ray_t1,
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


def render_forward(p, planes_cl, wt, ro, rd, u_c, u_f, ws, out):
    """p3d_render_forward as _RenderFunction calls it; u_c / u_f None: the kernel draws its own jitter."""
    from panic3d_b200 import _lib
    _lib.check(_lib.lib().p3d_render_forward(
        C.byref(p), planes_cl.data_ptr(), *[t.data_ptr() for t in wt], ro.data_ptr(), rd.data_ptr(), _lib.ptr(u_c),
        _lib.ptr(u_f), ws.data_ptr(), ws.numel(), *[o.data_ptr() for o in out], _lib.stream_ptr(planes_cl.device)))


def decode_points_call(p, planes_cl, wt, coords, rgb, sigma):
    """p3d_decode_points of coords (N,K,3) contiguous into rgb (N,K,32) and sigma."""
    from panic3d_b200 import _lib
    _lib.check(_lib.lib().p3d_decode_points(
        C.byref(p), planes_cl.data_ptr(), *[t.data_ptr() for t in wt], coords.data_ptr(), coords.shape[1], rgb.data_ptr(),
        sigma.data_ptr(), _lib.stream_ptr(planes_cl.device)))


def twice(call, outs, slot=None, prefill=(), checks_later=False, int_fill=0xFF):
    """call() twice, `outs` and `prefill` refilled before each run (floats with NaN, integers with int_fill), so an
    element the call never writes is NaN.  With `slot`, each run is exactly one launch in that profile slot.  Returns both runs'
    copies of `outs`; unless checks_later (the caller compares the values first: a kernel that reads memory it never
    wrote may still repeat itself), the second must equal the first bit for bit."""
    runs = []
    for _ in range(2):
        for t in (*outs, *prefill):
            if t is not None:
                t.fill_(float('nan') if t.is_floating_point() else int_fill)
        torch.cuda.synchronize()
        _, prof = profiled(call)
        if slot is not None:
            assert prof[slot] == 1, prof
        runs.append([None if t is None else t.clone() for t in outs])
    if not checks_later:
        repeats(*runs)
    return runs


def repeats(first, second, names=None, nan=False):
    """Two runs bit-identical, output by output; with nan, no NaN in the first (an element never written, or read before
    it landed)."""
    for i, (a, b) in enumerate(zip(first, second)):
        key = i if names is None else names[i]
        if nan:
            assert not torch.isnan(a).any(), f'{key} has NaN (an element never written, or read before it landed)'
        assert (a is None and b is None) or torch.equal(a, b), f'two runs differ in {key}'


# ------------------------------------------------------------------------------------------------- the tensor-core decode
def renderer(bf16, mode):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    r = ImportanceRenderer(use_triplane=True)
    r.planes_bf16 = bf16
    r.mlp_mode = mode
    return r


def decode_params(r, cl, decoder, n_points):
    """p3d_render_params as run_model / query_volume make them; 'auto' must pick the tensor-core decode for them."""
    from panic3d_b200 import _lib
    mode, r.mlp_mode = r.mlp_mode, 'auto'
    p, _ = r._params(cl, cl.shape[0], 0, dict(orc.DEFAULT_OPTS), decoder, None, None, None, n_points=n_points)
    assert p.mlp_mode == _lib.P3D_MLP_TC_3XBF16
    r.mlp_mode = mode
    p, wts = r._params(cl, cl.shape[0], 0, dict(orc.DEFAULT_OPTS), decoder, None, None, None, n_points=n_points)
    assert p.mlp_mode == mode
    return p, [t.detach().float().contiguous() for t in wts]


def decode_points(x, dec, coords, mode, bf16=False):
    """p3d_decode_points on planes `x` (device, any layout) -> rgb (N,K,32), sigma (N,K,1), twice: one launch in the
    decode slot each, bit-identical."""
    N, K, _ = coords.shape
    r = renderer(bf16, mode)
    decoder = make_decoder(dec, DEV)
    with torch.no_grad(), torch.cuda.device(DEV):
        cl = r._planes_cl(x)
        p, wt = decode_params(r, cl, decoder, N * K)
        c = coords.to(DEV).contiguous()
        rgb = torch.empty((N, K, 32), device=DEV)
        sigma = torch.empty((N, K, 1), device=DEV)
        return twice(lambda: decode_points_call(p, cl, wt, c, rgb, sigma), [rgb, sigma], PROF_SAMPLE_DECODE)[0]


def single_pass_bars(p64, d64, x64):
    """Per-point bars (rgb (N,K,32), sigma (N,K,1)) for mlp_mode 2, from the roundings the kernel makes.

    The kernel decodes in base 2 (fused_common.cuh stage_w1_biases / stage_w2): the A1 row a is the sum of the three
    planes' bilinear features, W1' = W1 g1 log2(e) / 3, b1' = b1 g1' log2(e), x' = a W1'^T + b1', h' = softplus2(x') =
    log2(1 + 2^x') = softplus(x) log2(e); sigma = h' . (W2_0 g2 ln 2) + b2_0, colour = rcp(1 + ex2(h' . (-W2_c g2) + b2c')).
    Single pass multiplies only the bf16 `hi` halves (split2 / split1): a, W1', h' and W2' are each rounded to bf16, u =
    2^-8 relative each, so a product of two rounded operands is off by at most e = 2u + u^2 of |product|:
      layer 1:  |dx'_j| <= e (|a| . |W1'_j|)
      hidden:   softplus2' = sigmoid <= 1, so |dh'_j| <= |dx'_j|; the rounded h'~ times rounded W2' is then off by
                dh_j = e |h'_j| + (1 + e) |dx'_j| per unit |W2'|
      sigma:    ln 2 * sum_j |W2_0j g2| dh_j
      colour:   |d(1.002 s - 0.001) / d logit'| <= 1.002 ln 2 / 4, times sum_j |W2_cj g2| dh_j
    plus the fp32 / MUFU term: everything mode 1 also does (fp32 gather and accumulation, ex2 / lg2 / rcp.approx, the
    biases), which mode 1's bar of 1e-4 covers."""
    C_ = d64['w1'].shape[1]
    lr = d64.get('lr_mul', 1.0)
    g1, g2 = lr / math.sqrt(C_), lr / math.sqrt(d64['w2'].shape[1])
    a = orc.sample_planes(p64, x64, BW, True).sum(1)                          # (N,K,C)
    w1p = d64['w1'] * (g1 * LOG2E / 3)
    x2 = a @ w1p.t() + d64['b1'] * (lr * LOG2E)
    h2 = F.softplus(x2 * LN2) * LOG2E
    e = 2 * U_BF16 + U_BF16 ** 2
    dh = e * h2.abs() + (1 + e) * e * (a.abs() @ w1p.abs().t())
    w2 = (d64['w2'] * g2).abs()
    return 1.002 * LN2 / 4 * (dh @ w2[1:].t()) + BAR, LN2 * (dh @ w2[:1].t()) + BAR


def three_pass_bars(p64, d64, x64, force_sigmoid=False, use_triplane=True):
    """Per-point bars (rgb (N,K,32), sigma (N,K,1)) for mlp_mode 1 (3-pass split bf16), at exact fp32 point coordinates.
    The error of the coordinates themselves (ray_point, the grid transform) is the caller's: it moves the point.

    In the base-2 form of `single_pass_bars`, with u = 2^-8 (bf16) and v = 2^-24 (fp32):
      gather    A1 = sum over 3 planes x 4 taps of w t (one fp32 fma chain, weights from three roundings):
                |dA1_c| <= 16 v sum |w| |t_c|
      split     an operand x = hi + lo + r, |lo| <= u |x|, |r| <= u |lo| <= u^2 |x|; the kernel forms hi hi + hi lo + lo hi
                and drops lo lo, r_a b and a r_b: e3 = 3 u^2 (+ O(u^3)) of |a| |b| per product
      accumulation  fp32 in the wgmma, 3K products: <= 3K v of sum |a| |b| (K = 32 for layer 1, 64 for layer 2)
      staging   W1' and the biases carry <= 3 roundings (v each) of their own magnitude, W2' <= 2
      layer 1   |dx'_j| <= (e3 + 100 v) sum_c |A1_c| |W1'_jc| + sum_c |dA1_c| |W1'_jc| + 4 v (|b1'_j| + |x'_j|)
      hidden    h' = max(x', 0) + lg2(1 + ex2(-|x'|)), slope <= 1: |dh'_j| <= |dx'_j| + (ex2 + 2 v) / ln 2 + lg2 + v |h'_j|
                with the MUFU bounds of the PTX ISA (ex2.approx.f32: relative error 2^-22, lg2.approx.f32: absolute 2^-22,
                rcp.approx.f32: 1 ulp = relative 2^-23)
      layer 2   |dl_k| <= (e3 + 200 v) sum_j |h'_j| |W2'_kj| + sum_j |dh'_j| |W2'_kj| + 3 v (|b2'_k| + |l_k|)
      sigma     dl_0 (the sigma row is the plain sum)
      colour    s = rcp(1 + ex2(l')): |ds| <= s (1 - s) (ln 2 |dl| + ex2) + s (v + rcp), times 1.002 for the colour map
    """
    C_ = d64['w1'].shape[1]
    lr = d64.get('lr_mul', 1.0)
    g1, g2 = lr / math.sqrt(C_), lr / math.sqrt(d64['w2'].shape[1])
    a = orc.sample_planes(p64, x64, BW, use_triplane).sum(1)                  # (N,K,C)
    # sum over planes and taps of |w| |t|: the bilinear gather of |planes| (weights are non-negative)
    a_abs = orc.sample_planes(p64.abs(), x64, BW, use_triplane).sum(1)
    da = 16 * U32 * a_abs
    e3 = 3 * U_BF16 ** 2
    w1p = d64['w1'] * (g1 * LOG2E / 3)
    b1p = d64['b1'] * (lr * LOG2E)
    x2 = a @ w1p.t() + b1p
    dx = (e3 + 100 * U32) * (a.abs() @ w1p.abs().t()) + da @ w1p.abs().t() + 4 * U32 * (b1p.abs() + x2.abs())
    h2 = F.softplus(x2 * LN2) * LOG2E
    dh = dx + (MUFU_EX2 + 2 * U32) / LN2 + MUFU_LG2 + U32 * h2.abs()
    w2p = d64['w2'] * g2
    w2p = torch.cat([w2p[:1] * LN2, -w2p[1:]], 0)                             # sigma row, then the colour rows
    b2p = d64['b2'] * lr
    b2p = torch.cat([b2p[:1], -b2p[1:] * LOG2E], 0)
    lg = h2 @ w2p.t() + b2p
    dl = (e3 + 200 * U32) * (h2.abs() @ w2p.abs().t()) + dh @ w2p.abs().t() + 3 * U32 * (b2p.abs() + lg.abs())
    s = torch.sigmoid(-lg[..., 1:] * LN2)
    ds = s * (1 - s) * (LN2 * dl[..., 1:] + MUFU_EX2) + s * (U32 + MUFU_RCP)
    return (ds if force_sigmoid else 1.002 * ds), dl[..., :1]


def simt_bars(p64, d64, x64, force_sigmoid=False, use_triplane=True):
    """Per-point bars (rgb (N,K,32), sigma (N,K,1)) for mlp_mode 0 (k_sample_decode, all fp32), at exact fp32 point
    coordinates (their rounding, and the grid transform's, are the caller's, as for `three_pass_bars`).  v = 2^-24:
      gather    per plane 4 fmaf of taps and weights that carry <= 2 roundings each, then (f0 + f1 + f2) / 3 in 3 roundings:
                |da_c| <= 12 v mean over planes of sum |w| |t_c|
      layer 1   W1 g1 and b1 lr each rounded once, then 32 fmaf from the bias: |dx_j| <= 34 v (|a| . |W1'_j| + |b1'_j|) +
                |da| . |W1'_j|
      hidden    softplus_t = log1pf(expf(x)), slope <= 1; expf and log1pf 2 ulp each: |dh_j| <= |dx_j| + 2^-22 (1 + |h_j|)
      layer 2   64 fmaf from the rounded bias: |do_k| <= 66 v (|h| . |W2'_k| + |b2'_k|) + |dh| . |W2'_k|
      sigma     do_0
      colour    s = 1 / (1 + expf(-o)) (the division and the add rounded): |ds| <= s (1 - s) (|do| + 2^-22) + 2 v s, then
                1.002 s - 0.001 in two roundings: 1.002 |ds| + v (1.002 s + |colour|)"""
    C_ = d64['w1'].shape[1]
    lr = d64.get('lr_mul', 1.0)
    g1, g2 = lr / math.sqrt(C_), lr / math.sqrt(d64['w2'].shape[1])
    a = orc.sample_planes(p64, x64, BW, use_triplane).mean(1)                 # (N,K,C)
    da = 12 * U32 * orc.sample_planes(p64.abs(), x64, BW, use_triplane).mean(1)
    w1p, b1p = (d64['w1'] * g1).abs(), (d64['b1'] * lr).abs()
    x = a @ (d64['w1'] * g1).t() + d64['b1'] * lr
    dx = 34 * U32 * (a.abs() @ w1p.t() + b1p) + da @ w1p.t()
    h = F.softplus(x)
    dh = dx + ULP2 * (1 + h.abs())
    w2p, b2p = (d64['w2'] * g2).abs(), (d64['b2'] * lr).abs()
    o = h @ (d64['w2'] * g2).t() + d64['b2'] * lr
    do = 66 * U32 * (h.abs() @ w2p.t() + b2p) + dh @ w2p.t()
    s = torch.sigmoid(o[..., 1:])
    ds = s * (1 - s) * (do[..., 1:] + ULP2) + 2 * U32 * s
    if not force_sigmoid:
        ds = 1.002 * ds + U32 * (1.002 * s + (1.002 * s - 0.001).abs())
    return ds, do[..., :1]


# ------------------------------------------------------------------------------------------------- per-ray bars of a render
class Arith:
    """The rounding model of one renderer kernel, for `ray_oracle`:
      sample_bars(p64, d64, x64, force_sigmoid, use_triplane) -> per-sample (rgb, sigma) bars of the decoder;
      alpha = (e_exp, e_sp_rel, e_sp_abs): alpha = 1 - exp(-softplus(smid) dt) with exp relative error e_exp and softplus
              error e_sp_rel softplus + e_sp_abs (see `alpha_bar`);
      cdf(S) -> the bar of every importance cdf entry of a ray with S coarse samples."""

    def __init__(self, sample_bars, alpha, cdf):
        self.sample_bars, self.alpha, self.cdf = sample_bars, alpha, cdf


# the fused kernel, mode 1 / mode 2 (tests/test_render_fused_paths_gpu.py): ex2.approx / lg2.approx in the interval alpha
# and the softplus, and (2 S + 40) v on every cdf entry (fp32 weights, their sum, the division and the scans)
FUSED_ALPHA = (MUFU_EX2, 4 * MUFU_EX2, 2 * MUFU_EX2)
FUSED_CDF = lambda S: (2 * S + 40) * U32
FUSED_MODE1 = Arith(three_pass_bars, FUSED_ALPHA, FUSED_CDF)
FUSED_MODE2 = Arith(lambda p64, d64, x64, force_sigmoid, use_triplane: single_pass_bars(p64, d64, x64), FUSED_ALPHA, FUSED_CDF)


def simt_cdf(S):
    """The fp32 SIMT importance cdf (render_device.cuh importance_ray), nb = S - 3 bins in nc = ceil(nb / 32) warp chunks:
    the coarse weights carry ~(5 + nc) v of their transmittance scan, each pooled pdf value 3 v (pooled add, + 0.01,
    + 1e-5), the total (nc + 5) v (8 lane adds, 5 butterflies), the division v: (2 nc + 14) v relative on every pdf,
    so as much absolute on a cdf entry <= 1; the in-chunk scan adds <= 5 roundings and every chunk's carry one more, of
    partial sums <= 1: 6 nc v.  Doubled for the orders this does not follow exactly."""
    nc = -(-(S - 3) // 32)
    return 2 * (8 * nc + 14) * U32


# k_sample_decode / k_ray_importance / k_ray_composite: expf (2 ulp) and softplus_t = log1pf(expf(x)) (2 ulp each)
SIMT = Arith(simt_bars, (ULP2, ULP2, ULP2), simt_cdf)


def alpha_bar(sig, t, e_exp, e_sp_rel, e_sp_abs):
    """Bound of a kernel's alpha error per interval, from the fp64 sigma and depths (..,L,1): the exp's relative error
    on 1 - alpha, the rounding of 1 - exp, and, scaled by (1 - alpha) dt, the softplus error, the rounding of smid =
    (s_a + s_b) / 2 - 1 through its slope sigmoid(smid), and 6 v of softplus dt for dt and the product."""
    dt = t[..., 1:, :] - t[..., :-1, :]
    smid = (sig[..., 1:, :] + sig[..., :-1, :]) / 2 - 1
    sp = F.softplus(smid)
    alpha = 1 - torch.exp(-sp * dt)
    spread = sig[..., 1:, :].abs() + sig[..., :-1, :].abs() + 2
    return (e_exp * (1 - alpha) + U32 * alpha +
            (1 - alpha) * (dt.abs() * (e_sp_rel * sp + e_sp_abs + torch.sigmoid(smid) * U32 * spread) + 6 * U32 * sp * dt.abs()))


def render_graph(ro, rd, d_c, u_f, c0, f0, white, leaves, importance=orc.importance_depths, left=False):
    """The oracle's render of a chunk of rays as a function of zero-valued perturbation leaves.  c0 / f0: (sigma masked,
    colour, slope of sigma, slope of colour, mask) of the coarse samples and of the fine samples at the unperturbed fine
    depths f0['t'] (f0 None: no fine pass).  `importance(z, w, u, cdf_eps=)` draws the fine depths.  Returns the
    outputs (m, 37) and the intermediate values the bars need."""
    e = leaves
    t_c = d_c + e['t_c']
    s_c = c0['sig'] + torch.where(c0['mask'], 0, c0['g_sig']) * e['t_c'] + e['s_c']
    col_c = c0['rgb'] + c0['g_rgb'] * e['t_c'] + e['c_c']
    x_c = ro[:, None] + t_c * rd[:, None]
    inf = torch.tensor(float('inf'), device=DEV, dtype=torch.float64)
    if f0 is None:
        out, depth, w = orc.march(torch.cat([col_c, x_c], -1)[None], s_c[None], t_c[None], white, -inf, inf,
                                  alpha_eps=e['a'][None], left_colours=left)
        o = torch.cat([out[0, :, :32], depth[0], w[0].sum(1), out[0, :, 32:]], -1)
        return o, dict(t_all=t_c, sig=s_c, col=torch.cat([col_c, x_c], -1), w=w[0], t_f=None)
    _, _, w = orc.march(torch.cat([col_c, x_c], -1)[None], s_c[None], t_c[None], white, alpha_eps=e['a_c'][None])
    t_f = importance(t_c[..., 0], w[0, ..., 0], u_f, cdf_eps=e['cdf'])[..., None] + e['t_f']
    dtf = t_f - f0['t']
    s_f = f0['sig'] + torch.where(f0['mask'], 0, f0['g_sig']) * dtf + e['s_f']
    col_f = f0['rgb'] + f0['g_rgb'] * dtf + e['c_f']
    x_f = ro[:, None] + t_f * rd[:, None]
    t_all = torch.cat([t_c, t_f], -2)
    order = torch.sort(t_all.detach(), dim=-2, stable=True)[1]
    t_all = torch.gather(t_all, -2, order)
    col = torch.gather(torch.cat([torch.cat([col_c, x_c], -1), torch.cat([col_f, x_f], -1)], -2), -2,
                       order.expand(-1, -1, 35))
    sig = torch.gather(torch.cat([s_c, s_f], -2), -2, order)
    out, depth, w = orc.march(col[None], sig[None], t_all[None], white, -inf, inf, alpha_eps=e['a'][None], left_colours=left)
    o = torch.cat([out[0, :, :32], depth[0], w[0].sum(1), out[0, :, 32:]], -1)
    return o, dict(t_all=t_all, sig=sig, col=col, w=w[0], t_f=t_f)


def zero_leaves(m, S, Sf, grad=False):
    """The perturbation leaves of `render_graph` for m rays of S coarse and Sf fine samples: coarse depth, sigma and
    colour, coarse alpha, cdf, fine depth, sigma and colour, merged alpha."""
    L = S + Sf
    shapes = dict(t_c=(m, S, 1), s_c=(m, S, 1), c_c=(m, S, 32))
    if Sf:
        shapes.update(a_c=(m, S - 1, 1), cdf=(m, S - 2), t_f=(m, Sf, 1), s_f=(m, Sf, 1), c_f=(m, Sf, 32))
    shapes['a'] = (m, L - 1, 1)
    return {k: torch.zeros(s, device=DEV, dtype=torch.float64, requires_grad=grad) for k, s in shapes.items()}


def decoded(arith, p64, d64, opts, use_triplane, xyz, rd_s, ray_point=True):
    """sigma (1,K,1) and colour (1,K,32) in fp64 at points xyz (1,K,3) of one view's planes p64; their slopes along the
    ray direction rd_s (central differences); their bars: the decoder's (arith) plus the points' fp32 rounding (ray_point
    and the grid transform: 4 v (|x| + box) per coordinate) times one-sided slopes.  ray_point False: points given
    exactly in fp32 (p3d_decode_points), so only the grid transform rounds.  bilinear_footprint forms
    fx = ((x cs + 1) W - 1) / 2 with cs = 2 / box rounded: 2 v |gx| + v (|gx| + 1) before the factor W / 2 and
    v (|gx| + 1) W after it, which is v (5 |x| + 2.5 box) in units of x: 5 v (|x| + box / 2)."""
    run = lambda x: orc.run_model(p64, d64, x, opts, use_triplane)
    rgb, sig = run(xyz)
    b_rgb, b_sig = arith.sample_bars(p64, d64, xyz, bool(d64.get('force_sigmoid', False)), use_triplane)
    h = 1e-7
    beta_x = 4 * U32 * (xyz.abs() + BW) if ray_point else 5 * U32 * (xyz.abs() + BW / 2)
    g_sig, g_rgb = torch.zeros_like(sig), torch.zeros_like(rgb)
    for i in range(3):
        e = torch.zeros_like(xyz)
        e[..., i] = h
        rp, sp = run(xyz + e)
        rm, sm = run(xyz - e)
        b_sig = b_sig + torch.maximum((sp - sig).abs(), (sig - sm).abs()) / h * beta_x[..., i:i + 1]
        b_rgb = b_rgb + torch.maximum((rp - rgb).abs(), (rgb - rm).abs()) / h * beta_x[..., i:i + 1]
        g_sig = g_sig + (sp - sm) / (2 * h) * rd_s[..., i:i + 1]
        g_rgb = g_rgb + (rp - rm) / (2 * h) * rd_s[..., i:i + 1]
    return sig, rgb, g_sig, g_rgb, b_sig, b_rgb


def ray_oracle(arith, p64, d64, opts, flags, use_triplane, ro, rd, d_c, t0, t1, u_f, Sf, with_bars=True, fine_bars=False):
    """The fp64 oracle's render of m rays of one view (ro, rd (m,3) fp64, coarse depths d_c (m,S,1), coarse limits t0, t1
    (m,1), fine uniforms u_f (m,Sf)) with a bar per ray and output component for a kernel of rounding model `arith`.

    The kernel's error is bounded per sample and propagated to first order through the oracle:
      * per sample: arith.sample_bars plus the point's fp32 rounding times the sigma and colour slopes (`decoded`);
      * per depth: coarse 16 v (|t| + |t0| + |t1|); fine 8 v (|t| + |t1 - t0|) for the lerp, and arith.cdf(S) on every
        cdf entry;
      * per interval alpha: `alpha_bar` with arith.alpha, in both marches.
    The render is restated as a graph of these perturbations (zero-valued leaves, `render_graph`): the coarse sigma /
    colour / depth perturbations move the coarse weights, the importance depths (kept differentiable) and, through each
    fine sample's slope along its ray, the fine sigma and colour.  For each output component o_k of a ray (32 rgb, depth,
    wsum, 3 xyz), one vector-Jacobian product per component over the chunk (rays are independent) gives
        bar_k = 2 (sum over leaves |do_k / d leaf| beta_leaf) + floor_k
    floor_k covers the roundings of the sums that form the output ((L + 8) v relative on each weight and on every partial
    sum; L = S + Sf).  The factor 2 covers second-order terms.  A fine depth's own bar (`fine_move`, (m, Sf)) is the same
    sum over the leaves that move it, doubled.
    Masks: a cull, binarize or crop decision is a jump.  A ray is `near` when one of its samples' fp64 sigma lies within
    its sigma bar (plus the rounding of the host's sigma_cull) of the threshold, or its |x| / |z| within the position bar
    of the crop bound.

    Returns (res, ctx): res has o (m,37), t_max, t_min, illdef (rays whose importance pdf is not positive: their cdf is not
    monotone and searchsorted's result depends on its probe order) and, with_bars, bar (m,37), near (m,), cull_share,
    fine_move; ctx has what mutated oracles need: samples(t), c0, f0, w (coarse weights), zero leaves, white."""
    m, S = d_c.shape[:2]
    white = bool(opts.get('white_back', False))

    def samples(t):
        xyz = (ro[:, None] + t * rd[:, None]).reshape(1, -1, 3)
        rd_s = rd[:, None].expand(-1, t.shape[1], -1).reshape(1, -1, 3)
        sig, rgb, g_sig, g_rgb, b_sig, b_rgb = decoded(arith, p64, d64, opts, use_triplane, xyz, rd_s)
        sig_m = orc.apply_masks(sig, xyz, BW, flags.get('triplane_crop'), flags.get('cull_clouds'), flags.get('binarize_clouds'))
        mask = sig_m != sig
        r = lambda x: x.reshape(m, t.shape[1], -1)
        return dict(sig=r(sig_m), raw=r(sig), rgb=r(rgb), g_sig=r(g_sig), g_rgb=r(g_rgb), b_sig=r(torch.where(mask, 0, b_sig)),
                    b_sig_raw=r(b_sig), g_sig_raw=r(g_sig), b_rgb=r(b_rgb), mask=r(mask), xyz=r(xyz), t=t)

    c0 = samples(d_c)
    w = t_f0 = f0 = None
    illdef = torch.zeros(m, dtype=torch.bool, device=DEV)
    if Sf:
        _, _, w = orc.march(torch.cat([c0['rgb'], c0['xyz']], -1)[None], c0['sig'][None], d_c[None], white)
        w = w[0, ..., 0]
        t_f0 = orc.importance_depths(d_c[..., 0], w, u_f)[..., None]
        wp = F.avg_pool1d(F.max_pool1d(w[:, None], 2, 1, padding=1), 2, 1)[:, 0] + 0.01
        illdef = (wp[:, 1:-1] + 1e-5).min(1).values <= 1e-6
        f0 = samples(t_f0)
    zero = zero_leaves(m, S, Sf)
    o, mid = render_graph(ro, rd, d_c, u_f, c0, f0, white, zero)
    res = dict(o=o, t_max=mid['t_all'].max(), t_min=mid['t_all'].min(), illdef=illdef, t_f=t_f0)
    ctx = dict(samples=samples, c0=c0, f0=f0, w=w, zero=zero, white=white)
    if not with_bars:
        return res, ctx
    leaves = zero_leaves(m, S, Sf, grad=True)
    o, mid = render_graph(ro, rd, d_c, u_f, c0, f0, white, leaves)
    # beta of every leaf
    L = S + Sf
    span = (t1 - t0).abs()[:, None]
    beta = dict(t_c=16 * U32 * (d_c.abs() + t0.abs()[:, None] + t1.abs()[:, None]), s_c=c0['b_sig'], c_c=c0['b_rgb'],
                a=alpha_bar(mid['sig'], mid['t_all'], *arith.alpha))
    if Sf:
        beta.update(a_c=alpha_bar(c0['sig'], d_c, *arith.alpha), cdf=torch.full((m, S - 2), arith.cdf(S), device=DEV, dtype=torch.float64),
                    t_f=8 * U32 * (t_f0.abs() + span), s_f=f0['b_sig'], c_f=f0['b_rgb'])
    names = list(leaves)
    bar = torch.zeros(m, 37, device=DEV, dtype=torch.float64)
    for k in range(37):
        gs = torch.autograd.grad(o[:, k].sum(), [leaves[n] for n in names], retain_graph=True, allow_unused=True)
        for n, gk in zip(names, gs):
            if gk is not None:
                bar[:, k] += (gk.abs() * beta[n]).reshape(m, -1).sum(1)
    fine_move = None
    if Sf and (flags or fine_bars):                 # the fine depths' own bars, for the mask borders and the depth check
        fine_move = torch.zeros(m, Sf, device=DEV, dtype=torch.float64)
        tf = mid['t_f'][..., 0]
        moving = ('t_c', 's_c', 'a_c', 'cdf', 't_f')
        for f in range(Sf):
            gs = torch.autograd.grad(tf[:, f].sum(), [leaves[n] for n in moving], retain_graph=True, allow_unused=True)
            for n, gk in zip(moving, gs):
                if gk is not None:
                    fine_move[:, f] += (gk.abs() * beta[n]).reshape(m, -1).sum(1)
        fine_move = 2 * fine_move
    res['fine_move'] = fine_move
    # floors: the roundings of the sums that form each output
    wts = mid['w'][..., 0].detach()
    W = wts.sum(1)
    tm = (mid['t_all'][:, 1:] + mid['t_all'][:, :-1])[..., 0] / 2
    om = torch.cat([wts[:, :1] * 0, wts], 1) / 2 + torch.cat([wts, wts[:, :1] * 0], 1) / 2
    rel = 2 * (L + 8) * U32
    fW = rel * W
    fD = rel * (wts * tm.abs()).sum(1)
    floor = torch.zeros_like(bar)
    floor[:, :32] = 2 * rel * (om[..., None] * (mid['col'][..., :32].detach().abs() + 0.002)).sum(1) + (2 * fW[:, None] if white else 0) + 8 * U32
    dep = (wts * tm).sum(1) / W
    floor[:, 32] = (fD + dep.abs() * fW) / W + U32 * dep.abs()
    floor[:, 33] = fW
    floor[:, 34:] = 2 * (ro.abs() * fW[:, None] + rd.abs() * fD[:, None] + 3 * U32 * (ro.abs() * W[:, None] + rd.abs() * (wts * tm).sum(1)[:, None])
                         + (fW[:, None] if white else 0)) + 4 * U32
    res['bar'] = 2 * bar + floor
    # rays with a sample within its bar of a jump
    near = torch.zeros(m, dtype=torch.bool, device=DEV)
    smps = ((c0, beta['t_c'][..., 0]),) + (((f0, fine_move),) if Sf else ())
    if flags.get('cull_clouds') or flags.get('binarize_clouds'):
        thr = cull_sigma(flags.get('cull_clouds') or flags.get('binarize_clouds'))
        for smp, move in smps:
            cropped = orc.crop_mask(smp['xyz'].reshape(1, -1, 3), flags['triplane_crop'], BW).reshape(m, -1) if flags.get('triplane_crop') \
                else torch.zeros(m, smp['t'].shape[1], dtype=torch.bool, device=DEV)
            # the slope of the unmasked sigma along the ray, times how far the sample's depth may move
            g_raw = smp['g_sig_raw'][..., 0].abs()
            b = smp['b_sig_raw'][..., 0] + g_raw * move + 2 * U32 * abs(thr) + 1e-12
            near |= (~cropped & ((smp['raw'][..., 0] - thr).abs() <= b)).any(1)
    if flags.get('triplane_crop'):
        lim = BW / 2 - flags['triplane_crop']
        for smp, move in smps:
            bx = 4 * U32 * (smp['xyz'].abs() + BW) + rd.abs()[:, None] * move[..., None] + 2 * U32 * lim
            near |= ((smp['xyz'][..., [0, 2]].abs() - lim).abs() <= bx[..., [0, 2]]).any(-1).any(1)
    res['near'] = near
    res['cull_share'] = None
    if flags.get('cull_clouds'):
        unc = ~orc.crop_mask(c0['xyz'].reshape(1, -1, 3), flags['triplane_crop'], BW).reshape(m, -1) if flags.get('triplane_crop') else \
            torch.ones(m, S, dtype=torch.bool, device=DEV)
        res['cull_share'] = ((c0['mask'][..., 0] & unc).sum().item(), unc.sum().item())
    return res, ctx


# ------------------------------------------------------------------------------------------------- the training path
def per_channel(cnt, D):
    """Tap counts (N,3,H,W) at D = 1, (N,3,D,H,W) above -> (N,3,32 D,H,W), the planes' indexing (channel c D + d)."""
    N, P, H, W = cnt.shape[0], cnt.shape[1], cnt.shape[-2], cnt.shape[-1]
    return cnt.view(N, P, 1, D, H, W).expand(N, P, 32, D, H, W).reshape(N, P, 32 * D, H, W)


class TrainKernel:
    """One forward of the training path (kept with its workspace) and any number of backwards, through the C ABI as
    _RenderFunction calls it: p3d_render_forward in fp32 SIMT mode into NaN outputs and a 0xFF workspace, twice and
    bit-identical, then p3d_render_backward into NaN-prefilled scratch.  `inputs` are (planes (N,3,32 D,H,W), dec, opts,
    ro, rd, u_c, u_f); case keys D (slabs, default 1), flags, eg3d, strided and bf16 (D > 1)."""

    def __init__(self, case, inputs, strided=None):
        from panic3d_b200 import _lib
        from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
        planes, dec, opts, ro, rd, u_c, u_f = inputs
        strided = case.get('strided', False) if strided is None else strided
        bf16 = case.get('bf16', False)
        N, _, CD, H, W = planes.shape
        D = case.get('D', 1)
        M = ro.shape[1]
        self.case, self.dec, self.opts, self.ro, self.rd, self.D = case, dec, opts, ro, rd, D
        self.N, self.M, self.S, self.Sf, self.H, self.W = N, M, case['S'], case['Sf'], H, W
        self.flags = case.get('flags', {})
        self.use_triplane = not case.get('eg3d')
        self.planes_ref = planes.bfloat16().float() if bf16 else planes       # what the kernel reads
        self.planes64 = self.planes_ref.to(DEV, torch.float64)
        r = ImportanceRenderer(use_triplane=self.use_triplane)
        self.decoder = make_decoder(dec, DEV)
        p, wts = r._params(r._shape_probe(planes, opts), N, M, opts, self.decoder, self.flags.get('triplane_crop'),
                           self.flags.get('cull_clouds'), self.flags.get('binarize_clouds'))
        # (N,3,D,H,W,C) texels: feature c of slab d is input channel c D + d; one-slab planes are (N,3,H,W,C)
        cl = planes.to(DEV).reshape(N, 3, CD // D, D, H, W).permute(0, 1, 3, 4, 5, 2).contiguous()
        if D == 1:
            cl = cl[:, :, 0]
        else:
            assert p.plane_depth == D
        if strided:
            # 64-channel texels sliced to their first 32, and one padding row after each plane's slab stack; NaN wherever
            # the kernel must not read
            buf = torch.full((N, 3, D * H + 1, W, 64), float('nan'), device=DEV)
            buf[:, :, :D * H, :, :32] = cl.reshape(N, 3, D * H, W, 32)
            cl = buf[:, :, :D * H, :, :32]
        elif bf16:
            cl = cl.to(torch.bfloat16)
        p.stride_view, p.stride_plane, *_, p.stride_row, p.stride_col, _ = cl.stride()
        if strided:
            assert p.stride_plane > D * H * p.stride_row and p.stride_col == 64
        self.planes_cl = cl
        p.planes_bf16, p.mlp_mode, p.defer_depth_clamp = (1 if bf16 else 0), _lib.P3D_MLP_FP32_SIMT, 0
        self.p, self.wt = p, [t.detach().float().contiguous() for t in wts]
        self.u_c, self.u_f = u_c.to(DEV).contiguous(), u_f.to(DEV).contiguous()
        nbytes = int(_lib.lib().p3d_render_workspace_bytes(C.byref(p)))
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=DEV)
        out = [torch.empty(s, device=DEV) for s in ((N, M, 32), (N, M, 1), (N, M, 1), (N, M, 3))]
        first, second = twice(lambda: render_forward(p, cl, self.wt, ro, rd, self.u_c, self.u_f, ws, out), out + [ws],
                              checks_later=True)
        del ws, out
        repeats(first[:4], second[:4], OUTPUTS)
        self.out, self.ws = first[:4], first[4]
        self.v, total = workspace_views(self.ws, N, M, self.S, self.Sf)
        assert total == nbytes, (total, nbytes)
        again = workspace_views(second[4], N, M, self.S, self.Sf)[0]
        for k in ('depth_c', 'sigma_c', 'rgb_c', 'depth_f', 'sigma_f', 'rgb_f'):
            assert torch.equal(self.v[k], again[k]), k
            assert not torch.isnan(self.v[k]).any(), k

    def backward(self, grads):
        """(gradients {planes (N,3,32 D,H,W), w1, b1, w2, b2}, k_ray_backward's per-sample dsig)."""
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
        N, _, D, H, W, Cc = d_planes.shape
        return dict(zip(PARAMS, [d_planes.permute(0, 1, 5, 2, 3, 4).reshape(N, 3, Cc * D, H, W)] + d_w)), dsig

    # the kernel's constants, in the form the oracle takes them
    def depths(self):
        return self.v['depth_c'][..., None], (self.v['depth_f'][..., None] if self.Sf else None)

    def masks(self):
        N = self.N
        return (self.v['sigma_c'].reshape(N, -1, 1) == -1e3, self.v['sigma_f'].reshape(N, -1, 1) == -1e3 if self.Sf else None)

    def fwd_values(self):
        return [(self.v['sigma_c'][n], self.v['rgb_c'][n], self.v['sigma_f'][n], self.v['rgb_f'][n]) for n in range(self.N)]

    def samples(self, n):
        """Positions (K,3) of view n's samples, coarse then fine, as the kernel makes them."""
        return torch.cat([(self.ro[n, :, None] + d[n][..., None] * self.rd[n, :, None]).reshape(-1, 3)
                          for d in (self.v['depth_c'], self.v['depth_f'])])

    def merged_rank(self):
        """Rank of every sample (coarse then fine, (N*M, L)) in its ray's merged order."""
        t = torch.cat([self.v['depth_c'], self.v['depth_f']], -1).reshape(self.N * self.M, -1)
        order = torch.sort(t, dim=-1, stable=True)[1]
        return torch.empty_like(order).scatter_(1, order, torch.arange(t.shape[1], device=DEV).expand_as(order).contiguous())

    def oracle(self, grads, planes=None, **kw):
        """render_backward_oracle.render_backward in fp64 on the kernel's depths, masks and W == 0 gate."""
        return rbo.render_backward(self.planes64 if planes is None else planes, dec64(self.dec), self.ro, self.rd, self.opts,
                                   self.depths(), self.masks(), grads, use_triplane=self.use_triplane,
                                   dead=self.out[2][..., 0] == 0, depth=self.D, **self.flags, **kw)

    def bars(self, grads, c_tri=0):
        """(B64, bars, tap counts): bar = (k_i + c)(u A + TINY) + 2 |B64 - Bk|, c = 2 L + 192 + c_tri; bars[key + '_fwd']
        is the forward part 2 |B64 - Bk| alone."""
        c = 2 * (self.S + self.Sf) + 192 + c_tri
        b64 = self.oracle(grads)
        bk = self.oracle(grads, fwd=self.fwd_values())
        A = self.oracle(grads, mag=True, c=c)
        n_cta = -(-self.N * self.M * self.S // KT) + (-(-self.N * self.M * self.Sf // KT) if self.Sf else 0)
        cnt = rbo.texel_counts(self.ro, self.rd, self.depths(), self.H, self.W, self.opts['box_warp'], self.use_triplane, self.D)
        bars = {}
        for key in PARAMS:
            kk = per_channel(cnt, self.D).double() if key == 'planes' else float(KT + n_cta)
            bars[key + '_fwd'] = 2 * (b64[key] - bk[key]).abs()
            bars[key] = (kk + c) * (U * A[key] + TINY) + bars[key + '_fwd']
        return b64, bars, cnt


def compare(tag, got, want, bars, taps=None):
    """Worst err / bar of every parameter, printed; with `taps` (per_channel counts), the worst texel of a failing plane
    gradient too."""
    worst = {}
    for key in PARAMS:
        err, r = ratio(got[key], want[key], bars[key])
        print(f'{tag} d_{key}: max abs err {err:.3e}, worst err / bar {r:.4f}')
        worst[key] = r
        if r > 1 and key == 'planes' and taps is not None:
            err = (got[key].double() - want[key]).abs()
            e = torch.where(err == 0, torch.zeros_like(err), err / bars[key]).nan_to_num(nan=float('inf'))
            i = np.unravel_index(int(e.argmax()), e.shape)
            print(f'  worst texel {i}: got {got[key][i].item():.6e} want {want[key][i].item():.6e} bar '
                  f'{bars[key][i].item():.3e} (forward part {bars[key + "_fwd"][i].item():.3e}) taps {taps[i].item()}')
    return worst


def negative_control(label, tag, got, mut, bars):
    """The mutated oracle `mut` misses the kernel by >= 20x its bar somewhere."""
    for key in PARAMS:
        d = (got[key].double() - mut[key]).abs()
        i = int(d.argmax())
        print(f'  control {key}: max |got - mutant| {d.max().item():.3e} where bar {bars[key].reshape(-1)[i].item():.3e} '
              f'(forward part {bars[key + "_fwd"].reshape(-1)[i].item():.3e}), |grad| {mut[key].reshape(-1)[i].abs().item():.3e}')
    worst = max(ratio(got[key], mut[key], bars[key])[1] for key in PARAMS)
    print(f'negative control "{label}" on {tag}: worst err / bar {worst:.1f}')
    assert worst >= 20, (label, worst)


def pin_device_oracle(cases):
    """The device fp64 run of a render oracle, fed the CPU fp32 run's depths and masks, equals that run within its
    rounding; render_backward on the device equals its fp32 autograd gradients within 1e-5 of each tensor's largest
    element.  cases: (name, render, planes, dec, ro, rd, u_c, u_f, opts, kw, D, upstream(outputs))."""
    for name, render, planes, dec, ro, rd, u_c, u_f, opts, kw, D, up in cases:
        pl = planes.clone().requires_grad_(True)
        dref = {k: (v.clone().requires_grad_(True) if torch.is_tensor(v) else v) for k, v in dec.items()}
        out, smp = render(pl, dref, ro, rd, opts, u_c, u_f, return_samples=True, **kw)
        gw = up(out)
        ref = torch.autograd.grad(sum((o * g.to(o.device)).sum() for o, g in zip(out, gw)),
                                  [pl] + [dref[k] for k in ('w1', 'b1', 'w2', 'b2')])
        to = lambda t: None if t is None else t.to(DEV)
        dep, msk = tuple(map(to, smp['depths'])), tuple(map(to, smp['masks']))
        out64 = render(planes.to(DEV, torch.float64), dec64(dec), ro.to(DEV), rd.to(DEV), opts, None, None, depths=dep,
                       masks=msk, **kw)
        for a, b in zip(out64, out):
            assert a.dtype == torch.float64
            assert (a.cpu() - b.detach().double()).abs().max().item() <= 2e-6, name
        g64 = rbo.render_backward(planes.to(DEV, torch.float64), dec64(dec), ro.to(DEV), rd.to(DEV), opts, dep, msk,
                                  [g.to(DEV, torch.float64) for g in gw], depth=D, **kw)
        for key, r in zip(PARAMS, ref):
            err = (g64[key].cpu() - r.double()).abs().max().item()
            print(f'pin {name} d_{key}: {err:.2e} of max {r.abs().max().item():.2e}')
            assert err <= 1e-5 * r.abs().max().item(), (name, key, err)


GREG_POINTS, GREG_DIST = 1000, 0.004          # loss_orthocondA.py:592-593 (density_reg_p_dist)


def density_regularisation(run_model, D, mode, launches_ok, gate_share, c):
    """The Greg phase (loss_orthocondA.py:579-600) on D-slab planes: 4 views x (1000 points uniform in [-1, 1]^3 + the same
    points plus N(0, 0.004^2)) through run_model under autograd (_PointsFunction) on 256^2 planes with the training
    options, then the L1 between the two halves' sigma.  Asserts the forward's mlp_mode and its launches per profile
    slot (launches_ok), sigma against the fp64 oracle `run_model`, the pairs whose sign is within rounding of 0 (at most
    gate_share of those that read a texel), and the plane and decoder gradients per element against points_backward fed
    the kernel's signs, bar (k + c)(u A + TINY).  Returns (opts, p64, d64, coords, g_sigma, B64, A)."""
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    tag = 'Greg' if D == 1 else f'Greg D={D}'
    t0 = time.time()
    N, H = 4, 256
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=48, depth_resolution_importance=48, **({'triplane_depth': D} if D > 1 else {}))
    g = torch.Generator().manual_seed(1234)
    planes = torch.randn(N, 3, 32 * D, H, H, generator=g)
    _, dec, *_ = orc.synth_inputs(1234, 1, 1, 2, 0, 2)
    x = torch.rand(N, GREG_POINTS, 3, generator=g) * 2 - 1
    coords = torch.cat([x, x + torch.randn(x.shape, generator=g) * GREG_DIST], 1).to(DEV)
    r = ImportanceRenderer(use_triplane=True)
    d = make_decoder(dec, DEV).requires_grad_(True)
    pg = planes.to(DEV).requires_grad_(True)
    # the forward's mode is chosen as for a ray render with M = 0 rays (renderer.py run_model under autograd)
    p, _ = r._params(r._shape_probe(pg, opts), N, 0, dict(opts), d, None, None, None)
    print(f'{tag}: forward mlp_mode {p.mlp_mode} (0 fp32 SIMT, 1 tensor-core 3-pass)')
    assert p.mlp_mode == mode and (D == 1 or p.plane_depth == D), (p.plane_depth, p.mlp_mode)
    out, prof = profiled(lambda: r.run_model(pg, d, coords, None, opts))
    assert launches_ok(prof), prof
    sigma = out['sigma']
    p64, d64 = planes.to(DEV, torch.float64), dec64(dec)
    _, s64 = run_model(p64, d64, coords, opts, True)
    err = (sigma.detach().double() - s64).abs().nan_to_num(nan=float('inf')).max().item()
    print(f'{tag}: forward sigma max abs err {err:.3e}')
    assert err <= FWD_BAR, err
    diff_k = (sigma[:, :GREG_POINTS] - sigma[:, GREG_POINTS:]).detach()
    diff64 = s64[:, :GREG_POINTS] - s64[:, GREG_POINTS:]
    # a point with two coordinates outside the box reads no texel, so a pair of such points has exactly equal sigma in both
    # runs (sign 0, no gradient); the sign of every other pair is gated when its fp64 difference is within 2e-4 of 0
    blank = (diff64 == 0) & (diff_k == 0)
    gated = (diff64.abs() <= 2 * FWD_BAR) & ~blank
    flipped = torch.sign(diff_k.double()) != torch.sign(diff64)
    assert not (flipped & ~gated).any(), 'an L1 sign differs away from 0'
    print(f'{tag}: {blank.sum().item()} of {blank.numel()} pairs read no texel (difference exactly 0 in both); of the rest '
          f'{gated.sum().item()} lie within 2e-4 of 0 (sign gated), {flipped.sum().item()} signs differ from the fp64 ones')
    assert gated.sum().item() <= gate_share * (~blank).sum().item()
    loss = F.l1_loss(sigma[:, :GREG_POINTS], sigma[:, GREG_POINTS:])
    got = torch.autograd.grad(loss, [pg, d.net[0].weight, d.net[0].bias, d.net[2].weight, d.net[2].bias])
    # the upstream gradient is the kernel's sign: the oracle differentiates the same loss at the same sign pattern
    sgn = torch.sign(diff_k[..., 0].double()) / diff_k.numel()
    g_sigma = torch.cat([sgn, -sgn], 1)
    b64 = rbo.points_backward(p64, d64, coords, g_sigma, opts['box_warp'], depth=D)
    A = rbo.points_backward(p64, d64, coords, g_sigma, opts['box_warp'], mag=True, c=c, depth=D)
    # tap contributions per texel: texel_counts with origins at the points, zero directions and unit depths
    cnt = rbo.texel_counts(coords, torch.zeros_like(coords), (torch.ones(N, 2 * GREG_POINTS, 1, 1, device=DEV), None), H, H,
                           opts['box_warp'], True, D)
    taps = per_channel(cnt, D)
    n_cta = -(-N * 2 * GREG_POINTS // KT)
    worst = 0.0
    for key, gk in zip(PARAMS, got):
        kk = taps.double() if key == 'planes' else float(KT + n_cta)
        e, r_ = ratio(gk, b64[key], (kk + c) * (U * A[key] + TINY))
        print(f'{tag} d_{key}: max abs err {e:.3e}, worst err / bar {r_:.4f}')
        worst = max(worst, r_)
    assert worst <= 1.0, worst
    assert (got[0][taps == 0] == 0).all()
    print(f'{tag}: {time.time() - t0:.1f} s')
    return opts, p64, d64, coords, g_sigma, b64, A
