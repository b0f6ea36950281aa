"""GPU: the deterministic training backward (``torch.use_deterministic_algorithms(True)``).

p3d_render_backward_det, p3d_decode_points_backward_det and p3d_paste_front_backward_det replace the float atomics of the
training backward with fixed-order reductions (DESIGN.md section 4.3 and "Front-view paste"):
  * tri-plane gradient   one (texel, entry = (sample, plane, tap)) pair per tap, stably radix-sorted by texel; each texel
                         sums its run in entry order, acc = fl(acc + fl(w * dF))
  * decoder gradients    per-CTA partials, summed over CTA index by adjacent pairs, level by level
  * paste d_xyz          each texel gathers its stencil of output pixels row-major, taps (i0,i0), (i0,i1), (i1,i0), (i1,i1)

Checked here, through the C ABI and through the autograd Functions:
  1. three runs with scratch and outputs prefilled with NaN, 0xFF and zeros give the same bits;
  2. the order is the documented one: a numpy float32 restatement of the sort and the sums, fed the kernel's own recorded
     feature gradients, weights and CTA partials, reproduces every gradient bit for bit; three mutants of it (an unstable
     sort, a reversed run, a run without its last entry) do not;
  3. the gradients lie within the fp64-oracle bars of the training-path tests, and within the bound for k contributions
     summed in sequence of the atomic path's;
  4. with the switch on the autograd Functions run the deterministic entry points and repeat bit for bit; with it off they
     run the atomic kernels, as before.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import paste_oracle as po, renderer_oracle as orc
from tests import render_abi as ra
from tests.helpers import profiled
from tests.render_abi import DEV, PARAMS, U, TrainKernel, compare, dec64, make_decoder, upstream

pytestmark = pytest.mark.gpu
FREE_BYTES = 24 << 30
PROF_OTHER = 6                    # profile slot of the reductions (csrc/p3d_common.cuh)
KPARAMS = 64 * 32 + 64 + 33 * 64 + 33
FILLS = ('nan', 0xFF, 0)

TRAIN = dict(N=4, R=64, S=48, Sf=48, H=256, W=256)
CASES = {
    'train': dict(TRAIN),                                                   # config 5's training render
    'view128': dict(N=1, R=128, S=96, Sf=96, H=256, W=256),
    'contention': dict(N=2, R=64, S=48, Sf=48, H=9, W=13),                  # texels take thousands of contributions
    'multiplane_d2': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, D=2),
    'multiplane_d3': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, D=3),
    'auto_miss': dict(N=2, R=32, S=48, Sf=48, H=64, W=64, opts=dict(ray_start='auto', ray_end='auto', white_back=False),
                      eg3d=True, miss_view=1),
    'small': dict(N=1, R=8, S=48, Sf=48, H=64, W=64),
}
RESTATED = ('small', 'contention', 'multiplane_d2', 'auto_miss')        # small enough for the numpy restatement


@pytest.fixture
def deterministic():
    """torch.use_deterministic_algorithms(True) for the test; the previous setting comes back even when the test fails."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _a256(x):
    return (x + 255) // 256 * 256


def det_layout(head, samples, nt, ctas):
    """det_layout (render_backward.cu) restated: byte offsets of dx, w, key0, key1, id0, id1, part after `head` bytes."""
    entries = samples * nt
    sizes = [('dx', samples * 32 * 4), ('w', entries * 4), ('key0', entries * 4), ('key1', entries * 4), ('id0', entries * 4),
             ('id1', entries * 4), ('part', ctas * KPARAMS * 4)]
    off, offs = _a256(head), {}
    for k, b in sizes:
        offs[k] = off
        off += _a256(b)
    return offs


def records(scratch, head, samples, nt, ctas):
    """The kernel's records in its scratch, as numpy arrays."""
    o = det_layout(head, samples, nt, ctas)
    s = scratch.cpu().numpy()
    f = lambda k, n, dt: s[o[k]:o[k] + n * 4].view(dt)
    e = samples * nt
    return dict(dx=f('dx', samples * 32, np.float32).reshape(samples, 32), w=f('w', e, np.float32),
                key=(f('key0', e, np.uint32), f('key1', e, np.uint32)), id=(f('id0', e, np.uint32), f('id1', e, np.uint32)),
                part=f('part', ctas * KPARAMS, np.float32).reshape(ctas, KPARAMS))


# ------------------------------------------------------------------------------------------------- numpy restatements
def run_sums(keys, terms, n_out, variant='stable'):
    """Entries with key < n_out summed per key in a fixed order: stable order of entry index (variant 'unstable': numpy's
    quicksort; 'reverse': each run backwards; 'droplast': each run without its last entry); acc = fl32(acc + term)."""
    perm = np.argsort(keys, kind='quicksort' if variant == 'unstable' else 'stable')
    ks = keys[perm]
    live = ks < n_out
    perm, ks = perm[live], ks[live]
    t = np.arange(n_out)
    lo, hi = np.searchsorted(ks, t, 'left'), np.searchsorted(ks, t, 'right')
    lens = hi - lo - (1 if variant == 'droplast' else 0)
    out = np.zeros((n_out,) + terms.shape[1:], np.float32)
    for j in range(int(lens.max(initial=0))):
        sel = lens > j
        idx = (hi[sel] - 1 - j) if variant == 'reverse' else (lo[sel] + j)
        out[sel] = out[sel] + terms[perm[idx]]
    return out, hi - lo


def restate_planes(rec, nt, n_texels, variant='stable', terms=None):
    """d_planes (texels, 32) from the records: the unsorted keys come back from either sort buffer (both hold a permutation
    of the (key, entry) pairs), then sort + fixed-order sums."""
    keys = np.empty_like(rec['key'][0])
    keys[rec['id'][0]] = rec['key'][0]
    keys1 = np.empty_like(keys)
    keys1[rec['id'][1]] = rec['key'][1]
    assert np.array_equal(keys, keys1)
    if terms is None:
        terms = rec['w'][:, None] * rec['dx'][np.arange(keys.size) // nt]      # fl32(w * dF)
    return run_sums(keys, terms, n_texels, variant)


def restate_params(part):
    """The CTA partials summed by adjacent pairs, level by level -> (w1, b1, w2, b2)."""
    x = part
    while x.shape[0] > 1:
        y = x[0:x.shape[0] - 1:2] + x[1::2]
        x = np.concatenate([y, x[-1:]]) if x.shape[0] % 2 else y
    v = x[0]
    return v[:2048].reshape(64, 32), v[2048:2112], v[2112:4224].reshape(33, 64), v[4224:]


# ------------------------------------------------------------------------------------------------- render inputs
@functools.lru_cache(maxsize=None)
def _inputs(name):
    case = CASES[name]
    N, R, S, Sf, H, W = (case[k] for k in ('N', 'R', 'S', 'Sf', 'H', 'W'))
    D = case.get('D', 1)
    g = torch.Generator().manual_seed(1300 + sorted(CASES).index(name))
    planes = torch.randn(N, 3, 32 * D, H, W, generator=g)
    _, dec, *_ = orc.synth_inputs(1300, 1, 1, 2, 0, 2)
    opts = dict(dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=Sf), **case.get('opts', {}))
    if D > 1:
        opts['triplane_depth'] = D
    ro, rd = ra.rays_at(ra.spin12(N), R)
    if case.get('miss_view') is not None:
        v = case['miss_view']                      # this view looks away from the box: every ray misses it
        rd = rd.clone()
        rd[v] = -rd[v]
    M = R * R
    u_c = torch.rand(N, M, S, 1, generator=g)
    u_f = torch.rand(N * M, Sf, generator=g)
    return planes, dec, opts, ro, rd, u_c, u_f


class DetKernel(TrainKernel):
    """TrainKernel with the deterministic backward: outputs and scratch prefilled with `fill` before the call."""

    def backward_det(self, grads, fill):
        from panic3d_b200 import _lib
        L, p = _lib.lib(), self.p
        nbytes = int(L.p3d_render_backward_det_scratch_bytes(C.byref(p)))
        assert nbytes, L.p3d_last_error()
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        d_planes = torch.empty((self.N, 3, self.D, self.H, self.W, 32), device=DEV)
        d_w = [torch.empty_like(t) for t in self.wt]
        _fill([scratch, d_planes, *d_w], fill)
        g = [t.float().contiguous() for t in grads]
        n0 = _lib.launch_count()
        _lib.check(L.p3d_render_backward_det(C.byref(p), self.planes_cl.data_ptr(), *[t.data_ptr() for t in self.wt],
                                             self.ro.data_ptr(), self.rd.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                                             self.out[1].data_ptr(), *[t.data_ptr() for t in g], scratch.data_ptr(), scratch.numel(),
                                             d_planes.data_ptr(), *[t.data_ptr() for t in d_w], _lib.stream_ptr(DEV)))
        torch.cuda.synchronize()
        self.launches = _lib.launch_count() - n0
        N, _, D, H, W, Cc = d_planes.shape
        got = dict(zip(PARAMS, [d_planes.permute(0, 1, 5, 2, 3, 4).reshape(N, 3, Cc * D, H, W)] + d_w))
        return got, d_planes, scratch

    def det_sizes(self):
        nt = 24 if self.D > 1 else 12
        R_ = self.N * self.M
        ctas = -(-R_ * self.S // 128) + -(-R_ * self.Sf // 128)
        head = 2 * R_ * (self.S + self.Sf) * 4 + 1024
        return head, R_ * (self.S + self.Sf), nt, ctas, self.N * 3 * self.D * self.H * self.W


def _fill(ts, fill):
    for t in ts:
        if fill == 'nan':
            (t.view(torch.float32)[:t.numel() // 4] if t.dtype == torch.uint8 else t).fill_(float('nan'))
            if t.dtype == torch.uint8:
                t[t.numel() // 4 * 4:].fill_(0xFF)
        elif t.dtype == torch.uint8:
            t.fill_(fill)
        else:
            t.view(torch.int32).fill_(-1 if fill == 0xFF else 0)
    torch.cuda.synchronize()


def _three(call):
    """call(fill) under each prefill; every output of the three runs bit-identical.  Returns the first run."""
    runs = [call(f) for f in FILLS]
    for r in runs[1:]:
        for k in PARAMS:
            assert torch.equal(runs[0][0][k], r[0][k]), f'three prefills give different {k}'
    return runs[0]


def _order_checks(tag, got, d_planes_flat, rec, nt, n_texels, bars=None):
    """The documented order reproduces d_planes and the decoder gradients bit for bit; the three mutants miss."""
    terms = rec['w'][:, None] * rec['dx'][np.arange(rec['w'].size) // nt]
    mine, cnt = restate_planes(rec, nt, n_texels, terms=terms)
    assert np.array_equal(mine.view(np.uint32), d_planes_flat.view(np.uint32)), f'{tag}: d_planes is not the documented order'
    print(f'{tag}: {int((cnt > 0).sum())} texels touched, longest run {int(cnt.max())}')
    for key, want in zip(PARAMS[1:], restate_params(rec['part'])):
        assert np.array_equal(got[key].cpu().numpy().view(np.uint32), want.view(np.uint32)), f'{tag}: d_{key} is not the pairwise order'
    for variant in ('unstable', 'reverse'):
        mut, _ = restate_planes(rec, nt, n_texels, variant, terms)
        differ = int((mut.view(np.uint32) != d_planes_flat.view(np.uint32)).sum())
        print(f'  control {variant}: {differ} elements differ from the kernel')
        assert differ > 0, variant
    mut, _ = restate_planes(rec, nt, n_texels, 'droplast', terms)
    if bars is not None:
        b = bars.cpu().numpy()
        r = (np.abs(mut.astype(np.float64) - d_planes_flat) / np.maximum(b, 1e-300)).max()
        print(f'  control droplast: worst err / bar {r:.3g}')
        assert r > 1, r
    else:
        assert not np.array_equal(mut, d_planes_flat)


def _planes_flat(d_planes):
    return d_planes.reshape(-1, 32).cpu().numpy()


def _flat_bars(bars, k):
    """(N,3,32 D,H,W) plane bars -> (texels, 32) in the (N,3,D,H,W,C) texel order."""
    N, D, H, W = k.N, k.D, k.H, k.W
    return bars.reshape(N, 3, 32, D, H, W).permute(0, 1, 3, 4, 5, 2).reshape(-1, 32)


@pytest.mark.parametrize('name', sorted(CASES))
def test_render_backward_det(name):
    case = CASES[name]
    if case['H'] * case['W'] >= 256 * 256:
        ra.skip_unless_free(FREE_BYTES)
    k = DetKernel(case, _inputs(name))
    grads = upstream('all', k.N, k.M, 71)
    got, d_planes, scratch = _three(lambda f: k.backward_det(grads, f))
    det_launches = k.launches
    n0 = ra_launches()
    atomic, _ = k.backward(grads)
    atomic_launches = ra_launches() - n0
    print(f'{name}: deterministic backward {det_launches} launches, atomic {atomic_launches}')
    assert det_launches > atomic_launches
    b64, bars, cnt = k.bars(grads)
    w = compare(f'{name} [det]', got, b64, bars, ra.per_channel(cnt, k.D))
    assert max(w.values()) <= 1.0, w
    taps = ra.per_channel(cnt, k.D)
    assert (got['planes'][taps == 0] == 0).all(), 'a texel no sample touches got a gradient'
    # against the atomic path: both are sequential sums of the same terms in two orders
    head, samples, nt, ctas, n_texels = k.det_sizes()
    rec = records(scratch, head, samples, nt, ctas)
    if name in RESTATED:
        _order_checks(name, got, _planes_flat(d_planes), rec, nt, n_texels, _flat_bars(bars['planes'], k))
    bound = seq_bound(rec, nt, n_texels)
    ad = atomic['planes'].reshape(k.N, 3, 32, k.D, k.H, k.W).permute(0, 1, 3, 4, 5, 2).reshape(-1, 32)
    err = (ad.double() - d_planes.reshape(-1, 32).double()).abs()
    assert bool((err <= bound).all()), f'{name}: det and atomic d_planes differ by more than 2 k u sum|terms|: {(err - bound).max().item()}'
    pa = np.abs(rec['part'].astype(np.float64)).sum(0)
    for key, (lo_, hi_) in zip(PARAMS[1:], ((0, 2048), (2048, 2112), (2112, 4224), (4224, KPARAMS))):
        b = torch.from_numpy(2 * ctas * U * pa[lo_:hi_]).to(DEV).reshape(got[key].shape)
        assert bool(((atomic[key].double() - got[key].double()).abs() <= b).all()), key


def ra_launches():
    from panic3d_b200 import _lib
    return _lib.launch_count()


def _unsorted_keys(rec):
    keys = np.empty_like(rec['key'][0])
    keys[rec['id'][0]] = rec['key'][0]
    return keys


def seq_bound(rec, nt, n_texels):
    """2 k u sum|w dF| per texel element (texels, 32), fp64 on the device: how far two sequential sums of a texel's k terms in
    different orders may differ."""
    keys = torch.from_numpy(_unsorted_keys(rec).astype(np.int64)).to(DEV)
    w = torch.from_numpy(rec['w']).to(DEV).double().abs()
    dx = torch.from_numpy(rec['dx']).to(DEV).double().abs()
    A = torch.zeros(n_texels + 1, 32, dtype=torch.float64, device=DEV)
    for c0 in range(0, keys.numel(), 1 << 22):
        kc = keys[c0:c0 + (1 << 22)]
        ids = torch.arange(c0, c0 + kc.numel(), device=DEV) // nt
        A.index_add_(0, kc, w[c0:c0 + kc.numel(), None] * dx[ids])
    kk = torch.bincount(keys, minlength=n_texels + 1).double()
    return (2 * kk[:, None] * U * A)[:n_texels]


# ------------------------------------------------------------------------------------------------- point mode (Greg)
def _points_inputs(D=1):
    g = torch.Generator().manual_seed(1400)
    N, K, H, W = 4, 2 * 1000, 256, 256
    planes = torch.randn(N, 3, 32 * D, H, W, generator=g).to(DEV)
    _, dec, *_ = orc.synth_inputs(1400, 1, 1, 2, 0, 2)
    coords = ((torch.rand(N, K, 3, generator=g) * 2 - 1) * 0.3).to(DEV)
    g_rgb = torch.randn(N, K, 32, generator=g).to(DEV)
    g_sigma = torch.randn(N, K, 1, generator=g).to(DEV)
    return planes, dec, coords, g_rgb, g_sigma


def test_points_backward_det_greg_shape():
    """run_model's backward at the density-regularisation shape, 4 views x 2 x 1000 points: three prefills give the same
    bits; the documented order reproduces them; the atomic path agrees within the sequential-sum bound."""
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer, _fp32_texels
    planes, dec, coords, g_rgb, g_sigma = _points_inputs()
    N, K = coords.shape[:2]
    r = ImportanceRenderer(use_triplane=True)
    decoder = make_decoder(dec, DEV)
    opts = dict(orc.DEFAULT_OPTS)
    p, wts = r._params(r._shape_probe(planes, opts), N, 0, opts, decoder, None, None, None)
    cl = _fp32_texels(planes, p)
    wt = [t.detach().float().contiguous() for t in wts]
    L = _lib.lib()

    def det(fill):
        nbytes = int(L.p3d_decode_points_backward_det_scratch_bytes(C.byref(p), K))
        assert nbytes, L.p3d_last_error()
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        d_planes = torch.empty_like(cl)
        d_w = [torch.empty_like(t) for t in wt]
        _fill([scratch, d_planes, *d_w], fill)
        _lib.check(L.p3d_decode_points_backward_det(C.byref(p), cl.data_ptr(), *[t.data_ptr() for t in wt], coords.data_ptr(), K,
                                                    g_rgb.data_ptr(), g_sigma.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                                    d_planes.data_ptr(), *[t.data_ptr() for t in d_w], _lib.stream_ptr(DEV)))
        torch.cuda.synchronize()
        return dict(zip(PARAMS, [d_planes] + d_w)), d_planes, scratch

    got, d_planes, scratch = _three(det)
    d_pl = torch.zeros_like(cl)
    d_w = [torch.zeros_like(t) for t in wt]
    _lib.check(L.p3d_decode_points_backward(C.byref(p), cl.data_ptr(), *[t.data_ptr() for t in wt], coords.data_ptr(), K,
                                            g_rgb.data_ptr(), g_sigma.data_ptr(), d_pl.data_ptr(), *[t.data_ptr() for t in d_w],
                                            _lib.stream_ptr(DEV)))
    torch.cuda.synchronize()
    samples, nt, ctas, n_texels = N * K, 12, -(-N * K // 128), N * 3 * 256 * 256
    rec = records(scratch, 0, samples, nt, ctas)
    _order_checks('points', got, _planes_flat(d_planes), rec, nt, n_texels)
    err = (d_pl.reshape(-1, 32).double() - d_planes.reshape(-1, 32).double()).abs()
    assert bool((err <= seq_bound(rec, nt, n_texels)).all())
    pa = np.abs(rec['part'].astype(np.float64)).sum(0)
    for key, t, (lo_, hi_) in zip(PARAMS[1:], d_w, ((0, 2048), (2048, 2112), (2112, 4224), (4224, KPARAMS))):
        e = (t.double() - got[key].double()).abs().cpu().numpy().reshape(-1)
        assert (e <= 2 * ctas * U * pa[lo_:hi_]).all(), key


# ------------------------------------------------------------------------------------------------- paste 'Agrad'
PASTE = {'train_agrad': dict(seed=42, N=4, R=64, S=512), 'eval': dict(seed=41, N=8, R=128, S=512)}
BW = 0.7
EVAL = dict(thresh_weight=0.95, thresh_edges=0.02, thresh_occ=0.05, thresh_dxyz=0.000005)


def _lin_src(n_out, scale, n_in):
    """F.interpolate's source index / weights (paste_front.cu lin_src), fp32 with the contracted multiply-add."""
    d = np.arange(n_out, dtype=np.float64)
    s = (np.float64(scale) * (d + 0.5) - 0.5).astype(np.float32)      # one rounding, as the kernel's FFMA
    s = np.maximum(s, np.float32(0))
    i0 = np.minimum(s.astype(np.int64), n_in - 1)
    i1 = np.minimum(i0 + 1, n_in - 1)
    l1 = np.clip(s - i0.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float32)
    return i0, i1, (np.float32(1) - l1).astype(np.float32), l1


def restate_paste(g_v, R, S, variant='stable'):
    """d_xyz (N,2,R,R) from the recorded per-pixel gradients: pixels row-major, taps (i0,i0), (i0,i1), (i1,i0), (i1,i1)."""
    scale = np.float32(R) / np.float32(S)
    iy0, iy1, ly0, ly1 = _lin_src(S, scale, R)
    ix0, ix1, lx0, lx1 = _lin_src(S, scale, R)
    keys, ws = [], []
    for ry, ly in ((iy0, ly0), (iy1, ly1)):
        for cx, lx in ((ix0, lx0), (ix1, lx1)):
            keys.append((ry[:, None] * R + cx[None, :]).reshape(-1))
            ws.append((ly[:, None] * lx[None, :]).astype(np.float32).reshape(-1))
    key = np.stack(keys, 1).reshape(-1)                 # entry = pixel * 4 + tap
    w = np.stack(ws, 1).reshape(-1)
    out = np.zeros((g_v.shape[0], 2, R * R), np.float32)
    for n in range(g_v.shape[0]):
        for c in range(2):
            g = np.repeat(g_v[n, c].reshape(-1), 4)
            kk = np.where(g != 0, key, R * R)
            out[n, c] = run_sums(kk, (g * w).astype(np.float32)[:, None], R * R, variant)[0][:, 0]
    return out


@pytest.mark.parametrize('name', sorted(PASTE))
def test_paste_backward_det(name):
    """paste 'Agrad' backward: three prefills give the same d_image and d_xyz; d_image equals the atomic path's bit for bit;
    the documented gather order reproduces d_xyz from the recorded per-pixel gradients; the atomic d_xyz agrees within the
    bound for k contributions summed in sequence."""
    import panic3d_b200.paste as pp
    from panic3d_b200 import _lib
    c = PASTE[name]
    N, R, S = c['N'], c['R'], c['S']
    d = {k: v.to(DEV) for k, v in po.synth_paste_inputs(c['seed'], N, R, S, box_warp=BW, reach=1.2).items() if torch.is_tensor(v)}
    _, _, mask, _ = pp.paste_front_fused(d['image'], d['image_xyz'], d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'],
                                         BW, **EVAL)
    p = pp.PasteParams()
    p.n_views, p.res_render, p.res_image, p.res_front, p.normalize_images, p.box_warp = N, R, S, 0, 0, BW
    p.thresh_weight, p.thresh_edges, p.thresh_occ, p.thresh_dxyz = (EVAL[k] for k in ('thresh_weight', 'thresh_edges', 'thresh_occ', 'thresh_dxyz'))
    g = torch.Generator(device=DEV).manual_seed(5)
    g_img, g_paste = torch.randn(N, 3, S, S, generator=g, device=DEV), torch.randn(N, 3, S, S, generator=g, device=DEV)
    xyz, front = d['image_xyz'].contiguous(), d['front_rgb'].contiguous()
    L = _lib.lib()

    def det(fill):
        scratch = torch.empty(int(L.p3d_paste_front_backward_det_scratch_bytes(C.byref(p))), dtype=torch.uint8, device=DEV)
        d_img, d_xyz = torch.empty(N, 3, S, S, device=DEV), torch.empty(N, 3, R, R, device=DEV)
        _fill([scratch, d_img, d_xyz], fill)
        (_, prof) = profiled(lambda: _lib.check(L.p3d_paste_front_backward_det(
            C.byref(p), xyz.data_ptr(), front.data_ptr(), mask.data_ptr(), g_img.data_ptr(), g_paste.data_ptr(), scratch.data_ptr(),
            scratch.numel(), d_img.data_ptr(), d_xyz.data_ptr(), _lib.stream_ptr(DEV))))
        assert prof[PROF_OTHER] == 1, prof
        return d_img, d_xyz, scratch

    runs = [det(f) for f in FILLS]
    for r in runs[1:]:
        assert torch.equal(runs[0][0], r[0]) and torch.equal(runs[0][1], r[1])
    d_img, d_xyz, scratch = runs[0]
    a_img, a_xyz = torch.empty_like(d_img), torch.zeros_like(d_xyz)
    _lib.check(L.p3d_paste_front_backward(C.byref(p), xyz.data_ptr(), front.data_ptr(), mask.data_ptr(), g_img.data_ptr(),
                                          g_paste.data_ptr(), a_img.data_ptr(), a_xyz.data_ptr(), _lib.stream_ptr(DEV)))
    torch.cuda.synchronize()
    assert torch.equal(a_img, d_img)
    assert bool((d_xyz[:, 2] == 0).all())
    g_v = scratch[:N * 2 * S * S * 4].view(torch.float32).reshape(N, 2, S, S).cpu().numpy()
    mine = restate_paste(g_v, R, S)
    got = d_xyz[:, :2].reshape(N, 2, R * R).cpu().numpy()
    assert np.array_equal(mine.view(np.uint32), got.view(np.uint32)), 'd_xyz is not the documented gather order'
    for variant in ('reverse', 'droplast'):
        mut = restate_paste(g_v, R, S, variant)
        assert not np.array_equal(mut.view(np.uint32), got.view(np.uint32)), variant
    # sequential-sum bound against the atomic path: |scatter - gather| <= 2 k u sum|terms| per texel
    gabs = np.abs(g_v).astype(np.float64)
    scale = np.float32(R) / np.float32(S)
    iy0, iy1, ly0, ly1 = _lin_src(S, scale, R)
    A = np.zeros((N, 2, R * R))
    kk = np.zeros((N, 2, R * R))
    for ry, ly in ((iy0, ly0), (iy1, ly1)):
        for cx, lx in ((iy0, ly0), (iy1, ly1)):                     # square images: the column stencil is the row one
            idx = (ry[:, None] * R + cx[None, :]).reshape(-1)
            w = (ly[:, None] * lx[None, :]).reshape(-1).astype(np.float64)
            for n in range(N):
                for ch in range(2):
                    gv = gabs[n, ch].reshape(-1)
                    np.add.at(A[n, ch], idx, gv * w)
                    np.add.at(kk[n, ch], idx, (gv != 0).astype(np.float64))
    err = np.abs(a_xyz[:, :2].reshape(N, 2, -1).double().cpu().numpy() - got.astype(np.float64))
    assert (err <= 2 * kk * U * A).all(), float((err - 2 * kk * U * A).max())
    print(f'paste {name}: longest stencil {int(kk.max())}, max |det - atomic| {err.max():.3e}')


# ------------------------------------------------------------------------------------------------- selection
def _render_route(name, det_on):
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    planes, dec, opts, ro, rd, u_c, u_f = _inputs(name)
    r = ImportanceRenderer(use_triplane=not CASES[name].get('eg3d'))
    r.injected_noise = (u_c, u_f)
    grads_out = []
    launches = []
    for _ in range(2):
        d = make_decoder(dec, DEV).requires_grad_(True)
        pg = planes.to(DEV).requires_grad_(True)
        out = r(pg, d, ro.to(DEV), rd.to(DEV), opts)
        up = upstream('all', ro.shape[0], ro.shape[1], 3)
        loss = sum((o * u).sum() for o, u in zip(out, up))
        n0 = _lib.launch_count()
        (_, prof) = profiled(lambda: loss.backward())
        launches.append((_lib.launch_count() - n0, prof[PROF_OTHER]))
        grads_out.append([pg.grad] + [q.grad for q in d.parameters()])
    return grads_out, launches


def test_selection_render(deterministic):
    """ImportanceRenderer under autograd with the switch on: two backward passes give the same bits and the reductions ran
    (launches in the PROF_OTHER slot); with it off the atomic backward ran: one ray and two sample launches, none there."""
    grads, launches = _render_route('small', True)
    for a, b in zip(*grads):
        assert torch.equal(a, b)
    assert all(n > 3 and other >= 1 for n, other in launches), launches
    torch.use_deterministic_algorithms(False)
    _, launches_off = _render_route('small', False)
    assert all(n == 3 and other == 0 for n, other in launches_off), launches_off
    print(f'render route launches: on {launches}, off {launches_off}')


def test_selection_run_model(deterministic):
    from panic3d_b200 import _lib
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    planes, dec, coords, g_rgb, g_sigma = _points_inputs()
    r = ImportanceRenderer(use_triplane=True)

    def once():
        d = make_decoder(dec, DEV).requires_grad_(True)
        pg = planes.clone().requires_grad_(True)
        out = r.run_model(pg, d, coords, None, dict(orc.DEFAULT_OPTS))
        loss = (out['rgb'] * g_rgb).sum() + (out['sigma'] * g_sigma).sum()
        n0 = _lib.launch_count()
        loss.backward()
        torch.cuda.synchronize()
        return [pg.grad] + [q.grad for q in d.parameters()], _lib.launch_count() - n0

    (a, na), (b, nb) = once(), once()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    torch.use_deterministic_algorithms(False)
    _, n_off = once()
    print(f'run_model backward launches: on {na}, off {n_off}')
    assert na == nb and na > n_off and n_off == 1


def test_selection_paste(deterministic):
    import panic3d_b200.paste as pp
    c = PASTE['train_agrad']
    N, R, S = c['N'], c['R'], c['S']
    d = {k: v.to(DEV) for k, v in po.synth_paste_inputs(c['seed'], N, R, S, box_warp=BW, reach=1.2).items() if torch.is_tensor(v)}
    g = torch.Generator(device=DEV).manual_seed(9)
    g_img, g_paste = torch.randn(N, 3, S, S, generator=g, device=DEV), torch.randn(N, 3, S, S, generator=g, device=DEV)

    def once():
        image = d['image'].clone().requires_grad_(True)
        xyz = d['image_xyz'].clone().requires_grad_(True)
        img, paste, _, _ = pp.paste_front_fused(image, xyz, d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], BW,
                                                grad_sample=True, **EVAL)
        loss = (img * g_img).sum() + (paste * g_paste).sum()
        (_, prof) = profiled(lambda: loss.backward())
        return image.grad, xyz.grad, prof[PROF_OTHER]

    a, b = once(), once()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == 1
    torch.use_deterministic_algorithms(False)
    off = once()
    assert off[2] == 0 and torch.equal(off[0], a[0])
