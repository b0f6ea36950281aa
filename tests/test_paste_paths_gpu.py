"""GPU: the fused front-view paste (k_paste_front / k_paste_front_bwd, csrc/paste_front.cu) at the eval and training
sizes, against the fp64 oracle run on the device.

`p3d_paste_front` runs on every view of the eval sweep (8 views, 128^2 render -> 512^2 image, scale 1/4) and on every
generated image of the training modes 'A' / 'Agrad' (64^2 -> 512^2, scale 1/8), where `grad_sample=True` sends
`p3d_paste_front_backward` into `image_xyz`.  The fixture cases of tests/test_paste_gpu.py stop at 160^2 with every lookup
inside the box.  Here every case builds its inputs with `reach` 1.2 (tiny: 4), so bands of pixels on every side look the
front image and the eroded weights up outside the box and both border clips run, forward and backward:

    case         N   R    S    Rf   what it reaches
    eval         8   128  512  -    the eval sweep's shape and thresholds, scale 1/4
    train_agrad  4   64   512  -    training 'Agrad', scale 1/8: 64 output pixels add atomically into each d_xyz texel
    train_erode  2   64   512  128  erosion 3 with Rf > R: the eroded lookup's own size and stride
    ragged       3   48   500  37   scale 0.096 (not dyadic), partial 32 x 8 tiles in x and y, Rf < R, normalize_images
    same_res     1   37   37   37   scale 1, one partial tile, normalize_images
    down         2   96   64   -    R > S (scale 1.5)
    tiny_*       2   1/2  7/3  -    every bilinear tap of the render clamps to the same texel

Every forward goes through the C ABI with NaN-prefilled outputs, is made twice and must repeat bit for bit, and must be
exactly one launch in profile slot 6.  The backward's d_image must repeat bit for bit; d_xyz sums with atomics.

Bars (u = 2^-24).  Each is an upper bound on the fp32 error of the operations the kernel performs, restated next to the
kernel line it follows; none is fitted to a measurement.  Run with -s to see every worst error / bar and every
excluded share.
  * source coordinate of the bilinear up-sampling (`lin_src`): 0 where the kernel's fp32 `scale * (dst + 0.5) - 0.5` is
    exact (checked per index), else `(dst + 0.5) |fl(R/S) - R/S| + u |scale (dst + 0.5)| + u |s|` (`_lin_src_err`);
  * up-sampled values: that coordinate error times the largest difference of adjacent render texels, plus 6 u |value|
    (two levels of a two-tap blend, each weight `1 - l` rounded once);
  * lookup coordinate `ix` at size n (`_ix_err`): n / box_warp times the value error, plus 10 u W n for the ten
    roundings of `1 - (v + bw/2) / bw -> vij * 2 - 1 -> ((g + 1) n - 1) / 2`, every intermediate bounded by W = 1 + |vij|;
  * `paste`: 9 u max|tap| for the 4-tap blend (8 roundings, weights included, plus the weights' sum exceeding 1) plus the
    coordinate error of each axis times the largest difference between the texels of every cell the fp32 coordinate can
    fall in.  An axis whose fp64 coordinate lies clearly past a border contributes no coordinate term: the clip is exact;
  * `image`: the mask times the paste bar plus 4 u (|image| + |paste|) for the two-sided lerp;
  * `mask_occ`: the two source coordinate errors (a blend of exact 0 / 1) plus 6 u; `mask_frontweight` is a lookup of
    exact 0 / 1 at size Rf and gets the paste bar;
  * thresholded masks are exact except within a margin of the threshold: weights 6 u + the value error; edges
    sqrt(6) times the Sobel component error (|dq / dg| summed over six components <= sqrt(6)) plus 5 u q; both plus the
    fp32 rounding of the threshold.  `mask_dxyz` is compared with the fp32 oracle on the GPU (the reference's own
    arithmetic): the kernel rounds its subtractions, products and dot product in the eager ops' order, and only torch's
    sum of squares may contract into fmas: margin 4 u q.  `mask_dxyz` also excludes the `nearest` source index where
    `dst R / S` lies within `dst |fl(R/S) - R/S| + u |dst fl(R/S)|` of an integer (the product's rounding counts only
    where it is inexact), counted separately: only `ragged` has such indices;
  * d_xyz per texel: (k + 16) u A + the coordinate terms, A the fp64 adjoint of the absolute contributions, k the most
    contributions any texel receives (16: the roundings of one contribution, tallied at `_bwd_bars`).  Pixels whose fp64
    lookup coordinate lies within its error of an integer or a border get zero upstream gradient (the derivative jumps
    there), counted.

Negative controls (each must miss the kernel by >= 20 x its bar somewhere): the oracle's lookup shifted by half a texel,
the oracle's up-sampling with align_corners=True, the backward oracle without the normalize_images factor.
"""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import paste_oracle as po
from tests.helpers import profiled

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
PROF_OTHER = 6                    # profile slot (csrc/p3d_common.cuh)
BW = 0.7
EVAL = dict(thresh_weight=0.95, thresh_edges=0.02, thresh_occ=0.05, thresh_dxyz=0.000005)   # generate.py:59-65, loss_orthocondA.py:133-139
EROSION = 3
C_UP, C_IX, C_BLEND, C_LERP, C_G = 6, 10, 9, 4, 16
NEG_MARGIN = 20.0
BORDER_SHARE = 0.01

CASES = {
    'eval': dict(seed=41, N=8, R=128, S=512, Rf=0, normalize=False, reach=1.2),
    'train_agrad': dict(seed=42, N=4, R=64, S=512, Rf=0, normalize=False, reach=1.2),
    'train_erode': dict(seed=43, N=2, R=64, S=512, Rf=128, normalize=False, reach=1.2),
    'ragged': dict(seed=44, N=3, R=48, S=500, Rf=37, normalize=True, reach=1.2),
    'same_res': dict(seed=45, N=1, R=37, S=37, Rf=37, normalize=True, reach=1.2),
    'down': dict(seed=46, N=2, R=96, S=64, Rf=0, normalize=False, reach=1.2),
    'tiny_1x7': dict(seed=47, N=2, R=1, S=7, Rf=0, normalize=False, reach=4.0),
    'tiny_2x3': dict(seed=48, N=2, R=2, S=3, Rf=0, normalize=False, reach=4.0),
}
BWD_CASES = ('train_agrad', 'ragged', 'same_res', 'down', 'eval')     # eval: grad_sample=False, d_image only
UPSTREAM = ('image', 'paste', 'both')


def _lib():
    import panic3d_b200.paste  # noqa: F401  (binds the p3d_paste_* prototypes)
    from panic3d_b200 import _lib as lib
    return lib


# ------------------------------------------------------------------------------------------------- inputs and calls
@functools.lru_cache(maxsize=None)
def _inputs_cpu(name):
    c = CASES[name]
    inp = po.synth_paste_inputs(c['seed'], c['N'], c['R'], c['S'], box_warp=BW, reach=c['reach'])
    if c['Rf']:
        inp['frontw'] = F.interpolate(inp['frontw'], c['Rf'], mode='bilinear')
    return inp


def _inputs(name):
    import panic3d_b200.paste as pp
    c = CASES[name]
    d = {k: v.to(DEV) for k, v in _inputs_cpu(name).items() if torch.is_tensor(v)}
    d['eroded'] = pp.erode_front_weights(d['frontw'], EROSION) if c['Rf'] else None
    return d


def _params(c, n=None):
    import panic3d_b200.paste as pp
    p = pp.PasteParams()
    p.n_views, p.res_render, p.res_image, p.res_front = n or c['N'], c['R'], c['S'], c['Rf']
    p.normalize_images = int(c['normalize'])
    p.box_warp = BW
    p.thresh_weight, p.thresh_edges, p.thresh_occ, p.thresh_dxyz = (EVAL[k] for k in ('thresh_weight', 'thresh_edges', 'thresh_occ', 'thresh_dxyz'))
    return p


def _view(d, n):
    return {k: (None if v is None else v[n:n + 1].contiguous()) for k, v in d.items()}


def _forward(c, d, n_views=None, want_parts=True):
    """p3d_paste_front through the C ABI, outputs NaN-prefilled.  Made twice: the two runs must be equal bit for bit and
    each must be exactly one launch in profile slot 6."""
    lib = _lib()
    N, S = n_views or c['N'], c['S']
    runs = []
    for _ in range(2):
        o = {'image': torch.full((N, 3, S, S), float('nan'), device=DEV), 'paste': torch.full((N, 3, S, S), float('nan'), device=DEV),
             'mask': torch.full((N, 1, S, S), float('nan'), device=DEV),
             'parts': torch.full((5, N, 1, S, S), float('nan'), device=DEV) if want_parts else None}
        p = _params(c, N)

        def call():
            lib.check(lib.lib().p3d_paste_front(C.byref(p), d['image'].data_ptr(), d['image_xyz'].data_ptr(), d['image_weights'].data_ptr(),
                                                d['front_rgb'].data_ptr(), d['occ'].data_ptr(), d['ro'].data_ptr(), d['rd'].data_ptr(),
                                                lib.ptr(d['eroded']), o['image'].data_ptr(), o['paste'].data_ptr(), o['mask'].data_ptr(),
                                                lib.ptr(o['parts']), lib.stream_ptr(torch.device(DEV))))
        _, launches = profiled(call)
        assert launches[PROF_OTHER] == 1 and sum(launches) == 1, launches
        runs.append(o)
    for k, v in runs[0].items():
        if v is not None:
            assert not torch.isnan(v).any(), f'{k}: an element no thread wrote'
            assert torch.equal(v, runs[1][k]), f'{k}: two runs differ'
    return runs[0]


def _backward(c, d, mask, g_img, g_paste, want_xyz):
    """p3d_paste_front_backward through the C ABI: d_image NaN-prefilled, d_xyz zeroed (it accumulates).  Made twice;
    d_image must repeat bit for bit.  Returns d_image and both d_xyz runs."""
    lib = _lib()
    outs = []
    for _ in range(2):
        d_img = torch.full_like(g_img, float('nan'))
        d_xyz = torch.zeros_like(d['image_xyz']) if want_xyz else None
        p = _params(c)
        lib.check(lib.lib().p3d_paste_front_backward(C.byref(p), d['image_xyz'].data_ptr(), d['front_rgb'].data_ptr(), mask.data_ptr(),
                                                     g_img.data_ptr(), lib.ptr(g_paste), d_img.data_ptr(), lib.ptr(d_xyz),
                                                     lib.stream_ptr(torch.device(DEV))))
        torch.cuda.synchronize()
        outs.append((d_img, d_xyz))
    assert not torch.isnan(outs[0][0]).any() and torch.equal(outs[0][0], outs[1][0]), 'd_image'
    return outs[0][0], outs[0][1], outs[1][1]


def _oracle(c, d, dtype=torch.float64, up_shift=0.0, align_corners=False):
    """oracle.paste_oracle.paste_front on the device in `dtype`; the negative controls shift the up-sampled world x by
    `up_shift` or up-sample with align_corners=True."""
    t = {k: (None if v is None else v.to(dtype)) for k, v in d.items()}
    kw = dict(EVAL, frontw=t['frontw'] if c['Rf'] else None, normalize_images=c['normalize'], front_weight_erosion=EROSION if c['Rf'] else 0)
    if not (up_shift or align_corners):
        return po.paste_front(t['image'], t['image_xyz'], t['image_weights'], t['front_rgb'], t['occ'], t['ro'], t['rd'], BW, **kw)
    up = F.interpolate(t['image_xyz'], c['S'], mode='bilinear', align_corners=align_corners)
    up[:, 0] += up_shift
    tocopy = t['front_rgb'] * 2 - 1 if c['normalize'] else t['front_rgb']
    return {'paste': po.sample_orthofront(tocopy, up, BW)}


# ------------------------------------------------------------------------------------------------- bars
def _lin_src_err(R, S):
    """|s_fp32 - s| of lin_src (paste_front.cu:29-38) per destination index, in source texels: s = scale (dst + 0.5) - 0.5
    with the kernel's scale = fl(R / S).  Zero where each fp32 step is exact (fma contraction or not, the result is the
    exact value then); otherwise the scale's rounding times (dst + 0.5) plus one rounding of the product and one of the
    difference."""
    dst = np.arange(S, dtype=np.float64)
    sc32 = float(np.float32(R) / np.float32(S))
    prod = sc32 * (dst + 0.5)                                          # exact in fp64 (24 x 24 bits)
    prod_exact = prod.astype(np.float32).astype(np.float64) == prod
    s = prod - 0.5
    sub_exact = s.astype(np.float32).astype(np.float64) == s
    err = (dst + 0.5) * abs(sc32 - R / S) + np.where(prod_exact, 0.0, U * np.abs(prod)) + np.where(sub_exact, 0.0, U * np.abs(s))
    return torch.from_numpy(err).to(DEV)


def _up_matrices(R, S):
    """The (S, R) bilinear up-sampling matrix of F.interpolate(align_corners=False) in fp64 (aten UpSample.h
    area_pixel_compute_source_index + guard_index_and_lambda), and the matching tap-count matrix (an index tapped twice,
    i0 == i1, counts twice: the kernel adds twice)."""
    dst = torch.arange(S, dtype=torch.float64)
    s = ((dst + 0.5) * R / S - 0.5).clamp(min=0)
    i0 = s.floor().long().clamp(max=R - 1)
    i1 = (i0 + 1).clamp(max=R - 1)
    l1 = (s - i0).clamp(0, 1)
    W, Cn = torch.zeros(S, R, dtype=torch.float64), torch.zeros(S, R, dtype=torch.float64)
    W.index_put_((torch.arange(S), i0), 1 - l1, accumulate=True)
    W.index_put_((torch.arange(S), i1), l1, accumulate=True)
    Cn.index_put_((torch.arange(S), i0), torch.ones(S, dtype=torch.float64), accumulate=True)
    Cn.index_put_((torch.arange(S), i1), torch.ones(S, dtype=torch.float64), accumulate=True)
    return W.to(DEV), Cn.to(DEV)


def _adjoint(M, X):
    """M^T X M per image: the adjoint of the separable up-sampling M applied to X (N, C, S, S) -> (N, C, R, R)."""
    return M.t() @ X @ M


def _adjacent_diff(x):
    """Largest difference between horizontally or vertically adjacent texels of x (N, C, R, R), per view (N, 1, 1, 1)."""
    dx = (x[..., :, 1:] - x[..., :, :-1]).abs().flatten(1).amax(1) if x.shape[-1] > 1 else x.new_zeros(x.shape[0])
    dy = (x[..., 1:, :] - x[..., :-1, :]).abs().flatten(1).amax(1) if x.shape[-2] > 1 else x.new_zeros(x.shape[0])
    return torch.maximum(dx, dy).view(-1, 1, 1, 1)


def _value_err(c, x64, es):
    """Error bound of the kernel's fp32 bilinear up-sampling of x (N, C, R, R) at every output pixel (N, 1, S, S)."""
    return es * _adjacent_diff(x64) + C_UP * U * x64.abs().flatten(1).amax(1).view(-1, 1, 1, 1)


def _ix_err(n, src, dv):
    """Error bound of the kernel's lookup coordinate at size n (ortho_tap, paste_front.cu:49-63) given the error dv of the
    up-sampled world coordinate and the fp64 coordinate src."""
    W = 1 + ((src + 0.5) / n).abs()
    return n / BW * dv + C_IX * U * W * n


def _cells_gather(img, r, c, n):
    """Texels of img (N, C, n, n) at the 2 x 2 cell with corner (r, c) (N, 1, S, S long): the four taps, clamped like the
    kernel's r1 / c1."""
    N, Cc = img.shape[:2]
    flat = img.reshape(N, Cc, n * n)
    r1, c1 = (r + 1).clamp(max=n - 1), (c + 1).clamp(max=n - 1)
    g = lambda rr, cc: flat.gather(2, (rr * n + cc).reshape(N, 1, -1).expand(-1, Cc, -1)).reshape(N, Cc, *r.shape[-2:])
    return g(r, c), g(r1, c), g(r, c1), g(r1, c1)


def _lookup_bar(img, n, src_r, src_c, er, ec):
    """Bar of a bilinear lookup of img (N, C, n, n) at fp64 coordinates (src_r, src_c) with coordinate errors (er, ec): the
    blend's rounding on the largest tap plus each axis' error times the largest texel difference of every cell the fp32
    coordinate can fall in.  An axis clearly past a border gets no coordinate term.  Returns (bar, clipped_r, clipped_c)."""
    hi_b = n - 1
    clip_r = (src_r < -er) | (src_r > hi_b + er)
    clip_c = (src_c < -ec) | (src_c > hi_b + ec)
    cells = lambda s, e: [(s - e).clamp(0, hi_b).floor().long(), (s + e).clamp(0, hi_b).floor().long()]
    hi = lo = None
    for r in cells(src_r, er):
        for cc in cells(src_c, ec):
            for t in _cells_gather(img, r, cc, n):
                hi, lo = (t, t) if hi is None else (torch.maximum(hi, t), torch.minimum(lo, t))
    coord = torch.where(clip_r, 0.0, er) + torch.where(clip_c, 0.0, ec)
    return C_BLEND * U * torch.maximum(hi.abs(), lo.abs()) + coord * (hi - lo), clip_r, clip_c


def _ratio(err, bar):
    """Worst err / bar; NaN counts as a failure."""
    r = err / bar.clamp(min=1e-300)
    return float('inf') if torch.isnan(r).any() else float(r.max())


def _fwd_bars(c, d, o64, th=EVAL):
    """Every per-pixel bar and borderline set of the forward (see the module docstring); th: the thresholds."""
    N, R, S, Rf = c['N'], c['R'], c['S'], c['Rf']
    es1 = _lin_src_err(R, S)
    es = es1.view(1, 1, S, 1) + es1.view(1, 1, 1, S)                  # rows + columns
    xyz = d['image_xyz'].double()
    dv_xy = _value_err(c, xyz[:, :2], es)
    dv_all = _value_err(c, xyz, es)
    er, ec = _ix_err(S, o64['src_row'], dv_xy), _ix_err(S, o64['src_col'], dv_xy)
    front = d['front_rgb'].double()
    tocopy = front * 2 - 1 if c['normalize'] else front
    bar_paste, clip_r, clip_c = _lookup_bar(tocopy, S, o64['src_row'], o64['src_col'], er, ec)
    b = {'paste': bar_paste, 'clip_r': clip_r, 'clip_c': clip_c, 'er': er, 'ec': ec, 'es1': es1}
    if Rf:
        b['frontweight'] = _lookup_bar(d['eroded'].double(), Rf, o64['src_fw_row'], o64['src_fw_col'],
                                       _ix_err(Rf, o64['src_fw_row'], dv_xy), _ix_err(Rf, o64['src_fw_col'], dv_xy))[0]
    b['occ'] = es + C_UP * U
    w = d['image_weights'].double()
    t32 = lambda t: abs(float(np.float32(t)) - t)
    m_w = _value_err(c, w, es) + t32(th['thresh_weight'])
    # Sobel component: six up-sampled values with |coefficients| summing to 1, five roundings of differences of values at
    # most two output pixels (max(1, R / S) source texels) apart
    dg = dv_all + 5 * U * 2 * max(1.0, R / S) * _adjacent_diff(xyz)
    m_e = math.sqrt(6) * dg + 5 * U * th['thresh_edges'] + t32(th['thresh_edges'])
    b['border_w'] = (o64['q_weights'] - th['thresh_weight']).abs() <= m_w
    b['border_e'] = (o64['q_edges'] - th['thresh_edges']).abs() <= m_e
    # nearest source index floorf(dst * fl(R / S)) (paste_front.cu:127): the scale's rounding times dst plus one rounding of
    # the product, zero where the fp32 product is exact (then floorf sees the exact value)
    nn = o64['src_nearest']
    sc32 = float(np.float32(R) / np.float32(S))
    prod = torch.arange(S, device=DEV, dtype=torch.float64) * sc32
    exact = prod.float().double() == prod
    margin = torch.arange(S, device=DEV, dtype=torch.float64) * abs(sc32 - R / S) + torch.where(exact, 0.0, U * prod.abs())
    near = (nn - nn.round()).abs() < margin
    b['border_nearest'] = (near.view(1, 1, S, 1) | near.view(1, 1, 1, S)).expand(N, 1, S, S)
    return b


# ------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize('name', list(CASES))
def test_forward_against_fp64_oracle(name):
    torch.cuda.reset_peak_memory_stats()
    c = CASES[name]
    N, S = c['N'], c['S']
    d = _inputs(name)
    k = _forward(c, d)
    o64 = _oracle(c, d)
    o32 = _oracle(c, d, torch.float32)
    b = _fwd_bars(c, d, o64)
    parts = dict(zip(('weights', 'edges', 'occ', 'dxyz', 'frontweight'), k['parts']))
    report = {}

    # thresholded masks: exact away from their borderline sets
    m_d = (o32['q_dxyz'] - float(np.float32(EVAL['thresh_dxyz']))).abs() <= 4 * U * EVAL['thresh_dxyz']
    nearest = b['border_nearest']
    for key, excl in (('weights', b['border_w']), ('edges', b['border_e']), ('dxyz', m_d)):
        share = float(excl.double().mean())
        assert share < BORDER_SHARE, (key, share)
        ok = ~excl & ~nearest if key == 'dxyz' else ~excl
        ref = o32 if key == 'dxyz' else o64
        bad = int((parts[key].double() != ref[f'mask_{key}'].double())[ok].sum())
        assert bad == 0, (key, bad)
        report[f'excluded_{key}'] = share
    report['excluded_nearest'] = float(nearest.double().mean())
    assert report['excluded_nearest'] < 2 * BORDER_SHARE
    for key in ('weights', 'edges', 'dxyz'):
        assert set(parts[key].unique().tolist()) <= {0.0, 1.0}
    if N * S * S >= 4096:                                              # every mask takes both values
        # below scale 1/4 the inputs' depth step (0.12) spreads over more than 6 pixels: every Sobel magnitude is under 0.02
        for key in ('weights', 'occ', 'dxyz') + (('edges',) if 4 * c['R'] >= S else ()):
            assert 0.0 < float((parts[key] > 0.5).float().mean()) < 1.0, key

    # continuous masks
    report['occ'] = _ratio((parts['occ'].double() - o64['mask_occ']).abs(), b['occ'])
    assert report['occ'] <= 1.0
    if c['Rf']:
        report['frontweight'] = _ratio((parts['frontweight'].double() - o64['mask_frontweight']).abs(), b['frontweight'])
        assert report['frontweight'] <= 1.0
        assert 0.0 < float((parts['frontweight'] > 0.5).float().mean()) < 1.0
    else:
        assert bool((parts['frontweight'] == 1).all())
    assert torch.equal(k['mask'], parts['weights'] * parts['edges'] * parts['occ'] * parts['dxyz'] * parts['frontweight'])

    # paste and image
    err_p = (k['paste'].double() - o64['paste']).abs()
    report['paste'] = _ratio(err_p, b['paste'])
    assert report['paste'] <= 1.0, report
    m64 = k['mask'].double()
    img_ref = torch.lerp(d['image'].double(), o64['paste'], m64)
    bar_img = m64 * b['paste'] + C_LERP * U * (d['image'].double().abs() + o64['paste'].abs())
    report['image'] = _ratio((k['image'].double() - img_ref).abs(), bar_img)
    assert report['image'] <= 1.0, report

    # clipped regions: both lookups reach past every border of the box (tiny_1x7 has one world point, at the centre)
    clip_r, clip_c = b['clip_r'], b['clip_c']
    if c['R'] > 1:
        for clip, src in ((clip_r, o64['src_row']), (clip_c, o64['src_col'])):
            assert bool((clip & (src < 0)).any()) and bool((clip & (src > S - 1)).any())
        if c['Rf']:
            assert bool((o64['src_fw_row'] < 0).any()) and bool((o64['src_fw_col'] > c['Rf'] - 1).any())
        cl = (clip_r | clip_c).expand_as(err_p)
        report['paste_clipped'] = _ratio(err_p[cl], b['paste'][cl])
        report['clipped_share'] = float((clip_r | clip_c).double().mean())

    # negative controls
    if c['R'] > 2:
        for ctl, kw in (('shift', dict(up_shift=0.5 * BW / S)), ('align_corners', dict(align_corners=True))):
            if ctl == 'align_corners' and c['R'] == c['S']:
                continue                                               # identical up-sampling at scale 1
            miss = _ratio((k['paste'].double() - _oracle(c, d, **kw)['paste']).abs(), b['paste'])
            report[f'control_{ctl}'] = miss
            assert miss >= NEG_MARGIN, (ctl, miss)

    # views are independent: each view alone gives the batch's outputs bit for bit (per-view offsets, the N S^2 parts stride)
    for n in range(N):
        kn = _forward(c, _view(d, n), n_views=1)
        for key in ('image', 'paste', 'mask'):
            assert torch.equal(kn[key][0], k[key][n]), (n, key)
        assert torch.equal(kn['parts'][:, 0], k['parts'][:, n]), n
    # want_parts=False: the same outputs
    kp = _forward(c, d, want_parts=False)
    for key in ('image', 'paste', 'mask'):
        assert torch.equal(kp[key], k[key]), key
    report['peak_GB'] = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f'\n[paste fwd {name}] ' + ', '.join(f'{kk} {v:.3g}' for kk, v in report.items()))


# ------------------------------------------------------------------------------------------------- backward
def _upstream(c, which, zero):
    g = torch.Generator(device=DEV).manual_seed(c['seed'])
    shape = (c['N'], 3, c['S'], c['S'])
    g_img = torch.randn(shape, generator=g, device=DEV) if which in ('image', 'both') else torch.zeros(shape, device=DEV)
    g_paste = torch.randn(shape, generator=g, device=DEV) if which in ('paste', 'both') else None
    g_img = g_img.masked_fill(zero, 0.0)
    if g_paste is not None:
        g_paste = g_paste.masked_fill(zero, 0.0)
    return g_img, g_paste


def _zero_set(c, o64, er, ec):
    """Pixels whose fp64 lookup coordinate lies within its error bound of an integer (a cell boundary, 0 and S - 1
    included) on either axis without being clearly clipped: the derivative jumps there."""
    S = c['S']
    near = lambda s, e: (s > -e) & (s < S - 1 + e) & ((s - s.round()).abs() <= e)
    return near(o64['src_row'], er) | near(o64['src_col'], ec)


def _bwd_reference(c, d, mask, g_img, g_paste, normalize=None):
    """fp64 autograd through the oracle's interpolate -> sample_orthofront chain, fed the kernel's mask."""
    normalize = c['normalize'] if normalize is None else normalize
    xyz = d['image_xyz'].double().requires_grad_(True)
    front = d['front_rgb'].double()
    paste = po.sample_orthofront(front * 2 - 1 if normalize else front, F.interpolate(xyz, c['S'], mode='bilinear'), BW)
    gp = g_img.double() * mask.double() + (0 if g_paste is None else g_paste.double())
    (paste * gp).sum().backward()
    return xyz.grad


def _bwd_bars(c, d, o64, mask, g_img, g_paste, b):
    """Per-texel bar of d_xyz.  One contribution g_v * w of a pixel rounds: gp = g m + g_paste (2), four tap differences
    (1), (1 - f) and its product (2), the two-term sum (1), times gp (1), the three-channel sum (2), gmul = -(float)S *
    fl(1 / fl(bw)) (3) and its product (1), the weight by.l * bx.l (1) and its product (1): 15 u, taken as 16 u of the
    pixel's absolute contribution.  The atomic sum of k contributions adds (k - 1) u A at most.  Coordinate terms: the
    row fraction's error moves the column derivative by <= 2 * (largest tap difference) per channel and vice versa; the
    up-sampling weights' error (the source coordinate error) moves each tap's weight."""
    S, R = c['S'], c['R']
    Wm, Cm = _up_matrices(R, S)
    xyz = d['image_xyz'].double()
    assert torch.allclose(Wm @ xyz @ Wm.t(), F.interpolate(xyz, S, mode='bilinear'), rtol=0, atol=1e-12)   # the restatement is torch's
    ns = 2.0 if c['normalize'] else 1.0
    front = d['front_rgb'].double() * ns
    gabs = g_img.double().abs() * mask.double() + (0 if g_paste is None else g_paste.double().abs())
    r_, c_ = o64['src_row'].clamp(0, S - 1), o64['src_col'].clamp(0, S - 1)
    r0, c0 = r_.floor().long(), c_.floor().long()
    fr, fc = r_ - r0, c_ - c0
    f00, f10, f01, f11 = _cells_gather(front, r0, c0, S)
    in_r = (o64['src_row'] > 0) & (o64['src_row'] < S - 1)
    in_c = (o64['src_col'] > 0) & (o64['src_col'] < S - 1)
    st = torch.stack([f00, f10, f01, f11])
    rng = st.amax(0) - st.amin(0)
    M_col = S / BW * (gabs * ((f01 - f00).abs() * (1 - fr) + (f11 - f10).abs() * fr)).sum(1, keepdim=True) * in_c
    M_row = S / BW * (gabs * ((f10 - f00).abs() * (1 - fc) + (f11 - f01).abs() * fc)).sum(1, keepdim=True) * in_r
    E_col = S / BW * (gabs * 2 * rng).sum(1, keepdim=True) * b['er'] * in_c
    E_row = S / BW * (gabs * 2 * rng).sum(1, keepdim=True) * b['ec'] * in_r
    es = b['es1'].view(1, 1, S, 1) + b['es1'].view(1, 1, 1, S)
    k = int(Cm.sum(0).max().item()) ** 2
    A = torch.cat([_adjoint(Wm, M_col), _adjoint(Wm, M_row)], 1)
    coord = torch.cat([_adjoint(Wm, E_col) + _adjoint(Cm, M_col * es), _adjoint(Wm, E_row) + _adjoint(Cm, M_row * es)], 1)
    return (k + C_G) * U * A + coord, A, k


@pytest.mark.parametrize('which', UPSTREAM)
@pytest.mark.parametrize('name', BWD_CASES)
def test_backward_against_fp64_autograd(name, which):
    c = CASES[name]
    grad_sample = name != 'eval'
    d = _inputs(name)
    k = _forward(c, d)
    o64 = _oracle(c, d)
    b = _fwd_bars(c, d, o64)
    zero = _zero_set(c, o64, b['er'], b['ec'])
    zshare = float(zero.double().mean())
    assert zshare < BORDER_SHARE, zshare
    g_img, g_paste = _upstream(c, which, zero)
    gp_kernel = g_paste if grad_sample else None
    d_img, d_xyz, d_xyz2 = _backward(c, d, k['mask'], g_img, gp_kernel, grad_sample)
    assert torch.equal(d_img, g_img * (1 - k['mask'])), 'd_image'
    report = {'zeroed': zshare}
    if grad_sample:
        ref = _bwd_reference(c, d, k['mask'], g_img, gp_kernel)
        bar, A, kmax = _bwd_bars(c, d, o64, k['mask'], g_img, gp_kernel, b)
        assert bool((d_xyz[:, 2] == 0).all()) and bool((ref[:, 2] == 0).all())
        err = (d_xyz[:, :2].double() - ref[:, :2]).abs()
        report['d_xyz'] = _ratio(err, bar)
        assert report['d_xyz'] <= 1.0, report
        dead = A == 0                                                  # every contributing pixel clips (or was zeroed)
        assert bool((d_xyz[:, :2][dead] == 0).all()) and bool((ref[:, :2][dead] == 0).all())
        assert bool(dead[:, 0].any()) and bool(dead[:, 1].any())
        live = bool((~dead).any())
        assert live or which == 'image'                                # same_res's mask is 0 wherever the lookup is inside
        report['dead_texels'] = float(dead.double().mean())
        report['k'] = kmax
        # the two runs differ only by the order of the atomic sums
        assert bool(((d_xyz - d_xyz2)[:, :2].double().abs() <= 2 * kmax * U * A).all())
        if c['normalize'] and live:
            miss = _ratio((d_xyz[:, :2].double() - _bwd_reference(c, d, k['mask'], g_img, gp_kernel, normalize=False)[:, :2]).abs(), bar)
            report['control_no_normalize'] = miss
            assert miss >= NEG_MARGIN, miss
        # the autograd route (paste_front_fused) gives the same gradients; with g_image absent autograd materialises zeros
        ai, ax = _autograd_route(c, d, g_img if which != 'paste' else None, gp_kernel, grad_sample)
        assert torch.equal(ai, d_img)
        assert bool(((ax - d_xyz)[:, :2].double().abs() <= 2 * kmax * U * A).all()) and bool((ax[:, 2] == 0).all())
    else:
        ai, ax = _autograd_route(c, d, g_img if which != 'paste' else None, g_paste, grad_sample)
        assert ax is None and torch.equal(ai, d_img if which != 'paste' else torch.zeros_like(d_img))
    print(f'\n[paste bwd {name} {which}] ' + ', '.join(f'{kk} {v:.3g}' for kk, v in report.items()))


def _autograd_route(c, d, g_img, g_paste, grad_sample):
    import panic3d_b200.paste as pp
    image = d['image'].clone().requires_grad_(True)
    xyz = d['image_xyz'].clone().requires_grad_(True)
    img, paste, _, _ = pp.paste_front_fused(image, xyz, d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], BW,
                                            front_eroded=d['eroded'], normalize_images=c['normalize'], grad_sample=grad_sample, **EVAL)
    loss = 0
    if g_img is not None:
        loss = loss + (img * g_img).sum()
    if g_paste is not None:
        loss = loss + (paste * g_paste).sum()
    if g_img is None and (g_paste is None or not grad_sample):
        loss = loss + img.sum() * 0                                    # the image output carries a zero gradient
    loss.backward()
    return image.grad, xyz.grad


# ------------------------------------------------------------------------------------------------- call surface
def test_inputs_as_the_pipeline_hands_them_over():
    """image in fp16 and channels_last, image_xyz a non-contiguous view: outputs equal the run on contiguous fp32
    copies bit for bit, gradients arrive in each input's dtype and shape."""
    import panic3d_b200.paste as pp
    c = CASES['train_agrad']
    d = _inputs('train_agrad')
    N, R, S = c['N'], c['R'], c['S']
    g = torch.Generator(device=DEV).manual_seed(7)
    g_img, g_paste = torch.randn(N, 3, S, S, generator=g, device=DEV), torch.randn(N, 3, S, S, generator=g, device=DEV)
    img16 = d['image'].half().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    base = torch.zeros(N, 3, R, 2 * R, device=DEV)
    base[..., ::2] = d['image_xyz']
    xyz_view = base[..., ::2].detach().requires_grad_(True)
    assert not xyz_view.is_contiguous() and not img16.is_contiguous()
    img32 = img16.detach().float().contiguous().requires_grad_(True)
    xyz32 = d['image_xyz'].clone().requires_grad_(True)
    outs, grads = [], []
    for im, xy in ((img16, xyz_view), (img32, xyz32)):
        o = pp.paste_front_fused(im, xy, d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], BW, grad_sample=True, **EVAL)
        ((o[0] * g_img).sum() + (o[1] * g_paste).sum()).backward()
        outs.append(o)
        grads.append((im.grad, xy.grad))
    for a, b_ in zip(outs[0], outs[1]):
        assert torch.equal(a, b_)
    assert grads[0][0].dtype == torch.float16 and tuple(grads[0][0].shape) == (N, 3, S, S)
    assert grads[0][1].dtype == torch.float32 and tuple(grads[0][1].shape) == (N, 3, R, R)
    assert torch.equal(grads[0][0], grads[1][0].half())
    o64 = _oracle(c, d)
    b = _fwd_bars(c, d, o64)
    _, A, kmax = _bwd_bars(c, d, o64, outs[1][2], g_img, g_paste, b)
    assert bool(((grads[0][1] - grads[1][1])[:, :2].double().abs() <= 2 * kmax * U * A).all())


def test_dropin_paste_front_equals_the_fused_call():
    """panic3d_b200.paste.paste_front(G, x, out, grad_sample=True, **EVAL) at the training size: gradients into
    out['image'] and out['image_xyz'] equal paste_front_fused's (d_xyz up to the order of its atomic sums)."""
    import panic3d_b200.paste as pp
    from tests.helpers import StandInG
    c = CASES['train_agrad']
    inp = _inputs_cpu('train_agrad')
    d = _inputs('train_agrad')
    N, S = c['N'], c['S']
    g = torch.Generator(device=DEV).manual_seed(8)
    g_img, g_paste = torch.randn(N, 3, S, S, generator=g, device=DEV), torch.randn(N, 3, S, S, generator=g, device=DEV)
    G = StandInG(inp, DEV)
    x = {'cond': {'image_ortho_front': d['front_rgb']}, 'normalize_images': False,
         'force_rays': {'ray_origins': d['ro'], 'ray_directions': d['rd']}, 'paste_params': dict(EVAL)}
    out = {'image': d['image'].clone().requires_grad_(True), 'image_xyz': d['image_xyz'].clone().requires_grad_(True),
           'image_weights': d['image_weights']}
    res = pp.paste_front(G, x, out, grad_sample=True, **EVAL)
    ((res['image'] * g_img).sum() + (res['paste'] * g_paste).sum()).backward()
    image = d['image'].clone().requires_grad_(True)
    xyz = d['image_xyz'].clone().requires_grad_(True)
    ro, rd = pp.occlusion_rays(d['image_xyz'], inp['ray_start'], 0.01)
    assert torch.equal(G.seen['occ_ro'], ro) and torch.equal(G.seen['occ_rd'], rd)
    o = pp.paste_front_fused(image, xyz, d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], BW, grad_sample=True, **EVAL)
    ((o[0] * g_img).sum() + (o[1] * g_paste).sum()).backward()
    assert torch.equal(res['image'], o[0]) and torch.equal(res['mask'], o[2])
    assert torch.equal(out['image'].grad, image.grad)
    o64 = _oracle(c, d)
    _, A, kmax = _bwd_bars(c, d, o64, o[2], g_img, g_paste, _fwd_bars(c, d, o64))
    assert bool(((out['image_xyz'].grad - xyz.grad)[:, :2].double().abs() <= 2 * kmax * U * A).all())
    assert bool((out['image_xyz'].grad[:, 2] == 0).all())


def test_gpu_fp64_oracle_equals_cpu_oracle():
    """Pin the device fp64 oracle to the CPU fp32 oracle (the one the reference fixtures pin) on the six fixture cases,
    at the forward bars above; mask_dxyz pins the device fp32 run to the CPU run instead (in fp64 its quantity moves by
    ~1e-7 against a 5e-6 threshold)."""
    from tests.golden.cases_paste import PASTE_CASES, build_paste_inputs
    for name, case in sorted(PASTE_CASES.items()):
        inp = build_paste_inputs(case)
        p = {kk: v for kk, v in case['params'].items() if kk not in ('offset_occ', 'mode')}
        ero = p.get('front_weight_erosion', 0)
        run = lambda dev, dt: po.paste_front(*(inp[kk].to(dev, dt) for kk in ('image', 'image_xyz', 'image_weights', 'front_rgb', 'occ', 'ro', 'rd')),
                                             inp['box_warp'], frontw=inp['frontw'].to(dev, dt), normalize_images=case['normalize_images'], **p)
        cpu, g64, g32 = run('cpu', torch.float32), run(DEV, torch.float64), run(DEV, torch.float32)
        c = dict(N=case['N'], R=case['R'], S=case['S'], Rf=case['R'] if ero else 0, normalize=case['normalize_images'])
        d = {kk: inp[kk].to(DEV) for kk in ('image_xyz', 'image_weights', 'front_rgb')}
        d['eroded'] = po.erosion_ones((inp['frontw'] > 0.5).float(), ero).to(DEV) if ero else None
        b = _fwd_bars(c, d, g64, th=dict(thresh_weight=p.get('thresh_weight', 0.95), thresh_edges=p.get('thresh_edges', 0.02)))
        assert _ratio((cpu['paste'].to(DEV).double() - g64['paste']).abs(), b['paste']) <= 1.0, name
        assert _ratio((cpu['mask_occ'].to(DEV).double() - g64['mask_occ']).abs(), b['occ']) <= 1.0, name
        if ero:
            assert _ratio((cpu['mask_frontweight'].to(DEV).double() - g64['mask_frontweight']).abs(), b['frontweight']) <= 1.0, name
        for key, border in (('weights', b['border_w']), ('edges', b['border_e'])):
            ok = ~border
            assert torch.equal(cpu[f'mask_{key}'].to(DEV)[ok], g64[f'mask_{key}'].float()[ok]), (name, key)
        td = p.get('thresh_dxyz', 0.01)
        ok = (g32['q_dxyz'] - float(np.float32(td))).abs() > 4 * U * td        # same operations, same order; the norm may contract
        assert torch.equal(cpu['mask_dxyz'].to(DEV)[ok], g32['mask_dxyz'][ok]), name
        assert float((~ok).double().mean()) < BORDER_SHARE, name
