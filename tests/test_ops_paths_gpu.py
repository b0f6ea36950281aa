"""GPU: bias_act, upfirdn2d and filtered_lrelu at the shapes that select their fast kernels, against the fp64 oracle.

tests/test_ops_gpu.py runs every op at fixture sizes, which are too small to reach the kernels training actually runs:
row-mode bias_act, the persistent cp.async upfirdn2d kernel walking several tiles per CTA, the channels-last kernel's
grid-stride loop, the image laps past gridDim.y = 32768, and filtered_lrelu's sign bytes on tile seams; nor, at the sizes
generator layers run, bias_act's per-vector, generic and scalar-tail launches or upfirdn2d's tiled and strided kernels
with flip, gain and up-sampled phases.  tests/run_mutations.py's bias_act, upfirdn2d and filtered_lrelu mutants must
each fail this file.  Each test
below restates the dispatch rule its shape relies on (with the source lines) and asserts the property that matters.

Reference: ``oracle/ops_oracle.py`` in float64 on the inputs already rounded to the storage dtype, with the scalars
rounded to fp32 as they cross the C ABI.  It is plain torch, so the large shapes run it on the GPU, in channel chunks
to bound memory; ``test_gpu_oracle_equals_cpu_oracle`` pins that the GPU and CPU fp64 oracles agree.

Bars:
  * 16-bit outputs: every element within 1 ulp of the fp64 reference (plus, for the FIR ops, the fp32 accumulation
    bound below, which only matters where an output nearly cancels), and at least EXACT_SHARE of the elements equal
    to the reference rounded to the dtype.  The share catches a wrong rounding mode, which 1 ulp lets through.
  * fp32 / fp64 FIR outputs: |got - ref| <= (roundings + 1) * eps * (|x| (*) |w|), the oracle run on |x| and |w|.
  * fp32 / fp64 bias_act: a few ulps of the value.
Gated gradients are discontinuous at the lrelu kink and the clamp, so the inputs keep every pre-activation away
from them; the tests assert that margin from the fp64 reference.

Run with ``-rA`` to see the measured worst error / bar and exact-rounding share of every comparison.
"""
import math

import numpy as np
import pytest
import torch

from oracle import ops_oracle as oo
from tests.helpers import f32_scalars
from tests.render_abi import n_sm

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64
EXACT_SHARE = 0.99
MANT = {F16: 10, BF16: 7, F32: 23, F64: 52}
EMIN = {F16: -14, BF16: -126, F32: -126, F64: -1022}
EPS = {F32: 2.0 ** -24, F16: 2.0 ** -24, BF16: 2.0 ** -24, F64: 2.0 ** -53}   # unit roundoff of the accumulation type
CTAS_PER_SM_MAX = 8       # 256-thread CTAs: 2048 resident threads per SM on H100
CHUNK = 1 << 23           # elements per piece of a float64 comparison


def min_work():
    """Items / tiles that force every CTA of a persistent grid (<= 8 CTAs per SM) through at least three of them."""
    return 3 * CTAS_PER_SM_MAX * n_sm()


def ulp(v, dtype):
    """Unit in the last place of `dtype` at |v| (v float64; subnormal spacing below the smallest normal)."""
    _, e = torch.frexp(v)
    e = torch.where(v == 0, torch.full_like(e, EMIN[dtype]), torch.clamp(e - 1, min=EMIN[dtype]))
    return torch.exp2((e - MANT[dtype]).double())


class Meter:
    """Accumulates one comparison over pieces: worst |got - ref| / bar and, for 16-bit, the exact-rounding share."""

    def __init__(self, name, dtype):
        self.name, self.dtype, self.worst, self.n, self.exact = name, dtype, 0.0, 0, 0

    def add(self, got, ref, slack=None, n_ulp=4):
        """got: kernel output piece; ref: float64 reference piece; slack: float64 error bound (FIR accumulation)."""
        got, ref = got.reshape(-1), ref.reshape(-1)
        for i in range(0, got.numel(), CHUNK):
            g, r = got[i:i + CHUNK], ref[i:i + CHUNK]
            s = None if slack is None else slack.reshape(-1)[i:i + CHUNK]
            if self.dtype in (F16, BF16):
                bar = ulp(r, self.dtype) + (0 if s is None else s)
                self.exact += int((g == r.to(self.dtype)).sum())
            else:
                bar = s if s is not None else n_ulp * ulp(r, self.dtype)
            self.worst = max(self.worst, worst_ratio(g.double() - r, bar))
            self.n += g.numel()

    def done(self):
        share = self.exact / self.n if self.dtype in (F16, BF16) else None
        print(f'[ops-paths] {self.name}: worst |err|/bar = {self.worst:.3g}' +
              ('' if share is None else f', exact-rounding share = {share:.5f}') + f' ({self.n} elements)')
        assert self.worst <= 1.0, f'{self.name}: worst error is {self.worst:.3g} x the bar'
        if share is not None:
            assert share >= EXACT_SHARE, f'{self.name}: only {share:.4f} of the elements are correctly rounded'


def worst_ratio(err, bar):
    """max |err| / bar, where a NaN (an element the kernel never wrote may hold one) counts as infinitely wrong."""
    q = err.abs() / (bar + 1e-300)
    return torch.nan_to_num(q, nan=math.inf).max().item()


def chunks(n, step):
    return [slice(i, min(i + step, n)) for i in range(0, n, step)]


# ================================================================================================== bias_act
def _ba():
    from panic3d_b200.torch_utils.ops import bias_act
    return bias_act


def ba_dispatch(x, dim, grad):
    """Restates launch_bias_act_t / launch_bias_act_v (ops_bias_act.cu:167-195) for an aligned x with numel % VEC == 0:
    the BIAS variant, and the work the persistent grid walks (items of 256 * UNROLL vectors, UNROLL = 4 forward, 2 in
    the gradient modes; k_bias_act, lines 103-114)."""
    vec = 16 // x.element_size()
    assert x.numel() % vec == 0 and x.data_ptr() % 16 == 0
    step_b, nvec = x.stride(dim), x.numel() // vec
    if step_b % vec == 0 and step_b // vec >= 128 and nvec % (step_b // vec) == 0:
        mode = 'row'
    elif step_b % vec == 0:
        mode = 'per_vector'
    elif vec > 1 and step_b == 1 and x.shape[dim] % vec == 0:
        mode = 'bias_run'
    else:
        mode = 'generic'
    k_item = 256 * (4 if grad == 0 else 2)
    row_vecs = step_b // vec if mode == 'row' else nvec
    items_per_row = -(-row_vecs // k_item)
    return dict(mode=mode, items=(nvec // row_vecs) * items_per_row, items_per_row=items_per_row,
                last_item=row_vecs - (items_per_row - 1) * k_item, k_item=k_item,
                grid=min(-(-nvec // 256), CTAS_PER_SM_MAX * n_sm()))


def assert_row_mode(x, dim, grad):
    d = ba_dispatch(x, dim, grad)
    assert d['mode'] == 'row', d
    assert d['last_item'] < d['k_item'], d                   # the last item of every row is ragged
    assert d['items'] >= min_work(), d                      # every CTA walks >= 3 items (grid-stride loop)
    return d


def _bshape(ndim, dim):
    return [-1 if i == dim else 1 for i in range(ndim)]


def ba_inputs(shape, dim, dtype, act, kw, seed, fmt=torch.contiguous_format):
    """x, b in `dtype` with every pre-activation s = x + b at least 1e-3 from the lrelu kink and every gain * lrelu(s)
    at least max(1e-3, 1 ulp) from +-clamp, so the fp32 and fp64 gates agree (re-drawn until none is closer).
    tanh draws |s| <= 1, keeping 1 - y^2 >= 0.42 so the second derivative has no cancellation."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    draw = (lambda n: torch.rand(n, generator=g, device=DEV) * 1.8 - 0.9) if act == 'tanh' else \
        (lambda n: torch.randn(n, generator=g, device=DEV))
    x = draw(math.prod(shape)).reshape(shape).to(dtype).contiguous(memory_format=fmt)
    b = (draw(shape[dim]) * (0.1 if act == 'tanh' else 0.5)).to(dtype)
    for _ in range(30):
        bad = ba_near_kink(x, b, dim, act, kw) < 0
        n = int(bad.sum())
        if n == 0:
            return x, b
        x[bad] = draw(n).to(dtype)
    raise AssertionError('could not draw inputs away from the kinks')


def ba_near_kink(x, b, dim, act, kw):
    """Distance of each element from the nearest gate discontinuity (the lrelu kink, the clamp of any activation) minus
    the required margin (>= 0 is safe)."""
    k = f32_scalars(kw, act)
    s = x.double() + b.double().reshape(_bshape(x.ndim, dim))
    d = s.abs() - 1e-3 if act == 'lrelu' else torch.ones_like(s)
    if k.get('clamp') is not None:
        c = k['clamp']
        y = oo.bias_act(s, act=act, alpha=k['alpha'], gain=k['gain'])
        d = torch.minimum(d, (y.abs() - c).abs() - max(1e-3, ulp(torch.tensor(c, dtype=F64), x.dtype).item()))
    return d


def ba_ref(x, b, dim, kw, act, sl, cdim):
    """fp64 oracle on one slice along cdim (!= dim)."""
    idx = [slice(None)] * x.ndim
    idx[cdim] = sl
    return oo.bias_act(x[tuple(idx)].double(), b.double(), dim=dim, act=act, **f32_scalars(kw, act)), tuple(idx)


def ba_compare(name, y, x, b, dim, act, kw, n_ulp=4):
    m = Meter(name, y.dtype)
    cdim = 0 if dim != 0 else 1
    for sl in chunks(x.shape[cdim], max(1, x.shape[cdim] // 8)):
        ref, idx = ba_ref(x, b, dim, kw, act, sl, cdim)
        m.add(y[idx], ref, n_ulp=n_ulp)
    m.done()


ROW_N = {2: 12, 4: 6, 8: 3}          # (N, 96, 160, 200): H*W = 32000, 4000 / 8000 / 16000 vectors per row
BA_FWD = {'lrelu_clamp256': dict(act='lrelu', clamp=256.0), 'lrelu_clamp1': dict(act='lrelu', clamp=1.0),
          'linear_clamp': dict(act='linear', clamp=0.8)}
DT_ALL = [F32, F16, BF16, F64]
DT_IDS = ['fp32', 'fp16', 'bf16', 'fp64']


@pytest.mark.parametrize('dtype', DT_ALL, ids=DT_IDS)
@pytest.mark.parametrize('variant', sorted(BA_FWD))
def test_bias_act_row_mode_forward(variant, dtype):
    """NCHW conv outputs: one bias per (n, c) row of H*W elements, rows of 4 to 16 items with a ragged last item, and
    3 to 17 items per CTA.  lrelu with the generator's clamp 256 and with a clamp that bites, linear + clamp (ToRGB)."""
    kw = dict(BA_FWD[variant])
    act = kw.pop('act')
    shape = (ROW_N[torch.empty(0, dtype=dtype).element_size()], 96, 160, 200)
    x, b = ba_inputs(shape, 1, dtype, act, kw, seed=100)
    assert_row_mode(x, 1, 0)
    assert ba_near_kink(x, b, 1, act, kw).min().item() >= 0
    y = _ba().bias_act(x, b, dim=1, act=act, **kw)
    ba_compare(f'bias_act row fwd {variant} {dtype}', y, x, b, 1, act, kw)


@pytest.mark.parametrize('dtype', DT_ALL, ids=DT_IDS)
@pytest.mark.parametrize('dim', [0, 2])
def test_bias_act_row_mode_other_dims(dim, dtype):
    """Row mode also applies when the bias runs along dim 2 (rows of W elements) or dim 0 of an (N, F) tensor."""
    shape = (8, 12, 40, 1032) if dim == 2 else (3300, 1040)
    kw = dict(clamp=1.0)
    x, b = ba_inputs(shape, dim, dtype, 'lrelu', kw, seed=101 + dim)
    assert_row_mode(x, dim, 0)
    y = _ba().bias_act(x, b, dim=dim, act='lrelu', **kw)
    ba_compare(f'bias_act row fwd dim={dim} {dtype}', y, x, b, dim, 'lrelu', kw)


@pytest.mark.parametrize('dtype', [F32, F16, BF16], ids=DT_IDS[:3])
def test_bias_act_channels_last_at_size(dtype):
    """channels_last with C % VEC == 0: each 16-byte vector reads a contiguous run of biases (BIAS == 2)."""
    kw = dict(clamp=1.0)
    x, b = ba_inputs((12, 96, 40, 200), 1, dtype, 'lrelu', kw, seed=104, fmt=torch.channels_last)
    d = ba_dispatch(x, 1, 0)
    assert d['mode'] == 'bias_run' and x.stride(1) == 1, d
    y = _ba().bias_act(x, b, dim=1, act='lrelu', **kw)
    assert y.stride() == x.stride()
    ba_compare(f'bias_act channels_last {dtype}', y, x, b, 1, 'lrelu', kw)


BA_MODES = {
    # generator layers at 8x8: 16 (fp32) / 8 (16-bit) vectors per (n, c) row, too few for row mode (BIAS == 1)
    'per_vector': ((64, 512, 8, 8), torch.contiguous_format, 'per_vector'),
    # NCHW with an odd H*W: vectors straddle two rows, each element finds its own row ((ge + k) / step_b, BIAS == 3)
    'generic_strided': ((4, 64, 97, 101), torch.contiguous_format, 'generic'),
    # channels_last RGB (C = 3, not a multiple of VEC): each element's channel counted from its element index (BIAS == 3)
    'generic_run': ((16, 3, 256, 256), torch.channels_last, 'generic'),
    # an aligned tensor with numel % VEC != 0: its last numel % VEC elements go through the scalar tail launch, whose
    # bias index starts at base = main_n (ops_bias_act.cu:198-210)
    'tail': ((5, 37, 41, 43), torch.contiguous_format, 'tail'),
}


@pytest.mark.parametrize('dtype', DT_ALL, ids=DT_IDS)
@pytest.mark.parametrize('mode', list(BA_MODES))
def test_bias_act_other_modes_at_size(mode, dtype):
    """The per-vector, generic and scalar-tail bias indexing at generator sizes, lrelu with the generator's clamp 256
    (which never bites, so a wrong bias shows in every element it reaches, the tail's last one included)."""
    shape, fmt, want = BA_MODES[mode]
    kw = dict(clamp=256.0)
    x, b = ba_inputs(shape, 1, dtype, 'lrelu', kw, seed=105, fmt=fmt)
    if want == 'tail':
        assert x.numel() % (16 // x.element_size()) != 0 and x.data_ptr() % 16 == 0
    else:
        d = ba_dispatch(x, 1, 0)
        assert d['mode'] == want, d
    y = _ba().bias_act(x, b, dim=1, act='lrelu', **kw)
    assert y.stride() == x.stride()
    ba_compare(f'bias_act {mode} {dtype}', y, x, b, 1, 'lrelu', kw)


def ba_grad_ref(g, y, kw, act, order, dy=None):
    """The kernel's derivative formulas (ops_bias_act.cu:46-50, 82-85) in float64, gated on the op's own stored y.
    order 1: g * act'(s) * gain, zero where |y| >= clamp; order 2 (tanh): g * act''(s) * gain * dy."""
    k = f32_scalars(kw, act)
    y = y.double()
    yy = y / k['gain']
    if act == 'lrelu':
        r = g.double() * torch.where(yy > 0, 1.0, k['alpha'])
    elif order == 1:
        r = g.double() * (1 - yy * yy)
    else:
        r = g.double() * (1 - yy * yy) * (-2 * yy)
    r = r * k['gain'] * (1.0 if dy is None else dy.double())
    if k.get('clamp') is not None:
        r = torch.where(y.abs() < k['clamp'], r, 0.0)
    return r


GRAD_N = {2: 6, 4: 3, 8: 2}
BA_GRAD = {'lrelu': ('lrelu', dict(clamp=1.0)), 'tanh': ('tanh', {}),
           # the derivative's yy = yref / gain (ops_bias_act.cu:42) at a gain != 1, and the gradient clamp gate on yref
           # (:85) in both orders: 2 |tanh(s)| >= 1 on about 40 % of the elements
           'tanh_gain2_clamp1': ('tanh', dict(gain=2.0, clamp=1.0))}


@pytest.mark.parametrize('dtype', DT_ALL, ids=DT_IDS)
@pytest.mark.parametrize('variant', list(BA_GRAD))
def test_bias_act_row_mode_gradients(variant, dtype):
    """dx and db through row mode (grad = 1: UNROLL = 2, twice the items), then the R1 pattern: d/d(dy) of <dx, ddx>
    (grad = 1 again) and, for tanh, d/dx and d/db of it (grad = 2).  The gates must agree with the fp64 signs, which the
    input margin guarantees; the test checks that on the stored y too."""
    act, kw = BA_GRAD[variant]
    kw = dict(kw)
    shape = (GRAD_N[torch.empty(0, dtype=dtype).element_size()], 96, 160, 200)
    x, b = ba_inputs(shape, 1, dtype, act, kw, seed=110)
    assert ba_near_kink(x, b, 1, act, kw).min().item() >= 0
    d = assert_row_mode(x, 1, 1)
    g = torch.Generator(device=DEV).manual_seed(111)
    dy = torch.randn(shape, generator=g, device=DEV).to(dtype).requires_grad_(True)
    ddx = torch.randn(shape, generator=g, device=DEV).to(dtype)
    x.requires_grad_(True)
    b.requires_grad_(True)
    y = _ba().bias_act(x, b, dim=1, act=act, **kw)
    dx, db = torch.autograd.grad(y, [x, b], dy, create_graph=True)
    s = (dx * ddx).sum()
    second = torch.autograd.grad(s, [dy, x, b] if act == 'tanh' else [dy])
    y, dx, db = y.detach(), dx.detach(), db.detach()
    if act == 'lrelu':                                      # the stored y gates like the fp64 pre-activation
        k = f32_scalars(kw, act)
        s64 = x.detach().double() + b.detach().double().reshape(-1, 1, 1)
        want = (s64 > 0) & ((torch.where(s64 > 0, s64, s64 * k['alpha']) * k['gain']).abs() < k['clamp'])
        got = (y > 0) & (y.double().abs() < k['clamp'])
        assert torch.equal(want, got)
        assert 0.05 < (~want).double().mean().item() < 0.95   # both gates are taken
    elif kw.get('clamp') is not None:                       # the clamp gate is taken on both sides
        assert 0.05 < (y.double().abs() >= kw['clamp']).double().mean().item() < 0.95
    n_ulp = 8 if act == 'tanh' else 4
    m = Meter(f'bias_act row dx {variant} {dtype} ({d["items"]} items)', dtype)
    m.add(dx, ba_grad_ref(dy.detach(), y, kw, act, 1), n_ulp=n_ulp)
    m.done()
    m = Meter(f'bias_act row d(dy) R1 {variant} {dtype}', dtype)
    m.add(second[0], ba_grad_ref(ddx, y, kw, act, 1), n_ulp=n_ulp)
    m.done()
    _check_db(f'bias_act db {variant} {dtype}', db, dx)
    if act == 'tanh':
        m = Meter(f'bias_act row d(x) R1 {variant} {dtype}', dtype)
        m.add(second[1], ba_grad_ref(ddx, y, kw, act, 2, dy=dy.detach()), n_ulp=n_ulp)
        m.done()
        _check_db(f'bias_act d(b) R1 {variant} {dtype}', second[2], second[1])


def _check_db(name, db, dx):
    """db is the sum of the (already checked) dx over all but the bias dim: within 2 ulps + the fp32 summation bound."""
    ref = dx.double().sum([0, 2, 3])
    bound = 2 * ulp(ref, db.dtype) + 2.0 ** -20 * dx.double().abs().sum([0, 2, 3])
    err = worst_ratio(db.double() - ref, bound)
    print(f'[ops-paths] {name}: worst |err|/bar = {err:.3g}')
    assert err <= 1.0, name


# ================================================================================================== upfirdn2d
def _up():
    from panic3d_b200.torch_utils.ops import upfirdn2d
    return upfirdn2d


def _pad4(p):
    p = [p, p] if isinstance(p, int) else list(p)
    return p * 2 if len(p) == 1 else ([p[0], p[0], p[1], p[1]] if len(p) == 2 else p)


def out_size(H, W, f, up, down, pad):
    px0, px1, py0, py1 = _pad4(pad)
    fH, fW = f.shape
    return (H * up + py0 + py1 - fH + down) // down, (W * up + px0 + px1 - fW + down) // down


def upf_dispatch(x, f, up, down, pad):
    """Restates launch_upfirdn2d (ops_upfirdn2d.cu:360-372, 461-515) for a float32 2-D filter: 'fast' (4x4 persistent
    kernel, tile sizes from FastCfg, lines 125-149), 'cl' (channels_last_ok), 'tiled' or 'strided'."""
    px0, px1, py0, py1 = _pad4(pad)
    N, C, H, W = x.shape
    oh, ow = out_size(H, W, f, up, down, pad)
    es = x.element_size()
    cl = x.stride(1) == 1 and C > 1                         # the output follows x's layout (upfirdn2d.py:99)
    if es <= 4 and not cl and x.stride(3) == 1 and tuple(f.shape) == (4, 4) and (up, down) in ((1, 1), (2, 1), (1, 2)) \
            and px0 % up == 0 and py0 % up == 0:
        rpt = 8 if down == 1 else (2 if es == 4 else 4)
        tx, ty = -(-ow // 128), -(-oh // (8 * rpt))
        return dict(path='fast', tiles_per_img=tx * ty, total=N * C * tx * ty, out=(oh, ow),
                    pair_store=int(ow % 2 == 0 and (oh * ow) % 2 == 0))
    vec = 16 // es
    if es <= 4 and cl and C % vec == 0 and x.data_ptr() % 16 == 0:
        threads = N * oh * ow * (C // vec)
        return dict(path='cl', threads=threads, grid_threads=min(-(-threads // 256), n_sm() * 32) * 256, out=(oh, ow))
    return dict(path='tiled' if x.stride(3) == 1 else 'strided', out=(oh, ow), images=N * C)


def adjoint_kw(x_shape, y_shape, f, up, down, pad, flip):
    """The backward launch of upfirdn2d.py:146-149: up and down swapped, flipped filter, adjoint padding."""
    px0, px1, py0, py1 = _pad4(pad)
    fH, fW = f.shape
    ih, iw, oh, ow = x_shape[2], x_shape[3], y_shape[2], y_shape[3]
    p = [fW - px0 - 1, iw * up - ow * down + px0 - up + 1, fH - py0 - 1, ih * up - oh * down + py0 - up + 1]
    return dict(up=down, down=up, padding=p, flip_filter=not flip)


def upf_taps(f, up):
    return -(-f.shape[0] // up) * -(-f.shape[1] // up)


def upf_compare(name, y, x, f, kw, cdim=1, step=None, dtype=None):
    """y vs the fp64 oracle on x (same rounded values), piece by piece along cdim, with the fp32 accumulation bound."""
    m = Meter(name, dtype or y.dtype)
    f64 = f.double()
    taps = upf_taps(f, kw.get('up', 1))
    eps = EPS[y.dtype]
    kw_abs = dict(kw, gain=abs(kw.get('gain', 1)))
    for sl in chunks(x.shape[cdim], step or max(1, x.shape[cdim] // 8)):
        idx = [slice(None)] * 4
        idx[cdim] = sl
        xs = x[tuple(idx)].double()
        ref = oo.upfirdn2d(xs, f64, **kw)
        bound = (taps + 1) * eps * oo.upfirdn2d(xs.abs(), f64.abs(), **kw_abs) + 1e-30
        m.add(y[tuple(idx)], ref, slack=bound)
    m.done()


def rand_filter(seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(4, 4, generator=g) + 0.1).to(DEV)      # non-symmetric, so the flip matters


FAST = {'blur': dict(padding=[2, 1, 2, 1]), 'up2': dict(up=2, padding=[2, 1, 2, 1], gain=4.0),
        'up2_odd_width': dict(up=2, padding=[2, 2, 2, 1], gain=4.0), 'down2': dict(down=2, padding=[1, 1, 1, 1])}
DT3, DT3_IDS = [F32, F16, BF16], ['fp32', 'fp16', 'bf16']


def fast_batch(op, dtype, C=3, H=97, W=301, adjoint=False):
    """Batch size that gives >= 3 * 8 * n_sm tiles of (C, H, W) images (odd W: rows are not 16-byte aligned), in the
    forward launch and, with `adjoint`, in the backward launch too."""
    kw = FAST[op]
    f = torch.empty(4, 4)
    up, down = kw.get('up', 1), kw.get('down', 1)
    probe = torch.empty((1, C, H, W), dtype=dtype, device=DEV)
    tiles = [upf_dispatch(probe, f, up, down, kw['padding'])['tiles_per_img']]
    if adjoint:
        oh, ow = out_size(H, W, f, up, down, kw['padding'])
        a = adjoint_kw(probe.shape, (1, C, oh, ow), f, up, down, kw['padding'], False)
        probe = torch.empty((1, C, oh, ow), dtype=dtype, device=DEV)
        tiles.append(upf_dispatch(probe, f, a['up'], a['down'], a['padding'])['tiles_per_img'])
    return -(-min_work() // (min(tiles) * C))


@pytest.mark.parametrize('dtype', DT3, ids=DT3_IDS)
@pytest.mark.parametrize('op', sorted(FAST))
def test_upfirdn2d_fast_kernel_at_depth(op, dtype):
    """Every CTA of k_upfirdn2d_fast walks >= 3 tiles (so the two-slot ring alternates and the row bases of the tile
    after next are prefetched), and tiles per image x C < n_sm, so one grid-stride step moves to another image n:
    advance()'s carries reach every digit.  up2_odd_width stores its last column alone (pair_store == 0)."""
    kw = FAST[op]
    up, down = kw.get('up', 1), kw.get('down', 1)
    N = fast_batch(op, dtype)
    g = torch.Generator(device=DEV).manual_seed(200)
    x = torch.randn((N, 3, 97, 301), generator=g, device=DEV).to(dtype)
    f = rand_filter(201)
    d = upf_dispatch(x, f, up, down, kw['padding'])
    assert d['path'] == 'fast' and d['total'] >= min_work() and d['tiles_per_img'] * 3 < n_sm() and x.shape[3] % 2 == 1, d
    if op == 'up2_odd_width':
        assert d['out'][1] % 2 == 1 and d['pair_store'] == 0, d
    y = _up().upfirdn2d(x, f, **kw)
    assert tuple(y.shape[2:]) == d['out']
    upf_compare(f'upfirdn2d fast {op} {dtype} ({d["total"]} tiles)', y, x, f, kw, cdim=0)


REAL = {'blur_513': ((2, 128, 513, 513), 'filter2d', {}), 'upsample_128': ((8, 96, 128, 128), 'upsample2d', {}),
        'downsample_512': ((2, 128, 512, 512), 'downsample2d', {}), 'downsample_512_cl': ((2, 128, 512, 512), 'downsample2d', {})}


@pytest.mark.parametrize('dtype', [F32, F16], ids=['fp32', 'fp16'])
@pytest.mark.parametrize('case', sorted(REAL))
def test_upfirdn2d_real_sizes(case, dtype):
    """bench_ops.py's layer sizes through the public helpers with the [1,3,3,1] filter; the channels_last variant takes
    k_upfirdn2d_cl through more than one grid-stride pass."""
    shape, helper, extra = REAL[case]
    up = _up()
    f = up.setup_filter([1, 3, 3, 1], device=DEV)
    g = torch.Generator(device=DEV).manual_seed(210)
    x = torch.randn(shape, generator=g, device=DEV).to(dtype)
    if case.endswith('_cl'):
        x = x.contiguous(memory_format=torch.channels_last)
    fw = f.shape[0]
    kw = {'filter2d': dict(padding=[fw // 2, (fw - 1) // 2] * 2),
          'upsample2d': dict(up=2, padding=[(fw + 1) // 2, (fw - 2) // 2] * 2, gain=4.0),
          'downsample2d': dict(down=2, padding=[(fw - 1) // 2, (fw - 2) // 2] * 2)}[helper]
    d = upf_dispatch(x, f, kw.get('up', 1), kw.get('down', 1), kw['padding'])
    if case.endswith('_cl'):
        assert d['path'] == 'cl' and d['threads'] > d['grid_threads'], d
    else:
        assert d['path'] == 'fast' and d['total'] >= min_work(), d
    y = getattr(up, helper)(x, f)
    upf_compare(f'upfirdn2d {case} {dtype}', y, x, f, kw, cdim=1, step=16)


def oracle_vjp(x_shape, f, kw, dy):
    """dL/dx of <oracle(x), dy> in float64 by torch.autograd (no use of the op's own adjoint formula)."""
    xz = torch.zeros(x_shape, dtype=F64, device=DEV, requires_grad=True)
    return torch.autograd.grad(oo.upfirdn2d(xz, f, **kw), xz, dy)[0]


@pytest.mark.parametrize('dtype', [F32, F16], ids=['fp32', 'fp16'])
@pytest.mark.parametrize('op', ['blur', 'up2', 'down2'])
def test_upfirdn2d_fast_kernel_gradients(op, dtype):
    """First-order dx in the training dtypes: the adjoint of up2 is down2 and vice versa, with the adjoint padding;
    the backward launch takes the fast kernel at depth as well."""
    kw = FAST[op]
    up_, down = kw.get('up', 1), kw.get('down', 1)
    N = fast_batch(op, dtype, adjoint=True)
    g = torch.Generator(device=DEV).manual_seed(220)
    x = torch.randn((N, 3, 97, 301), generator=g, device=DEV).to(dtype).requires_grad_(True)
    f = rand_filter(221)
    y = _up().upfirdn2d(x, f, **kw)
    dy = torch.randn(y.shape, generator=g, device=DEV).to(dtype)
    akw = adjoint_kw(x.shape, y.shape, f, up_, down, kw['padding'], False)
    d = upf_dispatch(dy, f, akw['up'], akw['down'], akw['padding'])
    assert d['path'] == 'fast' and d['total'] >= min_work(), d
    dx, = torch.autograd.grad(y, x, dy)
    m = Meter(f'upfirdn2d fast dx {op} {dtype} (adjoint {d["total"]} tiles)', dtype)
    taps = upf_taps(f, akw['up'])
    for sl in chunks(N, max(1, N // 8)):
        ref = oracle_vjp((sl.stop - sl.start,) + tuple(x.shape[1:]), f.double(), kw, dy[sl].double())
        bound = (taps + 1) * EPS[dtype] * oracle_vjp((sl.stop - sl.start,) + tuple(x.shape[1:]), f.double().abs(),
                                                     dict(kw, gain=abs(kw.get('gain', 1))), dy[sl].double().abs())
        m.add(dx[sl], ref, slack=bound + 1e-30)
    m.done()


def test_upfirdn2d_double_backward_through_dy_at_size():
    """R1 in fp16 at depth: d/d(dy) of <dx, v> is upfirdn2d(v), the re-entered forward of the adjoint's adjoint."""
    kw = FAST['down2']
    N = fast_batch('down2', F16)
    g = torch.Generator(device=DEV).manual_seed(230)
    x = torch.randn((N, 3, 97, 301), generator=g, device=DEV).to(F16).requires_grad_(True)
    v = torch.randn(x.shape, generator=g, device=DEV).to(F16)
    f = rand_filter(231)
    y = _up().upfirdn2d(x, f, **kw)
    dy = torch.ones_like(y, requires_grad=True)
    gx, = torch.autograd.grad(y, x, dy, create_graph=True)
    g_dy, = torch.autograd.grad((gx * v).sum(), dy)
    upf_compare('upfirdn2d R1 d(dy) down2 fp16', g_dy, v, f, kw, cdim=0)


def test_upfirdn2d_more_than_32768_images():
    """The tiled kernel caps gridDim.y at 32768 and loops img += gridDim.y: every image is compared, including the
    1232 on the second lap."""
    g = torch.Generator(device=DEV).manual_seed(240)
    x = torch.randn((2, 17000, 9, 11), generator=g, device=DEV)
    f = torch.rand(3, 3, generator=torch.Generator().manual_seed(241)).to(DEV) + 0.1
    kw = dict(padding=[1, 1, 2, 0])
    d = upf_dispatch(x, f, 1, 1, kw['padding'])
    assert d['path'] == 'tiled' and d['images'] > 32768, d
    y = _up().upfirdn2d(x, f, **kw)
    upf_compare('upfirdn2d tiled 34000 images fp32', y, x, f, kw, cdim=1, step=4096)


GENERIC = {
    # a 5x5 / 3x5 filter (not the fast kernel's 4x4) on NCHW: the tiled kernel with flip (ops_upfirdn2d.cu:58), gain and
    # zero fill on every side of the up-sampled image, then decimation with a crop
    'tiled_up2_flip': ((8, 32, 97, 101), 'nchw', (5, 5), dict(up=2, padding=[3, 2, 2, 3], flip_filter=True, gain=4.0)),
    'tiled_down2_crop': ((8, 32, 97, 101), 'nchw', (3, 5), dict(down=2, padding=[-1, 3, 2, -2], gain=0.5)),
    # channels_last RGB (C = 3 < VEC, so x.stride(3) = 3): the strided kernel, channel-fastest, up 2 (column phases)
    'strided_up2_cl3': ((16, 3, 128, 129), 'cl', (4, 4), dict(up=2, padding=[2, 1, 2, 1], gain=4.0)),
    # every other column of an NCHW buffer (x.stride(3) = 2): the strided kernel, column-fastest, up 2 and flipped
    'strided_up2_flip_cols': ((8, 16, 64, 75), 'cols', (4, 4), dict(up=2, padding=[1, 2, 2, 1], flip_filter=True, gain=4.0)),
}


@pytest.mark.parametrize('dtype', DT3, ids=DT3_IDS)
@pytest.mark.parametrize('case', list(GENERIC))
def test_upfirdn2d_tiled_and_strided_kernels(case, dtype):
    """The kernels every non-4x4 filter and every layout without a unit column stride takes, with the inputs that tell
    their index maths apart: an asymmetric filter with flip, a gain, up-sampled column phases, padding and crops."""
    shape, layout, fshape, kw = GENERIC[case]
    g = torch.Generator(device=DEV).manual_seed(260)
    if layout == 'cols':
        x = torch.randn(shape[:3] + (2 * shape[3],), generator=g, device=DEV).to(dtype)[..., ::2]
    else:
        x = torch.randn(shape, generator=g, device=DEV).to(dtype)
        if layout == 'cl':
            x = x.contiguous(memory_format=torch.channels_last)
    f = (torch.rand(fshape, generator=torch.Generator().manual_seed(261)) + 0.1).to(DEV)
    d = upf_dispatch(x, f, kw.get('up', 1), kw.get('down', 1), kw['padding'])
    assert d['path'] == ('tiled' if layout == 'nchw' else 'strided'), d
    y = _up().upfirdn2d(x, f, **kw)
    assert tuple(y.shape[2:]) == d['out']
    upf_compare(f'upfirdn2d {case} {dtype}', y, x, f, kw, cdim=0)


def test_upfirdn2d_fast_kernel_64bit_offsets():
    """A fp16 tensor of more than 2^31 elements through the fast kernel; the last channel is compared with the oracle run
    on that channel alone.  Needs about 9 GB of device memory; skipped below 16 GB free."""
    free, _ = torch.cuda.mem_get_info()
    if free < 16 * 2 ** 30:
        print(f'[ops-paths] 64-bit offsets: SKIPPED, {free / 2 ** 30:.1f} GB free')
        pytest.skip('needs 16 GB of free device memory')
    shape = (1, 8200, 512, 512)
    assert math.prod(shape) > 2 ** 31
    x = torch.empty(shape, dtype=F16, device=DEV)
    x.normal_(generator=torch.Generator(device=DEV).manual_seed(250))
    f = rand_filter(251)
    kw = FAST['blur']
    d = upf_dispatch(x, f, 1, 1, kw['padding'])
    assert d['path'] == 'fast', d
    y = _up().upfirdn2d(x, f, **kw)
    last_x, last_y = x[:, -1:].clone(), y[:, -1:].clone()
    del x, y
    torch.cuda.empty_cache()
    print('[ops-paths] 64-bit offsets: ran')
    upf_compare('upfirdn2d fast 2^31+ elements, last channel fp16', last_y, last_x, f, kw)


# ================================================================================================== filtered_lrelu
def _fl():
    from panic3d_b200.torch_utils.ops import filtered_lrelu
    return filtered_lrelu


def fl_scalars(kw):
    """filtered_lrelu's keyword arguments with its defaults, gain / slope / clamp rounded to fp32 as they cross the ABI."""
    out = dict(dict(gain=math.sqrt(2), slope=0.2), **kw)
    for k in ('gain', 'slope', 'clamp'):
        if out.get(k) is not None:
            out[k] = float(np.float32(out[k]))
    return out


def fl_pre_activation(x, b, fu, kw):
    """(v, bound): the fp64 pre-activation gain * upFIR(x + b) that the kernel compares with 0 and the clamp, and the fp32
    error bound of the kernel's own v (its up-FIR roundings)."""
    k = fl_scalars(kw)
    up = k.get('up', 1)
    s = x.double() + b.double().reshape(1, -1, 1, 1)
    pad = _pad4(k.get('padding', 0))
    u = oo.upfirdn2d(s, fu.double(), up=up, padding=pad, gain=up ** 2)
    ua = oo.upfirdn2d(s.abs(), fu.double().abs(), up=up, padding=pad, gain=up ** 2)
    taps = (2 * -(-fu.shape[-1] // up)) if fu.ndim == 1 else upf_taps(fu, up)
    return u * k['gain'], (taps + 2) * 2.0 ** -24 * ua * k['gain']


def fl_codes(v, kw):
    """Sign codes of the forward (ops_filtered_lrelu.cu:155-158): 0 plain, 1 negative, 2 clamped."""
    k = fl_scalars(kw)
    a = torch.where(v < 0, v * k['slope'], v)
    codes = torch.where(v < 0, 1, 0)
    if k.get('clamp') is not None:
        codes = torch.where(a.abs() > k['clamp'], 2, codes)
    return codes, a


def fl_kink_margin(v, bound, kw):
    """min over pixels of (distance to the lrelu kink or the clamp) / (fp32 error bound of v): > 1 means the kernel's gates
    equal the fp64 ones.  Pixels no input reaches (bound 0: only padding under the filter) are exactly 0 in both and carry
    no gradient to x."""
    k = fl_scalars(kw)
    r = v.abs() / bound
    if k.get('clamp') is not None:
        _, a = fl_codes(v, kw)
        r = torch.minimum(r, (a.abs() - k['clamp']).abs() / (bound * torch.where(v < 0, k['slope'], 1.0)))
    return r[bound > 0].min().item()


def fl_filter_bound(fu, fd, up, down):
    nu = (2 * -(-fu.shape[-1] // up)) if fu.ndim == 1 else upf_taps(fu, up)
    nd = 2 * fd.shape[-1] if fd.ndim == 1 else fd.shape[0] * fd.shape[1]
    return nu + nd + 4


def fl_check(name, x, b, fu, fd, kw, dtype, seed, seams=None):
    """Forward y, dx and db of filtered_lrelu vs torch.autograd on the fp64 oracle."""
    k = fl_scalars(kw)
    fl = _fl()
    xg = x.to(DEV, dtype).requires_grad_(True)
    bg = b.to(DEV, dtype).requires_grad_(True)
    fu, fd = fu.to(DEV), fd.to(DEV)
    y = fl.filtered_lrelu(xg, fu, fd, bg, **kw)
    g = torch.Generator(device=DEV).manual_seed(seed)
    dy = torch.randn(y.shape, generator=g, device=DEV).to(dtype)
    dx, db = torch.autograd.grad(y, [xg, bg], dy)

    x64 = xg.detach().double().requires_grad_(True)
    b64 = bg.detach().double().requires_grad_(True)
    ref = oo.filtered_lrelu(x64, fu.double(), fd.double(), b64, **k)
    dx_ref, db_ref = torch.autograd.grad(ref, [x64, b64], dy.double())
    # error bounds: the same linear chain with |filters|, slope 1, no clamp, on |x + b| (forward) and |dy| (backward)
    kl = dict(k, slope=1.0, clamp=None)
    xa = (x64.detach() + b64.detach().reshape(1, -1, 1, 1)).abs().requires_grad_(True)
    ya = oo.filtered_lrelu(xa, fu.double().abs(), fd.double().abs(), None, **kl)
    dxa, = torch.autograd.grad(ya, xa, dy.double().abs())
    K = fl_filter_bound(fu, fd, k.get('up', 1), k.get('down', 1)) * 2.0 ** -24

    v, vb = fl_pre_activation(xg.detach(), bg.detach(), fu, kw)
    margin = fl_kink_margin(v, vb, kw)
    codes, _ = fl_codes(v, kw)
    print(f'[ops-paths] {name}: kink margin / fp32 bound of the pre-activation = {margin:.3g}')
    assert margin > 1.0, 'an up-sampled pixel lies within rounding of a gate: pick another seed'
    for c in (0, 1, 2) if k.get('clamp') is not None else (0, 1):
        assert (codes == c).any(), f'sign code {c} never occurs'
    if seams is not None:                                   # the last sign byte each non-last tile owns, every code
        cols = torch.tensor([c for s in seams for c in range(s - 4, s)], device=DEV)
        on_seam = codes.index_select(3, cols)
        for c in (0, 1, 2):
            assert (on_seam == c).any(), f'sign code {c} never occurs in the last byte of a tile'
    for what, got, r, bound in (('y', y.detach(), ref.detach(), K * ya.detach()), ('dx', dx, dx_ref, K * dxa)):
        m = Meter(f'filtered_lrelu {name} {what} {dtype}', dtype)
        m.add(got, r, slack=bound + 1e-30)
        m.done()
    dbb = (K * dxa).sum([0, 2, 3]) + 2.0 ** -20 * dx_ref.abs().sum([0, 2, 3])
    if dtype != F32:                                        # dx and db are themselves rounded to the dtype
        dbb = dbb + ulp(dx_ref, dtype).sum([0, 2, 3]) + ulp(db_ref, dtype)
    err = worst_ratio(db.double() - db_ref, dbb)
    print(f'[ops-paths] filtered_lrelu {name} db {dtype}: worst |err|/bar = {err:.3g}')
    assert err <= 1.0


def _fl_case(seed, shape, taps):
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    b = torch.from_numpy(rng.standard_normal(shape[1]).astype(np.float32))
    mk = lambda t: oo.setup_filter(rng.uniform(0.1, 1.0, t).astype(np.float32))
    return x, b, mk(taps[0]), mk(taps[1])


SEP12 = dict(up=2, down=2, padding=[9, 10, 9, 10], clamp=0.5)
FL_SEEDS = {'sep12_fp32': 304, 'sep12_fp16': 304, 'full2d': 310}


@pytest.mark.parametrize('dtype', [F32, F16], ids=['fp32', 'fp16'])
def test_filtered_lrelu_multi_tile_gradients_separable(dtype):
    """12-tap separable up 2 / down 2 over 3 x 6 output tiles, clamp 0.5: sign bytes written by the CTA owning each part
    of the up-sampled image are read back by the backward pass at an offset; all three codes sit on the tile seams."""
    x, b, fu, fd = _fl_case(FL_SEEDS['sep12_' + ('fp32' if dtype == F32 else 'fp16')], (1, 5, 70, 90), (12, 12))
    assert fu.ndim == 1 and fd.ndim == 1
    fl_check('sep12 up2/down2 (1,5,70,90)', x, b, fu, fd, SEP12, dtype, seed=301, seams=[64, 128])


def test_filtered_lrelu_multi_tile_gradients_full_2d():
    """Non-separable 4x4 up-FIR, 3x3 down-FIR, up 2 / down 1, over 5 x 5 output tiles."""
    x, b, fu, fd = _fl_case(FL_SEEDS['full2d'], (1, 3, 40, 70), ((4, 4), (3, 3)))
    assert fu.ndim == 2 and fd.ndim == 2
    fl_check('full2d up2/down1 (1,3,40,70)', x, b, fu, fd, dict(up=2, down=1, padding=[3, 2, 2, 3], gain=1.3, slope=0.1, clamp=0.5),
             F32, seed=311, seams=[32, 64, 96, 128])


def test_filtered_lrelu_more_than_32768_images():
    """(2, 16500, 8, 8), up 2 / down 2: the grid covers 32768 images and loops; each image has its own sign plane.
    A 2x2 box up-FIR makes every up-sampled pixel gain * (x + b) of one input, so the inputs alone keep every pixel
    1e-3 away from the kink and the clamp."""
    kw = dict(up=2, down=2, padding=[1, 0, 1, 0], clamp=0.5)
    k = fl_scalars(dict(kw, gain=math.sqrt(2), slope=0.2))
    g = torch.Generator().manual_seed(320)
    x = torch.randn((2, 16500, 8, 8), generator=g)
    b = torch.randn(16500, generator=g) * 0.5
    for _ in range(30):
        s = x.double() + b.double().reshape(1, -1, 1, 1)
        v = s * k['gain']
        a = torch.where(v < 0, v * k['slope'], v)
        bad = (v.abs() < 1e-3) | ((a.abs() - k['clamp']).abs() < 1e-3)
        if not bad.any():
            break
        x[bad] = torch.randn(int(bad.sum()), generator=g)
    assert not bad.any()
    fu = oo.setup_filter([1, 1])
    fd = oo.setup_filter([1, 3, 3, 1])
    assert x.shape[0] * x.shape[1] > 32768 and tuple(fu.shape) == (2, 2)
    fl_check('box up2/down2 33000 images', x, b, fu, fd, kw, F32, seed=321)


# ================================================================================================== the oracle on the GPU
def test_gpu_oracle_equals_cpu_oracle():
    """The large-shape tests run ops_oracle in float64 on the GPU; on a moderate shape it agrees with the CPU run within
    1e-12 relative for all three ops."""
    g = torch.Generator().manual_seed(400)
    x = torch.randn((3, 16, 33, 41), generator=g, dtype=F64)
    b = torch.randn(16, generator=g, dtype=F64)
    f = torch.rand(4, 4, generator=g, dtype=F64) + 0.1
    fu = oo.setup_filter(torch.rand(12, generator=g).numpy() + 0.1).double()
    runs = {
        'bias_act': lambda d: oo.bias_act(x.to(d), b.to(d), act='lrelu', clamp=1.0),
        'upfirdn2d': lambda d: oo.upfirdn2d(x.to(d), f.to(d), up=2, padding=[2, 1, 2, 1], gain=4.0),
        'filtered_lrelu': lambda d: oo.filtered_lrelu(x.to(d), fu.to(d), fu.to(d), b.to(d), up=2, down=2, padding=[9, 10, 9, 10], clamp=0.5),
    }
    for name, run in runs.items():
        cpu, gpu = run('cpu'), run(DEV).cpu()
        rel = worst_ratio(gpu - cpu, cpu.abs().max())
        print(f'[ops-paths] oracle {name}: GPU vs CPU fp64 relative difference {rel:.3g}')
        assert rel <= 1e-12, name
