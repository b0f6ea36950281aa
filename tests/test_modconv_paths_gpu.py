"""GPU: the modulated convolution (csrc/modconv.cu: k_modconv_prep, k_modconv<F16, BN>) across the envelope
p3d_modconv_supported accepts, and the SR head's up-2 route through synthesis_layer_forward, against fp64 oracles with a
bar per element.

The kernels are called through the C ABI (p3d_modconv_prep, then p3d_modconv_forward) into a workspace filled with 0xFF
bytes and an output filled with NaN, each call twice and bit-identical (the kernels have no atomics).  The prep writes every
byte of its workspace, so no NaN may survive it, and the rows past Cout (the N tile's padding) and the channels past Cin
(the K chunk's padding) must be exactly +0.

Per weight: the prepared operand, read back positionally (modconv.unpack_workspace: slot -> kernel tap by tap_slots),
equals mo.per_sample_weights rounded to the compute type, except for a share below 1 % one rounding away (the fp32
demodulation sum order).  This pins the prep's tap layout independently of the conv, which reads only the tap offsets.
It runs on every eval layer shape (N = 3) and on every case below.

Per output element: the fp64 conv of the kernel's own rounded operands (the prepared weights read back, the activations
rounded to fp16 / tf32-rna), then the epilogue in fp64 (oracle.modconv_oracle.oracle_conv / epilogue64):

    bar = |gain| (K 2^-23 S + 2^-22 (|noise| + |bias|)) + u(ref) + 2^-24

with S the oracle on |x| and |w|, K = Cin k^2 and u(ref) one rounding of the output dtype at the reference value (the
rule of tests/test_modconv_gpu.py, plus the two fp32 additions of noise and bias).  lrelu and the clamp are 1-Lipschitz,
so a reference within the bar of +-clamp accepts either side.  The worst error as a fraction of the bar is printed (-s).

Cases (each at N = 1 and N = 3, in fp16 and in fp32 with TF32 unless noted; y is channels_last for channels_last inputs):

  k3_cin16_cout1_5x37         one fp16 K-step / half an fp32 chunk; Cout 1 on the BN = 8 tile; wide; per-sample noise,
                              lrelu, gain sqrt(1/2)
  k3_cin48_cout9_37x5         three fp16 K-steps; Cout 9 (BN = 128, one row group live); tall; channels_last (16-byte
                              vector gather); broadcast noise, linear
  k3_cin112_cout127_300x1     W = 1: both side columns of taps are off the edge; a channel slice of a wider NCHW tensor;
                              lrelu, gain 2 and a clamp that binds
  k3_cin80_cout255_7x13       channels_last channel slice x[:, 4:4 + Cin] of a wider tensor: base 8 bytes off 16 in fp16
                              (scalar gather, unit channel stride), 16-byte aligned in fp32 (vector gather, row stride > Cin)
  k3_cin16_cout4096_3x4       Cout at the 4096 limit (32 N tiles); channels_last based 8 bytes off 16 (scalar gather)
  k3_cin16_cout3_4096x3       H at the 4096 limit; 96 M tiles
  k1_cin80_cout4_1x300        H = 1; ToRGB form (no demodulation, styles x weight_gain); Cin 80 = one full and one 1-step
                              fp16 chunk; Cout 4 on BN = 8; channels_last 8 bytes off 16; a clamp that binds
  k1_cin48_cout129_9x20       a second, one-row-live N tile; spatially strided view x[:, :, ::2]; per-sample noise
  up2_cin16_cout8_11x11       the four phases are 12x12 / 12x11 / 11x12 / 11x11 = 144 / 132 / 132 / 121 pixels: two M
                              tiles for three phases, one for the last; channels_last channel slice
  up2_cin48_cout129_5x37      non-square up 2 (the phase widths come from W, the heights from H); strided view;
                              per-sample noise on the (2H+1) x (2W+1) grid
  up2_cin80_cout255_1x9       H = 1 up 2 (phase rows 2 / 1); broadcast noise; a clamp that binds
  up2_cin112_cout4_6x13       Cin 112 = one full fp16 chunk and one of 3 K-steps; channels_last 8 bytes off 16
  up2_cin16_cout9_2x4096      W at the 4096 limit (phase width 4097)
  deep_k1_cin65536            fp16 only: Cin at the 65536 limit at k = 1, 1024 K chunks through the 3-stage ring
  deep_k3_cin4096             fp32 only: 128 chunks x 9 taps = 1152 K iterations
  gridz_up2_n16383            fp16, N = 16383 only: batch x phases = 65532 grid z
  gridz_k3_n65535             fp32, N = 65535 only: grid z at the 65535 limit

Every up-2 case has H <= W (tests/run_mutations.py modconv_paths: the phase-width-from-H mutant stays in bounds).

The production route: modconv.synthesis_layer_forward (what install_modconv binds; measured_faster sends the fp16 up-2
layers to the kernel) on sr256_conv0 and sr512_conv0 at their eval sizes, N = 1 and 3, NCHW and channels_last, noise
random / const / none, gain 1 and sqrt(1/2), against the fp64 route bias_act(upfirdn2d(P64, f, pad 1, gain 4) + noise),
P64 the fp64 pre-filter of the kernel's own prepared weights.  Its bar follows the route's roundings:

    e_P   = K 2^-23 S + u16 |P| + 2^-24                     the pre-filter (fp16 store)
    e_F   = FIR4(e_P) + 16 2^-23 FIR4(|P| + e_P) + u16 |F|   through |f| x 4, fp32 accumulation, one fp16 rounding
    e_V   = e_F + u16 |V| + 2^-24                           V = F + noise, one fp16 rounding
    e_out = g s (e_V + 2^-22 (|V| + |b|)) + u16 |out| + 2^-24

u16 = 2^-10, g = act_gain x gain, s = 1 or the slope 0.2 where V + b + e_V < 0.  Negative controls on sr256_conv0, each
missing the kernel by >= 20x the bar somewhere: the FIR padding shifted by one, the noise added after bias_act, and the
bias added before the FIR as b / 4 (the FIR's DC gain is 4, so it agrees in the interior and differs only on the border
rows and columns, where the zero padding cuts the filter's support).  tests/test_modconv_gpu.py keeps the comparison
with the reference's own cuDNN order.
"""
import ctypes as C
import functools
import math
import time
import zlib

import pytest
import torch

from oracle import modconv_oracle as mo, ops_oracle
from oracle.modconv_oracle import EVAL_SHAPES, epilogue64, oracle_conv
from tests import render_abi as ra
from tests.helpers import profiled

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U16, U32, TINY = 2.0 ** -10, 2.0 ** -23, 2.0 ** -24
PROF_MODCONV = 7                 # profile slot (csrc/p3d_common.cuh)
SQRT_HALF = math.sqrt(0.5)
UP2_PAD = [1, 1, 1, 1]           # conv2d_resample's FIR padding after the 3x3 stride-2 transposed conv (4-tap filter, padding 1)
ES = {torch.float16: 2, torch.float32: 4}

# name: Cin, Cout, H, W, mode (k3: kernel 3 up 1, k1: kernel 1 without demodulation, up2: kernel 3 up 2), input layout,
# epilogue (noise: sample [N,1,H,W] / bcast [H,W]; act; gain; clamp); dtypes and N when not all (see the docstring)
CASES = {
    'k3_cin16_cout1_5x37': dict(cin=16, cout=1, h=5, w=37, mode='k3', layout='nchw', noise='sample', act='lrelu', gain=SQRT_HALF),
    'k3_cin48_cout9_37x5': dict(cin=48, cout=9, h=37, w=5, mode='k3', layout='cl', noise='bcast'),
    'k3_cin112_cout127_300x1': dict(cin=112, cout=127, h=300, w=1, mode='k3', layout='slice_nchw', act='lrelu', gain=2.0, clamp=0.5),
    'k3_cin80_cout255_7x13': dict(cin=80, cout=255, h=7, w=13, mode='k3', layout='slice_cl', noise='sample', act='lrelu', gain=SQRT_HALF),
    'k3_cin16_cout4096_3x4': dict(cin=16, cout=4096, h=3, w=4, mode='k3', layout='cl_off8', act='lrelu'),
    'k3_cin16_cout3_4096x3': dict(cin=16, cout=3, h=4096, w=3, mode='k3', layout='nchw', noise='bcast', act='lrelu'),
    'k1_cin80_cout4_1x300': dict(cin=80, cout=4, h=1, w=300, mode='k1', layout='cl_off8', clamp=0.5),
    'k1_cin48_cout129_9x20': dict(cin=48, cout=129, h=9, w=20, mode='k1', layout='strided', noise='sample', act='lrelu', gain=SQRT_HALF),
    'up2_cin16_cout8_11x11': dict(cin=16, cout=8, h=11, w=11, mode='up2', layout='slice_cl'),
    'up2_cin48_cout129_5x37': dict(cin=48, cout=129, h=5, w=37, mode='up2', layout='strided', noise='sample', act='lrelu', gain=SQRT_HALF),
    'up2_cin80_cout255_1x9': dict(cin=80, cout=255, h=1, w=9, mode='up2', layout='cl', noise='bcast', clamp=0.5),
    'up2_cin112_cout4_6x13': dict(cin=112, cout=4, h=6, w=13, mode='up2', layout='cl_off8', act='lrelu'),
    'up2_cin16_cout9_2x4096': dict(cin=16, cout=9, h=2, w=4096, mode='up2', layout='nchw', noise='sample'),
    'deep_k1_cin65536': dict(cin=65536, cout=9, h=12, w=11, mode='k1', layout='cl', dtypes=('f16',), free=4 << 30),
    'deep_k3_cin4096': dict(cin=4096, cout=8, h=5, w=6, mode='k3', layout='nchw', act='lrelu', dtypes=('f32',)),
    'gridz_up2_n16383': dict(cin=16, cout=8, h=2, w=3, mode='up2', layout='nchw', noise='bcast', dtypes=('f16',), ns=(16383,),
                             free=8 << 30),
    'gridz_k3_n65535': dict(cin=16, cout=4, h=3, w=2, mode='k3', layout='nchw', act='lrelu', dtypes=('f32',), ns=(65535,),
                            free=12 << 30),
}
DTYPES = {'f16': torch.float16, 'f32': torch.float32}
PARAMS = [(name, dt, n) for name, c in CASES.items() for dt in c.get('dtypes', ('f16', 'f32')) for n in c.get('ns', (1, 3))]
assert all(c['h'] <= c['w'] for c in CASES.values() if c['mode'] == 'up2')


@pytest.fixture(scope='module')
def mc():
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.modconv as mc
    return mc


def _lib():
    from panic3d_b200 import _lib
    return _lib


def _strides(t):
    return (C.c_int64 * 4)(*t.stride())


def _params(mc, n, cin, cout, h, w, mode, dtype):
    p = mc.ModconvParams()
    p.batch, p.in_channels, p.out_channels, p.in_h, p.in_w = n, cin, cout, h, w
    p.kernel_size = 1 if mode == 'k1' else 3
    p.up, p.down = (2 if mode == 'up2' else 1), 1
    p.dtype = mc.P3D_F16 if dtype == torch.float16 else mc.P3D_F32
    p.demodulate = int(mode != 'k1')
    p.allow_tf32 = 1
    assert mc.supported(p)
    return p


def _input(layout, n, cin, h, w, dtype, g):
    """x (N, Cin, H, W) of dtype in `layout`: nchw, cl (channels_last), cl_off8 (channels_last based 8 bytes past a
    16-byte boundary), slice_nchw / slice_cl (channels [c0, c0 + Cin) of a wider tensor), strided (x[:, :, ::2])."""
    r = lambda *s: torch.randn(*s, generator=g, device=DEV).to(dtype)
    cl = torch.channels_last
    if layout == 'nchw':
        return r(n, cin, h, w)
    if layout == 'cl':
        return r(n, cin, h, w).to(memory_format=cl)
    if layout == 'cl_off8':
        off = 8 // ES[dtype]
        return r(n * h * w * cin + off)[off:].as_strided((n, cin, h, w), (h * w * cin, 1, w * cin, cin))
    if layout == 'slice_nchw':
        return r(n, cin + 24, h, w)[:, 8:8 + cin]
    if layout == 'slice_cl':
        return r(n, cin + 12, h, w).to(memory_format=cl)[:, 4:4 + cin]
    assert layout == 'strided'
    return r(n, cin, 2 * h, w)[:, :, ::2]


def _vector_gather(x):
    """The conv's choice of 16-byte vector loads for A (p3d_modconv_forward)."""
    ue = 16 // x.element_size()
    s = x.stride()
    return s[1] == 1 and x.data_ptr() % 16 == 0 and s[0] % ue == 0 and s[2] % ue == 0 and s[3] % ue == 0


def prep_twice(mc, p, weight, styles):
    """p3d_modconv_prep into a 0xFF workspace, twice, bit-identical, one launch each; no NaN survives, the N-tile and
    K-chunk padding is exactly +0.  Returns the workspace."""
    lib = _lib()
    L = lib.lib()
    ws = torch.empty(int(L.p3d_modconv_workspace_bytes(C.byref(p))), dtype=torch.uint8, device=DEV)
    w32, s32 = weight.float().contiguous(), styles.float().contiguous()
    call = lambda: lib.check(L.p3d_modconv_prep(C.byref(p), w32.data_ptr(), s32.data_ptr(), ws.data_ptr(), lib.stream_ptr(DEV)))
    ws = ra.twice(call, [ws], PROF_MODCONV)[0][0]
    rows = mc.workspace_rows(p, ws)
    assert not torch.isnan(rows).any(), 'a workspace byte the prep never wrote'
    bits = rows.view(torch.int16 if p.dtype == mc.P3D_F16 else torch.int32)
    assert (bits[:, p.out_channels:] == 0).all() and (bits[..., p.in_channels:] == 0).all(), 'padding is not +0'
    return ws


def check_prep_weights(mc, p, ws, weight, styles, tag):
    """The prepared weights, positionally, against the fp64 oracle rounded to the compute type: at most one rounding off,
    on fewer than 1 % of them."""
    f16 = p.dtype == mc.P3D_F16
    dtype = torch.float16 if f16 else torch.float32
    got = mc.unpack_workspace(p, ws).double()
    want = mo.round_operand(mo.per_sample_weights(weight, styles, bool(p.demodulate), f16 and bool(p.demodulate)), dtype)
    ulp = (U16 if f16 else 2.0 ** -10) * want.abs().clamp_min(2.0 ** -14)
    diff = (got - want).abs()
    share = float((diff > 0).double().mean())
    worst = float((diff / ulp).max())
    print(f'{tag} prep: {share:.2e} of the weights one rounding away, worst {worst:.3f} rounding')
    assert worst <= 1.0001 and share < 0.01, (tag, worst, share)


def conv_twice(mc, p, x, ws, bias, noise, act, gain, clamp, y):
    """p3d_modconv_forward into a NaN-filled y, twice, one launch each: both runs, for the caller to compare the first with
    the oracle before it requires the second to equal it bit for bit (an element never written stays NaN in both)."""
    lib = _lib()
    L = lib.lib()
    ns = None
    if noise is not None:
        ns = (C.c_int64 * 3)(*((noise.stride(0), noise.stride(2), noise.stride(3)) if noise.dim() == 4 else (0, *noise.stride())))
    call = lambda: lib.check(L.p3d_modconv_forward(
        C.byref(p), x.data_ptr(), _strides(x), ws.data_ptr(), lib.ptr(bias), lib.ptr(noise), ns, y.data_ptr(), _strides(y),
        mc._ACTS[act], float(gain), -1.0 if clamp is None else float(clamp), lib.stream_ptr(DEV)))
    return ra.twice(call, [y], PROF_MODCONV, checks_later=True)


@pytest.mark.parametrize('name,dt,n', PARAMS, ids=[f'{a}-{b}-N{c}' for a, b, c in PARAMS])
def test_envelope_case_against_the_oracle(mc, name, dt, n):
    c = CASES[name]
    if 'free' in c:
        ra.skip_unless_free(c['free'])
    t0 = time.time()
    dtype = DTYPES[dt]
    cin, cout, h, w, mode = c['cin'], c['cout'], c['h'], c['w'], c['mode']
    k = 1 if mode == 'k1' else 3
    act, gain, clamp = c.get('act', 'linear'), c.get('gain', 1.0), c.get('clamp')
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(f'{name} {dt} {n}'.encode()))
    p = _params(mc, n, cin, cout, h, w, mode, dtype)
    x = _input(c['layout'], n, cin, h, w, dtype, g)
    assert tuple(x.shape) == (n, cin, h, w)
    if c['layout'] in ('cl', 'cl_off8'):
        assert _vector_gather(x) == (c['layout'] == 'cl')
    weight = torch.randn(cout, cin, k, k, generator=g, device=DEV)
    styles = torch.randn(n, cin, generator=g, device=DEV) * 0.5 + 1.0
    if mode == 'k1':
        styles = styles / math.sqrt(cin)                           # ToRGB: styles x weight_gain
    oh, ow = (2 * h + 1, 2 * w + 1) if mode == 'up2' else (h, w)
    bias = (torch.randn(cout, generator=g, device=DEV) * 0.5).to(dtype)
    noise = None
    if c.get('noise') == 'sample':
        noise = torch.randn(n, 1, oh, ow, generator=g, device=DEV) * 0.5
    elif c.get('noise') == 'bcast':
        noise = torch.randn(oh, ow, generator=g, device=DEV) * 0.5
    fmt = torch.channels_last if c['layout'] in ('cl', 'cl_off8', 'slice_cl') else torch.contiguous_format
    y = torch.empty(n, cout, oh, ow, dtype=dtype, device=DEV, memory_format=fmt)
    with torch.no_grad():
        ws = prep_twice(mc, p, weight, styles)
        check_prep_weights(mc, p, ws, weight, styles, f'{name} {dt} N={n}')
        runs = conv_twice(mc, p, x, ws, bias, noise, act, gain, clamp, y)
        y = runs[0][0]
        wk = mc.unpack_workspace(p, ws).double()
        x64 = mo.round_operand(x, dtype)
        acc = oracle_conv(x64, wk, p.up, k)
        s_abs = oracle_conv(x64.abs(), wk.abs(), p.up, k)
        ref = epilogue64(acc, bias, noise, act, gain, clamp)
        extra = bias.double().abs().reshape(1, -1, 1, 1) + (0.0 if noise is None else noise.double().abs())
        bar = abs(gain) * (cin * k * k * U32 * s_abs + 2 * U32 * extra) + (U16 if dtype == torch.float16 else U32) * ref.abs() + TINY
        err, frac = ra.ratio(y, ref, bar)
    if clamp is not None:
        share = float((ref.abs() == clamp).double().mean())
        assert share > 0.02, f'the clamp binds on only {share:.3f} of the outputs'
    print(f'{name} {dt} N={n} (vector gather {int(_vector_gather(x))}): max err {err:.3e}, {frac:.3f} of the bar, '
          f'{time.time() - t0:.1f} s')
    assert frac <= 1.0, (name, dt, n, frac)
    ra.repeats(*runs, nan=True)


@pytest.mark.parametrize('shape', EVAL_SHAPES, ids=[s[0] for s in EVAL_SHAPES])
def test_prep_weights_at_every_eval_shape(mc, shape):
    name, cin, cout, res, up, kind, dtype, clamp = shape
    layer = mo.make_layer(*shape).to(DEV).requires_grad_(False)
    g = torch.Generator(device=DEV).manual_seed(11)
    x = torch.empty(3, cin, res // up, res // up, dtype=dtype, device=DEV)
    w = torch.randn(3, 64, generator=g, device=DEV)
    with torch.no_grad():
        p = mc.make_params(x, layer.weight, kind == 'layer', up=up, allow_tf32=True)
        styles = layer.affine(w) * (layer.weight_gain if kind == 'torgb' else 1)
        ws = prep_twice(mc, p, layer.weight, styles)
        check_prep_weights(mc, p, ws, layer.weight, styles, name)


# ------------------------------------------------------------------------------------------ the SR head's up-2 route
SR = {s[0]: s for s in EVAL_SHAPES if s[0] in ('sr256_conv0', 'sr512_conv0')}
ROUTE = [(name, n, cl) for name in SR for n in (1, 3) for cl in (False, True)]


@functools.lru_cache(maxsize=1)
def _layer(name):
    return mo.make_layer(*SR[name]).to(DEV).requires_grad_(False)


def _route_inputs(name, n, channels_last):
    layer = _layer(name)
    g = torch.Generator(device=DEV).manual_seed(21 + n)
    x = torch.randn(n, layer.in_channels, layer.resolution // 2, layer.resolution // 2, generator=g, device=DEV).half()
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    return layer, x, torch.randn(n, 64, generator=g, device=DEV)


def _prefilter64(mc, layer, x, w):
    """(P64, e_P): the fp64 pre-filter of the kernel's own prepared weights, and its per-element bar."""
    p = mc.make_params(x, layer.weight, True, up=2, allow_tf32=True)
    wk = mc.unpack_workspace(p, mc.prep(p, layer.weight, layer.affine(w))).double()
    x64 = x.double()
    P = mo.transposed_prefilter(x64, wk)
    eP = layer.in_channels * 9 * U32 * mo.transposed_prefilter(x64.abs(), wk.abs())
    return P, eP.add_(U16 * P.abs()).add_(TINY)


def _fir(layer, t, pad=UP2_PAD):
    return ops_oracle.upfirdn2d(t, layer.resample_filter.double(), padding=pad, gain=4)


def _route64(layer, P, eP, noise, gain, variant=None):
    """The fp64 route bias_act(upfirdn2d(P, f, gain 4) + noise) and its bar (see the docstring); `variant` names a negative
    control: 'pad' (FIR padding shifted by one), 'noise_after' (noise added after bias_act), 'bias_first' (b / 4 added
    before the FIR)."""
    b = layer.bias.half().double().reshape(1, -1, 1, 1)
    g, c = layer.act_gain * gain, layer.conv_clamp * gain
    nz = 0.0 if noise is None else noise.double()
    F_ = _fir(layer, P + b / 4 if variant == 'bias_first' else P, [2, 0, 2, 0] if variant == 'pad' else UP2_PAD)
    eF = _fir(layer, eP) + 16 * U32 * _fir(layer, P.abs() + eP) + U16 * F_.abs()
    V = F_ if variant == 'noise_after' else F_ + nz
    eV = eF + U16 * V.abs() + TINY
    pre = V if variant == 'bias_first' else V + b
    out = (torch.where(pre > 0, pre, 0.2 * pre) * g).clamp(-c, c)
    if variant == 'noise_after':
        out = out + nz
    slope = torch.where(pre + eV < 0, 0.2, 1.0)
    bar = g * slope * (eV + 2 * U32 * (V.abs() + b.abs())) + U16 * out.abs() + TINY
    return out, bar


def _run_route(mc, layer, x, w, noise_mode, gain):
    """synthesis_layer_forward under a fixed seed: (y, the noise it drew or used, launches in the modulated-conv slot)."""
    torch.manual_seed(5)
    y, prof = profiled(lambda: mc.synthesis_layer_forward(layer, x, w, noise_mode=noise_mode, gain=gain))
    torch.manual_seed(5)
    noise = None
    if noise_mode == 'random':
        noise = torch.randn([x.shape[0], 1, layer.resolution, layer.resolution], device=DEV) * layer.noise_strength
    elif noise_mode == 'const':
        noise = layer.noise_const * layer.noise_strength
    return y, noise, prof[PROF_MODCONV]


def test_route_padding_is_conv2d_resamples():
    """UP2_PAD and the oracle's FIR equal the oracle's conv2d_resample up > 1 route (CPU, fp64)."""
    torch.manual_seed(0)
    x, w = torch.randn(2, 16, 5, 7, dtype=torch.float64), torch.randn(2, 8, 16, 3, 3, dtype=torch.float64)
    f = ops_oracle.setup_filter([1, 3, 3, 1]).double()
    want = mo.conv2d_resample(x.reshape(1, -1, 5, 7), w.reshape(-1, 16, 3, 3), f, up=2, padding=1, groups=2, flip_weight=False)
    got = ops_oracle.upfirdn2d(mo.transposed_prefilter(x, w), f, padding=UP2_PAD, gain=4)
    assert float((got.reshape(want.shape) - want).abs().max()) <= 1e-12 * float(want.abs().max())


@pytest.mark.parametrize('name,n,channels_last', ROUTE, ids=[f'{a}-N{b}-{"cl" if c else "nchw"}' for a, b, c in ROUTE])
def test_up2_route_per_element(mc, name, n, channels_last):
    ra.skip_unless_free(24 << 30)
    t0 = time.time()
    layer, x, w = _route_inputs(name, n, channels_last)
    with torch.no_grad():
        P, eP = _prefilter64(mc, layer, x, w)
        for noise_mode in ('random', 'const', 'none'):
            for gain in (1.0, SQRT_HALF):
                y, noise, launches = _run_route(mc, layer, x, w, noise_mode, gain)
                assert launches == 2 and y.dtype == torch.float16          # prep + conv: the kernel route
                ref, bar = _route64(layer, P, eP, noise, gain)
                assert y.shape == ref.shape
                err, frac = ra.ratio(y, ref, bar)
                print(f'{name} N={n} {"cl" if channels_last else "nchw"} noise={noise_mode} gain={gain:.3f}: '
                      f'max err {err:.3e}, {frac:.3f} of the bar')
                assert frac <= 1.0, (noise_mode, gain, frac)
    print(f'{name} N={n}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GB')


@pytest.mark.parametrize('variant', ['pad', 'noise_after', 'bias_first'])
def test_route_negative_controls(mc, variant):
    layer, x, w = _route_inputs('sr256_conv0', 1, False)
    with torch.no_grad():
        P, eP = _prefilter64(mc, layer, x, w)
        y, noise, _ = _run_route(mc, layer, x, w, 'random', 1.0)
        _, bar = _route64(layer, P, eP, noise, 1.0)
        mut, _ = _route64(layer, P, eP, noise, 1.0, variant)
        d = (y.double() - mut).abs()
        if variant == 'bias_first':                                       # agrees in the interior
            assert float((d[..., 1:-1, 1:-1] / bar[..., 1:-1, 1:-1]).max()) <= 1.0
        _, frac = ra.ratio(y, mut, bar)
    print(f'negative control {variant}: worst err / bar {frac:.1f}')
    assert frac >= 20, (variant, frac)
