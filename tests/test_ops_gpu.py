"""GPU parity of the StyleGAN ops (through the C-ABI) vs the reference impl='ref' fixtures and vs the CPU oracle,
forward + first/second-order gradients (R1 regularisation double-backward goes through bias_act and upfirdn2d)."""
import os

import numpy as np
import pytest
import torch

from oracle import ops_oracle as oo
from tests.golden.cases_ops import BIAS_ACT_CASES, UPFIRDN_CASES, FLRELU_CASES, make_input, make_filter
from tests.helpers import f32_scalars

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ops_golden.npz'))
DEV = 'cuda:0'


def _ba():
    from panic3d_b200.torch_utils.ops import bias_act
    return bias_act


# ------------------------------------------------------------------------------------------ bias_act
@pytest.mark.parametrize('name', sorted(BIAS_ACT_CASES))
def test_bias_act_forward_matches_reference_fixture(name):
    c = BIAS_ACT_CASES[name]
    x, b = make_input(c)
    kw = dict(dim=c.get('dim', 1), act=c['act'], alpha=c.get('alpha'), gain=c.get('gain'), clamp=c.get('clamp'))
    y = _ba().bias_act(x.to(DEV), None if b is None else b.to(DEV), **kw)
    assert y.shape == x.shape and y.dtype == x.dtype
    assert np.abs(y.cpu().numpy() - G['ba_' + name]).max() < 1e-5


@pytest.mark.parametrize('dtype,tol', [(torch.float16, 2e-3), (torch.bfloat16, 2e-2), (torch.float64, 1e-12)])
@pytest.mark.parametrize('name', ['lrelu_conv', 'linear_torgb', 'swish', 'softplus'])
def test_bias_act_dtypes(name, dtype, tol):
    c = BIAS_ACT_CASES[name]
    x, b = make_input(c)
    kw = dict(dim=c.get('dim', 1), act=c['act'], alpha=c.get('alpha'), gain=c.get('gain'), clamp=c.get('clamp'))
    xd, bd = x.to(dtype), b.to(dtype)
    y = _ba().bias_act(xd.to(DEV), bd.to(DEV), **kw)
    ref = oo.bias_act(xd.double(), bd.double(), **f32_scalars(kw, c['act']))
    assert y.dtype == dtype
    assert (y.cpu().double() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('name', ['lrelu_conv', 'linear_torgb', 'tanh'])
def test_bias_act_channels_last_and_unaligned(name):
    c = BIAS_ACT_CASES[name]
    x, b = make_input(c)
    kw = dict(dim=1, act=c['act'], clamp=c.get('clamp'))
    ref = oo.bias_act(x, b, **kw)
    xc = x.to(DEV).contiguous(memory_format=torch.channels_last)
    y = _ba().bias_act(xc, b.to(DEV), **kw)
    assert y.stride() == xc.stride()
    assert (y.cpu() - ref).abs().max().item() < 1e-5
    # misaligned storage offset -> scalar path
    buf = torch.zeros(x.numel() + 1, device=DEV)
    xs = buf[1:].view(x.shape)
    xs.copy_(x)
    y2 = _ba().bias_act(xs, b.to(DEV), **kw)
    assert (y2.cpu() - ref).abs().max().item() < 1e-5


@pytest.mark.parametrize('name', sorted(BIAS_ACT_CASES))
def test_bias_act_gradients(name):
    """dx, db and (where the activation has one) the double-backward, vs torch.autograd on the oracle (fp64 inputs)."""
    c = BIAS_ACT_CASES[name]
    x, b = make_input(c)
    kw = dict(dim=c.get('dim', 1), act=c['act'], alpha=c.get('alpha'), gain=c.get('gain'), clamp=c.get('clamp'))
    rng = np.random.default_rng(c['seed'] + 99)
    dy = torch.from_numpy(rng.standard_normal(c['shape']))
    ddx = torch.from_numpy(rng.standard_normal(c['shape']))

    def run(fn, xin, bin_, dy_, ddx_):
        xin = xin.clone().requires_grad_(True)
        bin_ = None if bin_ is None else bin_.clone().requires_grad_(True)
        y = fn(xin, bin_, **kw)
        ins = [xin] + ([bin_] if bin_ is not None else [])
        g1 = torch.autograd.grad(y, ins, dy_, create_graph=True)
        # R1-style second order: differentiate <dx, ddx> w.r.t. the incoming gradient path and x
        s = (g1[0] * ddx_).sum()
        g2 = torch.autograd.grad(s, ins, allow_unused=True) if s.requires_grad else [None] * len(ins)
        return [y] + list(g1) + [g for g in g2]

    kw_gpu, kw = kw, f32_scalars(kw, c['act'])
    if c['act'] == 'linear' and kw.get('clamp') is not None:
        # quirk of the reference CUDA path that this op reproduces on purpose: 'linear' saves neither x nor y
        # (activation_funcs['linear'].ref == '', bias_act.py:24,153-156), so its backward kernel sees yref = 0 and
        # never gates the gradient by the clamp (bias_act.cu:141-146) - unlike autograd through impl='ref'.
        y_fwd = oo.bias_act(x.double(), None if b is None else b.double(), **kw)
        kw = dict(kw, clamp=None)
    ref = run(oo.bias_act, x.double(), None if b is None else b.double(), dy, ddx)
    if c['act'] == 'linear' and kw_gpu.get('clamp') is not None:
        ref[0] = y_fwd
    kw = kw_gpu
    got = run(_ba().bias_act, x.double().to(DEV), None if b is None else b.double().to(DEV), dy.to(DEV), ddx.to(DEV))
    for r, g_ in zip(ref, got):
        if r is None:
            assert g_ is None or g_.abs().max().item() == 0
            continue
        assert g_ is not None
        assert (g_.cpu() - r).abs().max().item() < 1e-9 * max(1.0, r.abs().max().item()), name


def test_bias_act_empty_and_errors():
    ba = _ba()
    y = ba.bias_act(torch.zeros(0, 4, device=DEV), torch.zeros(4, device=DEV), act='lrelu')
    assert y.shape == (0, 4)
    with pytest.raises(RuntimeError):
        ba.bias_act(torch.zeros(2, 4), torch.zeros(4))                       # CPU tensor: no fallback
    with pytest.raises(RuntimeError):
        ba.bias_act(torch.zeros(2, 4, device=DEV), torch.zeros(5, device=DEV))  # wrong bias length


# ------------------------------------------------------------------------------------------ upfirdn2d
def _up():
    from panic3d_b200.torch_utils.ops import upfirdn2d
    return upfirdn2d


def _up_kw(c):
    return dict(up=c.get('up', 1), down=c.get('down', 1), padding=c.get('padding', 0), flip_filter=c.get('flip', False), gain=c.get('gain', 1))


@pytest.mark.parametrize('name', sorted(UPFIRDN_CASES))
def test_upfirdn2d_forward_matches_reference_fixture(name):
    c = UPFIRDN_CASES[name]
    x, _ = make_input(c)
    f = make_filter(c, _up().setup_filter)
    y = _up().upfirdn2d(x.to(DEV), None if f is None else f.to(DEV), **_up_kw(c))
    assert tuple(y.shape) == G['up_' + name].shape
    assert np.abs(y.cpu().numpy() - G['up_' + name]).max() < 1e-5


def test_upfirdn2d_helpers_match_reference_fixture():
    up = _up()
    x, _ = make_input(dict(seed=77, shape=(2, 3, 9, 8)))
    f = up.setup_filter([1, 3, 3, 1], device=DEV)
    assert np.abs(up.filter2d(x.to(DEV), f).cpu().numpy() - G['hl_filter2d']).max() < 1e-5
    assert np.abs(up.upsample2d(x.to(DEV), f, up=2).cpu().numpy() - G['hl_upsample2d']).max() < 1e-5
    assert np.abs(up.downsample2d(x.to(DEV), f, down=2).cpu().numpy() - G['hl_downsample2d']).max() < 1e-5
    assert torch.equal(up.setup_filter([1, 3, 3, 1]), oo.setup_filter([1, 3, 3, 1]))


@pytest.mark.parametrize('dtype,tol', [(torch.float16, 3e-3), (torch.bfloat16, 3e-2), (torch.float64, 1e-6)])
@pytest.mark.parametrize('name', ['blur_after_tconv', 'up2_skip', 'down2_skip', 'asym_updown_flip'])
def test_upfirdn2d_dtypes_and_channels_last(name, dtype, tol):
    c = UPFIRDN_CASES[name]
    x, _ = make_input(c)
    f = make_filter(c, oo.setup_filter)
    xd = x.to(dtype)
    ref = oo.upfirdn2d(xd.double(), f, **_up_kw(c))
    for fmt in (torch.contiguous_format, torch.channels_last):
        xg = xd.to(DEV).contiguous(memory_format=fmt)
        y = _up().upfirdn2d(xg, f.to(DEV), **_up_kw(c))
        assert y.dtype == dtype and y.shape == ref.shape
        if fmt == torch.channels_last and x.shape[1] > 1:
            assert y.stride(1) == 1
        assert (y.cpu().double() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('name', sorted(UPFIRDN_CASES))
def test_upfirdn2d_gradients_first_and_second_order(name):
    c = UPFIRDN_CASES[name]
    x, _ = make_input(c)
    f = make_filter(c, oo.setup_filter)
    rng = np.random.default_rng(c['seed'] + 7)

    def run(fn, xin, fin):
        xin = xin.clone().requires_grad_(True)
        y = fn(xin, fin, **_up_kw(c))
        dy = torch.from_numpy(rng_dy).to(y.device, y.dtype)
        gx, = torch.autograd.grad(y, xin, dy, create_graph=True)
        v = torch.from_numpy(rng_v).to(y.device, y.dtype)
        ggy, = torch.autograd.grad(gx, xin, v, allow_unused=True) if gx.requires_grad else (None,)
        return y, gx, ggy

    y_shape = oo.upfirdn2d(x.double(), f, **_up_kw(c)).shape
    rng_dy = rng.standard_normal(tuple(y_shape))
    rng_v = rng.standard_normal(tuple(x.shape))
    ref = run(oo.upfirdn2d, x.double(), f)
    got = run(_up().upfirdn2d, x.double().to(DEV), None if f is None else f.to(DEV))
    assert (got[0].cpu() - ref[0]).abs().max().item() < 1e-6
    assert (got[1].cpu() - ref[1]).abs().max().item() < 1e-6
    # upfirdn2d is linear in x: the second derivative w.r.t. x vanishes (autograd returns None/zeros on both sides)
    assert ref[2] is None or ref[2].abs().max().item() == 0
    assert got[2] is None or got[2].abs().max().item() == 0


def test_upfirdn2d_double_backward_through_dy():
    """R1-style: d/d(dy) of <dx, v> equals upfirdn2d(v) - exercises the re-entrant autograd Function."""
    c = UPFIRDN_CASES['down2_skip']
    x, _ = make_input(c)
    f = make_filter(c, oo.setup_filter)

    def run(fn, xin, fin, dev):
        xin = xin.clone().requires_grad_(True)
        y = fn(xin, fin, **_up_kw(c))
        dy = torch.ones_like(y, requires_grad=True)
        gx, = torch.autograd.grad(y, xin, dy, create_graph=True)
        s = (gx * torch.arange(gx.numel(), device=dev, dtype=gx.dtype).reshape(gx.shape)).sum()
        g_dy, = torch.autograd.grad(s, dy)
        return g_dy

    ref = run(oo.upfirdn2d, x.double(), f, 'cpu')
    got = run(_up().upfirdn2d, x.double().to(DEV), f.to(DEV), DEV)
    assert (got.cpu() - ref).abs().max().item() < 1e-6 * ref.abs().max().item()


def test_upfirdn2d_large_image_tiles():
    """512x512 fp16 conv-output sized tensor (networks_stylegan2.py:352 scale): tile seams / multi-tile grid."""
    up = _up()
    torch.manual_seed(0)
    x = torch.randn(2, 16, 200, 333, device=DEV)
    f = up.setup_filter([1, 3, 3, 1], device=DEV)
    for kw in (dict(up=2, padding=[2, 1, 2, 1], gain=4.0), dict(down=2, padding=[1, 1, 1, 1]), dict(padding=[1, 2, 2, 1])):
        y = up.upfirdn2d(x, f, **kw)
        ref = oo.upfirdn2d(x.cpu(), f.cpu(), up=kw.get('up', 1), down=kw.get('down', 1), padding=kw['padding'], gain=kw.get('gain', 1))
        assert (y.cpu() - ref).abs().max().item() < 1e-4


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 2e-5), (torch.float16, 2e-3), (torch.bfloat16, 2e-2)])
@pytest.mark.parametrize('kw', [dict(padding=[1, 1, 1, 1], gain=4.0), dict(up=2, padding=[2, 1, 2, 1], gain=4.0),
                                dict(down=2, padding=[1, 1, 1, 1]), dict(padding=[-1, 2, 3, -2], flip_filter=True),
                                dict(up=2, padding=[4, 3, 0, 5], flip_filter=True), dict(down=2, padding=[0, 3, -2, 4])],
                         ids=['blur', 'up2', 'down2', 'crop_flip', 'up2_asym_flip', 'down2_crop'])
def test_upfirdn2d_fast_path_misaligned_rows_and_views(kw, dtype, tol):
    """4x4-filter fast kernel: odd widths (rows not 16-byte aligned), several tiles per image, a non-symmetric 2-D
    filter (so flip matters), odd storage offsets and row strides (views of a larger buffer)."""
    up = _up()
    g = torch.Generator().manual_seed(11)
    f = torch.rand(4, 4, generator=g) + 0.1
    big = torch.randn(3, 5, 71, 275, generator=g).to(dtype)
    big_d = big.to(DEV)
    for take in (lambda t: t[:, :, :, :273], lambda t: t[:, 1:4, 3:70, 1:274], lambda t: t[:, :, ::2, 5:150]):
        view, xv = take(big), take(big_d)
        assert xv.stride(3) == 1 and not xv.is_contiguous()
        y = up.upfirdn2d(xv, f.to(DEV), **kw)
        ref = oo.upfirdn2d(view.double(), f.double(), up=kw.get('up', 1), down=kw.get('down', 1), padding=kw['padding'],
                           flip_filter=kw.get('flip_filter', False), gain=kw.get('gain', 1))
        assert y.shape == ref.shape and y.dtype == dtype
        assert (y.cpu().double() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 2e-5), (torch.float16, 2e-3), (torch.bfloat16, 2e-2)])
@pytest.mark.parametrize('kw', [dict(padding=[1, 1, 1, 1], gain=4.0), dict(up=2, padding=[2, 1, 2, 1], gain=4.0), dict(down=2, padding=[1, 1, 1, 1]),
                                dict(up=2, down=3, padding=[4, -1, 0, 5], flip_filter=True)], ids=['blur', 'up2', 'down2', 'up2_down3_crop_flip'])
def test_upfirdn2d_channels_last_vector_kernel(kw, dtype, tol):
    """channels_last tensors whose channel count fills whole 16-byte groups take the vectorised kernel (one 128-bit load of 4 / 8
    channels per tap): odd image sizes, a non-symmetric 2-D filter, and a channels_last VIEW (batch slice) of a larger buffer."""
    up = _up()
    g = torch.Generator().manual_seed(13)
    f = torch.rand(4, 4, generator=g) + 0.1
    big = torch.randn(3, 32, 37, 53, generator=g).to(dtype)
    xcl = big.to(DEV).contiguous(memory_format=torch.channels_last)
    for view, xv in ((big, xcl), (big[1:3], xcl[1:3])):
        assert xv.stride(1) == 1
        y = up.upfirdn2d(xv, f.to(DEV), **kw)
        ref = oo.upfirdn2d(view.double(), f.double(), up=kw.get('up', 1), down=kw.get('down', 1), padding=kw['padding'],
                           flip_filter=kw.get('flip_filter', False), gain=kw.get('gain', 1))
        assert y.shape == ref.shape and y.dtype == dtype and y.stride(1) == 1
        assert (y.cpu().double() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


# ------------------------------------------------------------------------------------------ filtered_lrelu
def _fl():
    from panic3d_b200.torch_utils.ops import filtered_lrelu
    return filtered_lrelu


def _fl_args(c):
    fu = make_filter(dict(c, filter=c.get('fu')), oo.setup_filter)
    fd = make_filter(dict(c, filter=c.get('fd')), oo.setup_filter)
    kw = dict(up=c.get('up', 1), down=c.get('down', 1), padding=c.get('padding', 0), gain=c.get('gain', np.sqrt(2)),
              slope=c.get('slope', 0.2), clamp=c.get('clamp'), flip_filter=c.get('flip', False))
    return fu, fd, kw


@pytest.mark.parametrize('name', sorted(FLRELU_CASES))
def test_filtered_lrelu_forward_matches_reference_fixture(name):
    c = FLRELU_CASES[name]
    x, b = make_input(c)
    fu, fd, kw = _fl_args(c)
    dev = lambda t: None if t is None else t.to(DEV)
    y = _fl().filtered_lrelu(dev(x), dev(fu), dev(fd), dev(b), **kw)
    assert tuple(y.shape) == G['fl_' + name].shape
    assert np.abs(y.cpu().numpy() - G['fl_' + name]).max() < 2e-5


@pytest.mark.parametrize('name', sorted(FLRELU_CASES))
def test_filtered_lrelu_gradients(name):
    """dx, db through the stored 2-bit sign tensor vs autograd on the oracle composition; plus a second-order
    product (the op is piecewise linear: d/dx of <dx, v> is zero, d/d(dy) re-enters the op)."""
    c = FLRELU_CASES[name]
    x, b = make_input(c)
    fu, fd, kw = _fl_args(c)
    rng = np.random.default_rng(c['seed'] + 3)
    y_ref0 = oo.filtered_lrelu(x, fu, fd, b, **kw)
    dy_np = rng.standard_normal(tuple(y_ref0.shape)).astype(np.float32)

    def run(fn, dev_):
        to = lambda t: None if t is None else t.to(dev_)
        xin = to(x).clone().requires_grad_(True)
        bin_ = None if b is None else to(b).clone().requires_grad_(True)
        y = fn(xin, to(fu), to(fd), bin_, **kw)
        dy = torch.from_numpy(dy_np).to(dev_).requires_grad_(True)
        ins = [xin] + ([bin_] if bin_ is not None else [])
        g = torch.autograd.grad(y, ins, dy, create_graph=True)
        s = (g[0] * torch.linspace(-1, 1, g[0].numel(), device=dev_).reshape(g[0].shape)).sum()
        g_dy, = torch.autograd.grad(s, dy)
        return [y] + list(g) + [g_dy]

    ref = run(oo.filtered_lrelu, 'cpu')
    got = run(_fl().filtered_lrelu, DEV)
    for r, g_ in zip(ref, got):
        scale = max(1.0, r.abs().max().item())
        assert (g_.cpu() - r).abs().max().item() < 2e-4 * scale, name


@pytest.mark.parametrize('dtype,tol', [(torch.float16, 5e-3), (torch.bfloat16, 4e-2)])
def test_filtered_lrelu_low_precision_and_channels_last(dtype, tol):
    c = FLRELU_CASES['up2_down2_sep']
    x, b = make_input(c)
    fu, fd, kw = _fl_args(c)
    xd, bd = x.to(dtype), b.to(dtype)
    ref = oo.filtered_lrelu(xd.float(), fu, fd, bd.float(), **kw)
    for fmt in (torch.contiguous_format, torch.channels_last):
        y = _fl().filtered_lrelu(xd.to(DEV).contiguous(memory_format=fmt), fu.to(DEV), fd.to(DEV), bd.to(DEV), **kw)
        assert y.dtype == dtype
        assert (y.float().cpu() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())


def test_filtered_lrelu_multi_tile_image():
    torch.manual_seed(1)
    x = torch.randn(1, 5, 70, 90, device=DEV)
    b = torch.randn(5, device=DEV)
    fu = oo.setup_filter(np.hanning(14)[1:-1])      # 12 taps, separable
    fd = oo.setup_filter(np.hanning(14)[1:-1])
    kw = dict(up=2, down=2, padding=[9, 10, 9, 10], clamp=256.0)
    y = _fl().filtered_lrelu(x, fu.to(DEV), fd.to(DEV), b, **kw)
    ref = oo.filtered_lrelu(x.cpu(), fu, fd, b.cpu(), **kw)
    assert y.shape == ref.shape
    assert (y.cpu() - ref).abs().max().item() < 1e-4
