"""GPU: the fp32 training convolutions (panic3d_b200.conv, csrc/conv_fp32.cu) against the fp64 oracle (oracle/conv_oracle.py)
- per-element bars on every backbone layer shape at batch 4 and on ragged shapes, no worse than torch fp32 with TF32 off,
gradients through a restated non-fused synthesis layer and an R1-style double backward, no_weight_gradients(), bitwise
repeats, and the routing of conv2d_gradfix calls."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import conv_oracle as co

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module', autouse=True)
def _fp32_strict():
    import __graft_entry__ as g
    g.build()
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True               # torch fp32 as the training loop runs it (cudnn.benchmark on)
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark = old


def _conv():
    import panic3d_b200.conv as pc
    return pc


def _ch(res):                                       # backbone channels: channel_base 32768, channel_max 512
    return min(32768 // res, 512)


# (name, transpose, N, Cin, Cout, H, W, k, stride, padding, output_padding): every conv of the 256^2 backbone at batch 4
# (conv0 of an up block is conv_transpose2d 3/2/0 from the previous resolution, conv1 conv2d 3/1/1, ToRGB 1x1 to 96)
BACKBONE = [('b4_conv1', False, 4, 512, 512, 4, 4, 3, 1, 1, 0), ('b4_torgb', False, 4, 512, 96, 4, 4, 1, 1, 0, 0)]
for _r in (8, 16, 32, 64, 128, 256):
    BACKBONE += [(f'b{_r}_conv0', True, 4, _ch(_r // 2), _ch(_r), _r // 2, _r // 2, 3, 2, 0, 0),
                 (f'b{_r}_conv1', False, 4, _ch(_r), _ch(_r), _r, _r, 3, 1, 1, 0),
                 (f'b{_r}_torgb', False, 4, _ch(_r), 96, _r, _r, 1, 1, 0, 0)]
RAGGED = [
    ('c3_to_100_odd', False, 5, 3, 100, 17, 13, 3, 1, 1, 0),
    ('c100_to_3_up2', True, 1, 100, 3, 9, 7, 3, 2, 0, 0),
    ('c96_to_3_k1', False, 1, 96, 3, 13, 11, 1, 1, 0, 0),
    ('c100_to_96_down2', False, 5, 100, 96, 15, 14, 3, 2, 0, 0),
    ('c96_to_100_t_s1', True, 5, 96, 100, 11, 9, 3, 1, 1, 0),
    ('c3_to_96_up2_opad', True, 1, 3, 96, 6, 7, 3, 2, 0, (1, 0)),
    ('c3_to_3_t_k1', True, 5, 3, 3, 5, 5, 1, 1, 0, 0),
]
CASES = {c[0]: c for c in BACKBONE + RAGGED}


def _inputs(case, seed=0):
    _, tr, n, cin, cout, h, w, k, s, p, op = case
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(n, cin, h, w, generator=g, device=DEV)
    wshape = (cin, cout, k, k) if tr else (cout, cin, k, k)
    wt = torch.randn(wshape, generator=g, device=DEV) / math.sqrt(cin * k * k)
    return x, wt, g


def _ours(case, x, w, dy):
    pc = _conv()
    _, tr, _, _, _, _, _, k, s, p, op = case
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = pc.conv_transpose2d_kernel(xg, wg, s, p, op) if tr else pc.conv2d_kernel(xg, wg, s, p)
    gx, gw = torch.autograd.grad(y, (xg, wg), dy)
    return y.detach(), gx, gw


def _torch32(case, x, w, dy):
    _, tr, _, _, _, _, _, k, s, p, op = case
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = F.conv_transpose2d(xg, wg, stride=s, padding=p, output_padding=op) if tr else F.conv2d(xg, wg, stride=s, padding=p)
    gx, gw = torch.autograd.grad(y, (xg, wg), dy)
    return y.detach(), gx, gw


def _check(what, ours, t32, ref, bound, K, floor):
    """The per-element bar, and our max error against twice torch fp32's.  `floor`: also allow the 3xTF32 representation
    error 3 * 2^-22 conv(|x|, |w|), which alone exceeds 2x fp32's error when a dot product has only a few terms (the
    ragged shapes with 3 channels or a handful of pixels); the backbone shapes take the plain 2x rule."""
    err = (ours.double() - ref).abs()
    bar = co.bar_constant(K) * bound + 1e-30
    worst = float((err / bar).max())
    assert worst <= 1.0, f'{what}: error reaches {worst:.3f} of the per-element bar'
    e_ours, e_t32 = float(err.max()), float((t32.double() - ref).abs().max())
    slack = 3 * 2.0 ** -22 * float(bound.max()) if floor else 1e-12 * float(bound.max())
    assert e_ours <= 2 * e_t32 + slack, f'{what}: max error {e_ours:.3e} vs torch fp32 {e_t32:.3e}'


@pytest.mark.parametrize('name', sorted(CASES))
def test_forward_and_gradients_per_element(name):
    case = CASES[name]
    _, tr, n, cin, cout, h, w_, k, s, p, op = case
    x, w, g = _inputs(case)
    y64 = co.conv(x, w, s, p, tr, op)
    dy = torch.randn(y64.shape, generator=g, device=DEV)
    ours, t32 = _ours(case, x, w, dy), _torch32(case, x, w, dy)
    assert ours[0].shape == y64.shape and ours[1].shape == x.shape and ours[2].shape == w.shape
    ax, aw, ady = x.double().abs(), w.double().abs(), dy.double().abs()
    floor = case in RAGGED
    _check(f'{name} forward', ours[0], t32[0], y64, co.conv(ax, aw, s, p, tr, op), cin * k * k, floor)
    _check(f'{name} input gradient', ours[1], t32[1], co.input_grad(x.shape, w, dy, s, p, tr, op),
           co.input_grad(x.shape, aw, ady, s, p, tr, op), cout * k * k, floor)
    _check(f'{name} weight gradient', ours[2], t32[2], co.weight_grad(x, w.shape, dy, s, p, tr, op),
           co.weight_grad(ax, w.shape, ady, s, p, tr, op), n * max(h * w_, y64.shape[2] * y64.shape[3]), floor)


@pytest.mark.parametrize('name', ['b64_conv0', 'b128_conv1', 'c100_to_96_down2'])
def test_two_runs_are_bitwise_equal(name):
    case = CASES[name]
    x, w, g = _inputs(case, seed=3)
    y = co.conv(x, w, case[8], case[9], case[1], case[10])
    dy = torch.randn(y.shape, generator=g, device=DEV)
    a, b = _ours(case, x, w, dy), _ours(case, x, w, dy)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ through layers
def _synthesis_layer(conv, convt, x, weight, styles, bias, r, up):
    """SynthesisLayer.forward on the non-fused route (networks_stylegan2.py:40-98, 334-354 with fused_modconv False):
    x * styles -> conv2d_resample (up 1: conv2d 3/1/1; up 2: conv_transpose2d 3/2/0 then the [1,3,3,1] FIR with gain 4
    and padding 1) -> * dcoefs -> bias, lrelu, gain sqrt(2).  `conv` / `convt` are the convolutions under test."""
    n = x.shape[0]
    dcoefs = (weight[None] * styles[:, None, :, None, None]).square().sum(dim=[2, 3, 4]).add(1e-8).rsqrt()
    xs = x * styles.reshape(n, -1, 1, 1)
    if up == 1:
        y = conv(xs, weight, 1, 1)
    else:
        y = convt(xs, weight.transpose(0, 1), 2, 0)
        f1 = torch.tensor([1., 3., 3., 1.], dtype=y.dtype, device=y.device)
        f = (f1[:, None] * f1[None, :]) / f1.sum() ** 2 * 4
        c = y.shape[1]
        y = F.conv2d(F.pad(y, [1, 1, 1, 1]), f.expand(c, 1, 4, 4), groups=c)
    y = y * dcoefs.reshape(n, -1, 1, 1) + bias.reshape(1, -1, 1, 1)
    y = F.leaky_relu(y, 0.2) * math.sqrt(2)
    return (y * r).sum()


@pytest.mark.parametrize('up', [1, 2])
def test_synthesis_layer_gradients_against_fp64(up):
    pc = _conv()
    g = torch.Generator(device=DEV).manual_seed(11 + up)
    n, cin, cout, res = 4, 96, 100, 32
    x = torch.randn(n, cin, res // up, res // up, generator=g, device=DEV)
    weight = torch.randn(cout, cin, 3, 3, generator=g, device=DEV)
    styles = torch.randn(n, cin, generator=g, device=DEV) * 0.5 + 1
    bias = torch.randn(cout, generator=g, device=DEV) * 0.1
    r = torch.randn(n, cout, res, res, generator=g, device=DEV)
    outs = {}
    for name, dt, conv, convt in (('ours', torch.float32, lambda a, b, s, p: pc.conv2d_kernel(a, b, s, p),
                                   lambda a, b, s, p: pc.conv_transpose2d_kernel(a, b, s, p)),
                                  ('fp64', torch.float64, lambda a, b, s, p: F.conv2d(a, b, stride=s, padding=p),
                                   lambda a, b, s, p: F.conv_transpose2d(a, b, stride=s, padding=p))):
        leaves = [t.to(dt).clone().requires_grad_(True) for t in (x, weight, styles, bias)]
        loss = _synthesis_layer(conv, convt, *leaves, r.to(dt), up)
        outs[name] = torch.autograd.grad(loss, leaves)
    for label, a, b in zip(('x', 'weight', 'styles', 'bias'), outs['ours'], outs['fp64']):
        rel = float((a.double() - b).abs().max() / b.abs().max())
        assert rel < 2e-5, (label, rel)


def _d_block(conv, x, w0, w1, wskip):
    """A discriminator-like block on the fp32 route: conv 3/1/1 -> softplus -> conv 3/2/0 -> softplus, plus a 1x1 skip
    on every other pixel; `conv(x, w, stride, padding)` is the convolution under test."""
    h = F.softplus(conv(x, w0, 1, 1))
    h = F.softplus(conv(h, w1, 2, 0))
    skip = conv(x[:, :, 1::2, 1::2][:, :, :h.shape[2], :h.shape[3]].contiguous(), wskip, 1, 0)
    return h + skip


def test_r1_double_backward_against_fp64():
    pc = _conv()
    g = torch.Generator(device=DEV).manual_seed(5)
    n, c0, c1, res = 4, 64, 96, 33
    x = torch.randn(n, c0, res, res, generator=g, device=DEV)
    ws = [torch.randn(c0, c0, 3, 3, generator=g, device=DEV) / math.sqrt(c0 * 9),
          torch.randn(c1, c0, 3, 3, generator=g, device=DEV) / math.sqrt(c0 * 9),
          torch.randn(c1, c0, 1, 1, generator=g, device=DEV) / math.sqrt(c0)]
    v = torch.randn(n, c1, 16, 16, generator=g, device=DEV)
    grads = {}
    for name, dt, conv in (('ours', torch.float32, lambda a, b, s, p: pc.conv2d_kernel(a, b, s, p)),
                           ('fp64', torch.float64, lambda a, b, s, p: F.conv2d(a, b, stride=s, padding=p))):
        img = x.to(dt).clone().requires_grad_(True)
        params = [w.to(dt).clone().requires_grad_(True) for w in ws]
        logits = (_d_block(conv, img, *params) * v.to(dt)).sum()
        (gi,) = torch.autograd.grad(logits, img, create_graph=True)
        pen = gi.square().sum()
        grads[name] = torch.autograd.grad(pen, params)
    for i, (a, b) in enumerate(zip(grads['ours'], grads['fp64'])):
        rel = float((a.double() - b).abs().max() / b.abs().max())
        assert rel < 2e-5, (i, rel)


# ------------------------------------------------------------------------------------------ routing
def _stub_gradfix(calls):
    """A stand-in for torch_utils.ops.conv2d_gradfix whose two functions record their calls and run torch's."""
    m = types.ModuleType('stub_conv2d_gradfix')
    m.enabled, m.weight_gradients_disabled = True, False
    m._should_use_custom_op = lambda t: m.enabled and torch.backends.cudnn.enabled and t.device.type == 'cuda'

    def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
        calls.append('conv2d')
        return F.conv2d(input, weight, bias, stride, padding, dilation, groups)

    def conv_transpose2d(input, weight, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
        calls.append('conv_transpose2d')
        return F.conv_transpose2d(input, weight, bias, stride, padding, output_padding, groups, dilation)
    m.conv2d, m.conv_transpose2d = conv2d, conv_transpose2d
    return m


@pytest.fixture()
def stub(monkeypatch):
    import panic3d_b200.dropin as dropin
    pc = _conv()
    calls = []
    m = _stub_gradfix(calls)
    monkeypatch.setattr(pc, '_gradfix', None)
    dropin.install_conv2d(m)
    yield m, calls, pc


def test_routed_away_calls_reach_the_original(stub, monkeypatch):
    m, calls, pc = stub
    x, w = torch.randn(2, 32, 8, 8, device=DEV), torch.randn(48, 32, 3, 3, device=DEV)
    key = (False, 3, 1, 32, 48, 8)
    assert pc.eligible(x, w, None, 1, 1, 1, 1, False) is not None
    m.conv2d(x, w, None, 1, 1)                                      # eligible, but not measured faster
    assert calls == ['conv2d']
    monkeypatch.setattr(pc, 'MEASURED_FASTER', frozenset([key]))
    y = m.conv2d(x, w, None, 1, 1)                                  # routed: the kernels, not the original
    assert calls == ['conv2d']
    ref = F.conv2d(x.double(), w.double(), padding=1)
    assert float((y.double() - ref).abs().max() / ref.abs().max()) < 1e-6
    torch.backends.cudnn.allow_tf32 = True
    try:
        m.conv2d(x, w, None, 1, 1)
    finally:
        torch.backends.cudnn.allow_tf32 = False
    m.conv2d(x.double(), w.double(), None, 1, 1)
    m.conv2d(x, w, torch.zeros(48, device=DEV), 1, 1)
    m.conv_transpose2d(x, w.transpose(0, 1).contiguous(), None, 1, 1, 0, 2)   # groups 2
    assert calls == ['conv2d'] * 4 + ['conv_transpose2d']


def test_no_weight_gradients_is_honoured(stub):
    m, calls, pc = stub
    x = torch.randn(2, 32, 8, 8, device=DEV, requires_grad=True)
    w = torch.randn(48, 32, 3, 3, device=DEV, requires_grad=True)
    m.weight_gradients_disabled = True
    pc.conv2d_kernel(x, w, 1, 1).square().sum().backward()
    assert w.grad is None and x.grad is not None
    m.weight_gradients_disabled = False
    pc.conv2d_kernel(x, w, 1, 1).square().sum().backward()
    assert w.grad is not None
