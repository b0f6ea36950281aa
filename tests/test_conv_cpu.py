"""CPU: the routing rule of panic3d_b200.conv at every edge of its envelope, install_conv2d() on a stand-in module, and
the C ABI of include/p3d_conv.h (struct layout, symbols, the supported envelope and workspace sizes)."""
import ctypes as C
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def pc():
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.conv as conv
    return conv


def _stub(calls, cuda_like=True):
    """A stand-in for torch_utils.ops.conv2d_gradfix.  `cuda_like`: its _should_use_custom_op accepts CPU tensors as if
    they were on CUDA, so that the rule's other conditions can be reached without a device; otherwise it is the
    reference's predicate (enabled, cuDNN enabled, a CUDA tensor)."""
    m = types.ModuleType('stub_conv2d_gradfix')
    m.enabled, m.weight_gradients_disabled = True, False
    m._should_use_custom_op = (lambda t: m.enabled and torch.backends.cudnn.enabled) if cuda_like else \
        (lambda t: m.enabled and torch.backends.cudnn.enabled and t.device.type == 'cuda')
    m.conv2d = lambda *a, **k: calls.append(('conv2d', a, k)) or 'original conv2d'
    m.conv_transpose2d = lambda *a, **k: calls.append(('conv_transpose2d', a, k)) or 'original conv_transpose2d'
    return m


@pytest.fixture()
def installed(pc, monkeypatch):
    import panic3d_b200.dropin as dropin
    calls = []
    m = _stub(calls)
    monkeypatch.setattr(pc, '_gradfix', None)
    monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
    dropin.install_conv2d(m)
    return m, calls


def test_install_conv2d_rebinds_and_keeps_the_originals(pc, monkeypatch):
    import panic3d_b200.dropin as dropin
    monkeypatch.setattr(pc, '_gradfix', None)
    m = _stub([])
    o2, ot = m.conv2d, m.conv_transpose2d
    assert dropin.install_conv2d(m) == ['conv2d', 'conv_transpose2d']
    dropin.install_conv2d(m)                                        # idempotent: the saved originals survive
    assert m.conv2d is pc.conv2d and m.conv_transpose2d is pc.conv_transpose2d
    assert m._p3d_reference_conv2d is o2 and m._p3d_reference_conv_transpose2d is ot
    assert pc._gradfix is m


X = dict(shape=(2, 32, 8, 8))
# (label, transpose, x kwargs, weight shape, call kwargs): each is one step outside the rule from an eligible call
BASE = (False, (2, 32, 8, 8), (48, 32, 3, 3), dict(stride=1, padding=1))
EDGES = [
    ('fp64 input', dict(dtype=torch.float64)),
    ('fp16 input', dict(dtype=torch.float16)),
    ('groups 2', dict(groups=2)),
    ('dilation 2', dict(dilation=2)),
    ('bias', dict(bias=True)),
    ('stride 2 with padding 1', dict(stride=2)),
    ('padding 0 with kernel 3 stride 1', dict(padding=0)),
    ('padding 2', dict(padding=2)),
    ('kernel 5', dict(wshape=(48, 32, 5, 5), padding=2)),
    ('kernel 2', dict(wshape=(48, 32, 2, 2), padding=0)),
    ('non-square kernel', dict(wshape=(48, 32, 3, 1))),
    ('channels_last input', dict(channels_last=True)),
    ('non-contiguous weight', dict(weight_t=True)),
]


def _call(pc, m, label, transpose=False, dtype=torch.float32, groups=1, dilation=1, bias=False, stride=1, padding=1,
          wshape=(48, 32, 3, 3), channels_last=False, weight_t=False, output_padding=0, xshape=(2, 32, 8, 8)):
    x = torch.randn(xshape, dtype=dtype)
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    w = torch.randn(wshape, dtype=dtype)
    if weight_t:
        w = torch.randn(wshape[1], wshape[0], *wshape[2:], dtype=dtype).transpose(0, 1)
    b = torch.zeros(wshape[0], dtype=dtype) if bias else None
    return pc.eligible(x, w, b, stride, padding, dilation, groups, transpose, output_padding)


def test_the_base_call_is_eligible(pc, installed):
    m, _ = installed
    p = _call(pc, m, 'base')
    assert p is not None and (p.kernel_size, p.stride, p.padding, p.transpose) == (3, 1, 1, 0)


@pytest.mark.parametrize('label,kw', EDGES, ids=[e[0] for e in EDGES])
def test_each_edge_is_routed_to_the_original(pc, installed, label, kw):
    m, calls = installed
    assert _call(pc, m, label, **kw) is None, label


def test_allow_tf32_enabled_flag_and_cpu_tensor_route_to_the_original(pc, installed, monkeypatch):
    m, calls = installed
    monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', True)
    assert _call(pc, m, 'tf32') is None
    monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
    m.enabled = False
    assert _call(pc, m, 'disabled') is None
    m.enabled = True
    m._should_use_custom_op = lambda t: m.enabled and torch.backends.cudnn.enabled and t.device.type == 'cuda'
    assert _call(pc, m, 'cpu tensor') is None
    x, w = torch.randn(2, 32, 8, 8), torch.randn(48, 32, 3, 3)
    assert m.conv2d(x, w, None, 1, 1) == 'original conv2d'          # a CPU call runs the original, arguments unchanged
    assert m.conv_transpose2d(x, w.transpose(0, 1), None, 1, 1, 0, 1, 1) == 'original conv_transpose2d'
    assert [c[0] for c in calls] == ['conv2d', 'conv_transpose2d'] and calls[0][1][0] is x


@pytest.mark.parametrize('transpose,k,s,p,op,ok', [
    (False, 3, 1, 1, 0, True), (False, 1, 1, 0, 0, True), (False, 3, 2, 0, 0, True),
    (True, 3, 2, 0, 0, True), (True, 3, 2, 0, 1, True), (True, 3, 2, 0, (1, 0), True), (True, 3, 1, 1, 0, True),
    (True, 1, 1, 0, 0, True), (True, 3, 2, 0, 2, False), (True, 3, 1, 1, 1, False), (False, 3, 2, 1, 0, False),
    (False, 1, 2, 0, 0, False), (False, 1, 1, 1, 0, False), (True, 3, 2, 1, 0, False), (False, 3, (1, 2), 1, 0, False),
])
def test_envelope_of_kernel_stride_padding(pc, installed, transpose, k, s, p, op, ok):
    m, _ = installed
    wshape = (32, 48, k, k) if transpose else (48, 32, k, k)
    got = _call(pc, m, 'env', transpose=transpose, wshape=wshape, stride=s, padding=p, output_padding=op)
    assert (got is not None) == ok


def test_routing_needs_a_measured_faster_entry(pc, installed, monkeypatch):
    m, calls = installed
    x, w = torch.randn(2, 32, 8, 8), torch.randn(48, 32, 3, 3)
    assert pc.eligible(x, w, None, 1, 1, 1, 1, False) is not None
    assert m.conv2d(x, w, None, 1, 1) == 'original conv2d'          # eligible but not in the table: the original
    assert not pc.measured_faster(pc.make_params(x.shape, w.shape, 1, 1, False))
    for key in pc.MEASURED_FASTER:                                   # every entry is a shape the kernels cover
        tr, k, s, cin, cout, h = key
        p = pc.make_params((4, cin, h, h), (cin, cout, k, k) if tr else (cout, cin, k, k), s, 1 if (k, s) == (3, 1) else 0, tr)
        assert pc.supported(p) and pc.measured_faster(p)


# ------------------------------------------------------------------------------------------ C ABI
def test_params_struct_matches_the_header(pc):
    hdr = open(os.path.join(ROOT, 'include', 'p3d_conv.h')).read()
    body = re.search(r'typedef struct p3d_conv_params \{(.*?)\} p3d_conv_params;', hdr, re.S).group(1)
    fields = []
    for line in body.splitlines():
        line = re.sub(r'/\*.*?\*/', '', line).strip()
        if line:
            ty, names = line.rstrip(';').split(None, 1)
            assert ty == 'int32_t', line
            fields += [n.strip() for n in names.split(',')]
    assert [f[0] for f in pc.ConvParams._fields_] == fields
    assert all(f[1] is C.c_int32 for f in pc.ConvParams._fields_)
    assert C.sizeof(pc.ConvParams) == 4 * len(fields)


def test_symbols_are_declared_bound_and_refuse_bad_calls(pc):
    from panic3d_b200 import _lib
    names = ['p3d_conv_supported', 'p3d_conv_out_size', 'p3d_conv_forward_workspace_bytes', 'p3d_conv_forward',
             'p3d_conv_weight_grad_workspace_bytes', 'p3d_conv_weight_grad']
    hdr = open(os.path.join(ROOT, 'include', 'p3d_conv.h')).read()
    L = _lib.lib()
    for n in names:
        assert n in _lib.declared_symbols() and getattr(L, n) is not None and n + '(' in hdr
    ok = pc.make_params((2, 32, 8, 8), (48, 32, 3, 3), 1, 1, False)
    bad = pc.make_params((2, 32, 8, 8), (48, 32, 5, 5), 1, 2, False)
    assert L.p3d_conv_forward_workspace_bytes(C.byref(ok)) == 48 * 32 * 9 * 4
    assert L.p3d_conv_forward_workspace_bytes(C.byref(bad)) == 0 and L.p3d_conv_weight_grad_workspace_bytes(C.byref(bad)) == 0
    assert L.p3d_conv_forward(C.byref(ok), None, None, None, 0, None, None) != 0 and b'NULL' in L.p3d_last_error()
    assert L.p3d_conv_forward(C.byref(bad), None, None, None, 0, None, None) != 0 and b'unsupported' in L.p3d_last_error()
    assert L.p3d_conv_weight_grad(C.byref(ok), None, None, None, 0, None, None) != 0 and b'NULL' in L.p3d_last_error()


@pytest.mark.parametrize('field,value,ok', [
    ('batch', 0, False), ('batch', 1, True), ('batch', 16384, True), ('batch', 16385, False),
    ('in_channels', 0, False), ('in_channels', 8192, True), ('in_channels', 8193, False),
    ('out_channels', 0, False), ('out_channels', 8192, True), ('out_channels', 8193, False),
    ('in_h', 0, False), ('in_h', 4096, True), ('in_h', 4097, False), ('in_w', 4097, False),
    ('transpose', 2, False), ('transpose', -1, False),
])
def test_supported_at_each_boundary(pc, field, value, ok):
    p = pc.make_params((2, 32, 8, 8), (48, 32, 3, 3), 1, 1, False)
    setattr(p, field, value)
    assert pc.supported(p) == ok


@pytest.mark.parametrize('args,size', [
    (((4, 512, 32, 32), (512, 512, 3, 3), 2, 0, True, 0), (65, 65)),        # conv0 of the 64^2 block
    (((4, 512, 32, 33), (512, 512, 3, 3), 2, 0, True, (1, 0)), (66, 67)),   # output_padding per axis
    (((4, 128, 257, 257), (128, 128, 3, 3), 2, 0, False, 0), (128, 128)),   # input gradient of conv0
    (((4, 128, 256, 256), (96, 128, 1, 1), 1, 0, False, 0), (256, 256)),
    (((1, 3, 3, 3), (3, 3, 3, 3), 2, 0, False, 0), (1, 1)),
])
def test_out_size(pc, args, size):
    p = pc.make_params(*args)
    assert pc.supported(p) and pc.out_size(p) == size


@pytest.mark.parametrize('batch,ok', [(16383, True), (16384, False)])
def test_stride_2_transposed_conv_batch_fits_the_grid(pc, batch, ok):
    """The forward of a stride-2 conv_transpose2d launches batch x 4 phases along gridDim.z (at most 65535); conv2d and
    the stride-1 ops keep the plain limit of 16384."""
    assert pc.supported(pc.make_params((batch, 8, 4, 4), (8, 8, 3, 3), 2, 0, True)) == ok
    assert pc.supported(pc.make_params((batch, 8, 4, 4), (8, 8, 3, 3), 1, 1, True))
    assert pc.supported(pc.make_params((batch, 8, 4, 4), (8, 8, 3, 3), 2, 0, False))


def test_conv2d_stride_2_needs_the_kernel_to_fit(pc):
    assert not pc.supported(pc.make_params((1, 3, 2, 8), (3, 3, 3, 3), 2, 0, False))
    assert not pc.supported(pc.make_params((1, 3, 8, 8), (3, 4, 3, 3), 1, 1, False))      # weight Cin != x channels
