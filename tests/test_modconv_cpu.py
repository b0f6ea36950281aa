"""CPU: the modulated-convolution oracle against the reference's own layers (tests/golden/modconv_*.npz), the
install_modconv() contract, and the C-ABI symbols of include/p3d_modconv.h."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import modconv_oracle as mo
from tests.golden.cases_modconv import MODCONV_CASES, make_inputs

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _layer(module, c):
    if c['kind'] == 'torgb':
        layer = module.ToRGBLayer(c['cin'], c['cout'], c['w_dim'], conv_clamp=c.get('clamp'))
    else:
        layer = module.SynthesisLayer(c['cin'], c['cout'], c['w_dim'], c['res'], up=c['up'], conv_clamp=c.get('clamp'))
    return mo.init_layer_(layer, c['seed'])


def _run(layer, c, x, w, fused_modconv=True):
    torch.manual_seed(c['seed'])
    with torch.no_grad():
        if c['kind'] == 'torgb':
            return layer(x, w, fused_modconv=fused_modconv)
        return layer(x, w, noise_mode=c['noise'], fused_modconv=fused_modconv, gain=c.get('gain', 1))


@pytest.mark.parametrize('name', sorted(MODCONV_CASES))
def test_oracle_equals_the_reference_layers(name):
    c = MODCONV_CASES[name]
    g = np.load(os.path.join(HERE, f'modconv_{name}.npz'))
    x, w = make_inputs(c)
    assert np.array_equal(x.numpy(), g['x']) and np.array_equal(w.numpy(), g['w'])
    y = _run(_layer(mo, c), c, x, w)
    assert y.dtype == x.dtype
    want = g['y'].astype(np.float64)
    tol = 2e-5 if x.dtype == torch.float32 else 2.0 ** -10 * np.abs(want)          # fp16: one ulp
    assert (np.abs(y.double().numpy() - want) <= tol).all()
    if 'noise' in g:                                               # the layer draws its noise with the seeded torch.randn
        torch.manual_seed(c['seed'])
        assert np.array_equal(torch.randn(g['noise'].shape).numpy(), g['noise'])


def test_oracle_in_fp64_equals_the_reference_layers():
    c = MODCONV_CASES['up2_random']
    g = np.load(os.path.join(HERE, 'modconv_up2_random.npz'))
    x, w = make_inputs(c)
    layer = _layer(mo, c).double()
    with torch.no_grad():
        torch.manual_seed(c['seed'])
        y = layer(x.double(), w.double(), noise_mode='random')
    assert float(np.abs(y.numpy() - g['y']).max()) <= 2e-5


def test_tf32_rounding_is_nearest_ties_away():
    t = torch.tensor([1 + 2 ** -11, 1 + 2 ** -12, -(1 + 2 ** -11), 1 + 3 * 2 ** -11, 3.0, float('inf')])
    assert mo.tf32_rna(t).tolist() == [1 + 2 ** -10, 1.0, -(1 + 2 ** -10), 1 + 2 * 2 ** -10, 3.0, float('inf')]


@pytest.fixture()
def standins():
    """A module object holding fresh stand-in classes, so that install_modconv() never touches the shared ones."""
    import types
    mod = types.ModuleType('fake_networks_stylegan2')
    mod.SynthesisLayer = type('SynthesisLayer', (mo.SynthesisLayer,), {})
    mod.ToRGBLayer = type('ToRGBLayer', (mo.ToRGBLayer,), {})
    return mod


def test_install_modconv_rebinds_and_keeps_the_originals(standins):
    import panic3d_b200.dropin as dropin
    import panic3d_b200.modconv as mc
    orig_s, orig_t = standins.SynthesisLayer.forward, standins.ToRGBLayer.forward
    assert dropin.install_modconv(standins) == ['SynthesisLayer.forward', 'ToRGBLayer.forward']
    dropin.install_modconv(standins)                               # idempotent: the saved originals survive
    assert standins.SynthesisLayer.forward is mc.synthesis_layer_forward and standins.ToRGBLayer.forward is mc.torgb_forward
    assert standins.SynthesisLayer._p3d_reference_forward is orig_s and standins.ToRGBLayer._p3d_reference_forward is orig_t


@pytest.mark.parametrize('name', sorted(MODCONV_CASES))
def test_installed_cpu_and_training_calls_are_bit_identical(standins, name):
    import panic3d_b200.dropin as dropin
    c = MODCONV_CASES[name]
    x, w = make_inputs(c)
    before = [_run(_layer(standins, c), c, x, w, fused_modconv=f) for f in (True, False)]
    layer = _layer(standins, c)
    with torch.enable_grad():
        x_g = x.clone().requires_grad_(True)
        torch.manual_seed(c['seed'])
        train_before = layer(x_g, w) if c['kind'] == 'torgb' else layer(x_g, w, noise_mode=c['noise'])
    dropin.install_modconv(standins)
    after = [_run(_layer(standins, c), c, x, w, fused_modconv=f) for f in (True, False)]
    with torch.enable_grad():
        torch.manual_seed(c['seed'])
        train_after = layer(x_g, w) if c['kind'] == 'torgb' else layer(x_g, w, noise_mode=c['noise'])
    for a, b in zip(before + [train_before], after + [train_after]):
        assert torch.equal(a, b)
    assert train_after.requires_grad


def test_modconv_symbols_are_declared_and_bound():
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.modconv as mc
    from panic3d_b200 import _lib
    names = ['p3d_modconv_supported', 'p3d_modconv_out_size', 'p3d_modconv_workspace_bytes', 'p3d_modconv_prep', 'p3d_modconv_forward']
    assert set(names) <= set(_lib.declared_symbols())
    L = _lib.lib()
    hdr = open(os.path.join(os.path.dirname(HERE), '..', 'include', 'p3d_modconv.h')).read()
    for n in names:
        assert getattr(L, n) is not None and n + '(' in hdr
    # the eligibility rule, which needs no device
    x = torch.empty(1, 32, 8, 8)
    ok = mc.make_params(x, torch.empty(64, 32, 3, 3), True)
    assert mc.supported(ok) and L.p3d_modconv_workspace_bytes(C.byref(ok)) > 0
    for bad in (mc.make_params(x, torch.empty(64, 32, 3, 3), True, allow_tf32=False),      # fp32 without TF32
                mc.make_params(torch.empty(1, 24, 8, 8), torch.empty(64, 24, 3, 3), True),  # Cin not a multiple of 16
                mc.make_params(x, torch.empty(64, 32, 5, 5), True),                         # kernel 5
                mc.make_params(x, torch.empty(64, 32, 1, 1), True, up=2),                   # up 2 needs kernel 3
                mc.make_params(x, torch.empty(64, 32, 3, 3), True, down=2),
                mc.make_params(x.double(), torch.empty(64, 32, 3, 3), True)):
        assert not mc.supported(bad) and L.p3d_modconv_workspace_bytes(C.byref(bad)) == 0
    assert L.p3d_modconv_prep(C.byref(ok), None, None, None, None) != 0 and b'NULL' in L.p3d_last_error()
    oh, ow = C.c_int32(), C.c_int32()
    up2 = mc.make_params(x, torch.empty(64, 32, 3, 3), True, up=2)
    assert L.p3d_modconv_out_size(C.byref(up2), C.byref(oh), C.byref(ow)) == 0 and (oh.value, ow.value) == (17, 17)


# ------------------------------------------------------------------------------------------ the supported envelope
F32, F16 = 0, 1                 # P3D_F32 / P3D_F16 (include/p3d_ops.h)


def _envelope(p):
    """include/p3d_modconv.h restated: (supported, (out_h, out_w) or None, workspace bytes).  The workspace holds, per
    sample and N tile (8 rows when Cout <= 8, else 128), one 128-byte-per-row B tile per tap slot and K chunk (64 fp16 /
    32 fp32 channels); up 2 has 4 + 2 + 2 + 1 = 9 slots, like kernel 3."""
    nph = 4 if p.up == 2 else 1
    ok = ((p.kernel_size == 3 or (p.kernel_size == 1 and p.up == 1)) and p.up in (1, 2) and p.down == 1 and
          (p.dtype == F16 or (p.dtype == F32 and p.allow_tf32)) and p.demodulate in (0, 1) and
          0 < p.in_channels <= 65536 and p.in_channels % 16 == 0 and 1 <= p.out_channels <= 4096 and
          1 <= p.batch and p.batch * nph <= 65535 and 1 <= p.in_h <= 4096 and 1 <= p.in_w <= 4096)
    if not ok:
        return False, None, 0
    es = 2 if p.dtype == F16 else 4
    bn = 8 if p.out_channels <= 8 else 128
    nchunks = -(-p.in_channels * es // 128)
    ntaps = 1 if p.kernel_size == 1 else 9
    size = (2 * p.in_h + 1, 2 * p.in_w + 1) if p.up == 2 else (p.in_h, p.in_w)
    return True, size, p.batch * -(-p.out_channels // bn) * ntaps * nchunks * bn * 128


_BASE = dict(batch=2, in_channels=32, out_channels=64, in_h=8, in_w=8, kernel_size=3, up=1, down=1, dtype=F16,
             demodulate=1, allow_tf32=1)
# each boundary at, one below and one above; every row also runs in fp32, kernel 1 and up 2 (where those are supported)
_EDGES = [('in_channels', v) for v in (0, 15, 16, 17, 31, 32, 48, 65520, 65535, 65536, 65537, 65552)] + \
         [('out_channels', v) for v in (0, 1, 2, 7, 8, 9, 127, 128, 129, 4095, 4096, 4097)] + \
         [('in_h', v) for v in (0, 1, 2, 4095, 4096, 4097)] + [('in_w', v) for v in (0, 1, 2, 4095, 4096, 4097)] + \
         [('batch', v) for v in (0, 1, 16383, 16384, 65534, 65535, 65536)] + \
         [('demodulate', v) for v in (-1, 0, 1, 2)] + [('down', v) for v in (0, 2)] + [('kernel_size', v) for v in (0, 2, 5)] + \
         [('up', v) for v in (0, 3)] + [('dtype', v) for v in (2, 3, -1)] + [('allow_tf32', 0)]


@pytest.mark.parametrize('field,value', _EDGES, ids=[f'{f}={v}' for f, v in _EDGES])
def test_supported_out_size_and_workspace_at_each_boundary(field, value):
    """p3d_modconv_supported / _out_size / _workspace_bytes against the restatement at every boundary of the envelope, +-1,
    with a non-square input (in_h != in_w) so that a swapped out_size shows."""
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.modconv as mc
    from panic3d_b200 import _lib
    L = _lib.lib()
    for variant in (dict(), dict(dtype=F32), dict(kernel_size=1, demodulate=0), dict(up=2),
                    dict(in_h=5, in_w=37), dict(in_h=37, in_w=5, up=2), dict(dtype=F32, allow_tf32=0)):
        p = mc.ModconvParams(**{**_BASE, **variant, field: value})
        ok, size, nbytes = _envelope(p)
        assert bool(L.p3d_modconv_supported(C.byref(p))) == ok, (variant, field, value)
        assert int(L.p3d_modconv_workspace_bytes(C.byref(p))) == nbytes, (variant, field, value)
        oh, ow = C.c_int32(-1), C.c_int32(-1)
        rc = L.p3d_modconv_out_size(C.byref(p), C.byref(oh), C.byref(ow))
        assert (rc == 0) == ok and (not ok or (oh.value, ow.value) == size), (variant, field, value, oh.value, ow.value)
