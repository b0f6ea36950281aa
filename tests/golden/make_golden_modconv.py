"""Golden vectors for the modulated convolution: the UNMODIFIED reference's SynthesisLayer / ToRGBLayer
(_train/eg3dc/src/training/networks_stylegan2.py:304-380) on CPU, fused_modconv=True, seeded parameters and inputs.

    PROJECT_DN=/root/reference python tests/golden/make_golden_modconv.py

Parameters come from oracle.modconv_oracle.init_layer_ (the reference zero-initialises bias and noise_strength, which
would leave the epilogue unexercised); tests/test_modconv_cpu.py rebuilds the same layers as the oracle's stand-ins with
the same call and compares.  `random` noise is drawn by the layer itself under torch.manual_seed(seed) and stored.
The script also checks, on the reference's own module, that dropin.install_modconv() rebinds both forwards, keeps the
originals, and leaves these CPU calls bit-identical (CPU calls always run the original method).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference'
os.environ.setdefault('PROJECT_DN', REF)
sys.path[:0] = [ROOT, os.path.join(ROOT, 'baseline'), REF, REF + '/_train/eg3dc/src']

import ref_env  # noqa: E402,F401  (kornia stub)
import training.networks_stylegan2 as ref  # noqa: E402
from oracle import modconv_oracle as mo  # noqa: E402
from tests.golden.cases_modconv import MODCONV_CASES, make_inputs  # noqa: E402


def build(module, c):
    if c['kind'] == 'torgb':
        layer = module.ToRGBLayer(c['cin'], c['cout'], c['w_dim'], conv_clamp=c.get('clamp'))
    else:
        layer = module.SynthesisLayer(c['cin'], c['cout'], c['w_dim'], c['res'], up=c['up'], conv_clamp=c.get('clamp'))
    return mo.init_layer_(layer, c['seed'])


def run(layer, c, x, w):
    torch.manual_seed(c['seed'])
    with torch.no_grad():
        if c['kind'] == 'torgb':
            return layer(x, w, fused_modconv=True)
        return layer(x, w, noise_mode=c['noise'], fused_modconv=True, gain=c.get('gain', 1))


def main():
    import panic3d_b200.dropin as dropin
    for name, c in MODCONV_CASES.items():
        layer = build(ref, c)
        x, w = make_inputs(c)
        y = run(layer, c, x, w)
        out = {'x': x.numpy(), 'w': w.numpy(), 'y': y.numpy()}
        if c.get('noise') == 'random':
            torch.manual_seed(c['seed'])
            out['noise'] = torch.randn([x.shape[0], 1, c['res'], c['res']]).numpy()
        np.savez_compressed(os.path.join(HERE, f'modconv_{name}.npz'), **out)
        print(name, y.shape, float(y.abs().max()))
    names = dropin.install_modconv(ref)
    assert names == ['SynthesisLayer.forward', 'ToRGBLayer.forward']
    assert ref.SynthesisLayer._p3d_reference_forward is not ref.SynthesisLayer.forward
    for name, c in MODCONV_CASES.items():
        x, w = make_inputs(c)
        got = run(build(ref, c), c, x, w)
        assert np.array_equal(got.numpy(), np.load(os.path.join(HERE, f'modconv_{name}.npz'))['y']), name
    print('install_modconv on the reference module: CPU calls bit-identical')


if __name__ == '__main__':
    main()
