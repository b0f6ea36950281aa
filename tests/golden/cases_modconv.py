"""Cases of tests/golden/modconv_*.npz (written by make_golden_modconv.py from the reference's own layers)."""
import math

import torch

MODCONV_CASES = {
    'up1_const_gain': dict(kind='layer', cin=32, cout=48, w_dim=16, res=8, up=1, n=3, noise='const', gain=math.sqrt(0.5), clamp=2.0, seed=1),
    'up1_none': dict(kind='layer', cin=16, cout=24, w_dim=16, res=6, up=1, n=1, noise='none', seed=2),
    'up2_random': dict(kind='layer', cin=32, cout=16, w_dim=16, res=12, up=2, n=3, noise='random', seed=3),
    'up2_const_clamp': dict(kind='layer', cin=16, cout=32, w_dim=16, res=8, up=2, n=2, noise='const', clamp=0.5, seed=4),
    'torgb': dict(kind='torgb', cin=48, cout=3, w_dim=16, res=8, n=3, seed=5),
    'torgb_clamp': dict(kind='torgb', cin=32, cout=96, w_dim=16, res=4, n=3, clamp=0.05, seed=6),
    # fp16 layers called directly (a block would force fp32 on CPU): the inf-norm pre-normalisation of the fp16 branch
    'up1_fp16': dict(kind='layer', cin=32, cout=48, w_dim=16, res=8, up=1, n=3, noise='none', clamp=256, dtype='float16', seed=7),
    'up2_fp16': dict(kind='layer', cin=16, cout=32, w_dim=16, res=8, up=2, n=2, noise='const', clamp=256, dtype='float16', seed=8),
    'torgb_fp16': dict(kind='torgb', cin=32, cout=3, w_dim=16, res=8, n=2, clamp=256, dtype='float16', seed=9),
}


def make_inputs(c):
    g = torch.Generator().manual_seed(1000 + c['seed'])
    res_in = c['res'] // c.get('up', 1)
    x = torch.randn(c['n'], c['cin'], res_in, res_in, generator=g)
    w = torch.randn(c['n'], c['w_dim'], generator=g)
    return x.to(getattr(torch, c.get('dtype', 'float32'))), w
