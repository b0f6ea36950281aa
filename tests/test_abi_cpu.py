"""CPU: the C-ABI library builds (cross-compile), loads, and exports every symbol the headers
declare; pure-host entry points behave (no GPU compute here)."""
import ctypes as C
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _lib
    return _lib.lib()


def header_functions():
    names = []
    for h in glob.glob(os.path.join(ROOT, 'include', '*.h')):
        src = re.sub(r'/\*.*?\*/', '', open(h).read(), flags=re.S)
        names += re.findall(r'\b(p3d_[a-z0-9_]+)\s*\(', src)
    return sorted(set(names))


def test_every_declared_symbol_is_exported(lib):
    from panic3d_b200 import _lib
    from panic3d_b200.torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu   # noqa: F401  (register their prototypes)
    from panic3d_b200 import paste, imageio                                        # noqa: F401
    declared = header_functions()
    assert len(declared) >= 10
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in include/*.h but not exported by libp3d.so'
    # and the ctypes binding covers exactly the header surface
    assert sorted(_lib.declared_symbols()) == declared


def test_version_and_host_only_calls(lib):
    from panic3d_b200 import _lib
    assert b'sm_90a' in lib.p3d_version()
    p = _lib.RenderParams()
    p.n_views, p.n_rays, p.n_coarse, p.n_fine = 8, 128 * 128, 96, 96
    p.channels, p.hidden, p.out_dim, p.plane_h, p.plane_w = 32, 64, 33, 512, 512
    nbytes = lib.p3d_render_workspace_bytes(C.byref(p))
    rays = 8 * 128 * 128
    assert nbytes >= rays * (96 + 96) * 34 * 4          # depth + sigma + 32 colours per sample
    assert nbytes < rays * (96 + 96) * 34 * 4 * 1.05


def test_bad_arguments_fail_loudly(lib):
    from panic3d_b200 import _lib
    p = _lib.RenderParams()
    p.channels, p.hidden, p.out_dim = 16, 64, 33         # unsupported decoder shape
    p.box_warp = 0.7
    rc = lib.p3d_render_forward(C.byref(p), *([None] * 9), None, 0, *([None] * 5))
    assert rc != 0
    assert b'unsupported' in lib.p3d_last_error()
    with pytest.raises(RuntimeError):
        _lib.check(rc)


def test_no_cpu_fallback():
    import torch
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    from panic3d_b200.training.volumetric_rendering.ray_sampler import RaySampler
    from panic3d_b200.training.triplane import OSGDecoder
    dec = OSGDecoder(32, {'decoder_lr_mul': 1, 'decoder_output_dim': 32})
    assert [k for k, _ in dec.named_parameters()] == ['net.0.weight', 'net.0.bias', 'net.2.weight', 'net.2.bias']
    assert tuple(dec.net[0].weight.shape) == (64, 32) and tuple(dec.net[2].weight.shape) == (33, 64)
    r = ImportanceRenderer(use_triplane=True)
    assert len(list(r.parameters())) == 0 and len(list(RaySampler().parameters())) == 0
    opts = dict(box_warp=0.7, ray_start=0.5, ray_end=1.5, depth_resolution=4, depth_resolution_importance=4)
    with pytest.raises(RuntimeError), torch.no_grad():
        r(torch.zeros(1, 3, 32, 8, 8), dec, torch.zeros(1, 4, 3), torch.ones(1, 4, 3), opts)
    with pytest.raises(RuntimeError):
        RaySampler()(torch.eye(4)[None], torch.eye(3)[None], 4)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, 'panic3d-anime-reconstruction_b200')
    for path in glob.glob(os.path.join(pkg, '**', '*.py'), recursive=True):
        src = open(path).read()
        assert not re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M), f'{path} imports oracle/'
