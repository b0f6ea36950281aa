"""CPU: host-side contract of the front-view paste (no GPU compute): struct layout, loud failure without CUDA, drop-in rebinding."""
import ctypes as C
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_params_struct_matches_the_header():
    import panic3d_b200.paste as pp
    src = open(os.path.join(ROOT, 'include', 'p3d_paste.h')).read()
    body = re.search(r'typedef struct p3d_paste_params \{(.*?)\} p3d_paste_params;', src, flags=re.S).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = []
    for decl in body.split(';'):
        decl = decl.strip()
        if decl:
            typ, names = decl.split(None, 1)
            fields += [(n.strip(), typ) for n in names.split(',')]
    ctype = {'int32_t': C.c_int32, 'double': C.c_double}
    assert [(n, ctype[t]) for n, t in fields] == list(pp.PasteParams._fields_)
    assert C.sizeof(pp.PasteParams) == 64


def test_no_cpu_path():
    import panic3d_b200.paste as pp
    t = torch.zeros(1, 3, 8, 8)
    with pytest.raises(RuntimeError, match='CUDA'):
        pp.occlusion_rays(t, 0.5)
    with pytest.raises(RuntimeError, match='CUDA'):
        pp.erode_front_weights(torch.zeros(1, 1, 8, 8), 3)
    with pytest.raises(RuntimeError, match='CUDA'):
        pp.paste_front_fused(torch.zeros(1, 3, 16, 16), t, torch.zeros(1, 1, 8, 8), torch.zeros(1, 3, 16, 16), torch.zeros(1, 1, 8, 8), t, t, 0.7)


def test_bad_arguments_fail_loudly():
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.paste as pp
    from panic3d_b200 import _lib
    L = _lib.lib()
    p = pp.PasteParams()
    p.n_views, p.res_render, p.res_image, p.box_warp = 1, 8, 16, 0.7
    assert L.p3d_paste_front(C.byref(p), *([None] * 8), *([None] * 4), None) != 0 and b'NULL' in L.p3d_last_error()
    p.box_warp = 0.0
    assert L.p3d_paste_front(C.byref(p), *([None] * 8), *([None] * 4), None) != 0 and b'box_warp' in L.p3d_last_error()
    assert L.p3d_paste_erode(None, 1, 8, 8, 3, 0.5, None, None) != 0
    assert L.p3d_paste_occlusion_rays(None, 1, 8, 0.5, 0.01, None, None, None) != 0


@pytest.mark.parametrize('guard', ['image', 'render'])
def test_32bit_offset_guard_at_its_boundary(guard):
    """Offsets inside a view and the (5, N, 1, S, S) parts stride are 32-bit in the kernels; check_params refuses a batch
    with 5 * N * S^2 >= 2^31 or 3 * N * R^2 >= 2^31.  The largest N that passes gets as far as the NULL-input check."""
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.paste as pp
    from panic3d_b200 import _lib
    L = _lib.lib()
    S, R, n_ok = (512, 8, 1638) if guard == 'image' else (16, 512, 2730)
    assert 5 * n_ok * S * S < 2 ** 31 <= 5 * (n_ok + 1) * S * S if guard == 'image' else 3 * n_ok * R * R < 2 ** 31 <= 3 * (n_ok + 1) * R * R
    p = pp.PasteParams()
    p.res_render, p.res_image, p.box_warp = R, S, 0.7
    for n, want in ((n_ok, b'NULL'), (n_ok + 1, b'32-bit offsets')):
        p.n_views = n
        assert L.p3d_paste_front(C.byref(p), *([None] * 8), *([None] * 4), None) != 0
        assert want in L.p3d_last_error(), (n, L.p3d_last_error())
        assert L.p3d_paste_front_backward(C.byref(p), *([None] * 7), None) != 0
        assert want in L.p3d_last_error(), (n, L.p3d_last_error())


def test_install_paste_rebinds_and_keeps_the_original():
    import panic3d_b200.dropin as dropin
    import panic3d_b200.paste as pp
    mod = types.ModuleType('fake_training_triplane')
    mod.paste_front = mod.get_front_occlusion = mod.get_front_weights = lambda *a, **k: 'reference'
    dropin.install_paste(mod)
    dropin.install_paste(mod)                                                      # idempotent: the saved original survives
    assert mod.paste_front is pp.paste_front and mod.get_front_occlusion is pp.get_front_occlusion
    assert mod._p3d_reference_paste_front() == 'reference'


def test_stand_alone_helpers_equal_the_oracle_on_cpu():
    """sample_orthofront / get_xyz_discrepancy are plain torch ops kept for stand-alone callers."""
    import panic3d_b200.paste as pp
    from oracle import paste_oracle as po
    inp = po.synth_paste_inputs(3, 1, 12, 24)
    up = torch.nn.functional.interpolate(inp['image_xyz'], 24, mode='bilinear')
    assert torch.equal(pp.sample_orthofront(inp['front_rgb'], up, 0.7), po.sample_orthofront(inp['front_rgb'], up, 0.7))
    rays = {'ray_origins': inp['ro'], 'ray_directions': inp['rd']}
    assert torch.equal(pp.get_xyz_discrepancy(inp['image_xyz'], rays), po.xyz_discrepancy(inp['image_xyz'], inp['ro'], inp['rd']))
