"""CPU: the drop-in mechanism - install() serves this package's modules under the reference's import names."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_install_registers_modules():
    code = textwrap.dedent('''
        import sys
        sys.path.insert(0, %r)
        import panic3d_b200.dropin as d
        names = d.install()
        assert 'training.volumetric_rendering.renderer' in names, names
        import panic3d_b200.training.volumetric_rendering.renderer as ours
        assert sys.modules['training.volumetric_rendering.renderer'] is ours
        print('ok')
    ''' % ROOT)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True)
    assert r.returncode == 0 and 'ok' in r.stdout, r.stderr[-2000:]


def test_plane_reuse_memo_runs_backbone_once_per_subject():
    """SURVEY 8f-1: repeated G.f-style calls with the same (ws, cond) hit the memo; changed latents, in-place edits,
    training-mode calls and non-const noise do not."""
    import torch
    from panic3d_b200 import dropin

    class Backbone:
        def __init__(self):
            self.calls = 0

        def synthesis(self, ws, cond, update_emas=False, **kw):
            self.calls += 1
            return ws.sum() + torch.zeros(1, 96, 4, 4) + self.calls

    class G:
        pass
    g = G()
    g.backbone = Backbone()
    memo = dropin.enable_plane_reuse(g)
    assert dropin.enable_plane_reuse(g) is memo                                   # idempotent
    ws = torch.randn(1, 14, 512)
    cond = {'image': torch.randn(1, 3, 8, 8), 'levels': [torch.ones(2), torch.zeros(3)]}
    a = g.backbone.synthesis(ws, cond, update_emas=False, noise_mode='const')
    for _ in range(15):                                                           # the other views of the sweep: fresh, equal ws
        b = g.backbone.synthesis(ws.clone(), {'image': cond['image'].clone(), 'levels': cond['levels']}, update_emas=False, noise_mode='const')
        assert b is a
    assert (memo.misses, memo.hits) == (1, 15)
    ws2 = ws.clone(); ws2[0, 0, 0] += 1
    assert g.backbone.synthesis(ws2, cond, noise_mode='const') is not a           # different subject
    ws2.mul_(2.0)                                                                 # in-place edit of the cached key tensor's twin
    c = g.backbone.synthesis(ws2, cond, noise_mode='const')
    assert memo.misses == 3 and g.backbone.synthesis(ws2, cond, noise_mode='const') is c
    n = memo.misses
    g.backbone.synthesis(ws2, cond, noise_mode='random')                          # stochastic noise: never cached
    g.backbone.synthesis(ws2, cond, update_emas=True, noise_mode='const')
    wsg = ws2.clone().requires_grad_(True)
    g.backbone.synthesis(wsg, cond, noise_mode='const')                           # autograd call (training): bypass
    assert memo.misses == n
    with torch.no_grad():
        assert g.backbone.synthesis(wsg, cond, noise_mode='const') is c           # same values under no_grad: reuse
    big = {'image': torch.randn(1, 3, 256, 256)}                                  # kept by reference + version counter
    d = g.backbone.synthesis(ws2, big, noise_mode='const')
    assert g.backbone.synthesis(ws2, big, noise_mode='const') is d
    big['image'].add_(1.0)                                                        # in-place write -> value compare -> miss
    assert g.backbone.synthesis(ws2, big, noise_mode='const') is not d
    memo.clear()
    assert g.backbone.synthesis(ws2, cond, noise_mode='const') is not c


def test_plane_reuse_memo_noise_mode_of_calls_that_do_not_name_one():
    """G.f / G.synthesis never pass noise_mode (the reference's layers then draw fresh noise per call).  The memo either
    passes an explicit 'const' on (default: deterministic sweep, cached) or, with default_noise_mode=None, leaves the call
    alone and does not cache it - it never replays one random draw for all views."""
    import torch
    from panic3d_b200 import dropin

    class Backbone:
        def __init__(self):
            self.modes = []

        def synthesis(self, ws, cond, update_emas=False, noise_mode='random', **kw):
            self.modes.append(noise_mode)
            return ws.sum() + torch.zeros(1, 96, 4, 4) + len(self.modes)

    class G:
        pass
    ws = torch.randn(1, 14, 512)
    g = G(); g.backbone = Backbone()
    bb = g.backbone
    memo = dropin.enable_plane_reuse(g)
    a = g.backbone.synthesis(ws, None)
    assert g.backbone.synthesis(ws.clone(), None) is a
    assert bb.modes == ['const'] and (memo.misses, memo.hits) == (1, 1)
    g2 = G(); g2.backbone = Backbone()
    bb2 = g2.backbone
    memo2 = dropin.enable_plane_reuse(g2, default_noise_mode=None)
    x = g2.backbone.synthesis(ws, None)
    y = g2.backbone.synthesis(ws, None)
    assert x is not y and bb2.modes == ['random', 'random'] and (memo2.misses, memo2.hits) == (0, 0)
    z = g2.backbone.synthesis(ws, None, noise_mode='const')
    assert g2.backbone.synthesis(ws, None, noise_mode='const') is z and memo2.hits == 1
