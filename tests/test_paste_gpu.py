"""GPU: the fused front-view paste (panic3d_b200.paste -> p3d_paste_front, SURVEY 8f-3) against outputs of the
reference's own ``paste_front`` (tests/golden/paste_*.npz), the live oracle, properties at full size, and gradients."""
import os

import numpy as np
import pytest
import torch

from oracle import paste_oracle as po
from tests.golden.cases_paste import PASTE_CASES, OUT_KEYS, build_paste_inputs
from tests.helpers import StandInG

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
HERE = os.path.dirname(os.path.abspath(__file__))


def load(name):
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(HERE, 'golden', f'paste_{name}.npz')).items()}


def run_dropin(case, inp):
    import panic3d_b200.paste as pp
    G = StandInG(inp, DEV)
    x = {'cond': {'image_ortho_front': inp['front_rgb'].to(DEV)}, 'normalize_images': case['normalize_images'],
         'force_rays': {'ray_origins': inp['ro'].to(DEV), 'ray_directions': inp['rd'].to(DEV)}, 'paste_params': dict(case['params'])}
    out = {'image': inp['image'].to(DEV), 'image_xyz': inp['image_xyz'].to(DEV), 'image_weights': inp['image_weights'].to(DEV)}
    with torch.no_grad():
        res = pp.paste_front(G, x, out, **case['params'])
    torch.cuda.synchronize()
    return res, G


def borderline(case, inp):
    """Pixels where one of the thresholded quantities sits within rounding distance of its threshold (oracle, CPU)."""
    p = {k: v for k, v in case['params'].items() if k not in ('offset_occ', 'mode')}
    o = po.paste_front(inp['image'], inp['image_xyz'], inp['image_weights'], inp['front_rgb'], inp['occ'], inp['ro'], inp['rd'],
                       inp['box_warp'], frontw=inp['frontw'], normalize_images=case['normalize_images'], **p)
    tw, te, td = p.get('thresh_weight', 0.95), p.get('thresh_edges', 0.02), p.get('thresh_dxyz', 0.01)
    return ((o['q_weights'] - tw).abs() < 2e-6) | ((o['q_edges'] - te).abs() < 2e-7) | ((o['q_dxyz'] - td).abs() < max(2e-8, td * 1e-6))


@pytest.mark.parametrize('name', sorted(PASTE_CASES))
def test_paste_matches_reference_fixture(name):
    case = PASTE_CASES[name]
    inp = build_paste_inputs(case)
    gold = load(name)
    res, G = run_dropin(case, inp)
    # the rays handed to the occlusion render: exact (sign flips and one subtraction)
    assert torch.equal(G.seen['occ_ro'].cpu(), gold['occ_ro']) and torch.equal(G.seen['occ_rd'].cpu(), gold['occ_rd'])
    edge = borderline(case, inp)
    assert edge.float().mean().item() < 0.01
    ok = ~edge
    for k in ('mask_weights', 'mask_edges', 'mask_dxyz'):                         # hard thresholds: exact away from the threshold
        assert torch.equal(res[k].cpu()[ok], gold[k][ok]), k
    assert (res['mask_occ'].cpu() - gold['mask_occ']).abs().max().item() < 1e-6   # bilinear blend of exact 0/1
    assert (res['mask_frontweight'].cpu() - gold['mask_frontweight']).abs().max().item() < 1e-4
    assert (res['paste'].cpu() - gold['paste']).abs().max().item() < 1e-4
    ok3 = ok.expand(-1, 3, -1, -1)
    assert (res['mask'].cpu() - gold['mask'])[ok].abs().max().item() < 1e-4
    assert (res['image'].cpu() - gold['image'])[ok3].abs().max().item() < 2e-4
    assert set(OUT_KEYS) <= set(res.keys()) and res.image is res['image']
    if case['params'].get('front_weight_erosion', 0) >= 1:
        assert res['frontweight'] is not None
    else:
        assert res['frontweight'] is None and bool((res['mask_frontweight'] == 1).all())


def test_erosion_and_rays_equal_oracle_exactly():
    import panic3d_b200.paste as pp
    inp = po.synth_paste_inputs(5, 2, 40, 80)
    for e in (1, 2, 3, 4, 7):
        got = pp.erode_front_weights(inp['frontw'].to(DEV), e).cpu()
        assert torch.equal(got, po.erosion_ones((inp['frontw'] > 0.5).float(), e)), e
    ro, rd = pp.occlusion_rays(inp['image_xyz'].to(DEV), 0.5, 0.01)
    o_ro, o_rd = po.occlusion_rays(inp['image_xyz'], 0.5, 0.01)
    assert torch.equal(ro.cpu(), o_ro) and torch.equal(rd.cpu(), o_rd)


def test_full_size_properties():
    """Eval size (8 views, 128^2 render, 512^2 image): size-independent properties instead of an oracle run."""
    import panic3d_b200.paste as pp
    inp = po.synth_paste_inputs(21, 8, 128, 512)
    d = {k: v.to(DEV) for k, v in inp.items() if torch.is_tensor(v)}
    eroded = pp.erode_front_weights(d['frontw'], 3)
    with torch.no_grad():
        img, paste, mask, parts = pp.paste_front_fused(d['image'], d['image_xyz'], d['image_weights'], d['front_rgb'], d['occ'], d['ro'],
                                                      d['rd'], 0.7, front_eroded=eroded, thresh_dxyz=5e-6)
        img2, paste2, mask2, none = pp.paste_front_fused(d['image'], d['image_xyz'], d['image_weights'], d['front_rgb'], d['occ'], d['ro'],
                                                        d['rd'], 0.7, front_eroded=eroded, thresh_dxyz=5e-6, want_parts=False)
    assert none is None and torch.equal(img, img2) and torch.equal(paste, paste2) and torch.equal(mask, mask2)   # deterministic
    assert torch.equal(mask, parts[0] * parts[1] * parts[2] * parts[3] * parts[4])
    assert 0.02 < mask.mean().item() < 0.9 and mask.min().item() >= 0 and mask.max().item() <= 1
    m3 = mask.expand(-1, 3, -1, -1)
    assert torch.equal(img[m3 == 0], d['image'][m3 == 0])                          # untouched where the mask is 0
    assert torch.equal(img[m3 == 1], paste[m3 == 1])                               # the front image where it is 1
    lo, hi = torch.minimum(d['image'], paste), torch.maximum(d['image'], paste)
    assert bool(((img >= lo - 1e-6) & (img <= hi + 1e-6)).all())                   # a blend in between
    assert paste.min().item() >= 0 and paste.max().item() <= 1                     # convex combination of front-image texels
    for k in (0, 1, 3):
        assert set(parts[k].unique().tolist()) <= {0.0, 1.0}
    # pasting twice changes nothing where the mask is binary: lerp(lerp(a, p, m), p, m) = lerp(a, p, m) for m in {0, 1}
    with torch.no_grad():
        again = pp.paste_front_fused(img, d['image_xyz'], d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], 0.7,
                                     front_eroded=eroded, thresh_dxyz=5e-6, want_parts=False)[0]
    binary = (m3 == 0) | (m3 == 1)
    assert torch.equal(again[binary], img[binary])


@pytest.mark.parametrize('grad_sample', [False, True])
def test_gradients_match_oracle_autograd(grad_sample):
    import panic3d_b200.paste as pp
    case = PASTE_CASES['defaults_erode3']
    inp = build_paste_inputs(case)
    g = torch.Generator().manual_seed(3)
    g_img, g_paste = torch.randn(inp['image'].shape, generator=g), torch.randn(inp['image'].shape, generator=g)
    # oracle: torch autograd through the restated ops (masks under no_grad, like the reference)
    image, xyz = inp['image'].clone().requires_grad_(True), inp['image_xyz'].clone().requires_grad_(True)
    o = po.paste_front(image, xyz if grad_sample else xyz.detach(), inp['image_weights'], inp['front_rgb'], inp['occ'], inp['ro'], inp['rd'],
                       inp['box_warp'], frontw=inp['frontw'], front_weight_erosion=3)
    loss = (o['image'] * g_img).sum() + ((o['paste'] * g_paste).sum() if grad_sample else 0)
    loss.backward()
    # ours
    d = {k: v.to(DEV) for k, v in inp.items() if torch.is_tensor(v)}
    image2, xyz2 = d['image'].clone().requires_grad_(True), d['image_xyz'].clone().requires_grad_(True)
    eroded = pp.erode_front_weights(d['frontw'], 3)
    img, paste, mask, _ = pp.paste_front_fused(image2, xyz2, d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], inp['box_warp'],
                                              front_eroded=eroded, grad_sample=grad_sample)
    loss2 = (img * g_img.to(DEV)).sum() + ((paste * g_paste.to(DEV)).sum() if grad_sample else 0)
    loss2.backward()
    assert (image2.grad.cpu() - image.grad).abs().max().item() < 1e-5
    if grad_sample:
        ref = xyz.grad
        assert ref.abs().max().item() > 1.0 and bool((ref[:, 2] == 0).all())
        err = (xyz2.grad.cpu() - ref).abs().max().item()
        assert err < 2e-3 * ref.abs().max().item(), (err, ref.abs().max().item())
        assert bool((xyz2.grad[:, 2] == 0).all())
    else:
        assert xyz2.grad is None and xyz.grad is None
    with pytest.raises(RuntimeError):                                              # hand-written first-order backward
        image3 = d['image'].clone().requires_grad_(True)
        out = pp.paste_front_fused(image3, d['image_xyz'], d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], 0.7)[0]
        (gi,) = torch.autograd.grad(out.sum(), image3, create_graph=True)
        gi.sum().backward()


def test_reuse_triplane_renders_the_occlusion_pass_from_the_views_planes():
    """Opt-in route of get_front_occlusion: G.renderer on out['triplane'] instead of a second G.f."""
    import panic3d_b200.paste as pp
    inp = po.synth_paste_inputs(9, 2, 12, 24)
    calls = {}

    class G:
        rendering_kwargs = {'ray_start': 0.5, 'box_warp': 0.7}
        decoder = object()

        @staticmethod
        def renderer(planes, decoder, ro, rd, opts, **flags):
            calls.update(planes=planes, ro=ro, rd=rd, flags=flags)
            n, m, _ = ro.shape
            return None, None, torch.arange(n * m, device=ro.device, dtype=torch.float32).reshape(n, m, 1), None

        @staticmethod
        def f(*a, **k):
            raise AssertionError('G.f must not be called when the tri-planes are reused')

    out = {'image_xyz': inp['image_xyz'].to(DEV), 'triplane': torch.zeros(2, 3, 32, 8, 8, device=DEV)}
    pp.REUSE_TRIPLANE = True
    try:
        w = pp.get_front_occlusion(G, {'triplane_crop': 0.1, 'cull_clouds': 0.5}, out, offset=0.01)
    finally:
        pp.REUSE_TRIPLANE = False
    o_ro, o_rd = po.occlusion_rays(inp['image_xyz'], 0.5, 0.01)
    assert torch.equal(calls['ro'].cpu(), o_ro.permute(0, 2, 3, 1).reshape(2, 144, 3)) and torch.equal(calls['rd'].cpu(), o_rd.permute(0, 2, 3, 1).reshape(2, 144, 3))
    assert calls['planes'] is out['triplane'] and calls['flags'] == {'triplane_crop': 0.1, 'cull_clouds': 0.5, 'binarize_clouds': None}
    assert tuple(w.shape) == (2, 1, 12, 12) and torch.equal(w.flatten().cpu(), torch.arange(288, dtype=torch.float32))
