"""GPU: p3d_volume_query (through panic3d_b200.volume) against the reference fixtures, the oracle, and run_model."""
import numpy as np
import pytest
import torch

from oracle import volume_oracle as vo
from tests.golden.cases import VOLUME_CASES, build_case_inputs
from tests.helpers import load_golden
from tests.render_abi import make_decoder

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _query(case, **kw):
    import panic3d_b200.volume as pv
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    planes, dec, _, _, _, _, opts = build_case_inputs(case)
    r = ImportanceRenderer(use_triplane=case.get('use_triplane', True))
    out = pv.query_volume(planes.to(DEV), make_decoder(dec, DEV), opts, resolution=case['res'], triplane_crop=case.get('triplane_crop'),
                          cull_clouds=case.get('cull_clouds'), renderer=r, **kw)
    torch.cuda.synchronize()
    return out, (planes, dec, opts)


@pytest.mark.parametrize('name', sorted(VOLUME_CASES))
def test_volume_matches_reference_fixture(name):
    g = load_golden('volume', name)
    out, _ = _query(g['case'])
    assert torch.equal(out['coordinates'].cpu(), g['coordinates'])                # sheared lattice + flip, bit for bit
    for key in ('sigmas', 'rgbs'):
        assert out[key].shape == g[key].shape
        assert (out[key].cpu() - g[key]).abs().max().item() < 1e-4, key
    d, dg = out['densities'].cpu(), g['densities']
    agree = ((d == -1e3) == (dg == -1e3)).float().mean().item()
    assert agree > 0.999, agree                                                   # a threshold flip needs |alpha - thr| < 1e-6
    keep = (d != -1e3) & (dg != -1e3)
    assert (d[keep] - dg[keep]).abs().max().item() < 1e-4
    assert out.sigmas is out['sigmas']                                            # attribute access like addict.Dict


def test_volume_equals_run_model_on_the_same_lattice_at_64_cubed():
    """Property at a size the CPU oracle does not need to touch: the fused launch (in-kernel lattice, flipped writes)
    equals ImportanceRenderer.run_model fed with create_samples, re-shaped the reference's way."""
    import panic3d_b200.volume as pv
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = dict(VOLUME_CASES['vol_plain13'], res=64, P=128, seed=77)
    out, (planes, dec, opts) = _query(case)
    R = 64
    samples, _, _ = pv.create_samples(R, cube_length=opts['box_warp'])
    r = ImportanceRenderer(use_triplane=True)
    with torch.no_grad():
        pts = r.run_model(planes.to(DEV), make_decoder(dec, DEV), samples.to(DEV), None, opts)

    def shape(t, c):
        return t.reshape(1, R, R, R, c).flip(dims=(1,)).permute(0, 4, 1, 2, 3)
    assert torch.equal(out['sigmas'], shape(pts['sigma'], 1))
    assert torch.equal(out['rgbs'], shape(pts['rgb'], 32))
    assert torch.equal(out['coordinates'].cpu(), shape(samples, 3))
    assert (out['densities'] - pv.sigma2density(out['sigmas'])).abs().max().item() < 1e-6


def test_volume_optional_outputs_multi_subject_and_errors():
    import panic3d_b200.volume as pv
    case = dict(VOLUME_CASES['vol_plain13'], N=2, res=9)
    out, _ = _query(case, want_rgb=False, want_coordinates=False)
    assert out['rgbs'] is None and out['coordinates'] is None and out['sigmas'].shape == (2, 1, 9, 9, 9)
    planes, dec, _, _, _, _, opts = build_case_inputs(case)
    for i in range(2):                                                            # subject i of the pair = its own single-subject query
        one = pv.query_volume(planes[i:i + 1].to(DEV), make_decoder(dec, DEV), opts, resolution=9)
        assert torch.equal(out['sigmas'][i:i + 1], one['sigmas'])
        assert torch.equal(out['densities'][i:i + 1], one['densities'])
    with pytest.raises(RuntimeError, match='resolution'):
        pv.query_volume(planes.to(DEV), make_decoder(dec, DEV), opts, resolution=1)


def test_get_eg3d_volume_drop_in_runs_backbone_once():
    """get_eg3d_volume(G, xin) on a stand-in generator: f() resolves ws, the backbone is asked for planes exactly once."""
    import panic3d_b200.volume as pv
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = VOLUME_CASES['vol_crop_cull16']
    planes, dec, _, _, _, _, opts = build_case_inputs(case)
    calls = []

    class Backbone:
        def synthesis(self, ws, cond, update_emas=False, **kw):
            calls.append(kw)
            return planes.to(DEV).reshape(1, 96, planes.shape[-2], planes.shape[-1])

    class G(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.decoder = make_decoder(dec, DEV)
            self.backbone, self.renderer = Backbone(), ImportanceRenderer(use_triplane=True)
            self.triplane_width, self.rendering_kwargs = 32, opts

        def f(self, xin):
            xin['ws'] = torch.zeros(1, 14, 512, device=DEV)
    vol = pv.get_eg3d_volume(G(), {'cond': None, 'triplane_crop': case['triplane_crop'], 'cull_clouds': case['cull_clouds']},
                             resolution=case['res'])
    assert len(calls) == 1 and calls[0] == {'noise_mode': 'const'}
    g = load_golden('volume', 'vol_crop_cull16')
    assert (vol.sigmas.cpu() - g['sigmas']).abs().max().item() < 1e-4
    assert (((vol.densities.cpu() == -1e3) == (g['densities'] == -1e3)).float().mean().item()) > 0.999
