"""GPU: p3d_mc_count / p3d_mc_emit (through panic3d_b200.mesh) against the numpy oracle, the colour route of extract_mesh
against the colour volume, the drop-ins, a full-size sphere and the error paths."""
import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from tests import mesh_fields as mf
from tests.golden.cases import VOLUME_CASES, build_case_inputs
from tests.render_abi import make_decoder

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _query(case, res, **kw):
    import panic3d_b200.volume as pv
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    planes, dec, _, _, _, _, opts = build_case_inputs(case)
    r = ImportanceRenderer(use_triplane=case.get('use_triplane', True))
    args = (planes.to(DEV), make_decoder(dec, DEV), opts)
    kw = dict(resolution=res, triplane_crop=case.get('triplane_crop'), cull_clouds=case.get('cull_clouds'), renderer=r, **kw)
    return pv.query_volume(*args, **kw), args, kw


def _fields():
    out = {'sphere48': mf.sphere(48, 20.0), 'torus48': mf.torus(48), 'noise24': mf.noise(24, seed=3),
           'sphere_uneven': mf.sphere(48, 20.0)[3:40, :29, 5:]}
    return out


def _check_against_oracle(v, level=0.5):
    import panic3d_b200.mesh as pm
    d = torch.from_numpy(v).to(DEV)
    m = pm.mesh_index(d, level)
    m2 = pm.mesh_index(d, level)
    ours = {k: t.cpu().numpy() for k, t in m.items()}
    for k in ours:                                                                    # deterministic order: bit-identical calls
        assert np.array_equal(ours[k], m2[k].cpu().numpy()), k
    ref = mo.marching_cubes_index(v, level)
    assert len(ours['verts']) > 0 and len(ref['faces']) > 0
    assert np.array_equal(_bits(ours['verts']), _bits(ref['verts']))
    assert np.array_equal(_bits(ours['values']), _bits(ref['values']))
    assert np.array_equal(ours['floor_node'], ref['floor_node'])
    assert np.abs(ours['normals'] - ref['normals']).max() < 1e-5
    assert np.array_equal(mo.canonical_faces(ours['faces']), mo.canonical_faces(ref['faces']))
    assert np.array_equal(ours['faces'], ref['faces'])                                # the stated triangle order, too
    return ours


@pytest.mark.parametrize('name', sorted(_fields()))
def test_kernel_equals_oracle_on_analytic_and_noise_fields(name):
    _check_against_oracle(_fields()[name])


@pytest.mark.parametrize('name', sorted(VOLUME_CASES))
def test_kernel_equals_oracle_on_query_volume_densities_at_64_cubed(name):
    case = VOLUME_CASES[name]
    vol, _, _ = _query(case, 64, want_rgb=False, want_coordinates=False)
    dens = vol['densities'][0, 0].cpu().numpy()
    assert (dens == -1e3).any() or name == 'vol_plain13'                             # crop / cull overwrites next to the surface
    # the random decoders of the other two cases never reach density 0.5: mesh them at the median of the kept densities
    level = 0.5 if name == 'vol_crop_cull16' else float(np.median(dens[dens != -1e3]))
    _check_against_oracle(dens, level)


def test_extract_mesh_colours_equal_the_colour_volume_bit_for_bit():
    import panic3d_b200.mesh as pm
    from panic3d_b200 import _lib
    case = VOLUME_CASES['vol_crop_cull16']
    vol, args, kw = _query(case, 64)
    n0 = _lib.launch_count()
    got = pm.extract_mesh(*args, **kw)
    assert _lib.launch_count() - n0 >= 6                                              # volume, count, scan (2), emit, lattice, decode
    want = pm.marching_cubes(vol['densities'][0, 0], vol['rgbs'][0, :3], args[2]['box_warp'])
    assert len(got['verts']) > 100
    for k in ('verts', 'faces', 'normals', 'values'):
        assert np.array_equal(got[k], want[k]), k
    vi = pm.mesh_index(vol['densities'][0, 0])['floor_node'].cpu().numpy()
    a, b, c = np.unravel_index(vi, (64, 64, 64))
    ref = vol['rgbs'][0, :3].cpu().numpy()[:, a, b, c].T
    assert got['colors'].dtype == np.float32 and np.array_equal(_bits(got['colors']), _bits(ref))
    assert np.array_equal(_bits(want['colors']), _bits(ref))


def test_marching_cubes_numpy_equals_cuda_tensors_and_returns_the_reference_dict():
    import panic3d_b200.mesh as pm
    v = mf.sphere(32, 12.0)
    rgbs = np.random.default_rng(2).random((3, 32, 32, 32), dtype=np.float32)
    a = pm.marching_cubes(v, rgbs, 0.7)
    b = pm.marching_cubes(torch.from_numpy(v).to(DEV), torch.from_numpy(rgbs).to(DEV), 0.7)
    assert sorted(a) == ['colors', 'faces', 'normals', 'values', 'verts'] and a.verts is a['verts']
    for k in a:
        assert isinstance(a[k], np.ndarray) and a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), k
    assert a['faces'].dtype == np.int32 and a['verts'].dtype == np.float32
    ref = mo.marching_cubes(v, rgbs, 0.7)
    for k in ('verts', 'values', 'colors'):
        assert np.array_equal(a[k], ref[k]), k
    empty = pm.marching_cubes(np.zeros((5, 5, 5), np.float32), np.zeros((3, 5, 5, 5), np.float32), 0.7)
    assert all(len(empty[k]) == 0 for k in empty) and empty['faces'].shape == (0, 3)


def test_get_eg3d_mesh_runs_the_backbone_once_and_equals_the_two_step_route():
    import panic3d_b200.mesh as pm
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
    xin = {'cond': None, 'triplane_crop': case['triplane_crop'], 'cull_clouds': case['cull_clouds']}
    mesh = pm.get_eg3d_mesh(G(), xin, resolution=40)
    assert len(calls) == 1 and calls[0] == {'noise_mode': 'const'}
    vol = pv.get_eg3d_volume(G(), xin, resolution=40)
    want = pm.marching_cubes(vol['densities'].cpu().numpy()[0, 0], vol['rgbs'].cpu().numpy()[0, :3], opts['box_warp'], level=0.5)
    assert len(mesh['faces']) > 0
    for k in want:
        assert np.array_equal(mesh[k], want[k]), k


def test_full_size_sphere_is_closed_with_area_and_normals():
    import panic3d_b200.mesh as pm
    r = 100.0
    v = torch.from_numpy(mf.sphere(256, r)).to(DEV)
    m = {k: t.cpu().numpy() for k, t in pm.mesh_index(v).items()}
    f, p = m['faces'], m['verts']
    assert len(f) > 100000
    assert mo.is_closed_oriented(f)
    assert mo.euler_characteristic(len(p), f) == 2
    area, vol = mo.area_and_volume(p, f)
    assert abs(area / (4 * np.pi * r * r) - 1) < 0.015 and vol > 0
    q = p.astype(np.float64)[f]
    fn = np.cross(q[:, 1] - q[:, 0], q[:, 2] - q[:, 0])
    vn = m['normals'].astype(np.float64)[f].mean(axis=1)
    assert ((fn * vn).sum(1) > 0).mean() >= 0.99


def test_errors():
    import panic3d_b200.mesh as pm
    rgbs = np.zeros((3, 4, 4, 4), np.float32)
    with pytest.raises(RuntimeError, match='CPU'):
        pm.marching_cubes(torch.zeros(4, 4, 4), rgbs, 0.7)
    with pytest.raises(RuntimeError, match='D0'):
        pm.marching_cubes(torch.zeros(4, 4, 4, 4, device=DEV), rgbs, 0.7)
    with pytest.raises(RuntimeError, match='>= 2'):
        pm.mesh_index(torch.zeros(4, 1, 4, device=DEV))
    with pytest.raises(RuntimeError, match='float32'):
        pm.mesh_index(torch.zeros(4, 4, 4, device=DEV, dtype=torch.float64))
    with pytest.raises(RuntimeError, match='rgbs'):
        pm.marching_cubes(np.zeros((4, 4, 4), np.float32), np.zeros((3, 4, 4, 5), np.float32), 0.7)
