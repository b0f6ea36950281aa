"""GPU: marching cubes (p3d_mc_count / CUB scan / p3d_mc_emit) through the C ABI at the eval size and on the volumes where
it can go wrong, against the table oracle (oracle/mesh_oracle.py) and against checks that use no oracle.

Every case: the kernel writes into oversized outputs prefilled with a sentinel (NaN floats, -7 integers) - rows [0, V) /
[0, F) all written, the guard rows after them untouched, two runs (count and emit) bit-identical, and an emit without
normals / values / floor nodes gives the same verts and faces.  Against the table oracle: verts, values, floor nodes and
faces (in order) bit-equal, normals within 1e-5.  Without the oracle:
  * closure: vertices with bit-identical positions merged, no triangle repeats a merged vertex and every undirected
    merged edge is used equally often in each direction unless both its ends lie in one volume-border plane.  This is
    the boundary-of-a-2-chain condition: it allows the edges two cells both fan across on a shared ambiguous face (two
    uses per direction) and it survives degenerate removal, since a dropped triangle has two merged-equal corners and
    contributes one use in each direction;
  * every vertex no triangle uses shares its position with another vertex or lies within one cell (max norm) of a
    position two vertices share: a triangle whose other two corners coincide is dropped, so a vertex all of whose
    triangles are like that is left unused (the zoo and ties256 have such vertices).  With no degenerate triangle
    dropped, every vertex is used;
  * each vertex lies on a sign-change lattice edge of the volume, in order, within the bar of its four fp32 roundings
    of the fp64 edge parameter (`_position_bar`);
  * on the smooth blob, the triangles face down the fp64 gradient.

Cases (each restated here: no bench module is imported):
  eval256     query_volume densities at 256^3 with the eval's crop 0.1 and cull 0.5, planes and decoder of bench_mesh.py's
              extract_mesh workload (vol_crop_cull16's decoder, seed 7, 512^2 planes) with a sigma bias that saturates
              the density (EVAL_SIGMA_BIAS).  Every vertex is a cliff next to a -1e3 node, at indices up to 255
  blob256     bench_mesh.py's seeded head-sized blob at 256^3; closed with Euler characteristic 2 after merging
  ties256     blob256 quantised to k/8 (nodes and deciders exactly at the level), its slab a >= 128 turned into -1e3 next
              to values in (0.5, 0.51] (t rounding onto nodes): degenerate triangles dropped
  zoo         every (case, decisions) configuration, each in its own block (tests/mesh_fields.py zoo_volume)
  shapes      blob at 257^3 (more than 2^24 nodes); 2x2x4099 and 4099x2x2; 3x517x33 (rows of 33 nodes); a sphere cut by
              all six borders - the scan across CTAs, warps straddling rows, the border guards of vertex_id and grad_at
  checker9    {0, 1} by node parity: V = 3 n^2 (n - 1), F = 4 (n - 1)^3, every decider ties
  checker815  the same at 815^3: V = 1.62e9 fits int32, F = 4 * 814^3 >= 2^31 does not - mesh_index refuses with both
              counts and p3d_mc_emit writes nothing
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import mesh_oracle as mo
from tests import mesh_fields as mf
from tests.render_abi import make_decoder, skip_unless_free, twice

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
LEVEL = 0.5
GUARD = 4096                    # sentinel rows after each output
INT_SENTINEL = -7
U = 2.0 ** -24
# eval256's triangle floor: 628066 triangles (365828 vertices) on an H100 SXM, recorded with 20 % margin
EVAL_MIN_F = 500000


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


# ------------------------------------------------------------------------------------------------- the C ABI
def _abi(v):
    """p3d_mc_count then p3d_mc_emit on the (D0,D1,D2) volume v (numpy or CUDA tensor), twice, into sentinel-filled outputs
    with GUARD extra rows; then once more without the optional outputs.  Returns the outputs' [0, V) / [0, F) rows as
    numpy."""
    from panic3d_b200 import _lib
    L = _lib.lib()
    vol = (torch.from_numpy(np.ascontiguousarray(v)) if isinstance(v, np.ndarray) else v).to(DEV).contiguous()
    D0, D1, D2 = vol.shape
    nbytes = int(L.p3d_mc_workspace_bytes(D0, D1, D2))
    assert nbytes, L.p3d_last_error()
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    counts = torch.empty(2, dtype=torch.int64, device=DEV)
    st = _lib.stream_ptr(DEV)

    def count():
        _lib.check(L.p3d_mc_count(vol.data_ptr(), D0, D1, D2, C.c_float(LEVEL), ws.data_ptr(), nbytes, counts.data_ptr(), st))

    count()
    V, F = (int(x) for x in counts.tolist())
    verts = torch.empty((V + GUARD, 3), device=DEV)
    faces = torch.empty((F + GUARD, 3), dtype=torch.int32, device=DEV)
    normals = torch.empty((V + GUARD, 3), device=DEV)
    values = torch.empty((V + GUARD,), device=DEV)
    floor = torch.empty((V + GUARD,), dtype=torch.int64, device=DEV)
    outs = [verts, faces, normals, values, floor]

    def emit(optional):
        _lib.check(L.p3d_mc_emit(vol.data_ptr(), D0, D1, D2, C.c_float(LEVEL), ws.data_ptr(), nbytes, verts.data_ptr(),
                                 faces.data_ptr(), *[t.data_ptr() if optional else None for t in (normals, values, floor)], st))

    first, second = twice(lambda: (count(), emit(True)), outs, checks_later=True, int_fill=INT_SENTINEL)
    assert counts.tolist() == [V, F]
    names = ('verts', 'faces', 'normals', 'values', 'floor_node')
    rows = (V, F, V, V, V)
    out = {}
    for name, n, a, b in zip(names, rows, first, second):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        assert np.array_equal(_bits(a), _bits(b)), f'two runs differ in {name}'
        unwritten = np.isnan(a) if a.dtype.kind == 'f' else a == INT_SENTINEL
        assert not unwritten[:n].any(), f'{name}: {int(unwritten[:n].sum())} of its first {n} elements never written'
        assert unwritten[n:].all(), f'{name}: written past row {n}'
        out[name] = a[:n]
    twice(lambda: emit(False), [verts, faces], checks_later=True, int_fill=INT_SENTINEL)
    assert np.array_equal(_bits(verts[:V].cpu().numpy()), _bits(out['verts'])), 'verts differ without the optional outputs'
    assert np.array_equal(faces[:F].cpu().numpy(), out['faces']), 'faces differ without the optional outputs'
    assert np.isnan(verts[V:].cpu().numpy()).all() and (faces[F:].cpu().numpy() == INT_SENTINEL).all()
    return out


# ------------------------------------------------------------------------------------------------- checks without the oracle
def _sign_change_edges(v):
    """(lower node (V,3) int64, axis (V,)) of every lattice edge whose end nodes straddle the level, in (flat node, axis)
    order - the order the vertices must come in."""
    inside = v > np.float32(LEVEL)
    nodes, axes, keys = [], [], []
    for ax in range(3):
        n = inside.shape[ax] - 1
        lo = np.argwhere(np.take(inside, range(n), ax) != np.take(inside, range(1, n + 1), ax))
        nodes.append(lo)
        axes.append(np.full(len(lo), ax))
        keys.append(np.ravel_multi_index(lo.T, v.shape) * 3 + ax)
    order = np.argsort(np.concatenate(keys), kind='stable')
    return np.concatenate(nodes)[order].astype(np.int64), np.concatenate(axes)[order]


def _position_bar(lo, t64):
    """Bound on |p - (lo + t)| for the kernel's p = fl(lo + fl(fl(level - v_lo) / fl(v_hi - v_lo))) against the exact
    t = (level - v_lo) / (v_hi - v_lo) (fp64, exact to 2^-53 from the fp32 inputs).  Each fl is one round to nearest,
    relative error <= u = 2^-24: the two differences and the quotient give t (1 + e1)(1 + e3) / (1 + e2), off by at most
    t ((1 + u)^2 / (1 - u) - 1) <= 3.0001 u t (0 <= t <= 1); the add then errs by at most u |lo + t~|.  Total
    u (lo + t) + 3.0001 u t (1 + u) <= u (lo + 4.0002 t), plus 1e-12 for the fp64 reference."""
    return U * (lo + 4.0002 * t64) + 1e-12


def _merge(verts):
    """Merged id of every vertex (bit-identical positions share one) and the merged positions."""
    uniq, inv = np.unique(_bits(verts), axis=0, return_inverse=True)
    return inv.reshape(-1), uniq.view(np.float32)


def _check_positions(v, m):
    """Vertices on their sign-change lattice edges, in order, within `_position_bar` of the fp64 edge point.  Returns the
    distance of each vertex from the nearer end node of its edge."""
    node, ax = _sign_change_edges(v)
    p = m['verts']
    assert len(p) == len(node), (len(p), len(node))
    V = len(p)
    other = np.ones((V, 3), dtype=bool)
    other[np.arange(V), ax] = False
    assert np.array_equal(p[other], node[other].astype(np.float32)), 'a vertex is off its lattice edge'
    hi = node.copy()
    hi[np.arange(V), ax] += 1
    vlo = v[tuple(node.T)].astype(np.float64)
    vhi = v[tuple(hi.T)].astype(np.float64)
    assert np.all((vlo > LEVEL) != (vhi > LEVEL))
    t64 = (LEVEL - vlo) / (vhi - vlo)
    lo = node[np.arange(V), ax].astype(np.float64)
    pa = p[np.arange(V), ax].astype(np.float64)
    assert np.all((pa >= lo) & (pa <= lo + 1)), 'a vertex outside its lattice edge'
    err = np.abs(pa - (lo + t64))
    worst = (err / _position_bar(lo, t64)).max()
    assert worst <= 1.0, worst
    return np.minimum(pa - lo, lo + 1 - pa)


def _check_closure(v, m):
    """The closure and unreferenced-vertex checks of the module docstring.  Returns the number of merged vertices and
    the number of unused vertices with a position of their own."""
    f = m['faces'].astype(np.int64)
    inv, P = _merge(m['verts'])
    mf_ = inv[f]
    assert np.all((mf_[:, 0] != mf_[:, 1]) & (mf_[:, 1] != mf_[:, 2]) & (mf_[:, 0] != mf_[:, 2])), 'a degenerate triangle'
    d = np.concatenate([mf_[:, [0, 1]], mf_[:, [1, 2]], mf_[:, [2, 0]]])
    a, b = d.min(1), d.max(1)
    key, kinv = np.unique(a * len(P) + b, return_inverse=True)
    fwd = np.bincount(kinv, weights=d[:, 0] < d[:, 1], minlength=len(key))
    bwd = np.bincount(kinv, weights=d[:, 0] > d[:, 1], minlength=len(key))
    bad = np.flatnonzero(fwd != bwd)
    ea, eb = P[key[bad] // len(P)], P[key[bad] % len(P)]
    top = np.array(v.shape, dtype=np.float32) - 1
    border = (((ea == 0) & (eb == 0)) | ((ea == top) & (eb == top))).any(1)
    assert border.all(), f'{int((~border).sum())} interior edges used unequally in the two directions, e.g. {ea[~border][:3]}'
    used = np.zeros(len(m['verts']), dtype=bool)
    used[f.reshape(-1)] = True
    mult = np.bincount(inv, minlength=len(P))
    lone = ~used & (mult[inv] < 2)
    if lone.any():
        dist, _ = cKDTree(P[mult >= 2]).query(m['verts'][lone], p=np.inf)
        assert np.all(dist <= 1), 'an unused vertex with a position of its own, away from every shared position'
    return len(P), int(lone.sum())


def _check_facing(v, m, share=0.99):
    """At least `share` of the triangles have a right-hand normal with a positive dot product with the negated fp64
    gradient at their centroid (central differences at the nodes, one-sided at the border, trilinear in between)."""
    q = m['verts'].astype(np.float64)[m['faces']]
    n = np.cross(q[:, 1] - q[:, 0], q[:, 2] - q[:, 0])
    cen = q.mean(1)
    v64 = v.astype(np.float64)
    D = np.array(v.shape)
    base = np.minimum(np.floor(cen).astype(np.int64), D - 2)
    w = cen - base
    g = np.zeros_like(cen)
    for k, off in enumerate(mo.CORNER_OFFSETS):
        node = base + off
        wk = np.prod(np.where(np.array(off) == 1, w, 1 - w), axis=1)
        for ax in range(3):
            up, dn = node.copy(), node.copy()
            up[:, ax] = np.minimum(node[:, ax] + 1, D[ax] - 1)
            dn[:, ax] = np.maximum(node[:, ax] - 1, 0)
            g[:, ax] += wk * (v64[tuple(up.T)] - v64[tuple(dn.T)]) / (up[:, ax] - dn[:, ax])
    frac = ((n * -g).sum(1) > 0).mean()
    assert frac >= share, frac
    return frac


def _run(name, v, smooth=False):
    """The kernel through the ABI against the table oracle and the oracle-free checks; prints and returns the case's
    figures."""
    t0 = time.time()
    m = _abi(v)
    t1 = time.time()
    ref = mo.marching_cubes_index(v, LEVEL)
    for k in ('verts', 'values', 'floor_node', 'faces'):
        assert np.array_equal(_bits(m[k]), _bits(ref[k])), k
    assert np.abs(m['normals'] - ref['normals']).max() < 1e-5
    t2 = time.time()
    near = _check_positions(v, m)
    merged, lone = _check_closure(v, m)
    stats = dict(V=len(m['verts']), F=len(m['faces']), dropped=mo.fan_triangles(v, LEVEL) - len(m['faces']),
                 cliffs=int((near < 1e-3).sum()), merged=merged, lone=lone)
    assert lone == 0 or stats['dropped'] > 0
    if smooth:
        stats['facing'] = _check_facing(v, m)
    print(f'{name} {tuple(v.shape)}: {stats}; kernel {t1 - t0:.1f} s, oracle {t2 - t1:.1f} s, checks {time.time() - t2:.1f} s')
    return m, stats


# ------------------------------------------------------------------------------------------------- cases
def test_zoo():
    v, where = mf.zoo_volume()
    _, st = _run('zoo', v)
    assert len(where) == 656 and st['dropped'] > 0


@pytest.mark.parametrize('n', [9])
def test_checker(n):
    m, st = _run(f'checker{n}', mf.checkerboard(n))
    assert st['V'] == 3 * n * n * (n - 1) and st['F'] == 4 * (n - 1) ** 3 and st['dropped'] == 0


SHAPES = {'border_sphere20': lambda: mf.sphere(20, 12.0),                # inside touches all six borders
          'rows2x2x4099': lambda: mf.noise((2, 2, 4099), seed=11),
          'cols4099x2x2': lambda: mf.noise((4099, 2, 2), seed=12),
          'odd3x517x33': lambda: mf.noise((3, 517, 33), seed=13),
          'blob257': lambda: mf.blob(257)}


@pytest.mark.parametrize('name', list(SHAPES))
def test_shapes(name):
    v = SHAPES[name]()
    if name == 'border_sphere20':
        assert (v[[0, -1]] > LEVEL).any() and (v[:, [0, -1]] > LEVEL).any() and (v[..., [0, -1]] > LEVEL).any()
    _, st = _run(name, v, smooth=name == 'blob257')
    assert st['F'] > 0


def test_ties256():
    v = mf.cliffs(mf.quantised(mf.blob(256)), 128)
    assert (v == LEVEL).any()
    _, st = _run('ties256', v)
    assert st['dropped'] >= 1 and st['cliffs'] > 0


def test_blob256():
    """The blob has one node exactly at the level, so 4 fan triangles are dropped and a few vertices coincide: closed,
    oriented and of Euler characteristic 2 once they are merged."""
    m, st = _run('blob256', mf.blob(256), smooth=True)
    inv, P = _merge(m['verts'])
    f = inv[m['faces']]
    assert mo.is_closed_oriented(f) and mo.euler_characteristic(len(P), f) == 2


# The eval's cull 0.5 runs on the density as if it were a sigma (eg3d_metrics3d.py:160-162): it keeps a node only when
# 1 - exp(-softplus(density - 1)) >= 0.5, i.e. when its density rounds to within 2 ulp of 1.  bench_mesh.py's decoder (sigma
# bias 1.5, sigma <= 3.3) never saturates, so its eval mesh is empty; a sigma bias of 17 saturates most of the uncropped
# box and leaves holes where sigma < ~18.3.
EVAL_SIGMA_BIAS = 17.0


def _eval_inputs():
    """bench_mesh.py's extract_mesh workload - vol_crop_cull16's decoder, seed 7, 512^2 planes - with sigma bias
    EVAL_SIGMA_BIAS, and the eval's crop 0.1 and cull 0.5 (bench.py's volume query)."""
    from oracle import renderer_oracle as orc
    from tests.golden.cases import VOLUME_CASES
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    case = VOLUME_CASES['vol_crop_cull16']
    planes, dec, *_ = orc.synth_inputs(7, 1, 1, 2, 0, 512, cameras=None)
    dec = dict(dec, lr_mul=1.0, force_sigmoid=False)
    dec['b2'] = dec['b2'].clone()
    dec['b2'][0] += EVAL_SIGMA_BIAS
    kw = dict(resolution=256, triplane_crop=0.1, cull_clouds=0.5, renderer=ImportanceRenderer(use_triplane=True))
    return planes.to(DEV), make_decoder(dec, DEV), dict(case['opts']), kw


def test_eval256():
    import panic3d_b200.volume as pv
    planes, dec, opts, kw = _eval_inputs()
    with torch.no_grad():
        dens = pv.query_volume(planes, dec, opts, want_rgb=False, want_coordinates=False, **kw)['densities'][0, 0]
    v = dens.cpu().numpy()
    kept = v[v != -1e3]
    assert kept.size and kept.min() >= np.float32(1 - 2 ** -23)
    _, st = _run('eval256', v)
    assert st['F'] >= EVAL_MIN_F
    # every vertex lies at t = 1000.5 / 1001 ~ 1 - 5e-4 from a culled node towards a kept one: within 1e-3 of a node, but
    # never rounded onto it, and no node is at the level - the eval's densities drop no degenerate triangle (ties256
    # carries that branch)
    assert st['cliffs'] == st['V'] and st['dropped'] == 0


def test_extract_mesh_colours_at_256():
    """extract_mesh with the eval's flags: its colours equal query_volume's colour volume at the floor nodes bit for bit,
    so k_mc_lattice maps floor nodes over the whole 256^3 index range."""
    import panic3d_b200.mesh as pm
    import panic3d_b200.volume as pv
    planes, dec, opts, kw = _eval_inputs()
    with torch.no_grad():
        got = pm.extract_mesh(planes, dec, opts, **kw)
        vol = pv.query_volume(planes, dec, opts, want_coordinates=False, **kw)
        fl = pm.mesh_index(vol['densities'][0, 0])['floor_node'].cpu().numpy()
        a, b, c = np.unravel_index(fl, (256, 256, 256))
        ref = vol['rgbs'][0, :3, torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV), torch.from_numpy(c).to(DEV)].T.cpu().numpy()
    assert len(got['verts']) == len(fl) > 1000 and a.max() > 200
    assert got['colors'].dtype == np.float32 and np.array_equal(_bits(got['colors']), _bits(ref))


def test_checker815_refuses_int32_overflow():
    """V = 3 * 815^2 * 814 < 2^31 but F = 4 * 814^3 >= 2^31: mesh_index raises with both exact counts, and p3d_mc_emit on
    the same workspace writes nothing into sentinel buffers."""
    from panic3d_b200 import _lib
    import panic3d_b200.mesh as pm
    n = 815
    skip_unless_free(8 << 30)
    V, F = 3 * n * n * (n - 1), 4 * (n - 1) ** 3
    assert V < 2 ** 31 <= F
    i = torch.arange(n, device=DEV)
    vol = ((i[:, None, None] + i[None, :, None] + i[None, None, :]) % 2).float()
    with pytest.raises(RuntimeError, match=f'{V} vertices / {F} triangles'):
        pm.mesh_index(vol)
    L = _lib.lib()
    nbytes = int(L.p3d_mc_workspace_bytes(n, n, n))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    counts = torch.empty(2, dtype=torch.int64, device=DEV)
    st = _lib.stream_ptr(DEV)
    _lib.check(L.p3d_mc_count(vol.data_ptr(), n, n, n, C.c_float(LEVEL), ws.data_ptr(), nbytes, counts.data_ptr(), st))
    assert counts.tolist() == [V, F]
    outs = [torch.full((GUARD, 3), float('nan'), device=DEV), torch.full((GUARD, 3), INT_SENTINEL, dtype=torch.int32, device=DEV),
            torch.full((GUARD, 3), float('nan'), device=DEV), torch.full((GUARD,), float('nan'), device=DEV),
            torch.full((GUARD,), INT_SENTINEL, dtype=torch.int64, device=DEV)]
    _lib.check(L.p3d_mc_emit(vol.data_ptr(), n, n, n, C.c_float(LEVEL), ws.data_ptr(), nbytes, *[t.data_ptr() for t in outs], st))
    torch.cuda.synchronize()
    for t in outs:
        assert (torch.isnan(t) if t.is_floating_point() else t == INT_SENTINEL).all()
