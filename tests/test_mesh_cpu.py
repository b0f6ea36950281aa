"""CPU: the marching-cubes rules of DESIGN.md section 2 on the numpy oracle (known answers, analytic fields, noise), the
oracle's configuration table against its per-cell walk, every configuration checked for closed loops and for agreement
with its neighbours across each face, the configuration zoo's coverage, the kernel's topology tables against the
oracle's derivation, the host-side scaling / colour lookup of panic3d_b200.mesh against the reference's own numpy
expressions, and the size guard of the C ABI."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import mesh_oracle as mo
from tests import mesh_fields as mf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cube(values):
    """2x2x2 volume from the 8 corner values, corner k at ((k >> 2) & 1, (k >> 1) & 1, k & 1)."""
    v = np.zeros((2, 2, 2), dtype=np.float32)
    for k, x in enumerate(values):
        v[(k >> 2) & 1, (k >> 1) & 1, k & 1] = x
    return v


def _tri_normals(m):
    p = m['verts'].astype(np.float64)[m['faces']]
    return np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), p.mean(axis=1)


def test_one_inside_corner_gives_one_outward_triangle():
    m = mo.marching_cubes_index(_cube([1, 0, 0, 0, 0, 0, 0, 0]))
    assert m['verts'].tolist() == [[0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.5]]          # node 0, axes 0, 1, 2
    assert m['faces'].tolist() == [[0, 1, 2]]
    n, _ = _tri_normals(m)
    assert np.allclose(n[0] / np.linalg.norm(n[0]), np.ones(3) / np.sqrt(3))        # away from the inside corner
    assert m['values'].tolist() == [1, 1, 1] and m['floor_node'].tolist() == [0, 0, 0]
    assert np.all(m['normals'] > 0)                                                   # descent: towards lower density
    # the opposite corner: the same triangle shape, normal towards -(1,1,1)
    m = mo.marching_cubes_index(_cube([0, 0, 0, 0, 0, 0, 0, 1]))
    n, _ = _tri_normals(m)
    assert len(m['faces']) == 1 and np.all(n[0] < 0)


@pytest.mark.parametrize('other, expect', [(0.2, 4), (-0.2, 2)])
def test_ambiguous_face_follows_the_decider(other, expect):
    """Corners 0 and 3 inside (diagonal on the face a = 0): s = (x^2 - y^2) / (2x - 2y) = (x + y) / 2 with x = 1, y = other.
    s > 0.5 connects them (a band of four triangles around a six-edge loop), otherwise two corner triangles."""
    v = _cube([1, other, other, 1, other, other, other, other])
    assert (mo.saddle(1, other, other, 1) > np.float32(0.5)) == (expect == 4)
    m = mo.marching_cubes_index(v)
    assert len(m['faces']) == expect
    n, centre = _tri_normals(m)
    inside = np.array([[0, 0, 0], [0, 1, 1]], dtype=np.float64)
    near = inside[np.argmin(((centre[:, None] - inside[None]) ** 2).sum(-1), axis=1)]
    if expect == 2:                                                                   # each triangle faces away from its corner
        assert np.all((n * (centre - near)).sum(1) > 0)
    else:                                                                             # the band faces away from the a-axis line
        axis_pt = np.stack([centre[:, 0], np.full(len(centre), 0.5), np.full(len(centre), 0.5)], 1)
        assert np.all((n * (centre - axis_pt)).sum(1) < 0) or np.all((n * (centre - axis_pt)).sum(1) > 0)


def test_level_node_drops_degenerate_triangles():
    """Corner 1 exactly at the level: the vertices of edges 0-1 (t = 1) and 1-3 (t = 0) coincide at node (0, 0, 1), and the
    one fan triangle holding both is dropped; nudging the corner below the level keeps all four."""
    m = mo.marching_cubes_index(_cube([1, 0.5, 0, 1, 0, 0, 0, 0]))
    pos = [tuple(p) for p in m['verts'].tolist()]
    assert pos.count((0.0, 0.0, 1.0)) == 2
    assert len(m['faces']) == 3
    for f in m['faces']:
        assert len({pos[i] for i in f}) == 3
    assert len(mo.marching_cubes_index(_cube([1, 0.49, 0, 1, 0, 0, 0, 0]))['faces']) == 4


def test_sphere_is_closed_with_euler_2_and_the_right_area():
    m = mo.marching_cubes_index(mf.sphere(48, 20.0))
    assert mo.is_closed_oriented(m['faces'])
    assert mo.euler_characteristic(len(m['verts']), m['faces']) == 2
    area, vol = mo.area_and_volume(m['verts'], m['faces'])
    assert abs(area / (4 * np.pi * 20.0 ** 2) - 1) < 0.03
    assert vol > 0                                                                    # outward winding


def test_torus_has_euler_0():
    m = mo.marching_cubes_index(mf.torus(48))
    assert mo.is_closed_oriented(m['faces'])
    assert mo.euler_characteristic(len(m['verts']), m['faces']) == 0


def test_noise_field_interior_edges_are_used_twice_and_both_decider_branches_run():
    """Away from the volume border every edge is used once in each direction.  The one exception the fan rule allows: two
    cells sharing an ambiguous face can both fan across the same pair of that face's vertices, so such a diagonal (both
    ends in one lattice plane) is used twice in each direction - the surface is still closed there."""
    v = mf.noise(24, seed=3)
    conn, sep = mf.ambiguous_face_decisions(v)
    assert conn > 50 and sep > 50
    m = mo.marching_cubes_index(v)
    use = mo.edge_use(m['faces'])
    P, D = m['verts'], np.array(v.shape) - 1
    shared = 0
    for (a, b), n in use.items():
        back = use.get((b, a), 0)
        if n == 1 and back == 1:
            continue
        if (((P[a] == 0) & (P[b] == 0)) | ((P[a] == D) & (P[b] == D))).any():
            continue                                                                  # open edge on the volume's border
        assert n == back == 2 and ((P[a] == P[b]) & (P[a] == np.round(P[a]))).any(), (a, b, n, back)
        shared += 1
    assert shared < 0.005 * len(use)


def test_kernel_topology_tables_match_the_oracle():
    src = open(os.path.join(ROOT, 'panic3d-anime-reconstruction_b200', 'csrc', 'marching_cubes.cu')).read()

    def table(name):
        body = re.search(name + r'(?:\[\d+\])+ = \{(.*?)\};', src, flags=re.S).group(1)
        return [int(x) for x in re.findall(r'\d+', body)]
    assert table('kEdgeCorner') == [k for k, _ in mo.EDGES]
    assert table('kEdgeAxis') == [ax for _, ax in mo.EDGES]
    assert table('kFaceCyc') == [q for cyc, _ in mo.FACES for q in cyc]
    assert table('kFaceEdge') == [mo._edge_between(cyc[k], cyc[(k + 1) % 4]) for cyc, _ in mo.FACES for k in range(4)]
    assert table('kFaceCanon') == [q for _, canon in mo.FACES for q in canon]


def test_scaling_and_colour_lookup_equal_the_reference_expressions():
    import panic3d_b200.mesh as pm
    v = mf.sphere(20, 7.0)
    rgbs = np.random.default_rng(1).random((3, 20, 20, 20), dtype=np.float32)
    m = mo.marching_cubes_index(v)
    mc_vert, bw, shape_res = m['verts'], 0.7, v.shape[-1]
    ref_verts = mc_vert / shape_res * bw - 0.5 * bw                                   # eg3d_metrics3d.py:203
    ref_colors = np.stack([rgbs[:3, a, b, c] for a, b, c in mc_vert.astype(int)])   # eg3d_metrics3d.py:197-200
    ours = pm.scale_verts(mc_vert, shape_res, bw)
    assert ours.dtype == ref_verts.dtype == np.float32 and np.array_equal(ours.view(np.uint32), ref_verts.view(np.uint32))
    col = pm.host_colors(rgbs, m['floor_node'], v.shape)
    assert col.dtype == ref_colors.dtype and np.array_equal(col, ref_colors)
    assert np.array_equal(m['floor_node'], np.ravel_multi_index(mc_vert.astype(int).T, v.shape))


def test_no_cpu_path_for_torch_cpu_tensors():
    import torch
    import panic3d_b200.mesh as pm
    with pytest.raises(RuntimeError, match='CPU'):
        pm.marching_cubes(torch.zeros(4, 4, 4), torch.zeros(3, 4, 4, 4), 0.7)
    with pytest.raises(RuntimeError, match='float32'):
        pm.marching_cubes(np.zeros((4, 4, 4)), np.zeros((3, 4, 4, 4)), 0.7)


# ---------------------------------------------------------------- the configuration table
def _table_fields():
    q = mf.quantised(mf.noise(20, seed=5))
    return {'sphere48': mf.sphere(48, 20.0), 'torus48': mf.torus(48), 'noise24': mf.noise(24, seed=3),
            'sphere_uneven': mf.sphere(48, 20.0)[3:40, :29, 5:],
            'quantised_noise20': q,                                       # nodes and saddles exactly at 0.5
            'cliffs_sphere40': mf.cliffs(mf.sphere(40, 15.0), 18, seed=1)}   # -1e3 next to values in (0.5, 0.51]


@pytest.mark.parametrize('name', sorted(_table_fields()))
def test_table_equals_the_walk_bit_for_bit(name):
    v = _table_fields()[name]
    table, walk = mo.marching_cubes_index(v), mo.marching_cubes_index(v, walk=True)
    assert len(table['faces']) > 100
    for k in walk:
        assert table[k].dtype == walk[k].dtype and np.array_equal(table[k].view(np.uint8), walk[k].view(np.uint8)), k
    dropped = mo.fan_triangles(v) - len(table['faces'])
    if name in ('quantised_noise20', 'cliffs_sphere40'):
        assert dropped > 0                                                # the degenerate branch runs
    if name == 'quantised_noise20':
        assert (v == 0.5).any() and (v > 0.5).any()


def _lattice(origin, e):
    k, ax = mo.EDGES[e]
    return tuple(o + d for o, d in zip(origin, mo.CORNER_OFFSETS[k])), ax


def _segments(loops):
    return {(lp[i], lp[(i + 1) % len(lp)]) for lp in loops for i in range(len(lp))}


def _face_edges(f):
    cyc = mo.FACES[f][0]
    return {mo._edge_between(cyc[k], cyc[(k + 1) % 4]) for k in range(4)}


def _sign_change_edges(case):
    return {e for e, (k, ax) in enumerate(mo.EDGES) if ((case >> k) ^ (case >> (k | mo._axis_bit(ax)))) & 1}


def _mirror(case, decisions, axis):
    """The configuration reflected across the plane normal to `axis`: corner k <-> k ^ bit, face (axis, s) <-> (axis, 1 - s)."""
    bit = mo._axis_bit(axis)
    c = sum(((case >> (k ^ bit)) & 1) << k for k in range(8))
    d = sum(((decisions >> (f ^ 1 if f // 2 == axis else f)) & 1) << f for f in range(6))
    return c, d


def test_every_configuration_closes_its_loops_and_agrees_with_its_neighbours():
    """For each of the 256 cases and every assignment of its ambiguous faces' decisions: the loops partition the cell's
    sign-change edges (each once, every loop >= 3 edges, so the kernel's walk of them ends), each face's segments pair up
    exactly that face's sign-change edges, and the cell across each face - the mirrored inside bits, the same decision on
    the shared face - has the same segments there, reversed, in lattice-edge terms.  With both, the surface is closed
    across every cell face: watertight as a statement over the whole configuration space."""
    configs = mo.configurations()
    assert len(configs) == sum(1 << bin(int(a)).count('1') for a in mo.AMBIGUOUS) == 656
    assert sorted(set(bin(int(a)).count('1') for a in mo.AMBIGUOUS)) == [0, 1, 2, 3, 6]
    for case, d in configs:
        loops = mo.loops_for(case, d)
        used = [e for lp in loops for e in lp]
        assert sorted(used) == sorted(_sign_change_edges(case)), (case, d)
        assert all(len(lp) >= 3 for lp in loops), (case, d)
        segs = _segments(loops)
        for f in range(6):
            axis, side = divmod(f, 2)
            fe = _face_edges(f)
            mine = {s for s in segs if s[0] in fe and s[1] in fe}
            assert sorted(e for s in mine for e in s) == sorted(_sign_change_edges(case) & fe), (case, d, f)
            nc, nd = _mirror(case, d, axis)
            origin = tuple((2 * side - 1) if a == axis else 0 for a in range(3))
            nfe = _face_edges(f ^ 1)
            theirs = {s for s in _segments(mo.loops_for(nc, nd)) if s[0] in nfe and s[1] in nfe}
            assert {(_lattice((0, 0, 0), a), _lattice((0, 0, 0), b)) for a, b in mine} == \
                   {(_lattice(origin, b), _lattice(origin, a)) for a, b in theirs}, (case, d, f)


# every (case, decisions) key the zoo's search reaches: all 656.  With continuous corner values alone, case 13 (the
# checkerboard cases 105 and 150, six ambiguous faces) realises 46 of its 64 decision patterns; the other 18 need a
# decider that ties with the level or divides by zero, which the tie values produce
ZOO_KEYS = 656


def test_configuration_zoo_reaches_every_case_and_every_configuration():
    found = mf.zoo_configurations()
    assert {c for c, _ in found} >= set(range(1, 255))
    assert len(found) == ZOO_KEYS == len(mo.configurations())
    for (case, d), cv in found.items():
        assert mo.inside_bits(cv, 0.5) == case and mo.face_decisions(cv, 0.5) == d
    v, where = mf.zoo_volume()
    idx, case, dec = mo.surface_cells(v)
    at = {tuple(p): (c, dd) for p, c, dd in zip(idx.tolist(), case.tolist(), dec.tolist())}
    for key, p in where.items():
        assert at.get(p, (key[0], 0)) == key, key                         # cases 0 and 255 are not surface cells


def test_continuous_corners_reach_46_of_case_13s_64_decision_patterns():
    rng = np.random.default_rng(0)
    ins = ((105 >> np.arange(8)) & 1).astype(bool)
    u = rng.random((200000, 8), dtype=np.float32) * np.float32(0.5)
    cv = np.where(ins, np.float32(1) - u, u)
    assert len(np.unique(mo.face_decisions(cv, 0.5))) == 46


# ---------------------------------------------------------------- the size guard of the C ABI
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _lib
    return _lib.lib()


@pytest.mark.parametrize('dims', [(2, 2, 2 ** 62 + 1), (2 ** 15, 2 ** 15, 2 ** 34), (2 ** 62, 2, 2), (2, 2 ** 40, 2 ** 24),
                                  (1025, 1024, 1024)])
def test_node_limit_is_checked_before_the_sides_are_multiplied(lib, dims):
    """The int64 product of the sides wraps for (2, 2, 2^62 + 1) (to 4) and (2^15, 2^15, 2^34) (to 0): every side and
    partial product is compared with 2^30 first, so these are refused instead of launched with truncated sides."""
    assert lib.p3d_mc_workspace_bytes(*dims) == 0
    assert b'at most 2^30 nodes' in lib.p3d_last_error()
    null = C.c_void_p(0)
    assert lib.p3d_mc_count(null, *dims, C.c_float(0.5), null, 0, null, null) != 0
    assert b'at most 2^30 nodes' in lib.p3d_last_error()
    assert lib.p3d_mc_emit(null, *dims, C.c_float(0.5), null, 0, *[null] * 6) != 0
    assert b'at most 2^30 nodes' in lib.p3d_last_error()
