"""TEST INFRASTRUCTURE ONLY - numpy restatement of the mesh extraction rules of DESIGN.md section 2 ("Marching cubes"),
written from the rules, not from the kernel.  Vertices are generated vectorised.  Triangles follow the per-cell rule: the
segments of the six faces (asymptotic decider on ambiguous faces) are chained into loops, each fanned from its smallest
vertex index.  That rule depends only on a cell's 8 inside bits and the decider's result on each of its ambiguous faces
(6 bits at most), so it is evaluated once per such configuration (`fan_table`, from `loops_for`) and gathered for every
surface cell at once: a 256^3 volume meshes in seconds.  The per-cell walk (`_faces_by_walk`, a Python loop over surface
cells, fine up to ~64^3) stays as the written-out definition the table is pinned against.

Only ``tests/`` (and the benchmark's reference arm) may import this module; the product path is ``panic3d_b200.mesh``.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32

# corner k of a cell sits at offset ((k >> 2) & 1, (k >> 1) & 1, k & 1) along axes (0, 1, 2)
CORNER_OFFSETS = [((k >> 2) & 1, (k >> 1) & 1, k & 1) for k in range(8)]


def _axis_bit(axis):
    return 1 << (2 - axis)


# local edges: (lower corner, axis), sorted by (corner, axis) - the same order as the global vertex indices they own
EDGES = sorted((k, ax) for k in range(8) for ax in range(3) if not k & _axis_bit(ax))
EDGE_ID = {e: i for i, e in enumerate(EDGES)}


def _edge_between(q0, q1):
    """Local edge joining two corners that differ along one axis."""
    diff = q0 ^ q1
    axis = 2 - diff.bit_length() + 1
    return EDGE_ID[(min(q0, q1), axis)]


def _faces():
    """The six faces as (corners in counter-clockwise order seen from outside the cell, canonical (u, w) corners).

    Face (axis f, side s) holds the corners whose coordinate along f is s; u < w are the two other axes.  Its outward
    normal is (2s - 1) e_f.  The cycle (0,0) -> (1,0) -> (1,1) -> (0,1) in (u, w) turns about e_u x e_w, which is +e_f for
    f in {0, 2} and -e_f for f = 1; it is reversed when that disagrees with the outward normal."""
    out = []
    for f in range(3):
        u, w = [a for a in range(3) if a != f]
        for s in (0, 1):
            def corner(iu, iw):
                return (_axis_bit(f) if s else 0) | (_axis_bit(u) if iu else 0) | (_axis_bit(w) if iw else 0)
            sigma = -1 if f == 1 else 1
            cyc = [(0, 0), (1, 0), (1, 1), (0, 1)] if sigma * (2 * s - 1) > 0 else [(0, 0), (0, 1), (1, 1), (1, 0)]
            out.append(([corner(*p) for p in cyc], (corner(0, 0), corner(0, 1), corner(1, 0), corner(1, 1))))
    return out


FACES = _faces()


def saddle(v00, v01, v10, v11):
    """Asymptotic decider value of a face, fp32 in this order: (v00*v11 - v01*v10) / (((v00 + v11) - v01) - v10)."""
    v00, v01, v10, v11 = F32(v00), F32(v01), F32(v10), F32(v11)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        return (v00 * v11 - v01 * v10) / (((v00 + v11) - v01) - v10)


def inside_bits(cv, level):
    """Case of cells with corner values cv (..., 8): bit k set when corner k is inside (v > level, fp32)."""
    cv = np.asarray(cv, dtype=F32)
    return ((cv > F32(level)).astype(np.int64) << np.arange(8)).sum(-1)


def _ambiguous(case):
    """6-bit mask of the faces of one case with exactly two diagonally opposite inside corners."""
    m = 0
    for f, (cyc, _) in enumerate(FACES):
        ins = [(case >> q) & 1 for q in cyc]
        m |= (sum(ins) == 2 and ins[0] == ins[2]) << f
    return m


AMBIGUOUS = np.array([_ambiguous(case) for case in range(256)], dtype=np.int64)


def face_decisions(cv, level):
    """Decision bits of cells with corner values cv (..., 8): bit f set when face f is ambiguous and its fp32 saddle value
    (`saddle`, at the face's canonical corners) exceeds the level, i.e. the inside corners are connected."""
    cv = np.asarray(cv, dtype=F32)
    level = F32(level)
    amb = AMBIGUOUS[inside_bits(cv, level)]
    d = np.zeros(cv.shape[:-1], dtype=np.int64)
    for f, (_, (c00, c01, c10, c11)) in enumerate(FACES):
        conn = saddle(cv[..., c00], cv[..., c01], cv[..., c10], cv[..., c11]) > level
        d |= ((amb >> f) & 1 & conn.astype(np.int64)) << f
    return d


def loops_for(case, decisions):
    """Closed loops of local edge ids of a cell with inside bits `case` whose ambiguous faces f are connected where bit f
    of `decisions` is set; each loop oriented so its right-hand normal points from inside to outside, starting at its
    smallest edge; loops ordered by that first edge."""
    nxt = {}
    for f, (cyc, _) in enumerate(FACES):
        ins = [bool((case >> q) & 1) for q in cyc]
        n_in = sum(ins)
        if n_in in (0, 4):
            continue
        fe = [_edge_between(cyc[k], cyc[(k + 1) % 4]) for k in range(4)]     # fe[k] joins cyc[k] and cyc[k+1]
        if n_in == 2 and ins[0] == ins[2]:                                    # two diagonally opposite inside corners
            connected = bool((decisions >> f) & 1)
            for k in range(4):
                if ins[k] and not connected:          # cut off the inside corner
                    nxt[fe[k - 1]] = fe[k]
                elif not ins[k] and connected:        # cut off the outside corner
                    nxt[fe[k]] = fe[k - 1]
        else:                                         # one segment: from the outside->inside edge to the inside->outside one
            start = [fe[k] for k in range(4) if not ins[k] and ins[(k + 1) % 4]]
            end = [fe[k] for k in range(4) if ins[k] and not ins[(k + 1) % 4]]
            assert len(start) == len(end) == 1
            nxt[start[0]] = end[0]
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        cur = nxt[e]
        while cur != e:
            assert cur not in seen and len(loop) <= 12, (case, decisions)
            loop.append(cur)
            seen.add(cur)
            cur = nxt[cur]
        loops.append(loop)
    return loops


def cell_loops(cv, level):
    """`loops_for` of one cell with corner values cv[8]."""
    return loops_for(int(inside_bits(cv, level)), int(face_decisions(cv, level)))


def configurations():
    """Every (case, decisions) key: decisions runs over the subsets of the case's ambiguous faces."""
    out = []
    for case in range(256):
        amb = int(AMBIGUOUS[case])
        sub = amb
        keys = []
        while True:                                   # the subsets of amb
            keys.append(sub)
            if sub == 0:
                break
            sub = (sub - 1) & amb
        out += [(case, d) for d in sorted(keys)]
    return out


MAX_FAN = 10                                          # fan triangles of one cell: 12 sign-change edges at most, minus 2 per loop


def _build_fan_table():
    tri = np.zeros((256, 64, MAX_FAN, 3), dtype=np.int8)
    cnt = np.zeros((256, 64), dtype=np.int64)
    for case, d in configurations():
        fan = [(lp[0], lp[i], lp[i + 1]) for lp in loops_for(case, d) for i in range(1, len(lp) - 1)]
        tri[case, d, :len(fan)] = np.reshape(fan, (-1, 3))
        cnt[case, d] = len(fan)
    return tri, cnt


_FAN = []


def fan_table():
    """(tri (256, 64, MAX_FAN, 3) int8, count (256, 64)): the fan triangles of every configuration as local-edge triples in
    (loop, fan position) order, from `loops_for`; built on first use."""
    if not _FAN:
        _FAN.append(_build_fan_table())
    return _FAN[0]


EDGE_CORNER = np.array([k for k, _ in EDGES], dtype=np.int64)
EDGE_AXIS = np.array([ax for _, ax in EDGES], dtype=np.int64)
OFFSETS = np.array(CORNER_OFFSETS, dtype=np.int64)


def _case_volume(v, level):
    inside = v > level
    D = v.shape
    cell_in = np.zeros((D[0] - 1, D[1] - 1, D[2] - 1), dtype=np.int64)
    for k, (dx, dy, dz) in enumerate(CORNER_OFFSETS):
        cell_in += inside[dx:dx + D[0] - 1, dy:dy + D[1] - 1, dz:dz + D[2] - 1].astype(np.int64) << k
    return cell_in


def surface_cells(v, level=0.5):
    """Surface cells in flat order: (lower-corner coordinates (n, 3), case (n,), decisions (n,))."""
    v = np.ascontiguousarray(v, dtype=F32)
    cell_in = _case_volume(v, F32(level))
    idx = np.argwhere((cell_in != 0) & (cell_in != 255))
    a, b, c = idx.T
    cv = np.stack([v[a + dx, b + dy, c + dz] for dx, dy, dz in CORNER_OFFSETS], -1)
    return idx, cell_in[a, b, c], face_decisions(cv, level)


def fan_triangles(v, level=0.5):
    """Fan triangles of the volume before degenerate removal (marching_cubes_index keeps those with 3 distinct positions)."""
    _, case, dec = surface_cells(v, level)
    return int(fan_table()[1][case, dec].sum())


def _faces_by_table(v, level, keys, verts):
    idx, case, dec = surface_cells(v, level)
    tri, cnt = fan_table()
    n = cnt[case, dec]
    e = tri[case, dec][np.arange(MAX_FAN) < n[:, None]].astype(np.int64)   # (F0, 3) local edges, cells in flat order
    cell = np.repeat(idx, n, axis=0)[:, None, :]                             # (F0, 1, 3)
    node = cell + OFFSETS[EDGE_CORNER[e]]                                    # (F0, 3, 3) owner nodes
    D = v.shape
    key = ((node[..., 0] * D[1] + node[..., 1]) * D[2] + node[..., 2]) * 3 + EDGE_AXIS[e]
    gid = np.searchsorted(keys, key)
    assert np.array_equal(keys[np.minimum(gid, len(keys) - 1)], key)
    p = verts[gid]
    same = lambda i, j: (p[:, i] == p[:, j]).all(-1)
    keep = ~(same(0, 1) | same(1, 2) | same(0, 2))                          # allow_degenerate=False
    return gid[keep].astype(np.int32).reshape(-1, 3)


def _faces_by_walk(v, level, keys, verts):
    D = v.shape
    cell_in = _case_volume(v, level)
    faces = []
    for a, b, c in np.argwhere((cell_in != 0) & (cell_in != 255)):
        cv = [v[a + dx, b + dy, c + dz] for dx, dy, dz in CORNER_OFFSETS]
        gid = []
        for k, ax in EDGES:
            dx, dy, dz = CORNER_OFFSETS[k]
            key = ((int(a) + dx) * D[1] + int(b) + dy) * D[2] + int(c) + dz
            i = np.searchsorted(keys, key * 3 + ax)
            gid.append(int(i) if i < len(keys) and keys[i] == key * 3 + ax else -1)
        for loop in cell_loops(cv, level):
            g = [gid[e] for e in loop]
            assert min(g) >= 0
            for i in range(1, len(g) - 1):
                tri = (g[0], g[i], g[i + 1])
                p0, p1, p2 = verts[tri[0]], verts[tri[1]], verts[tri[2]]
                if np.array_equal(p0, p1) or np.array_equal(p1, p2) or np.array_equal(p0, p2):
                    continue                                          # allow_degenerate=False
                faces.append(tri)
    return np.asarray(faces, dtype=np.int32).reshape(-1, 3)


def _gradient(v):
    """Per-node gradient (3, D0, D1, D2): central differences (v[i+1] - v[i-1]) * 0.5 inside, one-sided at the border."""
    g = np.empty((3,) + v.shape, dtype=F32)
    for ax in range(3):
        vm = np.moveaxis(v, ax, 0)
        gm = np.moveaxis(g[ax], ax, 0)
        gm[1:-1] = (vm[2:] - vm[:-2]) * F32(0.5)
        gm[0] = vm[1] - vm[0]
        gm[-1] = vm[-1] - vm[-2]
    return g


def marching_cubes_index(v, level=0.5, walk=False):
    """v (D0, D1, D2) fp32 -> dict of numpy arrays in index space:
    verts (V,3) fp32, faces (F,3) int32, normals (V,3) fp32, values (V,) fp32, floor_node (V,) int64.
    walk: triangles by the per-cell walk instead of the table (the same faces, bit for bit and in order; small volumes)."""
    v = np.ascontiguousarray(v, dtype=F32)
    assert v.ndim == 3 and min(v.shape) >= 2
    level = F32(level)
    D = v.shape
    inside = v > level
    grad = _gradient(v)
    # ---- vertices: one per sign-change lattice edge, ordered by (lower node flat index, axis)
    keys, pos_l, val_l, nrm_l = [], [], [], []
    for ax in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, D[ax] - 1), slice(1, D[ax])
        lo, hi = tuple(lo), tuple(hi)
        idx = np.argwhere(inside[lo] != inside[hi])                   # lower-node coordinates, C order
        a, b, c = idx.T
        h = idx.copy()
        h[:, ax] += 1
        vlo, vhi = v[a, b, c], v[h[:, 0], h[:, 1], h[:, 2]]
        with np.errstate(divide='ignore', invalid='ignore'):
            t = (level - vlo) / (vhi - vlo)
        p = idx.astype(F32)
        p[:, ax] = p[:, ax] + t
        glo = grad[:, a, b, c].T
        ghi = grad[:, h[:, 0], h[:, 1], h[:, 2]].T
        n = -(glo + t[:, None] * (ghi - glo))
        ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
        with np.errstate(divide='ignore', invalid='ignore'):
            n = np.where(ln[:, None] > 0, n / ln[:, None], F32(0)).astype(F32)
        flat = (a.astype(np.int64) * D[1] + b) * D[2] + c
        keys.append(flat * 3 + ax)
        pos_l.append(p)
        val_l.append(np.maximum(vlo, vhi))
        nrm_l.append(n)
    keys = np.concatenate(keys)
    order = np.argsort(keys, kind='stable')
    keys = keys[order]
    verts = np.concatenate(pos_l)[order].reshape(-1, 3).astype(F32)
    values = np.concatenate(val_l)[order].astype(F32)
    normals = np.concatenate(nrm_l)[order].reshape(-1, 3).astype(F32)
    fl = np.floor(verts).astype(np.int64)
    floor_node = (fl[:, 0] * D[1] + fl[:, 1]) * D[2] + fl[:, 2]
    # ---- triangles: surface cells in flat order, loops, fans
    faces = (_faces_by_walk if walk else _faces_by_table)(v, level, keys, verts)
    return dict(verts=verts, faces=faces, normals=normals, values=values, floor_node=floor_node)


def scale_verts(verts_index, shape_res, boxwarp):
    """The reference's ``mc_vert / shape_res * bw - 0.5*bw`` (eg3d_metrics3d.py:203) on fp32 vertices."""
    return verts_index / shape_res * boxwarp - 0.5 * boxwarp


def reference_colors(rgbs, verts_index):
    """The reference's per-vertex colour loop (eg3d_metrics3d.py:197-200)."""
    return np.stack([rgbs[:3, a, b, c] for a, b, c in verts_index.astype(int)])


def marching_cubes(vol, rgbs, boxwarp, level=0.5):
    """Host route of the reference's ``marching_cubes`` with this oracle in place of skimage (same returned keys)."""
    m = marching_cubes_index(vol, level)
    colors = reference_colors(rgbs, m['verts']) if len(m['verts']) else np.zeros((0, 3), dtype=rgbs.dtype)
    return dict(verts=scale_verts(m['verts'], vol.shape[-1], boxwarp), faces=m['faces'], normals=m['normals'],
                values=m['values'], colors=colors)


# ---------------------------------------------------------------- mesh checks shared by the tests
def edge_use(faces):
    """{(i, j): count} of directed edges."""
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    keys, counts = np.unique(e, axis=0, return_counts=True)
    return {(int(a), int(b)): int(n) for (a, b), n in zip(keys, counts)}


def is_closed_oriented(faces):
    """Every undirected edge used by exactly two triangles, once in each direction."""
    use = edge_use(faces)
    return all(n == 1 and use.get((b, a), 0) == 1 for (a, b), n in use.items())


def euler_characteristic(verts_count, faces):
    e = np.sort(np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]), axis=1)
    n_edges = len(np.unique(e, axis=0))
    used = len(np.unique(faces)) if len(faces) else 0
    del verts_count
    return used - n_edges + len(faces)


def area_and_volume(verts, faces):
    p = verts.astype(np.float64)[faces]
    cr = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    area = 0.5 * np.linalg.norm(cr, axis=1).sum()
    vol = np.einsum('ij,ij->i', p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0
    return float(area), float(vol)


def canonical_faces(faces):
    """Each triangle rotated so its smallest index comes first (winding kept), rows sorted."""
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    r = np.argmin(f, axis=1)
    rolled = np.stack([f[np.arange(len(f)), (r + k) % 3] for k in range(3)], axis=1)
    return rolled[np.lexsort(rolled.T[::-1])]
