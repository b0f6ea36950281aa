"""Seeded scalar fields for the marching-cubes tests (shared by test_mesh_cpu.py, test_mesh_gpu.py and
test_mesh_paths_gpu.py)."""
from __future__ import annotations

import numpy as np


def _centred(shape):
    return [np.arange(n, dtype=np.float64) - (n - 1) / 2 for n in shape]


def sphere(R=48, radius=20.0, width=1.0):
    """Density-like field: 1 / (1 + exp((|x| - radius) / width)), level 0.5 at |x| = radius voxels."""
    a, b, c = np.meshgrid(*_centred((R, R, R)), indexing='ij')
    d = np.sqrt(a * a + b * b + c * c)
    return (1.0 / (1.0 + np.exp((d - radius) / width))).astype(np.float32)


def torus(R=48, major=13.0, minor=5.0):
    a, b, c = np.meshgrid(*_centred((R, R, R)), indexing='ij')
    q = np.sqrt(b * b + c * c) - major
    d = np.sqrt(q * q + a * a)
    return (1.0 / (1.0 + np.exp(d - minor))).astype(np.float32)


def noise(R=24, seed=0):
    """i.i.d. uniform [0, 1) on an R^3 grid (or the shape R): every cell case and many ambiguous faces."""
    return np.random.default_rng(seed).random(R if isinstance(R, tuple) else (R, R, R), dtype=np.float32)


def blob(R, seed=0):
    """Seeded head-sized blob (bench_mesh.py's workload): density sigmoid(r - d) around a sphere of radius r = 0.35 R (1 +
    bumps) voxels, the bumps a few seeded low-frequency harmonics.  fp32 torch on the CPU."""
    import torch
    g = torch.Generator(device='cpu').manual_seed(seed)
    coef = (torch.rand(6, generator=g) - 0.5) * 0.16
    lin = torch.arange(R, dtype=torch.float32) - (R - 1) / 2
    a, b, c = torch.meshgrid(lin, lin, lin, indexing='ij')
    d = torch.sqrt(a * a + b * b + c * c)
    theta = torch.atan2(b, c)
    phi = torch.acos(torch.clamp(a / torch.clamp(d, min=1e-6), -1, 1))
    bumps = (coef[0] * torch.cos(2 * theta) + coef[1] * torch.sin(3 * theta) + coef[2] * torch.cos(2 * phi)
             + coef[3] * torch.sin(3 * phi) * torch.cos(theta) + coef[4] * torch.cos(4 * phi) + coef[5] * torch.sin(5 * theta) * torch.sin(phi))
    return torch.sigmoid(0.35 * R * (1 + bumps) - d).numpy()


def quantised(v, k=8):
    """v rounded to the grid j / k: with k even, nodes land exactly on 0.5 (outside) and so do many deciders (separated)."""
    return (np.round(v.astype(np.float64) * k) / k).astype(np.float32)


def cliffs(v, start, seed=0):
    """v with the slab of indices >= start along axis 0 replaced as crop / cull leave a volume: -1e3 where v <= 0.5, a
    value in (0.5, 0.51] where v > 0.5.  Every sign change there is a cliff: t within ~1e-5 of 0 or 1, which rounds onto
    the node for part of the values (index 128: when t is within 2^-17 of 1)."""
    v = v.copy()
    s = v[start:]
    up = 0.51 - 0.01 * np.random.default_rng(seed).random(s.shape)                # (0.5, 0.51]
    v[start:] = np.where(s > 0.5, up, -1e3).astype(np.float32)
    return v


def checkerboard(n):
    """{0, 1} by node parity: every lattice edge changes sign at t = 0.5, every face is ambiguous and its decider ties at
    (0 * 0 - 1 * 1) / (0 + 0 - 1 - 1) = 0.5 (separated): 3 n^2 (n - 1) vertices and 4 (n - 1)^3 triangles."""
    i = np.arange(n)
    return ((i[:, None, None] + i[None, :, None] + i[None, None, :]) % 2).astype(np.float32)


def ambiguous_face_decisions(v, level=0.5):
    """(connected, separated) counts over every lattice face with two diagonally opposite inside corners."""
    from oracle import mesh_oracle as mo
    v = v.astype(np.float32)
    conn = sep = 0
    for f in range(3):
        u, w = [x for x in range(3) if x != f]
        vm = np.moveaxis(v, (f, u, w), (0, 1, 2))
        v00, v01, v10, v11 = vm[:, :-1, :-1], vm[:, :-1, 1:], vm[:, 1:, :-1], vm[:, 1:, 1:]
        i00, i01, i10, i11 = (x > level for x in (v00, v01, v10, v11))
        amb = (i00 == i11) & (i01 == i10) & (i00 != i01)
        s = mo.saddle(v00[amb], v01[amb], v10[amb], v11[amb])
        conn += int((s > np.float32(level)).sum())
        sep += int((~(s > np.float32(level))).sum())
    return conn, sep


# the corner values the configuration zoo draws from besides continuous ones: level ties (0.5 and its neighbours), the
# values densities saturate at, and the crop / cull value
HALF = np.float32(0.5)
INSIDE_TIES = np.array([np.nextafter(HALF, np.float32(1)), 1], dtype=np.float32)
OUTSIDE_TIES = np.array([0, HALF, np.nextafter(HALF, np.float32(0)), -1e3], dtype=np.float32)


def zoo_configurations(seed=0, rounds=5, n=200000):
    """{(case, decisions): corner values (8,) fp32} - the first realisation at level 0.5 of every configuration a seeded
    search reaches.  A draw picks a case with probability proportional to 2^(its ambiguous faces), so case 13's 64 decision
    patterns get their share, then each corner from a per-draw mix of continuous values on its side of the level and the
    tie values above."""
    from oracle import mesh_oracle as mo
    rng = np.random.default_rng(seed)
    w = np.array([1 << bin(int(a)).count('1') for a in mo.AMBIGUOUS], dtype=np.float64)
    found = {}
    for _ in range(rounds):
        case = rng.choice(256, n, p=w / w.sum())
        ins = ((case[:, None] >> np.arange(8)) & 1).astype(bool)
        u = rng.random((n, 8), dtype=np.float32) * HALF
        cont = np.where(ins, np.float32(1) - u, u)
        tie = np.where(ins, INSIDE_TIES[rng.integers(0, len(INSIDE_TIES), (n, 8))],
                       OUTSIDE_TIES[rng.integers(0, len(OUTSIDE_TIES), (n, 8))])
        cv = np.where(rng.random((n, 8)) < rng.random((n, 1)), tie, cont)
        key = mo.inside_bits(cv, HALF) * 64 + mo.face_decisions(cv, HALF)
        uk, first = np.unique(key, return_index=True)
        for k, i in zip(uk.tolist(), first.tolist()):
            found.setdefault((k >> 6, k & 63), cv[i])
    return found


def zoo_volume(seed=0):
    """Every configuration of `zoo_configurations(seed)` in its own 2x2x2 block, blocks at stride 3 in key order; the
    filler nodes between blocks are seeded draws from the same values (continuous and ties).  Returns (volume, {key:
    lower corner of its block})."""
    found = zoo_configurations(seed)
    m = int(np.ceil(len(found) ** (1 / 3)))
    rng = np.random.default_rng(seed + 1)
    n = 3 * m - 1
    pool = np.concatenate([INSIDE_TIES, OUTSIDE_TIES])
    v = np.where(rng.random((n, n, n)) < 0.5, rng.random((n, n, n), dtype=np.float32), pool[rng.integers(0, len(pool), (n, n, n))])
    v = v.astype(np.float32)
    where = {}
    for i, key in enumerate(sorted(found)):
        a, b, c = 3 * (i // (m * m)), 3 * (i // m % m), 3 * (i % m)
        for k in range(8):
            v[a + ((k >> 2) & 1), b + ((k >> 1) & 1), c + (k & 1)] = found[key][k]
        where[key] = (a, b, c)
    return v, where
