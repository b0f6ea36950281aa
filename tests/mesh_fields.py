"""Seeded scalar fields for the marching-cubes tests (shared by test_mesh_cpu.py and test_mesh_gpu.py)."""
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
    """i.i.d. uniform [0, 1): every cell case and many ambiguous faces."""
    return np.random.default_rng(seed).random((R, R, R), dtype=np.float32)


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
