"""CPU restatement of the renderer's in-kernel jitter: Philox4x32-10 and the index rule of its call sites.

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle/``: nothing under the package imports it.

When ``p3d_render_forward`` gets NULL ``u_coarse`` / ``u_fine`` pointers (every production render: the default
``ImportanceRenderer`` path, ``_RenderFunction``, ``bench.py``), the kernels draw their own uniforms.  This module
gives every one of them, so the CPU oracle (``renderer_oracle.render``), fed ``render_uniforms(seed, ...)``, computes
what those renders must produce.

* ``philox4x32_10``  <- ``csrc/p3d_common.cuh:91-103`` (Salmon et al. 2011, Random123's Philox4x32 with 10 rounds)
* ``u01``            <- ``csrc/p3d_common.cuh:105``: the top 24 bits, times 2^-24
* ``uniforms``       <- ``csrc/p3d_common.cuh:106-110`` (``philox_uniform``): counter ``(lo(i>>2), hi(i>>2), stream,
  0x1BD11BDA)``, key ``(lo(seed), hi(seed))``, word ``i & 3``
* ``render_uniforms`` <- the call sites:
    coarse sample ``s`` of global ray ``r``: index ``r*S + s``, stream 0
    (``render_v1.cu:94`` in ``k_sample_decode``, ``render_fused_ws3.cu:165`` in ``k_render_ws3``);
    fine sample ``f``: index ``r*Sf + f``, stream 1
    (``render_device.cuh:280`` with ``rng_base = ray * Sf`` from ``render_v1.cu:244``, ``render_fused_ws3.cu:334``).
  ``r`` counts rays across views (``view * M + m``), as the kernels do.
* ``host_view_seed`` <- ``c_api.cu:591``: ``p3d_render_forward_host`` renders view ``v`` alone (ray indices restart at
  0) with seed ``seed + v * 0x9E3779B97F4A7C15`` mod 2^64.
* ``drawn_seed``     <- ``training/volumetric_rendering/renderer.py:251``: the seed ``ImportanceRenderer`` draws per
  render, one int64 ``random_()`` from torch's CPU generator.
"""
from __future__ import annotations

import numpy as np

MASK32 = 0xFFFFFFFF
MASK64 = 0xFFFFFFFFFFFFFFFF
PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57        # round multipliers
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85        # key bumps (Weyl sequence)
CTR_WORD3 = 0x1BD11BDA                               # fixed fourth counter word of philox_uniform
VIEW_SEED_STEP = 0x9E3779B97F4A7C15                  # per-view seed offset of the host entry point
STREAM_COARSE, STREAM_FINE = 0, 1


def philox4x32_10(ctr, key) -> np.ndarray:
    """Philox4x32-10 of counters ``ctr`` (..., 4) under keys ``key`` (..., 2), 32-bit words; broadcasts.  -> (..., 4)
    uint32.  The 32x32 -> 64-bit products are exact in uint64, so mulhi / mullo are a shift and a mask."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    c0, c1, c2, c3 = (ctr[..., j] for j in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    m32, s32 = np.uint64(MASK32), np.uint64(32)
    for _ in range(10):
        p0 = np.uint64(PHILOX_M0) * c0
        p1 = np.uint64(PHILOX_M1) * c2
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ k0, p1 & m32, (p0 >> s32) ^ c3 ^ k1, p0 & m32
        k0 = (k0 + np.uint64(PHILOX_W0)) & m32
        k1 = (k1 + np.uint64(PHILOX_W1)) & m32
    return np.stack(np.broadcast_arrays(c0, c1, c2, c3), -1).astype(np.uint32)


def u01(bits) -> np.ndarray:
    """32-bit words -> float32 in [0, 1): (bits >> 8) * 2^-24, exact in fp32 (0 reachable, maximum 1 - 2^-24)."""
    b = np.asarray(bits, dtype=np.uint32) >> np.uint32(8)
    return b.astype(np.float32) * np.float32(2.0 ** -24)


def uniforms(seed: int, index, stream: int) -> np.ndarray:
    """philox_uniform(seed, index, stream) for every element of ``index`` (non-negative integers) -> float32."""
    seed = int(seed) & MASK64
    idx = np.asarray(index, dtype=np.uint64)
    ctr = idx >> np.uint64(2)
    counter = np.stack([ctr & np.uint64(MASK32), ctr >> np.uint64(32),
                        np.full_like(ctr, stream), np.full_like(ctr, CTR_WORD3)], -1)
    words = philox4x32_10(counter, np.array([seed & MASK32, seed >> 32], dtype=np.uint64))
    lane = (idx & np.uint64(3)).astype(np.intp)
    return u01(np.take_along_axis(words, lane[..., None], -1)[..., 0])


def render_uniforms(seed: int, N: int, M: int, S: int, Sf: int):
    """The uniforms a render of N views x M rays with S coarse and Sf fine samples draws under ``seed``, in the
    shapes ``renderer_oracle.render`` takes: u_coarse (N, M, S, 1), u_fine (N*M, Sf), torch float32."""
    import torch
    u_c = uniforms(seed, np.arange(N * M * S, dtype=np.uint64), STREAM_COARSE).reshape(N, M, S, 1)
    u_f = uniforms(seed, np.arange(N * M * Sf, dtype=np.uint64), STREAM_FINE).reshape(N * M, Sf)
    return torch.from_numpy(u_c), torch.from_numpy(u_f)


def host_view_seed(seed: int, v: int) -> int:
    """The seed ``p3d_render_forward_host`` gives view v of a batch rendered under ``seed``."""
    return (int(seed) + int(v) * VIEW_SEED_STEP) & MASK64


def drawn_seed(k: int) -> int:
    """The seed an ``ImportanceRenderer`` render draws when it is the first draw after ``torch.manual_seed(k)``: one
    int64 ``random_()`` (in [0, 2^63)) from a CPU generator seeded with k, masked to 64 bits.  Uses a generator of
    its own, so the global one is not touched."""
    import torch
    g = torch.Generator().manual_seed(int(k))
    return int(torch.empty((), dtype=torch.int64).random_(generator=g).item()) & MASK64
