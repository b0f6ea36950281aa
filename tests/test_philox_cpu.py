"""CPU: the restatement of the renderer's in-kernel jitter (oracle/philox.py), which the production-path render tests
(tests/test_render_philox_gpu.py) feed to the oracle.  Pinned to Random123's published Philox4x32-10 known answers, to
the kernel's 24-bit float mapping, and to regression values of the kernel's counter layout; its statistics are checked on
2^20 draws of one fixed seed (deterministic, so no test here can flake)."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import philox as ph

N_DRAWS = 1 << 20
SEED = 0x5EED


def test_philox4x32_10_known_answers():
    """Random123's kat_vectors for philox4x32_10: counter words, key words -> output words."""
    kat = [([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
           ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
           ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
            [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1])]
    for ctr, key, want in kat:
        assert ph.philox4x32_10(ctr, key).tolist() == want
    # vectorised over a batch of counters and keys, each row equal to its scalar evaluation
    ctrs = np.array([k[0] for k in kat], dtype=np.uint64)
    keys = np.array([k[1] for k in kat], dtype=np.uint64)
    assert ph.philox4x32_10(ctrs, keys).tolist() == [k[2] for k in kat]


def test_u01_keeps_24_bits_and_never_reaches_one():
    bits = np.array([0, 0xFF, 0x100, 0x80000000, 0xFFFFFEFF, 0xFFFFFF00, 0xFFFFFFFF], dtype=np.uint32)
    u = ph.u01(bits)
    assert u.dtype == np.float32
    assert u.tolist() == [0.0, 0.0, 2.0 ** -24, 0.5, 1 - 2.0 ** -23, 1 - 2.0 ** -24, 1 - 2.0 ** -24]
    assert float(u.max()) < 1.0
    # every value is a multiple of 2^-24 below 1, exactly representable in fp32
    x = ph.uniforms(SEED, np.arange(N_DRAWS, dtype=np.uint64), 0).astype(np.float64) * 2 ** 24
    assert np.array_equal(x, np.floor(x)) and x.min() >= 0 and x.max() <= 2 ** 24 - 1


def test_kernel_layout_regression_values():
    """philox_uniform(seed, index, stream) at three points: low and high index words, both streams, the upper key word."""
    assert float(ph.uniforms(7, 0, 0)) == 0.5031725764274597
    assert float(ph.uniforms(7, 5, 1)) == 0.4604089856147766
    assert float(ph.uniforms(0x0123456789ABCDEF, 1000003, 0)) == 0.8772495985031128
    # the layout: index i reads word i & 3 of counter i >> 2
    seed, i = 0xFFFFFFFF00000001, (1 << 34) + 6
    words = ph.philox4x32_10([(i >> 2) & 0xFFFFFFFF, i >> 34, 1, ph.CTR_WORD3], [seed & 0xFFFFFFFF, seed >> 32])
    assert float(ph.uniforms(seed, i, 1)) == float(ph.u01(words[i & 3]))


def test_render_uniforms_shapes_and_index_rule():
    N, M, S, Sf, seed = 2, 5, 7, 3, 11
    u_c, u_f = ph.render_uniforms(seed, N, M, S, Sf)
    assert u_c.shape == (N, M, S, 1) and u_f.shape == (N * M, Sf)
    assert u_c.dtype == torch.float32 and u_f.dtype == torch.float32
    for n, m, s in ((0, 0, 0), (1, 3, 6), (1, 4, 2)):
        r = n * M + m                                      # global ray index across views
        assert u_c[n, m, s, 0].item() == float(ph.uniforms(seed, r * S + s, 0))
    for r, f in ((0, 0), (7, 2), (9, 1)):
        assert u_f[r, f].item() == float(ph.uniforms(seed, r * Sf + f, 1))
    assert ph.render_uniforms(seed, N, M, S, 0)[1].shape == (N * M, 0)


def _draws(seed, stream, n=N_DRAWS):
    return ph.uniforms(seed, np.arange(n, dtype=np.uint64), stream).astype(np.float64)


def test_uniforms_pass_kolmogorov_smirnov_and_chi_square():
    u = _draws(SEED, 0)
    assert stats.kstest(u, 'uniform').pvalue > 1e-3
    counts = np.bincount((u * 256).astype(np.int64), minlength=256)
    assert counts.shape == (256,)
    assert stats.chisquare(counts).pvalue > 1e-3


def _corr(a, b):
    return float(np.corrcoef(a, b)[0, 1])


def test_streams_lags_and_views_are_uncorrelated():
    bar = 5 / math.sqrt(N_DRAWS)
    u0, u1 = _draws(SEED, 0), _draws(SEED, 1)
    assert abs(_corr(u0[:-1], u0[1:])) < bar                      # lag 1 within the coarse stream
    assert abs(_corr(u1[:-1], u1[1:])) < bar                      # and within the fine stream
    assert abs(_corr(u0, u1)) < bar                               # coarse vs fine at the same index
    v1 = _draws(ph.host_view_seed(SEED, 1), 0)                    # view 0 vs view 1 of the host entry point
    assert abs(_corr(u0, v1)) < bar


def test_host_view_seed_wraps_and_is_distinct():
    s = 0xFFFFFFFF00000001
    assert ph.host_view_seed(s, 0) == s
    assert ph.host_view_seed(s, 1) == (s + ph.VIEW_SEED_STEP) % 2 ** 64
    assert 2 * ph.VIEW_SEED_STEP > 2 ** 64                                        # so v >= 2 wraps for every seed
    assert ph.host_view_seed(0, 2) == 2 * ph.VIEW_SEED_STEP - 2 ** 64
    assert ph.host_view_seed(s, 1) == s + ph.VIEW_SEED_STEP - 2 ** 64
    assert ph.host_view_seed(s, 2) == s + 2 * ph.VIEW_SEED_STEP - 2 * 2 ** 64
    seeds = [ph.host_view_seed(s, v) for v in range(1 << 16)]
    assert len(set(seeds)) == 1 << 16 and all(0 <= x < 2 ** 64 for x in seeds)


@pytest.mark.parametrize('k', [0, 1, 1234])
def test_drawn_seed_is_the_first_int64_draw_after_manual_seed(k):
    state = torch.get_rng_state()
    try:
        torch.manual_seed(k)
        first = int(torch.empty((), dtype=torch.int64).random_().item())
    finally:
        torch.set_rng_state(state)
    assert ph.drawn_seed(k) == first and 0 <= first < 2 ** 63
    assert ph.drawn_seed(1234) == 0x31076B2F7F66E2D3                         # regression value
