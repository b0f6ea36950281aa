"""CPU: the call surface of the deterministic training backward (p3d_render_backward_det, p3d_decode_points_backward_det,
p3d_paste_front_backward_det) - scratch-size queries at the edges of the 2^31 - 1 entry envelope and one past it, the
entry-count refusal on int64 shapes whose product wraps, and NULL / short-scratch errors, all before anything launches."""
from __future__ import annotations

import ctypes as C

import pytest

K = 2 ** 31 - 1                    # entry ids, texel keys and the sort's item count are 32-bit
KPARAMS = 64 * 32 + 64 + 33 * 64 + 33


@pytest.fixture(scope='module')
def lib():
    import panic3d_b200.paste  # noqa: F401  (binds the p3d_paste_* prototypes)
    from panic3d_b200 import _lib
    return _lib.lib()


def _params(N=1, M=1, S=1, Sf=0, H=2, W=2, D=0):
    from panic3d_b200 import _lib
    p = _lib.RenderParams()
    p.n_views, p.n_rays, p.n_coarse, p.n_fine, p.channels, p.plane_h, p.plane_w = N, M, S, Sf, 32, H, W
    p.hidden, p.out_dim, p.box_warp, p.plane_depth = 64, 33, 0.7, D
    p.stride_col, p.stride_row = 32, W * 32
    p.stride_plane = max(D, 1) * H * W * 32
    p.stride_view = 3 * p.stride_plane
    return p


def _err(lib):
    return lib.p3d_last_error().decode()


def test_render_scratch_covers_every_record(lib):
    """The scratch holds the atomic backward's per-sample scratch, then dF (32 floats per sample), weights, two key and
    two id buffers (one word per entry each), CTA partials and their pairwise levels, and the sort's temporaries."""
    p = _params(N=4, M=64 * 64, S=48, Sf=48, H=256, W=256)
    got = lib.p3d_render_backward_det_scratch_bytes(C.byref(p))
    samples = 4 * 64 * 64 * 96
    entries = samples * 12
    ctas = 2 * (4 * 64 * 64 * 48 // 128)
    least = lib.p3d_render_backward_scratch_bytes(C.byref(p)) + samples * 32 * 4 + 5 * entries * 4 + (2 * ctas + 64) * KPARAMS * 4
    assert least <= got <= least + (64 << 20), (got, least)


@pytest.mark.parametrize('D, nt', [(0, 12), (3, 24)])
def test_render_envelope_edges(lib, D, nt):
    """Exactly 2^31 - 1 entries is not reachable with 12 or 24 per sample; the largest sample count below it is accepted
    and one more sample is refused."""
    last = K // nt                               # samples
    ok = _params(N=1, M=last, S=1, Sf=0, D=D)
    assert lib.p3d_render_backward_det_scratch_bytes(C.byref(ok)) > last * nt * 4, _err(lib)
    over = _params(N=1, M=last + 1, S=1, Sf=0, D=D)
    assert lib.p3d_render_backward_det_scratch_bytes(C.byref(over)) == 0
    assert 'at most 2147483647 entries' in _err(lib)


def test_points_envelope_edges(lib):
    p = _params(N=3, D=0)
    last = K // 12 // 3
    assert lib.p3d_decode_points_backward_det_scratch_bytes(C.byref(p), last) > 0, _err(lib)
    assert lib.p3d_decode_points_backward_det_scratch_bytes(C.byref(p), last + 1) == 0
    assert 'at most 2147483647 entries' in _err(lib)
    assert lib.p3d_decode_points_backward_det_scratch_bytes(C.byref(p), -1) == 0
    assert 'negative point count' in _err(lib)


def test_texel_envelope(lib):
    """Keys run over every texel of the batch plus one for taps outside the plane: N x 3 x D x H x W < 2^31 - 1."""
    ok = _params(N=1, H=16384, W=16384)          # 3 x 2^28 texels
    assert lib.p3d_render_backward_det_scratch_bytes(C.byref(ok)) > 0, _err(lib)
    over = _params(N=3, H=16384, W=16384)
    assert lib.p3d_render_backward_det_scratch_bytes(C.byref(over)) == 0
    assert 'texels' in _err(lib)


@pytest.mark.parametrize('n_pts, N', [(2 ** 62 + 1, 4), (2 ** 61, 8), (2 ** 63 - 1, 2)])
def test_point_count_product_that_wraps_is_refused(lib, n_pts, N):
    """N x n_points wraps in int64 ((2^62 + 1) x 4 == 4, 2^61 x 8 == 0): the point count is bounded before it is multiplied."""
    p = _params(N=N)
    assert lib.p3d_decode_points_backward_det_scratch_bytes(C.byref(p), n_pts) == 0
    assert 'at most 2147483647 entries' in _err(lib)
    null = C.c_void_p(0)
    assert lib.p3d_decode_points_backward_det(C.byref(p), *[null] * 6, n_pts, null, null, null, 0, *[null] * 5, null) != 0
    assert 'at most 2147483647 entries' in _err(lib)


def test_render_rays_times_samples_that_overflow_is_refused(lib):
    p = _params(N=2 ** 31 - 1, M=2 ** 31 - 1, S=2 ** 30, Sf=2 ** 30)
    assert lib.p3d_render_backward_det_scratch_bytes(C.byref(p)) == 0
    assert 'at most 2147483647 entries' in _err(lib)


def test_null_and_short_scratch(lib):
    from panic3d_b200 import paste
    null = C.c_void_p(0)
    one = C.c_void_p(256)                        # never dereferenced: every check fails first
    p = _params(N=1, M=4, S=2, Sf=0)
    assert lib.p3d_render_backward_det(C.byref(p), *[null] * 8, 0, *[null] * 5, null, 0, *[null] * 5, null) == -1
    assert 'null input pointer' in _err(lib)
    assert lib.p3d_render_backward_det(None, *[null] * 8, 0, *[null] * 5, null, 0, *[null] * 5, null) == -1
    assert lib.p3d_render_backward_det_scratch_bytes(None) == 0
    assert lib.p3d_decode_points_backward_det(C.byref(p), *[one] * 6, 4, one, one, null, 0, *[one] * 5, null) == -1
    assert 'null output pointer' in _err(lib)
    assert lib.p3d_decode_points_backward_det(C.byref(p), *[one] * 6, 4, one, one, one, 16, *[one] * 5, null) == -3
    assert 'scratch too small' in _err(lib)
    pp = paste.PasteParams()
    pp.n_views, pp.res_render, pp.res_image, pp.box_warp = 2, 64, 512, 0.7
    need = lib.p3d_paste_front_backward_det_scratch_bytes(C.byref(pp))
    assert need == 2 * 2 * 512 * 512 * 4
    assert lib.p3d_paste_front_backward_det(C.byref(pp), one, one, one, one, null, one, need - 1, one, one, null) == -3
    assert 'scratch too small' in _err(lib)
    assert lib.p3d_paste_front_backward_det(C.byref(pp), null, one, one, one, null, one, need, one, one, null) == -1
    pp.n_views = 0
    assert lib.p3d_paste_front_backward_det_scratch_bytes(C.byref(pp)) == 0
    assert 'n_views' in _err(lib)
