"""CPU: the host side of the device PNG encoder (include/p3d_imageio.h) - its size queries at the edges of the envelope
and one past them, and the refusals of NULL pointers, short workspaces, short output strides and wrapping shapes, all
returned before anything reaches a device."""
import ctypes as C

import pytest

SEG = 16384
MAX_STREAM = 1 << 28


@pytest.fixture(scope='module')
def L():
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _lib, imageio  # noqa: F401  (register the p3d_png_* prototypes)
    return _lib.lib()


def bound(h, w, c):
    n = h * (1 + w * c)
    return 63 + n + 10 * (-(-n // SEG))


@pytest.mark.parametrize('h,w,c', [(1, 1, 1), (1, 1, 3), (1, 1, 4), (512, 512, 3), (128, 128, 4), (8192, 1, 1), (1, SEG - 2, 1),
                                   (SEG, SEG - 1, 1), (1, (MAX_STREAM - 1) // 4, 4)])
def test_bound_and_workspace_inside_the_envelope(L, h, w, c):
    n = h * (1 + w * c)
    assert n <= MAX_STREAM
    assert L.p3d_png_device_bound(h, w, c) == bound(h, w, c)
    nseg = -(-n // SEG)
    assert L.p3d_png_device_workspace_bytes(1, h, w, c) == nseg * (SEG + 32)
    assert L.p3d_png_device_workspace_bytes(65535, h, w, c) == 65535 * nseg * (SEG + 32)
    assert L.p3d_png_device_bound(h, w, c) >= L.p3d_png_scanline_bytes(h, w, c) + 63


@pytest.mark.parametrize('n,h,w,c', [(1, SEG + 1, SEG - 1, 1),           # one row past 2^28 bytes
                                     (1, 1, MAX_STREAM // 4, 4),            # one row of 2^28 + 1 bytes
                                     (1, 2 ** 31 - 1, 2 ** 31 - 1, 4),      # h * (1 + w * C) wraps 64 bits if multiplied first
                                     (1, 0, 5, 3), (1, 5, 0, 3), (1, -1, 5, 3), (1, 5, 5, 2), (1, 5, 5, 5),
                                     (0, 5, 5, 3), (65536, 5, 5, 3), (-1, 5, 5, 3)])
def test_outside_the_envelope_is_zero_and_refused(L, n, h, w, c):
    assert L.p3d_png_device_workspace_bytes(n, h, w, c) == 0
    if n == 1:
        assert L.p3d_png_device_bound(h, w, c) == 0
    fake = C.c_void_p(256)
    rc = L.p3d_png_encode_device(fake, n, h, w, c, fake, 1 << 40, fake, 1 << 30, fake, None)
    assert rc == -1 and b'envelope' in L.p3d_last_error()


def test_null_pointers_short_workspace_and_short_stride_are_refused(L):
    fake = C.c_void_p(256)
    ws = L.p3d_png_device_workspace_bytes(2, 512, 512, 3)
    b = L.p3d_png_device_bound(512, 512, 3)
    for i in (0, 5, 7, 9):
        args = [fake, 2, 512, 512, 3, fake, ws, fake, b, fake, None]
        args[i] = None
        assert L.p3d_png_encode_device(*args) == -1 and b'NULL' in L.p3d_last_error()
    assert L.p3d_png_encode_device(fake, 2, 512, 512, 3, fake, ws - 1, fake, b, fake, None) == -3      # P3D_EWORKSPACE
    assert b'workspace' in L.p3d_last_error()
    assert L.p3d_png_encode_device(fake, 2, 512, 512, 3, fake, ws, fake, b - 1, fake, None) == -1
    assert L.p3d_png_encode_device(fake, 2, 512, 512, 3, fake, ws, fake, 2 ** 63, fake, None) == -1     # n * stride wraps
    assert b'out_stride' in L.p3d_last_error()


def test_encoded_submission_refusals(L):
    h = C.c_void_p()
    assert L.p3d_png_writer_create(1, 3, C.byref(h)) == 0
    try:
        fake = C.c_void_p(256)
        assert L.p3d_png_writer_submit_encoded(h, fake, None, 4, 4, 3, b'/tmp/x.png', None) == -1
        assert L.p3d_png_writer_submit_encoded(h, None, fake, 4, 4, 3, b'/tmp/x.png', None) == -1
        assert L.p3d_png_writer_submit_encoded(h, fake, fake, 4, 4, 2, b'/tmp/x.png', None) == -1
        assert L.p3d_png_writer_submit_encoded(h, fake, fake, SEG + 1, SEG - 1, 1, b'/tmp/x.png', None) == -1
        assert b'envelope' in L.p3d_last_error()
        assert L.p3d_png_writer_submit_encoded(None, fake, fake, 4, 4, 3, b'/tmp/x.png', None) == -1
    finally:
        assert L.p3d_png_writer_destroy(h) == 0


def test_writer_encoder_argument(L):
    import panic3d_b200.imageio as pio
    with pytest.raises(ValueError):
        pio.AsyncImageWriter(encoder='gpu')
    w = pio.AsyncImageWriter(threads=1)
    assert w.encoder == 'host'
    w.close()
