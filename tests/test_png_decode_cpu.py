"""CPU: the host side of the device PNG decoder (include/p3d_imageio.h) and its oracle.

* The oracle (tests/png_oracle.py: zlib, numpy unfilter, PIL's nearest index, PIL's integer composite, / 255) equals PIL
  plus to_tensor's arithmetic on PIL-written and hand-filtered files, for every supported type and depth.
* p3d_png_inspect refuses each unsupported or malformed file with a message naming the field, and accepts split and
  empty IDATs and ancillary chunks.
* p3d_png_inflate_host, the device decoder's inflate built for the CPU, decodes what zlib writes and gives each
  malformed stream of png_oracle.malformed_streams its status code.
* The workspace query is 0 outside the envelope."""
import struct
import zlib

import numpy as np
import pytest
import torch

from tests import png_oracle as po

TYPES = [(1, 8), (3, 8), (4, 8), (3, 16), (4, 16)]
WIDTHS = [1, 2, 3, 31, 32, 33, 511, 512, 513]


@pytest.fixture(scope='module')
def L():
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _lib, imageio  # noqa: F401  (register the p3d_png_* prototypes)
    return _lib.lib()


def image(seed, h, w, c, depth):
    """Gradients + noise, and alpha drawn from 0, 255 and values in between."""
    g = np.random.default_rng(seed)
    top = 65535 if depth == 16 else 255
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    pix = np.stack([(xx * (7 + ch) + yy * 3 + ch * 40) % (top + 1) for ch in range(c)], -1)
    pix = np.where(g.random(pix.shape) < 0.3, g.integers(0, top + 1, pix.shape), pix)
    if c == 4:
        pix[..., 3] = g.choice([0, top, 1, top // 2, top - 1, 37 * (top // 255)], size=(h, w))
    return pix.astype(np.uint16 if depth == 16 else np.uint8)


def file_of(pix, depth, seed=0):
    h, w, c = pix.shape
    if depth == 8 and seed % 2 == 0:
        return po.pil_png(pix)                                              # PIL's own filters
    types = np.random.default_rng(seed).integers(0, 5, h)
    return po.png_file(h, w, c, depth, zlib.compress(po.filter_rows(pix, types)))


@pytest.mark.parametrize('c,depth', TYPES)
@pytest.mark.parametrize('w', WIDTHS)
def test_oracle_equals_pil(c, depth, w):
    for h, seed in ((1, w), (5, w + 1)):
        pix = image(seed, h, w, c, depth)
        f = file_of(pix, depth, seed)
        want = pix if depth == 8 else (pix >> 8).astype(np.uint8)
        assert np.array_equal(po.decode(f), want)
        for size in (None, 2 * w, max(1, w // 2), (3, 2 * w + 1), (7, max(1, (w * 2) // 3)), 1):
            for white in (False, True):
                a, b = po.chain(f, size, white), po.pil_chain(f, size, white)
                assert a.dtype == b.dtype == torch.float32 and a.shape == b.shape and torch.equal(a, b), (size, white)


def test_nearest_index_and_composite_against_pil():
    from PIL import Image
    for n_in in list(range(1, 40)) + [511, 512, 513, 1024]:
        for n_out in list(range(1, 40)) + [512, 1000]:
            im = Image.fromarray(np.arange(n_in, dtype=np.int32)[None], mode='I').resize((n_out, 1), Image.NEAREST)
            assert np.array_equal(np.asarray(im)[0], po.nearest_index(n_in, n_out)), (n_in, n_out)
    v, a = np.meshgrid(np.arange(256), np.arange(256), indexing='ij')
    src = Image.fromarray(np.stack([v, v, v, a], -1).astype(np.uint8), 'RGBA')
    got = np.asarray(Image.alpha_composite(Image.new('RGBA', (256, 256), (255, 255, 255, 255)), src))
    assert np.array_equal(got[..., 0], po.over_white(v, a)) and (got[..., 3] == 255).all()


# ---------------------------------------------------------------- p3d_png_inspect
def inspect(L, data):
    import ctypes as C
    from panic3d_b200 import imageio as pio
    buf = np.frombuffer(data, np.uint8)
    info = pio.PngInfo()
    rc = L.p3d_png_inspect(buf.ctypes.data, buf.size, C.byref(info), None)
    return rc, info, L.p3d_last_error().decode()


def ihdr(w=4, h=3, depth=8, color=2, comp=0, filt=0, interlace=0):
    return struct.pack('>IIBBBBB', w, h, depth, color, comp, filt, interlace)


GOOD = po.png_file(3, 4, 3, 8, zlib.compress(bytes(3 * 13)))


def refusals():
    s = zlib.compress(bytes(3 * 13))
    bad_crc = bytearray(GOOD)
    bad_crc[40] ^= 1
    no_iend = GOOD[:-12]
    after = po.png_file(3, 4, 3, 8, s, split=10)
    i = after.index(b'IDAT') - 4
    j = after.index(b'IDAT', i + 8) - 4
    split_by_text = after[:j] + po.chunk(b'tEXt', b'k\0v') + after[j:]
    return [
        ('signature', b'\x89PNG\r\n\x1a\x0b' + GOOD[8:]),
        ('CRC', bytes(bad_crc)),
        ('IHDR', GOOD[:8] + po.chunk(b'gAMA', b'\0\0\0\1') + GOOD[8:]),
        ('colour type 3', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(color=3))),
        ('colour type 4', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(color=4))),
        ('colour type 4', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(color=4, depth=16))),
        ('bit depth 16 with colour type 0', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(color=0, depth=16))),
        ('bit depth 4 with colour type 0', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(color=0, depth=4))),
        ('bit depth 1 with colour type 2', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(depth=1))),
        ('interlace method 1', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(interlace=1))),
        ('compression method 1', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(comp=1))),
        ('filter method 1', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(filt=1))),
        ('width 0', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(w=0))),
        ('envelope', po.png_file(3, 4, 3, 8, s, ihdr=ihdr(w=1 << 20, h=1 << 10))),
        ('tRNS chunk on colour type 2', po.png_file(3, 4, 3, 8, s, extra=[po.chunk(b'tRNS', bytes(6))])),
        ('tRNS chunk on colour type 0', po.png_file(3, 4, 1, 8, s, extra=[po.chunk(b'tRNS', bytes(2))])),
        ("unknown critical chunk 'ABCD'", po.png_file(3, 4, 3, 8, s, extra=[po.chunk(b'ABCD', b'x')])),
        ('IDAT chunks are not consecutive', split_by_text),
        ('no IDAT', GOOD[:33] + po.chunk(b'IEND', b'')),
        ('no IEND', no_iend),
        ('past the end of the file', GOOD[:45]),
    ]


@pytest.mark.parametrize('case', range(len(refusals())))
def test_inspect_refuses_with_the_field_named(L, case):
    what, data = refusals()[case]
    rc, _, msg = inspect(L, data)
    assert rc == -1 and what in msg, (what, msg)


def test_inspect_accepts_split_and_empty_idats_and_ancillary_chunks(L):
    pix = image(3, 9, 17, 4, 8)
    s = zlib.compress(po.filter_rows(pix, [4] * 9))
    anc = [po.chunk(b'gAMA', b'\0\0\xb1\x8f'), po.chunk(b'tEXt', b'a\0b'), po.chunk(b'tRNS', b'\0' * 8), po.chunk(b'prIv', b'x')]
    for split in (None, 1, 7, 8192):
        f = po.png_file(9, 17, 4, 8, s, split=split, extra=anc)
        if split == 7:                                                     # zero-length IDATs before, between and after
            i = f.index(b'IDAT') - 4
            e = po.chunk(b'IDAT', b'')
            f = f[:i] + e + f[i:i + 19] + e + f[i + 19:-12] + e + f[-12:]
        rc, info, msg = inspect(L, f)
        assert rc == 0, msg
        assert (info.h, info.w, info.channels, info.depth, info.stream_bytes) == (9, 17, 4, 8, len(s))
        assert info.n_idat == (1 if split is None else -(-len(s) // split) + (3 if split == 7 else 0))
        import ctypes as C
        buf = np.frombuffer(f, np.uint8)
        dst = np.zeros(len(s), np.uint8)
        assert L.p3d_png_inspect(buf.ctypes.data, buf.size, C.byref(info), dst.ctypes.data) == 0
        assert dst.tobytes() == s
        assert np.array_equal(po.decode(f), pix)


# ---------------------------------------------------------------- the decoder's inflate on the CPU
def inflate(L, stream, n):
    raw = np.zeros(n, np.uint8)
    s = np.frombuffer(stream, np.uint8)
    return L.p3d_png_inflate_host(s.ctypes.data if s.size else None, s.size, raw.ctypes.data, n), raw.tobytes()


@pytest.mark.parametrize('wbits', range(9, 16))
def test_host_inflate_decodes_every_zlib_setting(L, wbits):
    raw = po.filter_rows(image(wbits, 40, 300, 4, 8), np.arange(40) % 5)
    for level in range(10):
        for strategy in po.STRATEGIES:
            rc, out = inflate(L, po.zstream(raw, level, wbits, strategy), len(raw))
            assert rc == 0 and out == raw, (level, strategy)


def test_host_inflate_hand_built_streams(L):
    for name, (h, w, c, depth, stream, raw) in po.crafted_streams().items():
        rc, out = inflate(L, stream, len(raw))
        assert rc == 0 and out == raw, name


@pytest.mark.parametrize('name', list(po.malformed_streams()))
def test_host_inflate_malformed_streams(L, name):
    from panic3d_b200 import imageio as pio
    stream, n, code = po.malformed_streams()[name]
    rc, _ = inflate(L, stream, n)
    assert rc == code, (name, rc, pio.PNG_STATUS.get(rc))


# ---------------------------------------------------------------- size queries
@pytest.mark.parametrize('args', [(0, 5, 3, 8, 5, 5), (5, 0, 3, 8, 5, 5), (-1, 5, 3, 8, 5, 5), (5, 5, 2, 8, 5, 5), (5, 5, 1, 16, 5, 5),
                                  (5, 5, 3, 4, 5, 5), (5, 5, 3, 8, 0, 5), (5, 5, 3, 8, 5, 0), (5, 5, 3, 8, 32769, 5),
                                  (5, 5, 3, 8, 5, -3), (16384 + 1, 16383, 1, 8, 5, 5), (1, (1 << 28) // 8, 4, 16, 5, 5),
                                  (2 ** 31 - 1, 2 ** 31 - 1, 4, 16, 5, 5)])
def test_workspace_query_is_zero_outside_the_envelope(L, args):
    assert L.p3d_png_decode_workspace_bytes(*args) == 0


@pytest.mark.parametrize('h,w,c,d,oh,ow', [(1, 1, 1, 8, 1, 1), (512, 512, 3, 8, 512, 512), (1024, 1024, 4, 16, 512, 512),
                                           (16384, 16383, 1, 8, 32768, 32768), (1, ((1 << 28) - 1) // 8, 4, 16, 1, 1)])
def test_workspace_query_inside_the_envelope(L, h, w, c, d, oh, ow):
    raw = h * (1 + w * c * d // 8)
    assert raw <= 1 << 28
    a16 = lambda x: -(-x // 16) * 16
    assert L.p3d_png_decode_workspace_bytes(h, w, c, d, oh, ow) == a16(raw) + a16(4 * (oh + ow))


def test_device_entry_refuses_bad_batches_before_any_launch(L):
    import ctypes as C
    fake = C.c_void_p(256)
    args = [fake, 10, fake, 2, 8, 8, 3, 1, fake, 1 << 20, fake, fake, None]
    for i in (0, 2, 8, 10, 11):
        a = list(args)
        a[i] = None
        assert L.p3d_png_decode_device(*a) == -1 and b'NULL' in L.p3d_last_error()
    for i, v in ((3, 0), (3, 65536), (4, 0), (5, 32769), (6, 4), (6, 2)):
        a = list(args)
        a[i] = v
        assert L.p3d_png_decode_device(*a) == -1 and b'envelope' in L.p3d_last_error()
