"""Test-side restatement of the PNG input chain `I(src).resize(size)[.convert('RGBA').bg('w').convert('RGB')].t()`
(reference `_util/twodee_v1.py`) and the builders of the files and zlib streams the decoder tests feed it.

* ``decode``: zlib + a numpy unfilter (PNG specification 1.2 section 6.6, anti-diagonal wavefront) + the high byte of
  16-bit samples, the pixels PIL opens;
* ``nearest_index``: PIL's nearest resize (``ImagingScaleAffine``: the source coordinate accumulated in doubles);
* ``over_white``: PIL's integer ``Image.alpha_composite`` of a pixel over opaque white;
* ``chain``: all of it, then ``to_tensor``'s float32 / 255;
* ``png_file``, ``filter_rows`` and ``Deflate``: PNG files with chosen filters, zlib settings and IDAT splits, and
  hand-built deflate streams (fixed / dynamic / stored blocks, any match) for what zlib never emits.
"""
from __future__ import annotations

import io
import struct
import zlib

import numpy as np
import torch

COLOR = {1: 0, 3: 2, 4: 6}


# ---------------------------------------------------------------- the oracle
def unfilter(scan, h, w, bpp):
    """(h * (1 + w * bpp)) filtered bytes -> (h, w * bpp) uint8."""
    f = np.asarray(scan, dtype=np.uint8).reshape(h, 1 + w * bpp)
    types = f[:, 0].astype(np.int64)
    assert (types <= 4).all()
    f = f[:, 1:].reshape(h, w, bpp).astype(np.int64)
    out = np.zeros((h + 1, w + 1, bpp), dtype=np.int64)          # row 0 and column 0: the zeros above and left
    for s in range(h + w - 1):
        y = np.arange(max(0, s - w + 1), min(h, s + 1))
        x = s - y
        a, b, c = out[y + 1, x], out[y, x + 1], out[y, x]
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        t = types[y][:, None]
        pred = np.select([t == 0, t == 1, t == 2, t == 3], [np.zeros_like(a), a, b, (a + b) >> 1], paeth)
        out[y + 1, x + 1] = (f[y, x] + pred) & 255
    return out[1:, 1:].reshape(h, w * bpp).astype(np.uint8)


def chunks(data):
    o, res = 8, []
    while o < len(data):
        n, = struct.unpack('>I', data[o:o + 4])
        res.append((data[o + 4:o + 8], data[o + 8:o + 8 + n]))
        o += 12 + n
    return res


def decode(data):
    """PNG bytes -> (H, W, C) uint8, the pixels PIL opens (16-bit samples: their high byte)."""
    ch = chunks(data)
    w, h, depth, color = struct.unpack('>IIBB', ch[0][1][:10])
    c = {0: 1, 2: 3, 6: 4}[color]
    raw = zlib.decompress(b''.join(d for t, d in ch if t == b'IDAT'))
    bs = depth // 8
    pix = unfilter(np.frombuffer(raw, np.uint8), h, w, c * bs).reshape(h, w, c, bs)
    return np.ascontiguousarray(pix[..., 0])


def nearest_index(n_in, n_out):
    """PIL's nearest source index of every output index (-1: outside the source, PIL fills zeros)."""
    scale = n_in / n_out
    x, res = scale * 0.5, []
    for _ in range(n_out):
        v = -1 if x < 0 else int(x)
        res.append(v if v < n_in else -1)
        x += scale
    return np.array(res, dtype=np.int64)


def over_white(v, a):
    """libImaging/AlphaComposite.c for a destination of opaque white (7 bits of precision, rounded divisions)."""
    v, a = np.asarray(v, np.int64), np.asarray(a, np.int64)
    outa255 = a * 255 + 255 * (255 - a)
    coef1 = a * 255 * 255 * 128 // np.maximum(outa255, 1)
    tmp = v * coef1 + 255 * (255 * 128 - coef1) + (0x80 << 7)
    return np.where(a == 0, 255, (((tmp >> 8) + tmp) >> 8) >> 7)


def chain(data, size=None, white_background=False):
    """PNG bytes -> float32 (C, H, W): I(src).resize(size)[.convert('RGBA').bg('w').convert('RGB')].t()."""
    pix = decode(data)
    h, w, c = pix.shape
    oh, ow = (h, w) if size is None else (size, size) if isinstance(size, int) else size
    yi, xi = nearest_index(h, oh), nearest_index(w, ow)
    res = pix[np.clip(yi, 0, None)][:, np.clip(xi, 0, None)].astype(np.int64)
    res[(yi < 0)[:, None] | (xi < 0)[None, :]] = 0
    if white_background:
        if c == 1:
            res = np.repeat(res, 3, axis=2)
        elif c == 4:
            res = over_white(res[..., :3], res[..., 3:])
    return torch.from_numpy(res.astype(np.uint8)).permute(2, 0, 1).float().div(255)


def pil_chain(data, size=None, white_background=False):
    """The same through PIL itself and to_tensor's arithmetic (torchvision is not installed here)."""
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    assert im.mode in ('L', 'RGB', 'RGBA'), im.mode
    if size is not None:
        s = (size, size) if isinstance(size, int) else tuple(size)
        im = im.resize(s[::-1], resample=Image.NEAREST)
    if white_background:
        im = Image.alpha_composite(Image.new('RGBA', im.size, (255, 255, 255, 255)), im.convert('RGBA')).convert('RGB')
    a = np.asarray(im)
    a = a[..., None] if a.ndim == 2 else a
    return torch.from_numpy(a.copy()).permute(2, 0, 1).contiguous().float().div(255)


# ---------------------------------------------------------------- files
def filter_rows(pix, types):
    """(H, W, C) uint8 or uint16 (big-endian samples) and one filter type per row -> the filtered scan-line bytes."""
    h, w = pix.shape[:2]
    raw = (pix.astype('>u2') if pix.dtype == np.uint16 else pix).view(np.uint8).reshape(h, -1).astype(np.int64)
    bpp = raw.shape[1] // w
    out = np.zeros((h, 1 + raw.shape[1]), np.uint8)
    zero = np.zeros(raw.shape[1], np.int64)
    for y in range(h):
        x, b = raw[y], raw[y - 1] if y else zero
        a = np.concatenate([np.zeros(bpp, np.int64), x[:-bpp]])
        c = np.concatenate([np.zeros(bpp, np.int64), b[:-bpp]])
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        t = int(types[y])
        out[y, 0] = t
        out[y, 1:] = (x - [0 * x, a, b, (a + b) >> 1, paeth][t]) & 255
    return out.reshape(-1).tobytes()


def chunk(typ, data):
    return struct.pack('>I', len(data)) + typ + data + struct.pack('>I', zlib.crc32(typ + data))


def png_file(h, w, c, depth, stream, split=None, extra=(), ihdr=None):
    """A PNG around a zlib `stream`: IDATs of `split` bytes (None: one), `extra` chunks after IHDR."""
    head = chunk(b'IHDR', ihdr if ihdr is not None else struct.pack('>IIBBBBB', w, h, depth, COLOR[c], 0, 0, 0))
    parts = [stream] if not split else [stream[i:i + split] for i in range(0, len(stream), split)] or [b'']
    return b'\x89PNG\r\n\x1a\n' + head + b''.join(extra) + b''.join(chunk(b'IDAT', p) for p in parts) + chunk(b'IEND', b'')


def zstream(raw, level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY):
    z = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
    return z.compress(raw) + z.flush()


def pil_png(pix, **kw):
    """(H, W, C) uint8 -> PNG bytes written by PIL."""
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(pix[..., 0] if pix.shape[2] == 1 else pix, {1: 'L', 3: 'RGB', 4: 'RGBA'}[pix.shape[2]]).save(buf, 'PNG', **kw)
    return buf.getvalue()


# ---------------------------------------------------------------- hand-built deflate streams
LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


def canonical(lens):
    """Code lengths -> codes (RFC 1951 3.2.2)."""
    bl = [0] * 16
    for l in lens:
        bl[l] += 1
    bl[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for l in lens:
        out.append(nxt[l] if l else None)
        if l:
            nxt[l] += 1
    return out


class Deflate:
    """A raw deflate bit stream built block by block; `zlib()` wraps it with a header and an Adler-32."""

    def __init__(self):
        self.acc, self.n, self.out, self.raw = 0, 0, bytearray(), bytearray()

    def bits(self, v, k):
        self.acc |= v << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def huff(self, code, l):                                     # Huffman codes go most significant bit first
        if code is None:                                         # a symbol the block's code lacks (malformed streams)
            code, l = 0, 1
        self.bits(int(format(code, f'0{l}b')[::-1], 2), l)

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)

    def stored(self, data, final=False, nlen=None):
        self.bits(int(final), 1)
        self.bits(0, 2)
        self.align()
        self.bits(len(data), 16)
        self.bits((len(data) ^ 0xffff) if nlen is None else nlen, 16)
        self.out += data
        self.raw += data

    def _tokens(self, tokens, lcodes, llens, dcodes, dlens):
        for t in tokens:
            if isinstance(t, int):
                self.huff(lcodes[t], llens[t])
                if t < 256:
                    self.raw.append(t)
                continue
            length, dist = t
            s = max(i for i in range(29) if LBASE[i] <= length) if length < 258 else 28
            self.huff(lcodes[257 + s], llens[257 + s])
            self.bits(length - LBASE[s], LEXT[s])
            d = max(i for i in range(30) if DBASE[i] <= dist)
            self.huff(dcodes[d], dlens[d])
            self.bits(dist - DBASE[d], DEXT[d])
            for _ in range(length):
                self.raw.append(self.raw[-dist] if dist <= len(self.raw) else 0)

    def fixed(self, tokens, final=False, eob=True):
        """tokens: literal ints (256 = end of block, 286/287 allowed for malformed streams) and (length, distance)."""
        self.bits(int(final), 1)
        self.bits(1, 2)
        self._tokens(list(tokens) + ([256] if eob else []), canonical(FIXED_LIT), FIXED_LIT, canonical([5] * 32), [5] * 32)

    def dynamic(self, tokens, llens, dlens, final=False, cllens=None):
        """A dynamic block with the given code lengths (hlit = len(llens), hdist = len(dlens)), each length written as
        its own code-length symbol under a 4-bit code for 0..15 unless `cllens` (19 lengths) says otherwise."""
        self.bits(int(final), 1)
        self.bits(2, 2)
        cl = cllens if cllens is not None else [4] * 16 + [0] * 3
        self.bits(len(llens) - 257, 5)
        self.bits(len(dlens) - 1, 5)
        self.bits(19 - 4, 4)
        for i in CLORDER:
            self.bits(cl[i], 3)
        clc = canonical(cl)
        for l in list(llens) + list(dlens):
            self.huff(clc[l], cl[l])
        self._tokens(list(tokens) + [256], canonical(llens), llens, canonical(dlens), dlens)

    def zlib(self, cmf=0x78, flg=None, adler=None):
        self.align()
        if flg is None:
            flg = (31 - (cmf * 256) % 31) % 31
        return bytes([cmf, flg]) + bytes(self.out) + struct.pack('>I', zlib.adler32(bytes(self.raw)) if adler is None else adler)


def lit_lengths_286():
    """A complete literal/length code over all 286 symbols: 226 of 8 bits, 60 of 9."""
    return [8] * 226 + [9] * 60


STRATEGIES = (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED)


def crafted_streams():
    """Streams zlib never writes, each inflating to a valid filtered image: name -> (h, w, c, depth, zlib stream, raw).
    Grey images whose rows are w + 1 = 32768 or 65535 bytes long line matches and stored blocks up with rows."""
    g = np.random.default_rng(11)
    res = {}
    d = Deflate()                                                  # matches at the full window, 258 bytes long
    row = [0] + g.integers(0, 256, 32767).tolist()
    d.fixed(row)
    d.fixed([(258, 32768)] * 254 + [(4, 32768)], final=True)
    res['distance_32768_length_258'] = (3, 32767, 1, 8, d.zlib(), bytes(d.raw))
    runs = []
    for v in (7, 200, 0, 255):
        runs += [0, v, (258, 1), (258, 1), (83, 1)]
    d = Deflate()
    d.fixed(runs, final=True)
    res['distance_1_runs'] = (4, 600, 1, 8, d.zlib(), bytes(d.raw))
    d = Deflate()
    d.dynamic(runs, lit_lengths_286(), [1], final=True)            # one distance code (of one bit): distance 1
    res['one_distance_code'] = (4, 600, 1, 8, d.zlib(), bytes(d.raw))
    d = Deflate()
    pix = g.integers(0, 256, (2, 5, 3))
    d.dynamic([b for y in range(2) for b in [1] + pix[y].reshape(-1).tolist()], lit_lengths_286(), [0], final=True)
    res['zero_distance_codes'] = (2, 5, 3, 8, d.zlib(), bytes(d.raw))
    d = Deflate()
    rows = [bytes([0]) + bytes(g.integers(0, 256, 65534).astype(np.uint8)) for _ in range(2)]
    d.stored(rows[0])
    d.stored(b'')                                                  # an empty stored block: a sync flush
    d.stored(rows[1], final=True)
    res['stored_65535'] = (2, 65534, 1, 8, d.zlib(), bytes(d.raw))
    d = Deflate()                                                  # stored, fixed and dynamic blocks, matches across them
    row = bytes([0]) + bytes(g.integers(0, 256, 40).astype(np.uint8))
    d.stored(row)
    d.fixed([(41, 41)])
    d.dynamic([(164, 41)], lit_lengths_286(), [0] * 10 + [1], final=True)
    res['stored_fixed_dynamic'] = (6, 10, 4, 8, d.zlib(), bytes(d.raw))
    return res


def malformed_streams():
    """name -> (zlib stream, bytes the image should inflate to, the P3D_PNG_* status the decoder must give)."""
    n = 64
    raw = bytes([0]) + bytes(range(1, n))
    good = zlib.compress(raw)
    res = {}
    res['bad_fcheck'] = (good[:1] + bytes([good[1] ^ 1]) + good[2:], n, 2)
    res['cinfo_8'] = (bytes([0x88, (31 - (0x88 * 256) % 31) % 31]) + good[2:], n, 2)
    res['method_7'] = (bytes([0x77, (31 - (0x77 * 256) % 31) % 31]) + good[2:], n, 2)
    res['preset_dictionary'] = (bytes([0x78, 0x20 | (31 - (0x78 * 256 + 0x20) % 31) % 31]) + good[2:], n, 2)
    d = Deflate()
    d.bits(1, 1)
    d.bits(3, 2)
    res['block_type_3'] = (d.zlib(), n, 3)
    d = Deflate()
    d.stored(raw, final=True, nlen=len(raw))
    res['stored_nlen'] = (d.zlib(), n, 3)
    d = Deflate()
    d.dynamic(list(raw), lit_lengths_286(), [1], final=True, cllens=[1] * 19)
    res['oversubscribed_code_length_code'] = (d.zlib(), n, 4)
    d = Deflate()
    d.dynamic(list(raw), [9] * 286, [1], final=True)
    res['incomplete_literal_code'] = (d.zlib(), n, 4)
    d = Deflate()
    d.dynamic(list(raw), lit_lengths_286(), [1, 1, 1], final=True)
    res['oversubscribed_distance_code'] = (d.zlib(), n, 4)
    d = Deflate()
    d.dynamic(list(raw), [8] * 256 + [0], [1], final=True)
    res['no_end_of_block_code'] = (d.zlib(), n, 4)
    d = Deflate()
    d.fixed([0, 1, 286], final=True)
    res['literal_286'] = (d.zlib(), n, 5)
    d = Deflate()
    d.dynamic([0, 1, (10, 1)], lit_lengths_286(), [0], final=True)
    res['match_without_distance_codes'] = (d.zlib(), n, 5)
    d = Deflate()
    d.fixed([0, 1, (20, 3)], final=True)
    res['distance_past_start'] = (d.zlib(), n, 6)
    res['too_long'] = (zlib.compress(raw + b'x'), n, 7)
    res['too_short'] = (zlib.compress(raw[:-1]), n, 8)
    res['truncated_mid_block'] = (good[:len(good) // 2], n, 9)
    res['truncated_adler'] = (good[:-2], n, 9)
    res['empty_stream'] = (b'', n, 9)
    res['bad_adler'] = (good[:-1] + bytes([good[-1] ^ 0x40]), n, 10)
    return res
