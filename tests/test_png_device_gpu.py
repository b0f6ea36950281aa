"""GPU: the device PNG encoder (p3d_png_encode_device, csrc/png_deflate.cu) through the C ABI and the writer.  Every file is
taken apart here: chunk CRCs against zlib.crc32, the IDAT's zlib stream against zlib.decompress and its Adler-32, pixels
against PIL, and a small inflater below walks the deflate blocks to show which block types and matches the encoder chose.
Workspace and output are prefilled with 0xFF and NaN bytes, so a byte the encoder does not write shows."""
import io
import struct
import zlib

import numpy as np
import pytest
import torch

from tests.helpers import synth_image

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SEG = 16384                       # input bytes per encoder segment (include/p3d_imageio.h)
FILLS = (0xFF, 'nan')


# ---------------------------------------------------------------- encoder through the C ABI
def encode(scan, h, w, c, fill=0xFF):
    """(N, L) uint8 CUDA scan-lines -> list of N file bytes, workspace and output prefilled with `fill`."""
    from panic3d_b200 import _lib
    L = _lib.lib()
    n = scan.shape[0]
    bound, ws_bytes = L.p3d_png_device_bound(h, w, c), L.p3d_png_device_workspace_bytes(n, h, w, c)
    assert bound and ws_bytes

    def filled(nbytes):
        if fill == 'nan':
            t = torch.full(((nbytes + 3) // 4,), float('nan'), device=DEV).view(torch.uint8)[:nbytes]
        else:
            t = torch.full((nbytes,), fill, device=DEV, dtype=torch.uint8)
        return t
    ws, out = filled(ws_bytes), filled(n * bound)
    lens = torch.full((n,), -1, device=DEV, dtype=torch.int64)
    _lib.check(L.p3d_png_encode_device(scan.contiguous().data_ptr(), n, h, w, c, ws.data_ptr(), ws_bytes, out.data_ptr(), bound,
                                       lens.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    out, lens = out.cpu().numpy().reshape(n, bound), lens.cpu().tolist()
    assert all(0 < x <= bound for x in lens)
    return [out[i, :lens[i]].tobytes() for i in range(n)]


def chunks(png):
    """Parse a PNG into [(type, data)], checking the signature, every length and every CRC."""
    assert png[:8] == b'\x89PNG\r\n\x1a\n'
    o, res = 8, []
    while o < len(png):
        n, = struct.unpack('>I', png[o:o + 4])
        typ, data = png[o + 4:o + 8], png[o + 8:o + 8 + n]
        crc, = struct.unpack('>I', png[o + 8 + n:o + 12 + n])
        assert crc == zlib.crc32(typ + data), typ
        res.append((typ, data))
        o += 12 + n
    assert o == len(png)
    return res


def check_file(png, stream, h, w, c):
    """Container, zlib stream and Adler-32 of one file; returns the raw deflate data."""
    ch = chunks(png)
    assert [t for t, _ in ch] == [b'IHDR', b'IDAT', b'IEND']
    assert ch[0][1] == struct.pack('>IIBBBBB', w, h, 8, {1: 0, 3: 2, 4: 6}[c], 0, 0, 0)
    z = ch[1][1]
    assert (z[0] * 256 + z[1]) % 31 == 0 and z[0] & 15 == 8
    assert zlib.decompress(z) == stream
    assert struct.unpack('>I', z[-4:])[0] == zlib.adler32(stream)
    return z[2:-4]


# ---------------------------------------------------------------- a small inflater that records the blocks and matches
LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]


def walk(data):
    """Raw deflate -> (output bytes, [block type per block], [(output position, length, distance)])."""
    bits = np.unpackbits(np.frombuffer(data, np.uint8), bitorder='little')
    pos = 0

    def get(n):
        nonlocal pos
        v = int(sum(int(bits[pos + i]) << i for i in range(n)))
        pos += n
        return v

    def table(lens):
        count = [0] * 16
        for x in lens:
            count[x] += x > 0
        code, nxt, tab = 0, {}, {}
        for b in range(1, 16):
            code = (code + count[b - 1]) << 1
            nxt[b] = code
        for s, l in enumerate(lens):
            if l:
                tab[(l, nxt[l])] = s
                nxt[l] += 1
        return tab

    def sym(tab):
        code, l = 0, 0
        while True:
            code = code << 1 | get(1)
            l += 1
            if (l, code) in tab:
                return tab[(l, code)]
            assert l <= 15, 'bad code'

    out, types, matches = bytearray(), [], []
    while True:
        final, bt = get(1), get(2)
        types.append(bt)
        if bt == 0:
            pos = (pos + 7) // 8 * 8
            n, nn = get(16), get(16)
            assert n ^ nn == 0xFFFF
            out += bytes(np.packbits(bits[pos:pos + 8 * n], bitorder='little'))
            pos += 8 * n
        else:
            if bt == 1:
                lt = table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
                dt = table([5] * 30)
            else:
                assert bt == 2
                hlit, hdist, hclen = get(5) + 257, get(5) + 1, get(4) + 4
                order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
                cl = [0] * 19
                for i in range(hclen):
                    cl[order[i]] = get(3)
                ct, lens = table(cl), []
                while len(lens) < hlit + hdist:
                    s = sym(ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + get(2))
                    elif s == 17:
                        lens += [0] * (3 + get(3))
                    else:
                        lens += [0] * (11 + get(7))
                assert max(lens) <= 15 and len(lens) == hlit + hdist
                lt, dt = table(lens[:hlit]), table(lens[hlit:])
            while True:
                s = sym(lt)
                if s < 256:
                    out.append(s)
                elif s == 256:
                    break
                else:
                    ln = LBASE[s - 257] + get(LEXT[s - 257])
                    dc = sym(dt)
                    d = DBASE[dc] + get(DEXT[dc])
                    assert 1 <= d <= len(out) and d <= 32768
                    matches.append((len(out), ln, d))
                    for _ in range(ln):
                        out.append(out[-d])
        if final:
            return bytes(out), types, matches


# ---------------------------------------------------------------- cases
def scan_of(img):
    import panic3d_b200.imageio as pio
    return pio.png_scanlines(img.to(DEV))


def decode_pil(png):
    from PIL import Image
    im = Image.open(io.BytesIO(png))
    im.load()
    return np.asarray(im)


@pytest.mark.parametrize('fill', FILLS)
@pytest.mark.parametrize('n,c,h,w', [(1, 3, 1, 1), (1, 1, 1, 1), (1, 4, 1, 300), (1, 3, 257, 1), (2, 1, 3, 17), (3, 3, 40, 37),
                                     (2, 4, 33, 64), (1, 3, 2, 6000), (1, 4, 5, 4500)])
def test_files_decode_to_the_kernel_pixels(n, c, h, w, fill):
    import panic3d_b200.imageio as pio
    img = torch.stack([synth_image(7 * c + i, c, h, w) for i in range(n)])
    scan, _ = scan_of(img)
    pix = pio.to_uint8(img.to(DEV)).cpu().numpy()
    files = encode(scan, h, w, c, fill)
    s = scan.cpu().numpy()
    for i in range(n):
        check_file(files[i], s[i].tobytes(), h, w, c)
        assert np.array_equal(decode_pil(files[i]).reshape(h, w, c), pix[i])


def stream_case(name):
    """(h, w, c, (N, L) uint8 stream bytes) for the content cases; the bytes need not be valid scan-lines for zlib."""
    g = np.random.Generator(np.random.PCG64(11))
    if name == 'constant':
        h, w, c = 96, 400, 3
        s = np.zeros((h, 1 + w * c), np.uint8)
        s[:, 1:] = 77
    elif name == 'noise':
        h, w, c = 40, 1000, 3
        s = g.integers(0, 256, (h, 1 + w * c), dtype=np.uint8)
    elif name == 'noise_one_segment':                # 65,536 + 1 bytes of noise in one row
        h, w, c = 1, 16384, 4
        s = g.integers(0, 256, (h, 1 + w * c), dtype=np.uint8)
    elif name == 'window':                           # the same 300 random bytes 32,768 apart, zeros around them
        h, w, c = 3, 16383, 1
        s = np.zeros(h * (1 + w * c), np.uint8)
        blk = g.integers(1, 256, 300, dtype=np.uint8)
        s[1000:1300] = blk
        s[1000 + 32768:1300 + 32768] = blk
    return h, w, c, s.reshape(1, -1)


@pytest.mark.parametrize('name', ['constant', 'noise', 'noise_one_segment', 'window'])
def test_content_cases_round_trip_within_the_bound(name):
    from panic3d_b200 import _lib
    h, w, c, s = stream_case(name)
    scan = torch.from_numpy(s).to(DEV)
    png, = encode(scan, h, w, c)
    raw = check_file(png, s[0].tobytes(), h, w, c)
    assert len(png) <= _lib.lib().p3d_png_device_bound(h, w, c)
    out, types, matches = walk(raw)
    assert out == s[0].tobytes()
    nseg = -(-s.shape[1] // SEG)
    if name == 'constant':
        assert sum(1 for _, ln, _ in matches if ln == 258) > 100 and len(png) < s.size // 50
    if name.startswith('noise'):
        assert len(png) <= 63 + s.size + 10 * nseg                            # inside the bound
        assert len(types) == 2 * nseg - 1 and set(types[:-1]) == {0}          # stored segments + the sync flushes; the
                                                                              # last segment may be a few bytes (fixed)
    if name == 'noise_one_segment':
        assert s.size > 65535 and nseg >= 5
    if name == 'window':
        assert (1000 + 32768, 258, 32768) in matches                          # the full window and the longest match
        assert any(p // SEG != (p - d) // SEG for p, _, d in matches)         # matches reach back across a seam


def test_streams_ending_on_and_around_a_seam():
    """A stream one byte short of a segment, exactly one, exactly two, and one byte past two."""
    for L, (h, w) in ((SEG - 1, (1, SEG - 2)), (SEG, (8192, 1)), (2 * SEG, (16384, 1)), (2 * SEG + 1, (1, 2 * SEG))):
        s = ((np.arange(L) * 131) % 256).astype(np.uint8)
        assert h * (1 + w) == L
        png, = encode(torch.from_numpy(s[None]).to(DEV), h, w, 1)
        out, types, _ = walk(check_file(png, s.tobytes(), h, w, 1))
        assert out == s.tobytes() and len(types) == 2 * (-(-L // SEG)) - 1


def test_every_block_type_appears():
    seen = set()
    for h, w, c, s in [stream_case('noise'), stream_case('constant')]:
        seen |= set(walk(check_file(encode(torch.from_numpy(s).to(DEV), h, w, c)[0], s[0].tobytes(), h, w, c))[1])
    img = synth_image(3, 3, 64, 64)
    scan, _ = scan_of(img[None])
    seen |= set(walk(check_file(encode(scan, 64, 64, 3)[0], scan[0].cpu().numpy().tobytes(), 64, 64, 3))[1])
    one = torch.tensor([[0, 200, 100, 50]], dtype=torch.uint8, device=DEV)             # 1x1 RGB: fixed codes are smallest
    seen |= set(walk(check_file(encode(one, 1, 1, 3)[0], bytes([0, 200, 100, 50]), 1, 1, 3))[1])
    assert seen == {0, 1, 2}


@pytest.mark.parametrize('n', [8, 16])
def test_eval_shapes_deterministic_and_batch_independent(n):
    import panic3d_b200.imageio as pio
    for c, h in ((3, 512), (4, 128)):
        img = torch.stack([synth_image(100 + i, c, h, h) for i in range(n)])
        scan, _ = scan_of(img)
        a, b = encode(scan, h, h, c, 0xFF), encode(scan, h, h, c, 'nan')
        assert a == b
        assert encode(scan[3:4], h, h, c)[0] == a[3]
        s = scan.cpu().numpy()
        pix = pio.to_uint8(img.to(DEV)).cpu().numpy()
        for i in (0, n - 1):
            check_file(a[i], s[i].tobytes(), h, h, c)
            assert np.array_equal(decode_pil(a[i]).reshape(h, h, c), pix[i])
        dev = sum(map(len, a))
        z1 = sum(len(zlib.compress(s[i].tobytes(), 1)) for i in range(n))
        z6 = sum(len(zlib.compress(s[i].tobytes(), 6)) for i in range(n))
        assert dev < s.size
        print(f'{n} x {h}^2 C={c}: device {dev / n:.0f} B/view, {dev / z1:.3f} x zlib-1, {dev / z6:.3f} x zlib-6, '
              f'{dev / s.size:.3f} x raw')


def test_writer_device_files_decode_like_the_host_files(tmp_path):
    import panic3d_b200.imageio as pio
    img = torch.stack([synth_image(50 + i, 3, 96, 80) for i in range(3)]).to(DEV)
    xyz, wt = torch.rand(2, 3, 64, 64, device=DEV) - 0.5, torch.rand(2, 1, 64, 64, device=DEV)
    for enc in ('host', 'device'):
        with pio.AsyncImageWriter(threads=2, encoder=enc) as w:
            w.save(img, [tmp_path / f'{enc}_{i}.png' for i in range(3)])
            w.save_xyza(xyz, wt, 1.0, [tmp_path / f'{enc}_x{i}.png' for i in range(2)])
    for name in [f'{i}' for i in range(3)] + [f'x{i}' for i in range(2)]:
        a, b = (tmp_path / f'host_{name}.png').read_bytes(), (tmp_path / f'device_{name}.png').read_bytes()
        assert a != b
        assert np.array_equal(decode_pil(a), decode_pil(b))
    host = tmp_path / 'host_0.png'
    scan, _ = scan_of(img[:1].cpu())
    assert host.read_bytes() == pio.encode_png(scan[0].cpu().numpy(), 96, 80, 3, level=3)   # the default writer: zlib level 3
    with pytest.raises(ValueError):
        pio.AsyncImageWriter(encoder='gpu')
