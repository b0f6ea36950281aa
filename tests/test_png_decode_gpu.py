"""GPU: the device PNG decoder (p3d_png_decode_device, csrc/png_inflate.cu) through `panic3d_b200.imageio.load_images`,
bit-exact against tests/png_oracle.py (which tests/test_png_decode_cpu.py holds equal to PIL + to_tensor):
every zlib level, strategy and window size, IDATs split down to single bytes, rows forced to each filter, hand-built
streams zlib never writes (full-window 258-byte matches, distance-1 runs, one and zero distance codes, 65,535-byte stored
blocks), files from both AsyncImageWriter encoders, batch independence and repeatability, and malformed streams failing
alone in a batch whose other images still decode exactly."""
import os
import tempfile
import zlib

import numpy as np
import pytest
import torch

from tests import png_oracle as po
from tests.helpers import synth_image

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


def load(files, size=None, white=False):
    from panic3d_b200 import imageio as pio
    out = pio.load_images(files, size=size, white_background=white, device=DEV)
    torch.cuda.synchronize()
    return out.cpu()


def check(files, size=None, white=False):
    got = load(files, size, white)
    for i, f in enumerate(files):
        want = po.chain(f if isinstance(f, bytes) else open(f, 'rb').read(), size, white)
        assert torch.equal(got[i], want), (i, size, white, (got[i] != want).sum().item())
    return got


def image(seed, h, w, c, depth=8):
    g = np.random.default_rng(seed)
    top = 65535 if depth == 16 else 255
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing='ij')
    pix = np.stack([(np.sin(xx / (9 + ch)) * np.cos(yy / 13) * 0.5 + 0.5) * top for ch in range(c)], -1)
    pix = np.where(g.random(pix.shape) < 0.15, g.integers(0, top + 1, pix.shape), pix)
    pix[h // 3: h // 2, :] = (pix[h // 3: h // 2, :] // (top // 3)) * (top // 3)      # flat runs
    if c == 4:
        pix[..., 3] = g.choice([0, top, top // 2, 1, top - 3], size=(h, w))
    return pix.astype(np.uint16 if depth == 16 else np.uint8)


def raw_of(pix, types=None):
    h = pix.shape[0]
    return po.filter_rows(pix, np.arange(h) % 5 if types is None else types)


@pytest.mark.parametrize('white', [False, True])
def test_every_zlib_level_and_strategy(white):
    pix = image(1, 45, 70, 4)
    raw = raw_of(pix)
    files = [po.png_file(45, 70, 4, 8, po.zstream(raw, level, 15, s)) for level in range(10) for s in po.STRATEGIES]
    check(files, None, white)
    check(files, 64, white)


def test_every_window_size_and_idat_split():
    pix = image(2, 96, 130, 3)
    raw = raw_of(pix)
    files = [po.png_file(96, 130, 3, 8, po.zstream(raw, 9, wbits)) for wbits in range(9, 16)]
    files += [po.png_file(96, 130, 3, 8, zlib.compress(raw), split=s) for s in (1, 7, 8192)]
    check(files, None)
    check(files, 51, True)


@pytest.mark.parametrize('c,depth', [(1, 8), (3, 8), (4, 8), (3, 16), (4, 16)])
def test_rows_forced_to_each_filter(c, depth):
    h, w = 40, 77
    pix = image(3 + c + depth, h, w, c, depth)
    files = [po.png_file(h, w, c, depth, zlib.compress(raw_of(pix, [t] * h))) for t in range(5)]
    files.append(po.png_file(h, w, c, depth, zlib.compress(raw_of(pix, np.random.default_rng(c).integers(0, 5, h)))))
    check(files, None)
    check(files, (33, 120), True)


def test_widths_heights_and_resizes():
    files = []
    for w in (1, 2, 3, 31, 32, 33, 511, 512, 513):
        for c in (3, 4):
            pix = image(w + c, 1 if w % 2 else 9, w, c)
            files.append(po.pil_png(pix))
    for size in (1, 7, 256, 512, 700, (5, 1000)):
        check(files, size, True)


def test_hand_built_streams():
    for name, (h, w, c, depth, stream, raw) in po.crafted_streams().items():
        f = po.png_file(h, w, c, depth, stream)
        assert po.decode(f).size == h * w * c
        if w <= 32768:                                                     # the output side's envelope
            check([f], None)
        check([f], 97, True)
        check([f], (h, 20000))


@pytest.mark.parametrize('encoder', ['host', 'device'])
def test_writer_files_round_trip(encoder):
    import panic3d_b200.imageio as pio
    from oracle import imageio_oracle as io_orc
    imgs = [synth_image(s, c, 512, 512) for s, c in ((1, 3), (2, 4), (3, 1))] + [synth_image(4, 4, 128, 128)]
    with tempfile.TemporaryDirectory() as d:
        fns = [os.path.join(d, f'{encoder}{i}.png') for i in range(len(imgs))]
        with pio.AsyncImageWriter(threads=2, encoder=encoder) as wr:
            for img, fn in zip(imgs, fns):
                wr.save(img.to(DEV), fn)
        for img, fn in zip(imgs, fns):
            got = load([fn])[0]
            want = torch.from_numpy(io_orc.quantize(img)[0]).permute(2, 0, 1).float().div(255)
            assert torch.equal(got, want)
        check(fns, 256, True)


def test_batch_equals_each_image_alone_on_every_run():
    files = [po.pil_png(image(10 + i, 512, 512, 3 + i % 2)) for i in range(6)]
    files += [po.png_file(300, 200, 4, 16, zlib.compress(raw_of(image(20, 300, 200, 4, 16)))),
              po.pil_png(image(21, 1, 1, 1)), po.pil_png(image(22, 1024, 1024, 4)),
              po.png_file(61, 513, 3, 8, zlib.compress(raw_of(image(23, 61, 513, 3)), 1), split=7)]
    batch = [load(files, 512, True) for _ in range(3)]
    assert all(torch.equal(b, batch[0]) for b in batch[1:])
    for i, f in enumerate(files):
        assert torch.equal(load([f], 512, True)[0], batch[0][i])
        assert torch.equal(batch[0][i], po.chain(f, 512, True))


def test_malformed_streams_fail_alone():
    from panic3d_b200 import imageio as pio
    mal = po.malformed_streams()
    files, codes = [], []
    for name, (stream, n, code) in mal.items():
        files.append(po.png_file(1, n - 1, 1, 8, stream))
        codes.append(code)
    filt = bytes([5]) + bytes(20)
    files.append(po.png_file(1, 20, 1, 8, zlib.compress(filt)))
    codes.append(11)
    good = [po.png_file(5, 30, 1, 8, zlib.compress(raw_of(image(30 + i, 5, 30, 1)), i)) for i in range(4)]
    order = list(range(len(files) + len(good)))
    np.random.default_rng(0).shuffle(order)
    allf = files + good
    allc = codes + [0] * len(good)
    batch = [allf[k] for k in order]
    want_codes = [allc[k] for k in order]
    out, status, names = pio.decode_batch(batch, size=16, white_background=True, device=DEV)
    out = out.cpu()
    assert status == want_codes
    for j, k in enumerate(order):
        if allc[k] == 0:
            assert torch.equal(out[j], po.chain(allf[k], 16, True))
        else:
            assert (out[j] == 0).all()
    with pytest.raises(RuntimeError) as e:
        pio.load_images(batch, size=16, white_background=True, device=DEV)
    for j, c in enumerate(want_codes):
        assert (f'<bytes #{j}>: ' in str(e.value)) == (c != 0)
