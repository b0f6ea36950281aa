"""GPU: the device PNG decoder (csrc/png_inflate.cu) along the paths the zlib- and PIL-written files of
tests/test_png_decode_gpu.py never take, each output element for element against tests/png_oracle.py's chain and each
status code exactly.

* Streams zlib never writes (png_oracle.path_streams): dynamic -> fixed -> fixed -> dynamic -> stored -> fixed blocks with
  a match across every seam, 15-bit literal and distance codes at HLIT = 286 and HDIST = 30, a repeat 16 from the literal
  into the distance lengths, and a repeat 18 of 138.
* A 256 x 256 RGBA image whose pixel (x, y) has value x and alpha y, on white, at 8 and 16 bits (16-bit low bytes are
  noise): every (value, alpha) pair of the integer composite.
* Heights 31-33 and 63-65 with each filter forced on the rows either side of the unfilter's 32-row band seams, for every
  type and depth.
* Nearest resizes to 30,000 and 32,768 columns and rows, where a float accumulation of the source index goes wrong.
* Every malformed stream (png_oracle.malformed_streams and refusal_streams) and three refused job-table entries, shuffled
  into batches of good images: the failures give zeros and their codes, the good images equal the oracle.
The file is the target of `tests/run_png_mutations.py png_inflate`, which runs it once per mutant."""
import zlib

import numpy as np
import pytest
import torch

from tests import png_oracle as po

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TYPES = [(1, 8), (3, 8), (4, 8), (3, 16), (4, 16)]


@pytest.fixture(scope='module', autouse=True)
def built():
    import __graft_entry__ as g
    g.build()


def check(files, size=None, white=False):
    from panic3d_b200 import imageio as pio
    got = pio.load_images(files, size=size, white_background=white, device=DEV).cpu()
    for i, f in enumerate(files):
        want = po.chain(f, size, white)
        assert torch.equal(got[i], want), (i, size, white, (got[i] != want).sum().item())


@pytest.mark.parametrize('name', list(po.path_streams()))
def test_streams_zlib_never_writes(name):
    h, w, c, depth, stream, raw = po.path_streams()[name]
    f = po.png_file(h, w, c, depth, stream)
    check([f])
    check([f], (2, 777), True)


@pytest.mark.parametrize('depth', [8, 16])
def test_every_value_and_alpha_on_white(depth):
    y, x = np.meshgrid(np.arange(256), np.arange(256), indexing='ij')
    pix = np.stack([x, 255 - x, (x * 7 + y) & 255, y], -1)
    if depth == 16:
        pix = pix << 8 | np.random.default_rng(5).integers(0, 256, pix.shape)
    pix = pix.astype(np.uint16 if depth == 16 else np.uint8)
    f = po.png_file(256, 256, 4, depth, zlib.compress(po.filter_rows(pix, np.arange(256) % 5)))
    check([f], None, True)
    check([f], None, False)


@pytest.mark.parametrize('c,depth', TYPES)
def test_filters_on_the_band_seams(c, depth):
    g = np.random.default_rng(c * 100 + depth)
    w, top = 19, (1 << depth) - 1
    files = []
    for h in (31, 32, 33, 63, 64, 65):
        pix = g.integers(0, top + 1, (h, w, c)).astype(np.uint16 if depth == 16 else np.uint8)
        for t in range(5):
            types = g.integers(0, 5, h)
            types[[r for r in range(h) if r % 32 in (0, 31)]] = t             # rows 31 | 32 and 63 | 64: the seams
            files.append(po.png_file(h, w, c, depth, zlib.compress(po.filter_rows(pix, types))))
    check(files, (65, w))
    if c == 4:
        check(files, (65, w), True)


@pytest.mark.parametrize('n_in,n_out', [(4097, 32768), (1000, 30000)])
def test_nearest_resize_to_the_largest_sides(n_in, n_out):
    g = np.random.default_rng(n_in)
    row = po.png_file(1, n_in, 1, 8, zlib.compress(bytes([0]) + g.integers(0, 256, n_in).astype(np.uint8).tobytes()))
    check([row], (1, n_out))
    col = po.png_file(n_in, 1, 1, 8, zlib.compress(bytes(np.stack([np.zeros(n_in, np.int64), g.integers(0, 256, n_in)], 1)
                                                         .astype(np.uint8).tobytes())))
    check([col], (n_out, 2))


def good_images(k):
    g = np.random.default_rng(7)
    return [po.png_file(5, 30, 1, 8, zlib.compress(po.filter_rows(g.integers(0, 256, (5, 30, 1)).astype(np.uint8),
                                                                   g.integers(0, 5, 5)), i % 10)) for i in range(k)]


def test_malformed_streams_fail_alone():
    from panic3d_b200 import imageio as pio
    mal = dict(po.malformed_streams())
    mal.update(po.refusal_streams())
    files = [po.png_file(1, n - 1, 1, 8, s) for s, n, _ in mal.values()]
    codes = [code for _, _, code in mal.values()]
    good = good_images(8)
    allf, allc = files + good, codes + [0] * len(good)
    order = np.random.default_rng(1).permutation(len(allf))
    out, status, _ = pio.decode_batch([allf[k] for k in order], size=16, white_background=True, device=DEV)
    out = out.cpu()
    assert status == [allc[k] for k in order], [(list(mal)[k] if k < len(mal) else 'good', allc[k], s)
                                                for k, s in zip(order, status) if allc[k] != s]
    for j, k in enumerate(order):
        if allc[k]:
            assert (out[j] == 0).all()
        else:
            assert torch.equal(out[j], po.chain(allf[k], 16, True))


def test_refused_jobs_fail_alone():
    """check_job's three refusals, one job each, among good jobs:
    channels 2 (outside the envelope),
    input span past the buffer,
    workspace offset not 16-byte aligned."""
    from panic3d_b200 import imageio as pio
    files = good_images(6)
    st, _ = pio._stage(files, 16, True, DEV)
    jobs = (pio.PngDecodeJob * len(files)).from_address(st['pinned'].data_ptr())
    jobs[1].channels = 2
    jobs[3].in_bytes = 1 << 40
    jobs[4].ws_offset += 8
    out, status = pio._decode_staged(st)
    assert status.cpu().tolist() == [0, 1, 0, 1, 1, 0]
    out = out.cpu()
    for i, f in enumerate(files):
        assert torch.equal(out[i], torch.zeros_like(out[i]) if i in (1, 3, 4) else po.chain(f, 16, True)), i
