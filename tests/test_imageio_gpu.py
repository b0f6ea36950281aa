"""GPU: device half of the image output path (SURVEY 8f-4): quantise + PNG filter kernel against the numpy oracle (byte for
byte), files written by the asynchronous writer decoded with PIL, flat weight file onto the device."""
import os

import numpy as np
import pytest
import torch

from oracle import imageio_oracle as io_orc
from tests.helpers import TinyG, synth_image

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


@pytest.mark.parametrize('n,c,h,w', [(1, 3, 40, 37), (2, 4, 33, 64), (3, 1, 17, 5), (2, 3, 512, 512)])
def test_scanlines_equal_the_oracle_byte_for_byte(n, c, h, w):
    import panic3d_b200.imageio as pio
    img = torch.stack([synth_image(10 * c + i, c, h, w) for i in range(n)])
    scan, shape = pio.png_scanlines(img.to(DEV))
    assert shape == (h, w, c) and tuple(scan.shape) == (n, h * (1 + w * c))
    pix = io_orc.quantize(img)
    assert np.array_equal(pio.to_uint8(img.to(DEV)).cpu().numpy(), pix)
    for i in range(n):
        want = io_orc.png_filter_rows(pix[i])
        got = scan[i].cpu().numpy().reshape(h, 1 + w * c)
        assert np.array_equal(got[:, 0], want[:, 0]), 'filter choice'
        assert np.array_equal(got, want)


def test_special_values_and_filter_ties():
    """NaN -> 0, +-inf clamped, -0 -> 0, 1 -> 255 and 0.99999994 -> 254 (truncation, not rounding), in both kernels; and
    rows where filters tie (an all-zero first row: every sum 0; constant rows: Up and Paeth both 0), which go to the
    first minimum in the order none, sub, up, average, paeth."""
    import panic3d_b200.imageio as pio
    special = torch.tensor([float('nan'), float('inf'), float('-inf'), -0.0, 1.0, 0.99999994, 0.5, -1e-30, 2.0, 0.2])
    want = np.array([0, 255, 0, 0, 255, 254, 127, 0, 255, 51], np.uint8)
    w = 40
    img = torch.zeros(1, 3, 5, w)
    img[0, :, 1] = special.repeat(4)[None].roll(1, 1) * torch.ones(3, 1)
    img[0, 0, 1] = special.repeat(4)
    img[0, :, 2] = 0.5
    img[0, :, 3] = 0.5
    img[0, :, 4] = torch.linspace(0, 1, w)
    pix = io_orc.quantize(torch.nan_to_num(img, nan=0.0))
    assert np.array_equal(pix[0, 1, :, 0], np.tile(want, 4))
    assert np.array_equal(pio.to_uint8(img.to(DEV)).cpu().numpy(), pix)
    scan, _ = pio.png_scanlines(img.to(DEV))
    got = scan[0].cpu().numpy().reshape(5, 1 + w * 3)
    ref = io_orc.png_filter_rows(pix[0])
    assert list(ref[:, 0][[0, 3]]) == [0, 2]
    assert np.array_equal(got, ref)


def test_rows_beyond_the_shared_memory_staging_use_filter_none():
    import panic3d_b200.imageio as pio
    img = torch.rand(1, 4, 2, 30000)
    scan, _ = pio.png_scanlines(img.to(DEV))
    got = scan[0].cpu().numpy().reshape(2, 1 + 30000 * 4)
    assert (got[:, 0] == 0).all() and np.array_equal(got[:, 1:].reshape(2, 30000, 4), io_orc.quantize(img)[0])


def test_async_writer_files_decode_to_the_reference_pixels(tmp_path):
    from PIL import Image
    import panic3d_b200.imageio as pio
    imgs = torch.stack([synth_image(40 + i, 3, 128, 96) for i in range(6)])
    xyz = torch.stack([synth_image(50 + i, 3, 64, 64) for i in range(2)]) * 0.7 - 0.35
    wts = torch.stack([synth_image(60 + i, 1, 64, 64) for i in range(2)])
    with pio.AsyncImageWriter(threads=3, level=2) as w:
        w.save(imgs.to(DEV), [tmp_path / f'rgb{i}.png' for i in range(6)])                   # batch
        w.save(imgs[0].to(DEV), tmp_path / 'single.png')                                     # (C,H,W), like I(t).save(fn)
        w.save(imgs[1, 0].to(DEV), tmp_path / 'gray.png')                                    # (H,W) -> mode L
        for i in range(2):
            w.save_xyza(xyz[i:i + 1].to(DEV), wts[i:i + 1].to(DEV), 0.7, tmp_path / f'xyza{i}.png')
        w.flush()
        pix = io_orc.quantize(imgs)
        for i in range(6):
            assert np.array_equal(np.asarray(Image.open(tmp_path / f'rgb{i}.png')), pix[i])
        assert np.array_equal(np.asarray(Image.open(tmp_path / 'single.png')), pix[0])
        g = Image.open(tmp_path / 'gray.png')
        assert g.mode == 'L' and np.array_equal(np.asarray(g), pix[1][:, :, 0])
        for i in range(2):
            im = Image.open(tmp_path / f'xyza{i}.png')
            want = io_orc.quantize(io_orc.xyza(xyz[i:i + 1], wts[i:i + 1], 0.7))[0]
            got = np.asarray(im).astype(np.int32)
            assert im.mode == 'RGBA'
            # (x + bw/2) * (1/bw) on the device vs the eager division: a value within one ulp of a level boundary may land
            # on the other side - never more than one level, on a vanishing share of the pixels
            d = np.abs(got - want.astype(np.int32))
            assert d.max() <= 1 and (d > 0).mean() < 1e-3
        with pytest.raises(RuntimeError, match='PNG'):
            w.save(imgs[0].to(DEV), tmp_path / 'x.jpg')


def test_weight_file_loads_onto_the_device(tmp_path):
    import panic3d_b200.weights as pw
    torch.manual_seed(1)
    G = TinyG(8, depth=2, rendering_kwargs={'box_warp': 0.7})
    pw.export_generator(G, tmp_path / 'g.p3dw')
    tensors, meta = pw.load_weights(tmp_path / 'g.p3dw', device=DEV)
    ref = dict(list(G.named_parameters()) + list(G.named_buffers()))
    for k, t in ref.items():
        assert tensors[k].is_cuda and torch.equal(tensors[k].cpu(), t.detach()), k
    base = {t.untyped_storage().data_ptr() for t in tensors.values() if t.numel()}
    assert len(base) == 1                                                                  # one device buffer, views into it
    G2 = pw.build_generator(tmp_path / 'g.p3dw', TinyG, device=DEV)
    assert all(torch.equal(a.cpu(), b) for a, b in zip(G2.state_dict().values(), G.state_dict().values()))
