"""CPU: the host half of the image output path (SURVEY 8f-4) - PNG container + zlib on the thread pool, the numpy oracle of
the device filter kernel, the flat weight file.  No GPU compute here; the device kernels are tested in test_imageio_gpu.py."""
import io
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import imageio_oracle as io_orc
from tests.helpers import TinyG, synth_image


@pytest.fixture(scope='module')
def built():
    import __graft_entry__ as g
    g.build()


@pytest.mark.parametrize('c,h,w', [(3, 40, 37), (4, 33, 64), (1, 17, 5)])
def test_oracle_filters_round_trip_and_decode_with_pil(built, c, h, w):
    from PIL import Image
    import panic3d_b200.imageio as pio
    pix = io_orc.quantize(synth_image(c, c, h, w))[0]
    scan = io_orc.png_filter_rows(pix)
    assert np.array_equal(io_orc.png_unfilter(scan, h, w, c), pix)          # the filters invert
    assert len(set(scan[:, 0].tolist())) >= 2                               # more than one filter type in play
    for level in (0, 3, 9):
        png = pio.encode_png(scan, h, w, c, level=level)
        im = Image.open(io.BytesIO(png))
        im.load()
        assert im.mode == {1: 'L', 3: 'RGB', 4: 'RGBA'}[c] and im.size == (w, h)
        assert np.array_equal(np.asarray(im).reshape(h, w, c), pix)         # PIL decodes the exact pixels


def test_quantisation_rule():
    t = torch.tensor([[[-0.5, 0.0, 0.5 / 255, 0.999999 / 255 * 2, 127.5 / 255, 254.999 / 255, 1.0, 7.0]]])
    assert io_orc.quantize(t)[0, 0, :, 0].tolist() == [0, 0, 0, 1, 127, 254, 255, 255]   # clamp, x255, truncate


def test_writer_pool_writes_every_file_atomically(built, tmp_path):
    from PIL import Image
    import panic3d_b200.imageio as pio
    imgs = [io_orc.quantize(synth_image(s, 3, 24 + s, 31))[0] for s in range(12)]
    with pio.AsyncImageWriter(threads=3, level=1) as w:
        for i, pix in enumerate(imgs):
            w.submit_host(io_orc.png_filter_rows(pix), pix.shape[0], pix.shape[1], 3, tmp_path / f'v{i:02d}.png')
        w.flush()
        assert sorted(os.listdir(tmp_path)) == [f'v{i:02d}.png' for i in range(12)]      # no .tmp left behind
        for i, pix in enumerate(imgs):
            assert np.array_equal(np.asarray(Image.open(tmp_path / f'v{i:02d}.png')), pix)
        w.submit_host(io_orc.png_filter_rows(imgs[0]), imgs[0].shape[0], imgs[0].shape[1], 3, tmp_path / 'no_such_dir' / 'x.png')
        with pytest.raises(RuntimeError, match='cannot write'):
            w.flush()
        w.flush()                                                                         # the failure was reported once


def test_bad_arguments_fail_loudly(built):
    import ctypes as C
    import panic3d_b200.imageio as pio
    from panic3d_b200 import _lib
    L = _lib.lib()
    assert L.p3d_png_scanline_bytes(4, 5, 3) == 4 * 16 and L.p3d_png_scanline_bytes(0, 5, 3) == 0
    n = C.c_size_t(0)
    buf = np.zeros(64, np.uint8)
    assert L.p3d_png_encode_host(buf.ctypes.data, 4, 5, 2, 3, buf.ctypes.data, 64, C.byref(n)) != 0     # 2 channels: no PNG mode here
    assert L.p3d_png_encode_host(buf.ctypes.data, 4, 5, 3, 3, buf.ctypes.data, 8, C.byref(n)) == -3 and n.value > 8   # P3D_EWORKSPACE + size
    h = C.c_void_p()
    assert L.p3d_png_writer_create(0, 3, C.byref(h)) != 0 and L.p3d_png_writer_create(2, 11, C.byref(h)) != 0
    with pytest.raises(RuntimeError, match='CUDA'):
        pio.png_scanlines(torch.zeros(3, 8, 8))
    with pytest.raises(RuntimeError, match='CUDA'):
        pio.to_uint8(torch.zeros(3, 8, 8))


def test_async_pickle_writer(tmp_path):
    import panic3d_b200.imageio as pio
    w = pio.AsyncPickleWriter()
    obj = {'verts': np.arange(30, dtype=np.float32).reshape(10, 3), 'faces': np.arange(12).reshape(4, 3)}
    w.pdump(obj, tmp_path / 'mc.pkl')
    w.flush()
    back = pickle.load(open(tmp_path / 'mc.pkl', 'rb'))
    assert np.array_equal(back['verts'], obj['verts']) and np.array_equal(back['faces'], obj['faces'])
    w.pdump(obj, tmp_path / 'missing' / 'mc.pkl')
    with pytest.raises(OSError):
        w.flush()


def test_weight_file_round_trip_is_bit_exact(tmp_path):
    import panic3d_b200.weights as pw
    torch.manual_seed(0)
    rk = {'box_warp': 0.7, 'ray_start': 0.5, 'ray_end': 1.5, 'depth_resolution': 48, 'depth_resolution_importance': 48, 'clamp_mode': 'softplus',
          'white_back': True, 'sr_antialias': None}
    G = TinyG(6, depth=3, rendering_kwargs=rk)
    G.neural_rendering_resolution = 128
    path = tmp_path / 'g.p3dw'
    nbytes = pw.export_generator(G, path)
    assert os.path.getsize(path) == nbytes and nbytes % pw.ALIGN == 0
    tensors, meta = pw.load_weights(path, device='cpu')
    ref = dict(list(G.named_parameters()) + list(G.named_buffers()))
    assert list(tensors) == list(ref)
    for k, t in ref.items():
        assert tensors[k].dtype == t.dtype and tensors[k].shape == t.shape and torch.equal(tensors[k], t.detach()), k
    assert meta['init_args'] == [6] and meta['init_kwargs']['depth'] == 3 and meta['rendering_kwargs'] == rk
    G2 = pw.build_generator(path, TinyG, device='cpu', force_sigmoid=True)
    assert all(torch.equal(a, b) for a, b in zip(G.state_dict().values(), G2.state_dict().values()))
    assert G2.force_sigmoid and not G2.training and not any(p.requires_grad for p in G2.parameters())
    assert G2.neural_rendering_resolution == 128 and G2.rendering_kwargs['depth_resolution'] == 96 and G2.rendering_kwargs['box_warp'] == 0.7
    # require_all: a module with a tensor the file lacks must fail like misc.copy_params_and_buffers(require_all=True)
    G3 = TinyG(6, depth=4, rendering_kwargs=rk)
    with pytest.raises(RuntimeError, match='require_all'):
        pw.load_into(G3, path, device='cpu')
    pw.load_into(G3, path, device='cpu', require_all=False)
    with open(path, 'r+b') as f:
        f.truncate(nbytes - 100)
    with pytest.raises(RuntimeError, match='truncated'):
        pw.load_weights(path, device='cpu')
