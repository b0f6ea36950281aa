"""Image output behind the renderer - the H100 replacement for ``I(tensor).save(fn)`` at the end of every view of the
reference's eval sweep (``_scripts/eval/generate.py:141-148``; ``_util/twodee_v1.py:36-91,174-185,732-760``; SURVEY.md 8f-4).

The reference converts on the host: a blocking ``.cpu()`` of the fp32 image, ``to_pil_image(t.float().clamp(0,1))``
(x255, truncate) and PIL's PNG encoder, on the same Python thread that drives the GPU; with eight GPUs gathering views to
rank 0 that thread is the bottleneck.  Here quantisation, channel interleave and PNG scan-line filtering run on the device
(``p3d_image_to_png_scanlines``), the 8-bit stream is copied to pinned memory on a side stream, and a pool of host threads
(``p3d_png_writer_*``) deflates and writes the files.  The decoded pixels equal the reference's files (the byte stream does
not: filter choice and deflate level are not part of the image).

    ``to_uint8(img)``                       (C,H,W) / (N,C,H,W) float -> (N,H,W,C) uint8, the pixels ``I(img).pil()`` holds
    ``AsyncImageWriter(threads, level)``    ``.save(img, fn)``          drop-in for ``I(img).save(fn)`` (returns at once)
                                            ``.save_xyza(xyz, w, bw, fn)`` for ``I(cat([(xyz+bw/2)/bw, w])).save(fn)``
                                            (generate.py:141-147) without materialising the 4-channel image
                                            ``.flush()``                all files on disk (raises if one failed)
    ``load_images(sources, size, white_background)``  PNG files -> (N,C,H,W) float32 on the GPU: the training set's
                                            ``I(path).resize(size)[.convert('RGBA').bg('w').convert('RGB')].t()``
    ``AsyncPickleWriter``                   ``uutil.pdump(obj, fn)`` (generate.py:104-105, the marching-cubes dict) off-thread

No CPU path for the device kernels: images must be CUDA tensors and ``load_images`` decodes on a CUDA device (the numpy
restatements are ``oracle/imageio_oracle.py`` and ``tests/png_oracle.py``, tests only).  ``encode_png`` / ``submit_host`` are pure host code (zlib) and work anywhere.
"""
from __future__ import annotations

import ctypes as C
import os
import pickle
import threading

import torch

from . import _lib

_VP = C.c_void_p
_lib.register_protos({
    'p3d_png_scanline_bytes': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    'p3d_image_to_png_scanlines': (C.c_int, [_VP, _VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP, _VP, _VP, _VP]),
    'p3d_image_to_u8': (C.c_int, [_VP, _VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP, _VP, _VP, _VP]),
    'p3d_png_encode_bound': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    'p3d_png_encode_host': (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP, C.c_size_t, C.POINTER(C.c_size_t)]),
    'p3d_png_writer_create': (C.c_int, [C.c_int32, C.c_int32, C.POINTER(_VP)]),
    'p3d_png_writer_submit': (C.c_int, [_VP, _VP, C.c_int32, C.c_int32, C.c_int32, C.c_char_p, _VP]),
    'p3d_png_writer_submit_host': (C.c_int, [_VP, _VP, C.c_int32, C.c_int32, C.c_int32, C.c_char_p]),
    'p3d_png_writer_flush': (C.c_int, [_VP, C.POINTER(C.c_int32)]),
    'p3d_png_device_bound': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    'p3d_png_device_workspace_bytes': (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    'p3d_png_encode_device': (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP, C.c_size_t, _VP, C.c_size_t, _VP, _VP]),
    'p3d_png_writer_submit_encoded': (C.c_int, [_VP, _VP, _VP, C.c_int32, C.c_int32, C.c_int32, C.c_char_p, _VP]),
    'p3d_png_writer_destroy': (C.c_int, [_VP]),
})


class PngInfo(C.Structure):
    """Mirror of ``p3d_png_info`` (include/p3d_imageio.h)."""
    _fields_ = [('h', C.c_int32), ('w', C.c_int32), ('channels', C.c_int32), ('depth', C.c_int32), ('n_idat', C.c_int32),
                ('reserved', C.c_int32), ('stream_bytes', C.c_uint64)]


class PngDecodeJob(C.Structure):
    """Mirror of ``p3d_png_decode_job`` (include/p3d_imageio.h)."""
    _fields_ = [('in_offset', C.c_uint64), ('in_bytes', C.c_uint64), ('ws_offset', C.c_uint64), ('h', C.c_int32),
                ('w', C.c_int32), ('channels', C.c_int32), ('depth', C.c_int32), ('slot', C.c_int32), ('reserved', C.c_int32)]


_lib.register_protos({
    'p3d_png_inspect': (C.c_int, [_VP, C.c_size_t, C.POINTER(PngInfo), _VP]),
    'p3d_png_decode_workspace_bytes': (C.c_size_t, [C.c_int32] * 6),
    'p3d_png_decode_device': (C.c_int, [_VP, C.c_size_t, _VP, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _VP, C.c_size_t,
                                        _VP, _VP, _VP]),
    'p3d_png_inflate_host': (C.c_int, [_VP, C.c_size_t, _VP, C.c_size_t]),
})

# P3D_PNG_* status codes of p3d_png_decode_device
PNG_STATUS = {
    1: 'job outside the buffers or the envelope', 2: 'bad zlib header', 3: 'bad deflate block (type 3, or stored LEN/NLEN)',
    4: 'bad Huffman code lengths', 5: 'invalid Huffman code or symbol', 6: 'match distance past the start of the output',
    7: 'decompresses to more than h*(1+w*bytes per pixel) bytes', 8: 'decompresses to fewer than h*(1+w*bytes per pixel) bytes',
    9: 'zlib stream truncated', 10: 'Adler-32 mismatch', 11: 'scan-line filter byte above 4',
}


def _canon(img, name='image'):
    """The shapes ``I.__init__`` accepts for a torch tensor (twodee_v1.py:71-91): (H,W), (C,H,W), (1,C,H,W) - plus a
    batch (N,C,H,W), which the reference cannot save in one call."""
    if not (torch.is_tensor(img) and img.is_cuda):
        raise RuntimeError(f'panic3d_b200.imageio: {name} must be a CUDA tensor (there is no CPU path)')
    if img.dim() == 2:
        img = img[None, None]
    elif img.dim() == 3:
        img = img[None]
    if img.dim() != 4:
        raise RuntimeError(f'panic3d_b200.imageio: {name} must be (H,W), (C,H,W) or (N,C,H,W), got {tuple(img.shape)}')
    if img.dtype == torch.bool:
        img = img.float()
    return img.detach().float().contiguous()


def _affine(scale, shift, c, dev):
    if scale is None and shift is None:
        return None, None
    s = torch.ones(4) if scale is None else torch.as_tensor(scale, dtype=torch.float32).flatten()
    t = torch.zeros(4) if shift is None else torch.as_tensor(shift, dtype=torch.float32).flatten()
    pad = lambda v, fill: torch.cat([v, torch.full((4 - len(v),), fill)])[:4].contiguous()
    return pad(s, 1.0), pad(t, 0.0)                                           # host arrays: read by the launch, not the kernel


def png_scanlines(img, extra=None, scale=None, shift=None):
    """(N,C,H,W) float CUDA image(s) -> (N, H*(1+W*C)) uint8 CUDA tensor of filtered PNG scan-lines.
    ``extra``: optional (N,1,H,W) plane appended as the last channel; ``scale`` / ``shift``: per-channel affine
    ``(x + shift) * scale`` applied before the clamp."""
    img = _canon(img)
    N, c, H, W = img.shape
    if extra is not None:
        extra = _canon(extra, 'extra')
        if tuple(extra.shape) != (N, 1, H, W):
            raise RuntimeError(f'panic3d_b200.imageio: extra must be {(N, 1, H, W)}, got {tuple(extra.shape)}')
        c += 1
    if c not in (1, 3, 4):
        raise RuntimeError(f'panic3d_b200.imageio: {c} channels; PNG modes L / RGB / RGBA need 1, 3 or 4 (twodee_v1.py:88)')
    s, t = _affine(scale, shift, c, img.device)
    L = _lib.lib()
    out = torch.empty((N, L.p3d_png_scanline_bytes(H, W, c)), device=img.device, dtype=torch.uint8)
    with torch.cuda.device(img.device):
        _lib.check(L.p3d_image_to_png_scanlines(img.data_ptr(), _lib.ptr(extra), N, c, H, W, _lib.ptr(s), _lib.ptr(t), out.data_ptr(),
                                                _lib.stream_ptr(img.device)))
    return out, (H, W, c)


def to_uint8(img, extra=None, scale=None, shift=None):
    """(N,C,H,W) float CUDA image(s) -> (N,H,W,C) uint8: ``clamp(0,1) * 255`` truncated, the pixels ``I(img).pil()`` holds."""
    img = _canon(img)
    N, c, H, W = img.shape
    if extra is not None:
        extra = _canon(extra, 'extra')
        c += 1
    s, t = _affine(scale, shift, c, img.device)
    out = torch.empty((N, H, W, c), device=img.device, dtype=torch.uint8)
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().p3d_image_to_u8(img.data_ptr(), _lib.ptr(extra), N, c, H, W, _lib.ptr(s), _lib.ptr(t), out.data_ptr(),
                                              _lib.stream_ptr(img.device)))
    return out


def png_encode_device(scan, shape):
    """(N, H*(1+W*C)) uint8 CUDA scan-lines (``png_scanlines``' output) -> ``(files, lens)``: an (N, bound) uint8 CUDA
    tensor whose row i starts with PNG file i, and its (N,) int64 lengths, both on the device; deflated on the GPU
    (``p3d_png_encode_device``) on the current stream.  Workspace and output come from torch's caching allocator."""
    H, W, c = shape
    L = _lib.lib()
    N = scan.shape[0]
    bound, ws_bytes = L.p3d_png_device_bound(H, W, c), L.p3d_png_device_workspace_bytes(N, H, W, c)
    if not bound or not ws_bytes:
        raise RuntimeError(f'panic3d_b200.imageio: {N} image(s) of {H}x{W}x{c} are outside the device encoder\'s envelope')
    ws = torch.empty(ws_bytes, device=scan.device, dtype=torch.uint8)
    files = torch.empty((N, bound), device=scan.device, dtype=torch.uint8)
    lens = torch.empty(N, device=scan.device, dtype=torch.int64)
    with torch.cuda.device(scan.device):
        _lib.check(L.p3d_png_encode_device(scan.contiguous().data_ptr(), N, H, W, c, ws.data_ptr(), ws_bytes, files.data_ptr(), bound,
                                           lens.data_ptr(), _lib.stream_ptr(scan.device)))
    return files, lens


def png_inspect(data):
    """PNG file bytes -> ``PngInfo`` (``p3d_png_inspect``); RuntimeError naming the field for anything unsupported."""
    import numpy as np
    buf = np.frombuffer(data, dtype=np.uint8)
    info = PngInfo()
    _lib.check(_lib.lib().p3d_png_inspect(buf.ctypes.data, buf.size, C.byref(info), None))
    return info


def load_images(sources, size=None, white_background=False, device=None):
    """PNG files (paths or ``bytes``) -> float32 (N, C, H, W) on the device, decoded on the GPU (``p3d_png_decode_device``).

    Equal, element for element, to ``torch.stack([I(src).resize(size).t() ...])`` - with ``white_background``, to
    ``I(src).resize(size).convert('RGBA').bg('w').convert('RGB').t()`` (C = 3) - where ``I`` is the reference's
    ``_util/twodee_v1.py`` image class: PIL's nearest resize, PIL's integer alpha composite and ``to_tensor``'s / 255.
    ``size``: an int (square) or (H, W); None keeps the files' size, which must then be the same for all of them.
    Without ``white_background`` every file must have the same channel count (L: 1, RGB: 3, RGBA: 4).

    The files are read and inspected on the host, their IDAT payloads packed into one pinned buffer behind the job
    table, and one host-to-device copy and one decode launch sequence run on the current stream.  RuntimeError names
    every file that is refused or fails to decode.  There is no host fallback."""
    out, codes, names = decode_batch(sources, size, white_background, device)
    bad = [f'{names[i]}: {PNG_STATUS.get(s, f"status {s}")}' for i, s in enumerate(codes) if s]
    if bad:
        raise RuntimeError('panic3d_b200.imageio.load_images: ' + '; '.join(bad))
    return out


def decode_batch(sources, size=None, white_background=False, device=None):
    """``load_images`` without the raise on a failed decode: ``(out, status, names)``, with one ``P3D_PNG_*`` code per
    source (``PNG_STATUS`` names them) and the failed images' outputs zeroed.  Refused files still raise."""
    st, names = _stage(sources, size, white_background, device)
    out, status = _decode_staged(st)
    return out, status.cpu().tolist(), names


def _stage(sources, size, white_background, device):
    """Read and inspect the files and pack the job table and their zlib streams into one pinned buffer."""
    import numpy as np
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    if dev.type != 'cuda':
        raise RuntimeError('panic3d_b200.imageio.load_images: the decoder runs on a CUDA device (there is no CPU path)')
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    names, datas = [], []
    for i, src in enumerate(sources):
        if isinstance(src, (bytes, bytearray, memoryview)):
            names.append(f'<bytes #{i}>')
            datas.append(np.frombuffer(src, dtype=np.uint8))
        else:
            names.append(os.fspath(src))
            with open(names[-1], 'rb') as f:
                datas.append(np.frombuffer(f.read(), dtype=np.uint8))
    n = len(datas)
    if n < 1:
        raise RuntimeError('panic3d_b200.imageio.load_images: no sources')
    L = _lib.lib()
    infos, bad = [], []
    for name, buf in zip(names, datas):
        info = PngInfo()
        if L.p3d_png_inspect(buf.ctypes.data, buf.size, C.byref(info), None) != 0:
            bad.append(f'{name}: {L.p3d_last_error().decode("utf-8", "replace")}')
        infos.append(info)
    if bad:
        raise RuntimeError('panic3d_b200.imageio.load_images: ' + '; '.join(bad))
    if size is None:
        shapes = {(f.h, f.w) for f in infos}
        if len(shapes) != 1:
            raise RuntimeError(f'panic3d_b200.imageio.load_images: files of sizes {sorted(shapes)} need a size to resize to')
        out_h, out_w = shapes.pop()
    else:
        out_h, out_w = (size, size) if isinstance(size, int) else (int(size[0]), int(size[1]))
    if white_background:
        c = 3
    else:
        chans = {f.channels for f in infos}
        if len(chans) != 1:
            raise RuntimeError(f'panic3d_b200.imageio.load_images: files with {sorted(chans)} channels cannot be stacked '
                               '(white_background=True gives 3 channels for all of them)')
        c = chans.pop()
    jobs = (PngDecodeJob * n)()
    head = C.sizeof(jobs)
    off, ws_total = 0, 0
    for i, f in enumerate(infos):
        ws = L.p3d_png_decode_workspace_bytes(f.h, f.w, f.channels, f.depth, out_h, out_w)
        if not ws:
            raise RuntimeError(f'panic3d_b200.imageio.load_images: {names[i]}: output {out_h}x{out_w} outside the envelope')
        jobs[i] = PngDecodeJob(off, f.stream_bytes, ws_total, f.h, f.w, f.channels, f.depth, i, 0)
        off += f.stream_bytes
        ws_total += ws
    pinned = torch.empty(head + off, dtype=torch.uint8, pin_memory=True)
    base = pinned.data_ptr()
    C.memmove(base, C.addressof(jobs), head)
    for i, (buf, job) in enumerate(zip(datas, jobs)):
        _lib.check(L.p3d_png_inspect(buf.ctypes.data, buf.size, C.byref(infos[i]), base + head + job.in_offset))
    st = dict(dev=dev, pinned=pinned, head=head, in_bytes=off, n=n, out_h=out_h, out_w=out_w, c=c, white=int(bool(white_background)),
              ws_bytes=ws_total)
    return st, names


def _decode_staged(st):
    """One H2D copy of the packed jobs and streams, then the decode launch sequence, on the current stream of st['dev']."""
    dev = st['dev']
    with torch.cuda.device(dev):
        staged = st['pinned'].to(dev, non_blocking=True)
        ws = torch.empty(st['ws_bytes'], dtype=torch.uint8, device=dev)
        out = torch.empty((st['n'], st['c'], st['out_h'], st['out_w']), dtype=torch.float32, device=dev)
        status = torch.empty(st['n'], dtype=torch.int32, device=dev)
        _lib.check(_lib.lib().p3d_png_decode_device(staged.data_ptr() + st['head'], st['in_bytes'], staged.data_ptr(), st['n'], st['out_h'],
                                                    st['out_w'], st['c'], st['white'], ws.data_ptr(), st['ws_bytes'], out.data_ptr(),
                                                    status.data_ptr(), _lib.stream_ptr(dev)))
    return out, status


def encode_png(scanlines, h, w, c, level=3):
    """Filtered scan-lines (bytes / uint8 CPU tensor / numpy array) -> PNG file bytes.  Pure host code (zlib)."""
    import numpy as np
    buf = np.ascontiguousarray(np.frombuffer(scanlines, dtype=np.uint8) if isinstance(scanlines, (bytes, bytearray)) else
                               (scanlines.numpy() if torch.is_tensor(scanlines) else scanlines), dtype=np.uint8).reshape(-1)
    L = _lib.lib()
    if buf.size != L.p3d_png_scanline_bytes(h, w, c):
        raise RuntimeError(f'panic3d_b200.imageio: {buf.size} scan-line bytes for a {h}x{w}x{c} image, expected {L.p3d_png_scanline_bytes(h, w, c)}')
    cap = L.p3d_png_encode_bound(h, w, c)
    out = np.empty(cap, dtype=np.uint8)
    n = C.c_size_t(0)
    _lib.check(L.p3d_png_encode_host(buf.ctypes.data, h, w, c, int(level), out.ctypes.data, cap, C.byref(n)))
    return out[:n.value].tobytes()


def _png_name(fn):
    fn = os.fspath(fn)
    if not fn.lower().endswith('.png'):
        raise RuntimeError(f'panic3d_b200.imageio: only PNG output is implemented ({fn})')
    return fn


class AsyncImageWriter:
    """A pool of host threads that write PNGs while the GPU renders the next view.

        w = AsyncImageWriter(threads=4)
        w.save(out['image'], fn_rgb)                                  # = I(out['image']).save(fn_rgb), returns at once
        w.save_xyza(out['image_xyz'], out['image_weights'], bw, fn)   # = I(cat([(xyz+bw/2)/bw, weights], 1)).save(fn)
        w.flush()                                                     # before reading the files back / at the end of the sweep

    ``encoder`` picks where the deflate runs, a trade like zlib's ``level``:
      'host'    (default) the filtered scan-lines are copied to pinned memory and the pool's threads deflate them with zlib
                at ``level``: the smaller files, at host-core time per view on the process that writes (rank 0 when views
                are gathered there).
      'device'  ``p3d_png_encode_device`` deflates on the GPU, on the caller's stream, and the threads only copy the
                finished file to disk: no host deflate, for larger files (a greedy parse with per-16 KB Huffman codes)
                and a little GPU time per view.  ``level`` is unused.
    Measured (``bench_png_device.py``, NVIDIA H100 80GB HBM3, 700 W power limit, 1980 MHz max SM clock), per eval-shaped
    512^2 RGB view: 'device' takes 0.247 ms of GPU time and writes 148 KB, with 1.05 ms of writer-thread time; 'host'
    writes 110 KB at level 3 (131 KB at 1, 93 KB at 6), with 20.7 ms of writer-thread time (zlib level 1 / 3 / 6: 8.8 /
    15 / 42 ms of one core).  For a 128^2 RGBA xyza: 0.128 ms, 32 KB, 0.50 ms against 28 KB, 3.0 ms.  DESIGN.md 4.6 has
    the rest.
    """

    def __init__(self, threads=4, level=3, encoder='host'):
        if encoder not in ('host', 'device'):
            raise ValueError(f"panic3d_b200.imageio: encoder must be 'host' or 'device', got {encoder!r}")
        self._h = _VP()
        self.encoder = encoder
        _lib.check(_lib.lib().p3d_png_writer_create(int(threads), int(level), C.byref(self._h)))
        self._side = {}                                               # device -> side stream for the D2H copies

    def _stream(self, dev):
        s = self._side.get(dev)
        if s is None:
            s = self._side[dev] = torch.cuda.Stream(dev)
        return s

    def _submit(self, scan, shape, fns):
        H, W, c = shape
        fns = [fns] if isinstance(fns, (str, os.PathLike)) else list(fns)
        if len(fns) != scan.shape[0]:
            raise RuntimeError(f'panic3d_b200.imageio: {scan.shape[0]} image(s) but {len(fns)} file name(s)')
        dev = scan.device
        if self.encoder == 'device':
            files, lens = png_encode_device(scan, shape)              # on the caller's stream, behind the filter kernel
        side = self._stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))              # the copy follows the filter kernel, off the render stream
        L = _lib.lib()
        with torch.cuda.device(dev):
            if self.encoder == 'device':
                files.record_stream(side)
                lens.record_stream(side)
                for i, fn in enumerate(fns):
                    fn = _png_name(fn)
                    _lib.check(L.p3d_png_writer_submit_encoded(self._h, files[i].data_ptr(), lens[i:].data_ptr(), H, W, c, fn.encode(),
                                                               side.cuda_stream))
                return
            scan.record_stream(side)
            for i, fn in enumerate(fns):
                fn = _png_name(fn)
                _lib.check(L.p3d_png_writer_submit(self._h, scan[i].data_ptr(), H, W, c, fn.encode(), side.cuda_stream))

    def save(self, img, fn):
        """``I(img).save(fn)`` for a float CUDA tensor (C,H,W) / (1,C,H,W); a batch (N,C,H,W) takes a list of N names."""
        scan, shape = png_scanlines(img)
        self._submit(scan, shape, fn)

    def save_xyza(self, image_xyz, image_weights, box_warp, fn):
        """``I(torch.cat([(image_xyz + bw/2)/bw, image_weights], dim=1)).save(fn)`` (generate.py:141-147)."""
        bw = float(box_warp)
        scan, shape = png_scanlines(image_xyz, extra=image_weights, scale=[1.0 / bw] * 3 + [1.0], shift=[bw / 2] * 3 + [0.0])
        self._submit(scan, shape, fn)

    def submit_host(self, scanlines, h, w, c, fn):
        """Scan-lines already in host memory (numpy uint8); pure host path."""
        import numpy as np
        buf = np.ascontiguousarray(scanlines, dtype=np.uint8).reshape(-1)
        _lib.check(_lib.lib().p3d_png_writer_submit_host(self._h, buf.ctypes.data, h, w, c, os.fspath(fn).encode()))

    def flush(self):
        n = C.c_int32(0)
        _lib.check(_lib.lib().p3d_png_writer_flush(self._h, C.byref(n)))

    def close(self):
        if self._h:
            _lib.lib().p3d_png_writer_destroy(self._h)
            self._h = _VP()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        try:
            if exc[0] is None:
                self.flush()
        finally:
            self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class AsyncPickleWriter:
    """``uutil.pdump(obj, fn)`` (``_util/util_v1.py:275-277``; the marching-cubes dict of generate.py:104-105) on a
    background thread; the object must not be mutated until ``flush()``."""

    def __init__(self):
        self._threads, self._errors = [], []

    def pdump(self, obj, fn):
        def work():
            try:
                tmp = os.fspath(fn) + '.tmp'
                with open(tmp, 'wb') as handle:
                    pickle.dump(obj, handle)
                os.replace(tmp, fn)
            except Exception as e:                                            # surfaced by flush()
                self._errors.append(e)
        t = threading.Thread(target=work, daemon=True)
        t.start()
        self._threads.append(t)

    def flush(self):
        for t in self._threads:
            t.join()
        self._threads = []
        if self._errors:
            e, self._errors = self._errors[0], []
            raise e
