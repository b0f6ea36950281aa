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
    ``AsyncPickleWriter``                   ``uutil.pdump(obj, fn)`` (generate.py:104-105, the marching-cubes dict) off-thread

No CPU path for the device kernels: images must be CUDA tensors (the numpy restatement is ``oracle/imageio_oracle.py``,
tests only).  ``encode_png`` / ``submit_host`` are pure host code (zlib) and work anywhere.
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
    'p3d_png_writer_destroy': (C.c_int, [_VP]),
})


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


class AsyncImageWriter:
    """A pool of host threads that deflate and write PNGs while the GPU renders the next view.

        w = AsyncImageWriter(threads=4)
        w.save(out['image'], fn_rgb)                                  # = I(out['image']).save(fn_rgb), returns at once
        w.save_xyza(out['image_xyz'], out['image_weights'], bw, fn)   # = I(cat([(xyz+bw/2)/bw, weights], 1)).save(fn)
        w.flush()                                                     # before reading the files back / at the end of the sweep
    """

    def __init__(self, threads=4, level=3):
        self._h = _VP()
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
        side = self._stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))              # the copy follows the filter kernel, off the render stream
        scan.record_stream(side)
        L = _lib.lib()
        with torch.cuda.device(dev):
            for i, fn in enumerate(fns):
                fn = os.fspath(fn)
                if not fn.lower().endswith('.png'):
                    raise RuntimeError(f'panic3d_b200.imageio: only PNG output is implemented ({fn})')
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
