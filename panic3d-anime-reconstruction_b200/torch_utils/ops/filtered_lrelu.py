"""Drop-in for ``torch_utils/ops/filtered_lrelu.py`` (reference ops/filtered_lrelu.py:58-274).

``filtered_lrelu(x, fu, fd, b, up, down, padding, gain, slope, clamp, flip_filter, impl)`` over the sm_90a
kernel ``p3d_filtered_lrelu`` (include/p3d_ops.h).  One runtime-generic kernel covers every filter/up/down
combination, so the reference's "no optimised kernel -> generic fallback" branch does not exist here.  The
forward pass records 2 bits per up-sampled pixel (negative / clamped) so the backward pass - the same op with
filters and up/down swapped, reading those bits - never re-evaluates the non-linearity; gradients of any order
re-enter the same autograd Function.  No CPU path, no ``impl='ref'``.
"""
from __future__ import annotations

import numpy as np
import torch

from ... import _lib

_C = _lib.C
_P64 = _C.POINTER(_C.c_int64)
_lib.register_protos({
    'p3d_filtered_lrelu': (_C.c_int, [_lib._VP] * 6 + [_C.c_int32] * 5 + [_P64, _C.c_int32, _C.c_int32, _P64] + [_C.c_int32] * 16 +
                           [_C.c_float] * 3 + [_C.c_int32, _C.c_int32, _lib._VP]),
})
_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and 1 <= f.ndim <= 2
    return f.shape[-1], f.shape[0]     # width, height


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple)) and all(isinstance(x, (int, np.integer)) for x in padding)
    padding = [int(x) for x in padding]
    if len(padding) == 2:
        px, py = padding
        padding = [px, px, py, py]
    px0, px1, py0, py1 = padding
    return px0, px1, py0, py1


def _launch(x, fu, fd, b, si, up, down, px0, px1, py0, py1, sx, sy, gain, slope, clamp, flip, write_signs):
    """-> (y, signs or None).  fu / fd: fp32, rank 1 (separable) or 2; si: existing sign tensor (read mode) or None."""
    if x.dtype not in _DTYPES:
        raise TypeError(f'filtered_lrelu: unsupported dtype {x.dtype} (fp32 / fp16 / bf16)')
    N, Cc, H, W = x.shape
    fu = fu.to(x.device, torch.float32).contiguous()
    fd = fd.to(x.device, torch.float32).contiguous()
    fu_sep, fd_sep = int(fu.ndim == 1), int(fd.ndim == 1)
    fuw, fuh = fu.shape[-1], (fu.shape[-1] if fu_sep else fu.shape[0])
    fdw, fdh = fd.shape[-1], (fd.shape[-1] if fd_sep else fd.shape[0])
    cw, ch = W * up + px0 + px1 - (fuw - 1), H * up + py0 + py1 - (fuh - 1)
    if not (cw > fdw - 1 and ch > fdh - 1):
        raise RuntimeError('upsampled buffer must be at least the size of downsampling filter')
    yw, yh = (cw - (fdw - 1) + down - 1) // down, (ch - (fdh - 1) + down - 1) // down
    fmt = torch.channels_last if (x.stride(1) == 1 and Cc > 1) else torch.contiguous_format
    y = torch.empty((N, Cc, yh, yw), dtype=x.dtype, device=x.device, memory_format=fmt)
    mode, s = 0, None
    if si is not None:
        mode, s = 2, si
        assert s.dtype == torch.uint8 and s.is_contiguous() and s.dim() == 4 and s.shape[0] == N and s.shape[1] == Cc
    elif write_signs:
        sh = yh * down - (down - 1) + (fdh - 1)
        sw = (yw * down - (down - 1) + (fdw - 1) + 15) & ~15          # active width rounded up to 16 elements
        s = torch.zeros((N, Cc, sh, sw >> 2), dtype=torch.uint8, device=x.device)
        mode = 1
    s_h, s_w = (s.shape[2], s.shape[3] << 2) if s is not None else (0, 0)
    xs, ys = (_C.c_int64 * 4)(*x.stride()), (_C.c_int64 * 4)(*y.stride())
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().p3d_filtered_lrelu(
            x.data_ptr(), fu.data_ptr(), fd.data_ptr(), b.data_ptr(), _lib.ptr(s), y.data_ptr(), _DTYPES[x.dtype], N, Cc, H, W, xs,
            yh, yw, ys, 1 if fu_sep else fuh, fuw, fu_sep, 1 if fd_sep else fdh, fdw, fd_sep, up, down, px0, px1, py0, py1,
            s_h, s_w, sx, sy, gain, slope, clamp, 1 if flip else 0, mode, _lib.stream_ptr(x.device)))
    return y, (s if mode == 1 else None)


_cache = {}


def _op(up, down, padding, gain, slope, clamp, flip_filter):
    assert isinstance(up, int) and up >= 1 and isinstance(down, int) and down >= 1
    px0, px1, py0, py1 = _parse_padding(padding)
    assert gain == float(gain) and gain > 0 and slope == float(slope) and slope >= 0
    assert clamp is None or (clamp == float(clamp) and clamp >= 0)
    gain, slope = float(gain), float(slope)
    clamp = float(clamp if clamp is not None else 'inf')
    key = (up, down, px0, px1, py0, py1, gain, slope, clamp, flip_filter)
    if key in _cache:
        return _cache[key]

    class FilteredLRelu(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, fu, fd, b, si, sx, sy):
            assert isinstance(x, torch.Tensor) and x.ndim == 4
            one = lambda: torch.ones([1, 1], dtype=torch.float32, device=x.device)
            fu = one() if fu is None else fu
            fd = one() if fd is None else fd
            assert 1 <= fu.ndim <= 2 and 1 <= fd.ndim <= 2
            if up == 1 and fu.ndim == 1 and fu.shape[0] == 1:
                fu = fu.square()[None]
            if down == 1 and fd.ndim == 1 and fd.shape[0] == 1:
                fd = fd.square()[None]
            if b is None:
                b = torch.zeros([x.shape[1]], dtype=x.dtype, device=x.device)
            write_signs = si is None and (x.requires_grad or b.requires_grad)
            y, so = _launch(x, fu, fd, b.to(x.dtype).contiguous(), si, up, down, px0, px1, py0, py1, sx, sy, gain, slope, clamp,
                            flip_filter, write_signs)
            ctx.save_for_backward(fu, fd, si if si is not None else so)
            ctx.x_shape, ctx.y_shape, ctx.s_ofs = x.shape, y.shape, (sx, sy)
            return y

        @staticmethod
        def backward(ctx, dy):
            fu, fd, si = ctx.saved_tensors
            _, _, xh, xw = ctx.x_shape
            _, _, yh, yw = ctx.y_shape
            sx, sy = ctx.s_ofs
            fuw, fuh = _get_filter_size(fu)
            fdw, fdh = _get_filter_size(fd)
            if fu.ndim == 1:
                fuh = fuw
            if fd.ndim == 1:
                fdh = fdw
            dx = db = None
            for i in (1, 2, 4, 5, 6):
                assert not ctx.needs_input_grad[i]
            if ctx.needs_input_grad[0] or ctx.needs_input_grad[3]:
                pp = [(fuw - 1) + (fdw - 1) - px0, xw * up - yw * down + px0 - (up - 1),
                      (fuh - 1) + (fdh - 1) - py0, xh * up - yh * down + py0 - (up - 1)]
                gg = gain * (up ** 2) / (down ** 2)
                dx = _op(down, up, pp, gg, slope, None, not flip_filter).apply(dy, fd, fu, None, si, sx - (fuw - 1) + px0, sy - (fuh - 1) + py0)
            if ctx.needs_input_grad[3]:
                db = dx.sum([0, 2, 3])
            return dx, None, None, db, None, None, None

    _cache[key] = FilteredLRelu
    return FilteredLRelu


def filtered_lrelu(x, fu=None, fd=None, b=None, up=1, down=1, padding=0, gain=np.sqrt(2), slope=0.2, clamp=None,
                   flip_filter=False, impl='cuda'):
    """bias -> up-FIR (x up^2) -> gain*lrelu(slope) -> clamp -> down-FIR.  Reference filtered_lrelu.py:58-119."""
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        raise NotImplementedError("panic3d_b200 ships no impl='ref'; the PyTorch restatement is oracle/ops_oracle.py (tests only)")
    if not x.is_cuda:
        raise RuntimeError('panic3d_b200.filtered_lrelu has no CPU path: x must be on a CUDA device')
    return _op(up, down, padding, gain, slope, clamp, flip_filter).apply(x, fu, fd, b, None, 0, 0)
