"""Host mirror of ``torch_utils/ops/upfirdn2d.py`` (reference ops/upfirdn2d.py:37-389).

Interface contract, not an implementation: the argument-parsing helpers (``_parse_scaling``, ``_parse_padding``,
``_get_filter_size``), ``setup_filter`` and the padding arithmetic of ``filter2d`` / ``upsample2d`` / ``downsample2d`` below follow
the reference line for line because other reference modules import those private names (``conv2d_resample.py``,
``networks_stylegan2.py``) and any other arithmetic would change output sizes; everything that does work - the kernels, the autograd
formulation - is this repository's own.

Same public names and argument meaning - ``setup_filter``, ``upfirdn2d``, ``filter2d``, ``upsample2d``,
``downsample2d`` (+ the ``_parse_*`` / ``_get_filter_size`` helpers other reference modules import) - over the
sm_90a kernel ``p3d_upfirdn2d`` (include/p3d_ops.h).  upfirdn2d is linear, so its gradient of any order is
another upfirdn2d with up/down swapped, the filter flipped and the adjoint padding; the autograd Function below
re-enters itself for that, which is what makes R1's double-backward work.  No CPU path, no ``impl='ref'``.
"""
from __future__ import annotations

import numpy as np
import torch

from ... import _lib

_C = _lib.C
_lib.register_protos({
    'p3d_upfirdn2d': (_C.c_int, [_lib._VP, _lib._VP, _lib._VP, _C.c_int32] + [_C.c_int32] * 4 + [_C.POINTER(_C.c_int64)] +
                      [_C.c_int32, _C.c_int32, _C.c_int64, _C.c_int64, _C.c_int32, _C.c_int32, _C.POINTER(_C.c_int64)] +
                      [_C.c_int32] * 9 + [_C.c_float, _lib._VP]),
})
_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}


def _parse_scaling(scaling):
    if isinstance(scaling, int):
        scaling = [scaling, scaling]
    assert isinstance(scaling, (list, tuple)) and all(isinstance(x, int) for x in scaling)
    sx, sy = scaling
    assert sx >= 1 and sy >= 1
    return sx, sy


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple)) and all(isinstance(x, (int, np.integer)) for x in padding)
    padding = [int(x) for x in padding]
    if len(padding) == 2:
        padx, pady = padding
        padding = [padx, padx, pady, pady]
    padx0, padx1, pady0, pady1 = padding
    return padx0, padx1, pady0, pady1


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and f.ndim in [1, 2]
    fw, fh = int(f.shape[-1]), int(f.shape[0])
    assert fw >= 1 and fh >= 1
    return fw, fh


def setup_filter(f, device=torch.device('cpu'), normalize=True, flip_filter=False, gain=1, separable=None):
    """Build the fp32 FIR tensor upfirdn2d expects (reference upfirdn2d.py:72-116): outer product of 1-D taps unless
    separable (>= 8 taps by default), DC-normalised, optionally flipped, scaled by gain**(ndim/2)."""
    if f is None:
        f = 1
    f = torch.as_tensor(f, dtype=torch.float32)
    assert f.ndim in [0, 1, 2] and f.numel() > 0
    if f.ndim == 0:
        f = f[np.newaxis]
    if separable is None:
        separable = (f.ndim == 1 and f.numel() >= 8)
    if f.ndim == 1 and not separable:
        f = f.ger(f)
    assert f.ndim == (1 if separable else 2)
    if normalize:
        f = f / f.sum()
    if flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f * (gain ** (f.ndim / 2))
    return f.to(device=device)


def _launch(x, f2d, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip, gain):
    """One p3d_upfirdn2d call. x (N,C,H,W) any strides; f2d (fH,fW) fp32 on x.device."""
    if x.dtype not in _DTYPES:
        raise TypeError(f'upfirdn2d: unsupported dtype {x.dtype}')
    if x.dim() != 4:
        raise RuntimeError('x must be rank 4')
    if f2d.dim() != 2 or f2d.dtype != torch.float32 or f2d.device != x.device:
        raise RuntimeError('f must be a rank-2 float32 tensor on the same device as x')
    if x.numel() == 0:
        raise RuntimeError('x has zero size')
    N, Cc, H, W = x.shape
    fH, fW = f2d.shape
    outW = (W * upx + padx0 + padx1 - fW + downx) // downx
    outH = (H * upy + pady0 + pady1 - fH + downy) // downy
    if outW < 1 or outH < 1:
        raise RuntimeError('output must be at least 1x1')
    fmt = torch.channels_last if (x.stride(1) == 1 and Cc > 1) else torch.contiguous_format   # x.suggest_memory_format()
    y = torch.empty((N, Cc, outH, outW), dtype=x.dtype, device=x.device, memory_format=fmt)
    xs = (_C.c_int64 * 4)(*x.stride())
    ys = (_C.c_int64 * 4)(*y.stride())
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().p3d_upfirdn2d(x.data_ptr(), f2d.data_ptr(), y.data_ptr(), _DTYPES[x.dtype], N, Cc, H, W, xs,
                                            fH, fW, f2d.stride(0), f2d.stride(1), outH, outW, ys, upx, upy, downx, downy,
                                            padx0, padx1, pady0, pady1, 1 if flip else 0, float(gain), _lib.stream_ptr(x.device)))
    return y


_cache = {}


def _op(up, down, padding, flip_filter, gain):
    upx, upy = _parse_scaling(up)
    downx, downy = _parse_scaling(down)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    key = (upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain)
    if key in _cache:
        return _cache[key]

    class Upfirdn2d(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, f):
            assert isinstance(x, torch.Tensor) and x.ndim == 4
            if f is None:
                f = torch.ones([1, 1], dtype=torch.float32, device=x.device)
            if f.ndim == 1 and f.shape[0] == 1:
                f = f.square().unsqueeze(0)                    # separable single tap == full 1x1
            assert f.ndim in [1, 2]
            if f.ndim == 2:
                y = _launch(x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain)
            else:                                               # separable: row pass then column pass
                y = _launch(x, f.unsqueeze(0), upx, 1, downx, 1, padx0, padx1, 0, 0, flip_filter, 1.0)
                y = _launch(y, f.unsqueeze(1), 1, upy, 1, downy, 0, 0, pady0, pady1, flip_filter, gain)
            ctx.save_for_backward(f)
            ctx.x_shape = x.shape
            return y

        @staticmethod
        def backward(ctx, dy):
            f, = ctx.saved_tensors
            _, _, ih, iw = ctx.x_shape
            _, _, oh, ow = dy.shape
            fw, fh = _get_filter_size(f)
            dx = None
            if ctx.needs_input_grad[0]:                         # adjoint: swap up/down, flip the filter, adjoint padding
                p = [fw - padx0 - 1, iw * upx - ow * downx + padx0 - upx + 1,
                     fh - pady0 - 1, ih * upy - oh * downy + pady0 - upy + 1]
                dx = _op((downx, downy), (upx, upy), p, not flip_filter, gain).apply(dy, f)
            assert not ctx.needs_input_grad[1]
            return dx, None

    _cache[key] = Upfirdn2d
    return Upfirdn2d


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Pad, upsample, filter and downsample a batch of 2-D images.  Reference upfirdn2d.py:120-165."""
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        raise NotImplementedError("panic3d_b200 ships no impl='ref'; the PyTorch restatement is oracle/ops_oracle.py (tests only)")
    if not x.is_cuda:
        raise RuntimeError('panic3d_b200.upfirdn2d has no CPU path: x must be on a CUDA device')
    if f is not None and f.device != x.device:
        f = f.to(x.device)
    return _op(up, down, padding, flip_filter, gain).apply(x, f)


def filter2d(x, f, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Same-size FIR filtering (reference upfirdn2d.py:279-311)."""
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + fw // 2, padx1 + (fw - 1) // 2, pady0 + fh // 2, pady1 + (fh - 1) // 2]
    return upfirdn2d(x, f, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)


def upsample2d(x, f, up=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Integer up-sampling with FIR interpolation (reference upfirdn2d.py:315-350)."""
    upx, upy = _parse_scaling(up)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + (fw + upx - 1) // 2, padx1 + (fw - upx) // 2, pady0 + (fh + upy - 1) // 2, pady1 + (fh - upy) // 2]
    return upfirdn2d(x, f, up=up, padding=p, flip_filter=flip_filter, gain=gain * upx * upy, impl=impl)


def downsample2d(x, f, down=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Integer down-sampling with FIR anti-aliasing (reference upfirdn2d.py:354-389)."""
    downx, downy = _parse_scaling(down)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + (fw - downx + 1) // 2, padx1 + (fw - downx) // 2, pady0 + (fh - downy + 1) // 2, pady1 + (fh - downy) // 2]
    return upfirdn2d(x, f, down=down, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)
