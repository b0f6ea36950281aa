"""Drop-in for ``torch_utils/ops/bias_act.py`` (reference ops/bias_act.py:23-209).

Same call surface - ``bias_act(x, b, dim, act, alpha, gain, clamp, impl)`` and the ``activation_funcs`` table -
over the sm_90a kernel ``p3d_bias_act`` (include/p3d_ops.h).  First and second derivatives are the same fused
kernel in grad mode 1 / 2, wired through two autograd Functions exactly as the op's contract requires
(what gets saved is dictated by which of x / y each activation's derivative is expressed in).
No CPU path and no ``impl='ref'`` here: the PyTorch restatement lives in ``oracle/ops_oracle.py`` (tests only).
"""
from __future__ import annotations

import math
from types import SimpleNamespace as _NS

import torch

from ... import _lib

_sqrt2 = math.sqrt(2)
# name -> cuda_idx / defaults / which forward tensors the derivative formulas need (reference bias_act.py:23-33)
activation_funcs = {
    'linear':   _NS(def_alpha=0,   def_gain=1,      cuda_idx=1, ref='',  has_2nd_grad=False),
    'relu':     _NS(def_alpha=0,   def_gain=_sqrt2, cuda_idx=2, ref='y', has_2nd_grad=False),
    'lrelu':    _NS(def_alpha=0.2, def_gain=_sqrt2, cuda_idx=3, ref='y', has_2nd_grad=False),
    'tanh':     _NS(def_alpha=0,   def_gain=1,      cuda_idx=4, ref='y', has_2nd_grad=True),
    'sigmoid':  _NS(def_alpha=0,   def_gain=1,      cuda_idx=5, ref='y', has_2nd_grad=True),
    'elu':      _NS(def_alpha=0,   def_gain=1,      cuda_idx=6, ref='y', has_2nd_grad=True),
    'selu':     _NS(def_alpha=0,   def_gain=1,      cuda_idx=7, ref='y', has_2nd_grad=True),
    'softplus': _NS(def_alpha=0,   def_gain=1,      cuda_idx=8, ref='y', has_2nd_grad=True),
    'swish':    _NS(def_alpha=0,   def_gain=_sqrt2, cuda_idx=9, ref='x', has_2nd_grad=True),
}

_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3}

_lib.register_protos({
    'p3d_bias_act': (_lib.C.c_int, [_lib._VP] * 6 + [_lib.C.c_int64, _lib.C.c_int32, _lib.C.c_int32, _lib.C.c_int64,
                                    _lib.C.c_int32, _lib.C.c_int32, _lib.C.c_float, _lib.C.c_float, _lib.C.c_float, _lib._VP]),
})


def _is_dense(t):
    """non-overlapping and dense: some permutation of the dims is contiguous (any memory format)."""
    dims = sorted((st, sz) for st, sz in zip(t.stride(), t.shape) if sz > 1)
    expect = 1
    for st, sz in dims:
        if st != expect:
            return False
        expect *= sz
    return True


def _dense_like(t, fmt):
    return t.contiguous(memory_format=fmt)


def _launch(x, b, xref, yref, dy, grad, dim, spec, alpha, gain, clamp):
    """One call of p3d_bias_act; all tensor arguments share x's dense layout (None = absent)."""
    if x.dtype not in _DTYPES:
        raise TypeError(f'bias_act: unsupported dtype {x.dtype}')
    if not _is_dense(x):
        raise RuntimeError('x must be non-overlapping and dense')
    for name, t in (('xref', xref), ('yref', yref), ('dy', dy)):
        if t is not None and (t.shape != x.shape or t.stride() != x.stride() or t.dtype != x.dtype):
            raise RuntimeError(f'{name} must have the same shape, dtype and layout as x')
    if b is not None:
        if b.dim() != 1 or not (0 <= dim < x.dim()) or b.shape[0] != x.shape[dim]:
            raise RuntimeError('b must be a rank-1 tensor matching x.shape[dim]')
        if b.dtype != x.dtype or b.device != x.device:
            raise RuntimeError('b must have the same dtype and device as x')
        b = b.contiguous()
    y = torch.empty_like(x)            # preserves the dense layout (strides) of x
    if x.numel() == 0:
        return y
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().p3d_bias_act(
            x.data_ptr(), _lib.ptr(b), _lib.ptr(xref), _lib.ptr(yref), _lib.ptr(dy), y.data_ptr(), x.numel(),
            _DTYPES[x.dtype], grad, x.stride(dim) if b is not None else 1, b.numel() if b is not None else 1,
            spec.cuda_idx, alpha, gain, clamp, _lib.stream_ptr(x.device)))
    return y


_cache = {}


def _op(dim, act, alpha, gain, clamp):
    key = (dim, act, alpha, gain, clamp)
    if key in _cache:
        return _cache[key]
    spec = activation_funcs[act]
    trivial = act == 'linear' and gain == 1 and clamp < 0          # y = x + b only

    def fmt_of(t):
        return torch.channels_last if t.ndim > 2 and t.stride(1) == 1 else torch.contiguous_format

    class Fwd(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, b):
            ctx.fmt = fmt_of(x)
            x = _dense_like(x, ctx.fmt)
            y = x if (trivial and b is None) else _launch(x, b, None, None, None, 0, dim, spec, alpha, gain, clamp)
            need_x = 'x' in spec.ref or spec.has_2nd_grad
            ctx.has_b = b is not None
            ctx.save_for_backward(x if need_x else None, b if (need_x and b is not None) else None, y if 'y' in spec.ref else None)
            return y

        @staticmethod
        def backward(ctx, dy):
            x, b, y = ctx.saved_tensors
            dx = db = None
            if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
                dy = _dense_like(dy, ctx.fmt)
                dx = dy if trivial else Bwd.apply(dy, x, b, y)
            if ctx.has_b and ctx.needs_input_grad[1]:
                db = dx.sum([i for i in range(dx.ndim) if i != dim])
            return dx, db

    class Bwd(torch.autograd.Function):
        @staticmethod
        def forward(ctx, dy, x, b, y):
            ctx.fmt = fmt_of(dy)
            dx = _launch(dy, b, x, y, None, 1, dim, spec, alpha, gain, clamp)
            ctx.save_for_backward(dy if spec.has_2nd_grad else None, x, b, y)
            return dx

        @staticmethod
        def backward(ctx, d_dx):
            d_dx = _dense_like(d_dx, ctx.fmt)
            dy, x, b, y = ctx.saved_tensors
            d_dy = d_x = d_b = None
            if ctx.needs_input_grad[0]:
                d_dy = Bwd.apply(d_dx, x, b, y)
            if spec.has_2nd_grad and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
                d_x = _launch(d_dx, b, x, y, dy, 2, dim, spec, alpha, gain, clamp)
            if spec.has_2nd_grad and ctx.needs_input_grad[2] and b is not None:
                d_b = d_x.sum([i for i in range(d_x.ndim) if i != dim])
            return d_dy, d_x, d_b, None

    _cache[key] = Fwd
    return Fwd


def bias_act(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None, impl='cuda'):
    """Fused ``clamp(gain * act(x + b))`` with first and second order gradients.  Reference bias_act.py:54-88."""
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    assert clamp is None or clamp >= 0
    if impl == 'ref':
        raise NotImplementedError("panic3d_b200 ships no impl='ref'; the PyTorch restatement is oracle/ops_oracle.py (tests only)")
    if not x.is_cuda:
        raise RuntimeError('panic3d_b200.bias_act has no CPU path: x must be on a CUDA device')
    spec = activation_funcs[act]
    alpha = float(alpha if alpha is not None else spec.def_alpha)
    gain = float(gain if gain is not None else spec.def_gain)
    clamp = float(clamp if clamp is not None else -1)
    return _op(dim, act, alpha, gain, clamp).apply(x, b)
