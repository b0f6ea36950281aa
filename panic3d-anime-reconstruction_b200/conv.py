"""fp32 training convolutions on the tensor cores - the H100 replacement for the reference's
``torch_utils.ops.conv2d_gradfix.conv2d`` / ``conv_transpose2d`` (``_train/eg3dc/src/torch_utils/ops/conv2d_gradfix.py``)
at the shapes the generator's non-fused synthesis layers and the discriminator's fp32 blocks produce.

The kernels (``csrc/conv_fp32.cu``, ``include/p3d_conv.h``) compute in 3xTF32 on wgmma: fp32-class results on the tensor
cores, for training runs that turn TF32 off.  The autograd Functions mirror conv2d_gradfix's: the input gradient is the
opposite-transpose op, the weight gradient a ``GradWeight`` Function whose own backward runs these ops again, so gradients
of any order (R1's ``create_graph=True``) stay on the kernels.  ``weight_gradients_disabled`` is read from the reference
module at backward time, so its ``no_weight_gradients()`` keeps working.

``dropin.install_conv2d()`` rebinds the reference module's two functions to ``conv2d`` / ``conv_transpose2d`` below.  A call
takes the kernels only when the reference would use its custom op (``enabled``, cuDNN enabled, a CUDA tensor), x and the
weight are contiguous fp32, ``groups == 1``, ``dilation == 1``, there is no bias, ``torch.backends.cudnn.allow_tf32`` is
false, ``p3d_conv_supported`` accepts the shape, and the kernels measured faster than cuDNN on it (``measured_faster``).
Every other call runs the original function.  ``conv2d_kernel`` / ``conv_transpose2d_kernel`` run the kernels for any
supported call.  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


class ConvParams(C.Structure):
    """Mirror of ``p3d_conv_params`` (include/p3d_conv.h) - field order and types must match."""
    _fields_ = [
        ('batch', C.c_int32), ('in_channels', C.c_int32), ('out_channels', C.c_int32), ('in_h', C.c_int32), ('in_w', C.c_int32),
        ('kernel_size', C.c_int32), ('stride', C.c_int32), ('padding', C.c_int32), ('transpose', C.c_int32),
        ('output_padding_h', C.c_int32), ('output_padding_w', C.c_int32),
    ]


_VP = C.c_void_p
_P = C.POINTER(ConvParams)
_lib.register_protos({
    'p3d_conv_supported': (C.c_int, [_P]),
    'p3d_conv_out_size': (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    'p3d_conv_forward_workspace_bytes': (C.c_size_t, [_P]),
    'p3d_conv_forward': (C.c_int, [_P, _VP, _VP, _VP, C.c_size_t, _VP, _VP]),
    'p3d_conv_weight_grad_workspace_bytes': (C.c_size_t, [_P]),
    'p3d_conv_weight_grad': (C.c_int, [_P, _VP, _VP, _VP, C.c_size_t, _VP, _VP]),
})

_gradfix = None          # the reference's conv2d_gradfix module, set by dropin.install_conv2d()


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _same(v):
    a, b = _pair(v)
    return a if a == b else -1


def make_params(x_shape, w_shape, stride, padding, transpose, output_padding=0):
    """``p3d_conv_params`` of a conv2d (``transpose`` false, weight (Cout, Cin, k, k)) or conv_transpose2d (weight
    (Cin, Cout, k, k)) call on an input of ``x_shape``.  Non-square kernels, strides or paddings, and a weight whose
    input channels do not match x, become values the kernels refuse."""
    p = ConvParams()
    p.batch, p.in_channels, p.in_h, p.in_w = x_shape
    cin_w = w_shape[0] if transpose else w_shape[1]
    p.out_channels = w_shape[1] if transpose else w_shape[0]
    p.kernel_size = w_shape[2] if w_shape[2] == w_shape[3] and cin_w == x_shape[1] else -1
    p.stride, p.padding = _same(stride), _same(padding)
    p.transpose = int(bool(transpose))
    p.output_padding_h, p.output_padding_w = _pair(output_padding)
    return p


def supported(p) -> bool:
    return bool(_lib.lib().p3d_conv_supported(C.byref(p)))


def out_size(p):
    oh, ow = C.c_int32(), C.c_int32()
    _lib.check(_lib.lib().p3d_conv_out_size(C.byref(p), C.byref(oh), C.byref(ow)))
    return oh.value, ow.value


def _workspace(nbytes, device):
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def run_forward(p, x, w):
    """``p3d_conv_forward``: conv2d / conv_transpose2d of contiguous fp32 x and w, as a new contiguous tensor."""
    L = _lib.lib()
    oh, ow = out_size(p)
    x, w = x.contiguous(), w.contiguous()
    y = torch.empty([p.batch, p.out_channels, oh, ow], dtype=torch.float32, device=x.device)
    ws = _workspace(L.p3d_conv_forward_workspace_bytes(C.byref(p)), x.device)
    with torch.cuda.device(x.device):          # the launch and its per-device attributes go to x's device, not the current one
        _lib.check(L.p3d_conv_forward(C.byref(p), x.data_ptr(), w.data_ptr(), ws.data_ptr(), ws.numel(), y.data_ptr(),
                                      _lib.stream_ptr(x.device)))
    return y


def run_weight_grad(p, x, dy):
    """``p3d_conv_weight_grad``: the gradient of sum(y * dy) with respect to the weight of the call p on input x."""
    L = _lib.lib()
    x, dy = x.contiguous(), dy.contiguous()
    kk = p.kernel_size
    shape = [p.in_channels, p.out_channels, kk, kk] if p.transpose else [p.out_channels, p.in_channels, kk, kk]
    dw = torch.empty(shape, dtype=torch.float32, device=x.device)
    ws = _workspace(L.p3d_conv_weight_grad_workspace_bytes(C.byref(p)), x.device)
    with torch.cuda.device(x.device):
        _lib.check(L.p3d_conv_weight_grad(C.byref(p), x.data_ptr(), dy.data_ptr(), ws.data_ptr(), ws.numel(), dw.data_ptr(),
                                          _lib.stream_ptr(x.device)))
    return dw


# ------------------------------------------------------------------------------------------ autograd
_null_tensor = torch.empty([0])
_functions = {}


def _weight_gradients_disabled():
    return bool(getattr(_gradfix, 'weight_gradients_disabled', False))


def _function(transpose, weight_shape, stride, padding, output_padding):
    """The autograd Function of one op (conv2d_gradfix.py:_conv2d_gradfix restated on the kernels); cached per key."""
    key = (bool(transpose), tuple(weight_shape), stride, padding, _pair(output_padding))
    if key in _functions:
        return _functions[key]
    k = weight_shape[2]

    def params(x_shape):
        return make_params(x_shape, weight_shape, stride, padding, transpose, output_padding)

    def calc_output_padding(input_shape, output_shape):
        """output_padding of the opposite op that maps output_shape back to input_shape (conv2d_gradfix.py:95-104)."""
        if transpose:
            return (0, 0)
        return tuple(input_shape[i + 2] - (output_shape[i + 2] - 1) * stride - (1 - 2 * padding) - (k - 1) for i in range(2))

    class Conv2d(torch.autograd.Function):
        @staticmethod
        def forward(ctx, input, weight):
            ctx.save_for_backward(input if weight.requires_grad else _null_tensor, weight if input.requires_grad else _null_tensor)
            ctx.input_shape = input.shape
            return run_forward(params(input.shape), input, weight)

        @staticmethod
        def backward(ctx, grad_output):
            input, weight = ctx.saved_tensors
            grad_input = grad_weight = None
            if ctx.needs_input_grad[0]:
                op = calc_output_padding(ctx.input_shape, grad_output.shape)
                grad_input = _function(not transpose, weight_shape, stride, padding, op).apply(grad_output, weight)
                assert grad_input.shape == ctx.input_shape
            if ctx.needs_input_grad[1] and not _weight_gradients_disabled():
                grad_weight = Conv2dGradWeight.apply(grad_output, input)
                assert grad_weight.shape == weight_shape
            return grad_input, grad_weight

    class Conv2dGradWeight(torch.autograd.Function):
        @staticmethod
        def forward(ctx, grad_output, input):
            ctx.save_for_backward(grad_output if input.requires_grad else _null_tensor, input if grad_output.requires_grad else _null_tensor)
            ctx.grad_output_shape = grad_output.shape
            ctx.input_shape = input.shape
            return run_weight_grad(params(input.shape), input, grad_output)

        @staticmethod
        def backward(ctx, grad2_grad_weight):
            grad_output, input = ctx.saved_tensors
            grad2_grad_output = grad2_input = None
            if ctx.needs_input_grad[0]:
                grad2_grad_output = Conv2d.apply(input, grad2_grad_weight)
                assert grad2_grad_output.shape == ctx.grad_output_shape
            if ctx.needs_input_grad[1]:
                op = calc_output_padding(ctx.input_shape, ctx.grad_output_shape)
                grad2_input = _function(not transpose, weight_shape, stride, padding, op).apply(grad_output, grad2_grad_weight)
                assert grad2_input.shape == ctx.input_shape
            return grad2_grad_output, grad2_input

    _functions[key] = Conv2d
    return Conv2d


# ------------------------------------------------------------------------------------------ routing
# (transpose, kernel, stride, Cin, Cout, H) of the calls where the kernels' forward + input gradient + weight gradient
# measured faster than cuDNN fp32 with TF32 off in both of two runs of these kernels: the ToRGB convs at 64^2 and 128^2
# (bench_conv.py, batch 4, 1x H100 80GB HBM3 at a 700 W power limit: 0.25 / 0.25 ms vs 0.29 / 0.29 ms and
# 0.46 / 0.45 ms vs 0.51 / 0.52 ms).  Every other backbone shape was slower in at least one run (DESIGN.md 5) and keeps
# cuDNN.
MEASURED_FASTER = frozenset({(False, 1, 1, 512, 96, 64), (False, 1, 1, 256, 96, 128)})


def measured_faster(p) -> bool:
    return (bool(p.transpose), p.kernel_size, p.stride, p.in_channels, p.out_channels, p.in_h) in MEASURED_FASTER


def eligible(input, weight, bias, stride, padding, dilation, groups, transpose, output_padding=0):
    """Params of a call every routing condition admits except measured_faster, else None."""
    g = _gradfix
    if g is None or not torch.is_tensor(input) or not torch.is_tensor(weight) or not g._should_use_custom_op(input):
        return None
    if input.dtype != torch.float32 or weight.dtype != torch.float32 or input.dim() != 4 or weight.dim() != 4:
        return None
    if weight.device != input.device or not input.is_contiguous() or not weight.is_contiguous():
        return None
    if groups != 1 or _pair(dilation) != (1, 1) or bias is not None or torch.backends.cudnn.allow_tf32:
        return None
    p = make_params(input.shape, weight.shape, stride, padding, transpose, output_padding)
    return p if supported(p) else None


def _original(name):
    fn = getattr(_gradfix, '_p3d_reference_' + name, None)
    return fn if fn is not None else getattr(torch.nn.functional, name)


def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    """``conv2d_gradfix.conv2d``: same arguments and result; routed calls run the kernels, every other call the original."""
    p = eligible(input, weight, bias, stride, padding, dilation, groups, False)
    if p is None or not measured_faster(p):
        return _original('conv2d')(input, weight, bias, stride, padding, dilation, groups)
    return _function(False, weight.shape, p.stride, p.padding, 0).apply(input, weight)


def conv_transpose2d(input, weight, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
    """``conv2d_gradfix.conv_transpose2d``: same arguments and result; routed calls run the kernels."""
    p = eligible(input, weight, bias, stride, padding, dilation, groups, True, output_padding)
    if p is None or not measured_faster(p):
        return _original('conv_transpose2d')(input, weight, bias, stride, padding, output_padding, groups, dilation)
    return _function(True, weight.shape, p.stride, p.padding, output_padding).apply(input, weight)


def _kernel_call(transpose, input, weight, stride, padding, output_padding):
    if not (input.is_cuda and input.dtype == torch.float32 and weight.dtype == torch.float32 and input.dim() == 4 and weight.dim() == 4):
        raise RuntimeError('panic3d_b200.conv: the kernels take 4-D fp32 CUDA tensors')
    p = make_params(input.shape, weight.shape, stride, padding, transpose, output_padding)
    if not supported(p):
        raise RuntimeError('panic3d_b200.conv: this call is not covered by the kernels (see p3d_conv_supported)')
    return _function(transpose, weight.shape, p.stride, p.padding, output_padding).apply(input.contiguous(), weight.contiguous())


def conv2d_kernel(input, weight, stride=1, padding=0):
    """conv2d on the kernels, with autograd, for any supported call, whatever measured_faster says (raises otherwise)."""
    return _kernel_call(False, input, weight, stride, padding, 0)


def conv_transpose2d_kernel(input, weight, stride=1, padding=0, output_padding=0):
    """conv_transpose2d on the kernels, with autograd, for any supported call (raises otherwise)."""
    return _kernel_call(True, input, weight, stride, padding, output_padding)


def flops(p) -> int:
    """Multiply-adds x 2 of one forward call (equally of its input gradient or weight gradient), shape-computed."""
    oh, ow = out_size(p)
    pix = p.in_h * p.in_w if p.transpose else oh * ow
    return 2 * p.batch * pix * p.in_channels * p.out_channels * p.kernel_size * p.kernel_size
