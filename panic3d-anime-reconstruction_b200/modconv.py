"""Modulated convolution at inference - the H100 replacement for the fused branch of StyleGAN2's ``modulated_conv2d``
inside ``SynthesisLayer.forward`` / ``ToRGBLayer.forward`` (reference ``_train/eg3dc/src/training/networks_stylegan2.py``
:40-98, :334-354, :376-380).

Per layer call: ``styles = layer.affine(w)`` and the noise exactly as the reference draws them (same ``torch.randn`` call,
same order), then two launches - ``p3d_modconv_prep`` (per-sample modulated, demodulated weights in the conv kernel's
operand layout) and ``p3d_modconv_forward`` (implicit-GEMM conv on wgmma with the noise / bias / lrelu / gain / clamp
epilogue).  ``up=2`` layers store the transposed conv's pre-filter tensor and run the reference's own remaining sequence on
this package's ops: ``upfirdn2d`` (gain 4), ``+ noise``, ``bias_act``.

A call takes the kernel only when it is a CUDA call with ``fused_modconv`` true, nothing under autograd requires grad, the
layer shape is one ``p3d_modconv_supported`` accepts - for fp32 layers only with ``torch.backends.cudnn.allow_tf32`` true,
the same numeric class as the cuDNN route it replaces - and one where the kernel measured faster than the reference route
(``measured_faster``: today the fp16 up-2 layers).  Every other call runs the original method unchanged.
``synthesis_layer_kernel`` / ``torgb_kernel`` run the kernel route for any supported shape.
``dropin.install_modconv()`` rebinds the reference classes' ``forward`` to the two functions below.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .torch_utils.ops import bias_act as _bias_act
from .torch_utils.ops import upfirdn2d as _upfirdn2d

P3D_F32, P3D_F16 = 0, 1
P3D_ACT_LINEAR, P3D_ACT_LRELU = 1, 3
_ACTS = {'linear': P3D_ACT_LINEAR, 'lrelu': P3D_ACT_LRELU}
KB = 128                                       # bytes of one K chunk of an operand row (csrc/modconv.cu kKB)


class ModconvParams(C.Structure):
    """Mirror of ``p3d_modconv_params`` (include/p3d_modconv.h) - field order and types must match."""
    _fields_ = [
        ('batch', C.c_int32), ('in_channels', C.c_int32), ('out_channels', C.c_int32), ('in_h', C.c_int32), ('in_w', C.c_int32),
        ('kernel_size', C.c_int32), ('up', C.c_int32), ('down', C.c_int32), ('dtype', C.c_int32), ('demodulate', C.c_int32),
        ('allow_tf32', C.c_int32), ('reserved0', C.c_int32),
    ]


_VP = C.c_void_p
_P = C.POINTER(ModconvParams)
_I64P = C.POINTER(C.c_int64)
_lib.register_protos({
    'p3d_modconv_supported': (C.c_int, [_P]),
    'p3d_modconv_out_size': (C.c_int, [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    'p3d_modconv_workspace_bytes': (C.c_size_t, [_P]),
    'p3d_modconv_prep': (C.c_int, [_P, _VP, _VP, _VP, _VP]),
    'p3d_modconv_forward': (C.c_int, [_P, _VP, _I64P, _VP, _VP, _VP, _I64P, _VP, _I64P, C.c_int32, C.c_float, C.c_float, _VP]),
})


def make_params(x, weight, demodulate, up=1, down=1, allow_tf32=None):
    """``p3d_modconv_params`` of one layer call on input ``x`` with the (Cout, Cin, k, k) ``weight``."""
    cout, cin, kh, kw = weight.shape
    p = ModconvParams()
    p.batch, p.in_channels, p.out_channels = x.shape[0], cin, cout
    p.in_h, p.in_w = x.shape[2], x.shape[3]
    p.kernel_size = kh if kh == kw else -1
    p.up, p.down = up, down
    p.dtype = {torch.float32: P3D_F32, torch.float16: P3D_F16}.get(x.dtype, -1)
    p.demodulate = int(bool(demodulate))
    p.allow_tf32 = int(torch.backends.cudnn.allow_tf32 if allow_tf32 is None else allow_tf32)
    return p


def supported(p) -> bool:
    return bool(_lib.lib().p3d_modconv_supported(C.byref(p)))


def _strides(t):
    return (C.c_int64 * 4)(*t.stride())


def prep(p, weight, styles):
    """Per-sample operand of one layer: ``p3d_modconv_prep`` into a workspace from torch's caching allocator (capturable)."""
    L = _lib.lib()
    ws = torch.empty(int(L.p3d_modconv_workspace_bytes(C.byref(p))), dtype=torch.uint8, device=styles.device)
    w32 = weight.detach().to(torch.float32).contiguous()
    s32 = styles.detach().to(torch.float32).contiguous()
    _lib.check(L.p3d_modconv_prep(C.byref(p), w32.data_ptr(), s32.data_ptr(), ws.data_ptr(), _lib.stream_ptr(styles.device)))
    return ws


def _out_format(x):
    """The memory format the reference's grouped conv gives its output: the fused branch reshapes x to (1, N*C, H, W),
    which stays a channels_last view only for N = 1; cuDNN then writes its output in the input's format."""
    xr = x.reshape(1, -1, *x.shape[2:])
    cl = (not xr.is_contiguous()) and xr.is_contiguous(memory_format=torch.channels_last)
    return torch.channels_last if cl else torch.contiguous_format


def conv(p, x, ws, bias=None, noise=None, act='linear', gain=1.0, clamp=None):
    """``p3d_modconv_forward``: y = clamp(act(conv + noise + bias) * gain) in x's dtype (up 2: the pre-filter tensor)."""
    L = _lib.lib()
    oh, ow = C.c_int32(), C.c_int32()
    _lib.check(L.p3d_modconv_out_size(C.byref(p), C.byref(oh), C.byref(ow)))
    y = torch.empty([p.batch, p.out_channels, oh.value, ow.value], dtype=x.dtype, device=x.device, memory_format=_out_format(x))
    nz, nz_stride = None, None
    if noise is not None:                                          # [N, 1, H, W] per sample or [H, W] broadcast
        nz = noise.to(torch.float32)
        if nz.dim() == 4:
            nz = nz.expand(p.batch, 1, oh.value, ow.value)
            nz_stride = (C.c_int64 * 3)(nz.stride(0), nz.stride(2), nz.stride(3))
        else:
            nz_stride = (C.c_int64 * 3)(0, nz.stride(0), nz.stride(1))
    b = None if bias is None else bias.detach().to(x.dtype).contiguous()
    _lib.check(L.p3d_modconv_forward(C.byref(p), x.data_ptr(), _strides(x), ws.data_ptr(), _lib.ptr(b),
                                     _lib.ptr(nz), nz_stride, y.data_ptr(), _strides(y),
                                     _ACTS[act], float(gain), -1.0 if clamp is None else float(clamp),
                                     _lib.stream_ptr(x.device)))
    return y


def workspace_rows(p, ws):
    """The whole workspace as (N, Cout padded to the N tile, slot, Cin padded to the K chunk), in the compute type (fp16
    or tf32 as fp32): a view of its bytes, padding included."""
    f16 = p.dtype == P3D_F16
    es = 2 if f16 else 4
    kce = KB // es
    nchunks = -(-p.in_channels // kce)
    bn = 8 if p.out_channels <= 8 else 128
    nnb = -(-p.out_channels // bn)
    nslots = len(tap_slots(p))
    vals = ws.view(torch.float16 if f16 else torch.float32)
    # tile_byte(r, b) = (b >> 4) * (bn * 16) + (r >> 3) * 128 + (r & 7) * 16 + (b & 15): dims (kc, rg, r8, e) of one tile
    vals = vals.view(p.batch, nnb, nslots, nchunks, kce * es // 16, bn // 8, 8, 16 // es)
    return vals.permute(0, 1, 5, 6, 2, 3, 4, 7).reshape(p.batch, nnb * bn, nslots, nchunks * kce)


def unpack_workspace(p, ws):
    """The prepared operand as (N, Cout, Cin, k, k) fp32 (fp16 values widened): the weights the conv kernel multiplies."""
    slots = tap_slots(p)
    vals = workspace_rows(p, ws)[:, :p.out_channels, :, :p.in_channels].to(torch.float32)
    k = p.kernel_size
    out = torch.zeros(p.batch, p.out_channels, p.in_channels, k * k, dtype=torch.float32, device=ws.device)
    for s, t in enumerate(slots):
        out[:, :, :, t] = vals[:, :, s, :]
    return out.view(p.batch, p.out_channels, p.in_channels, k, k)


def tap_slots(p):
    """Kernel tap (ky * k + kx) of each operand slot, in the order csrc/modconv.cu make_taps() lays them out."""
    if p.up == 2:                                                  # phases (py, px) row-major; phase 0 rows ky = 0, 2
        ks1 = [[0, 2], [1]]
        return [ky * 3 + kx for py in range(2) for px in range(2) for ky in ks1[py] for kx in ks1[px]]
    return list(range(p.kernel_size * p.kernel_size))


# ------------------------------------------------------------------------------------------ eligibility
def _reference_forward(layer):
    cls = type(layer)
    return getattr(cls, '_p3d_reference_forward', None) or cls.forward


def _needs_autograd(layer, *tensors):
    if not torch.is_grad_enabled():
        return False
    return any(t.requires_grad for t in tensors) or any(q.requires_grad for q in layer.parameters())


def _up2_padding(layer, f):
    """conv2d_resample's FIR padding after its stride-2 transposed conv (conv2d_resample.py up > 1 branch); None when that
    conv would need padding (pxt / pyt > 0), which the kernel does not implement."""
    fw, fh = _upfirdn2d._get_filter_size(f)
    kh, kw = layer.weight.shape[2:]
    px0 = px1 = py0 = py1 = layer.padding
    up = layer.up
    px0 += (fw + up - 1) // 2; px1 += (fw - up) // 2
    py0 += (fh + up - 1) // 2; py1 += (fh - up) // 2
    px0 -= kw - 1; px1 -= kw - up; py0 -= kh - 1; py1 -= kh - up
    if max(min(-px0, -px1), 0) or max(min(-py0, -py1), 0):
        return None
    return [px0, px1, py0, py1]


def measured_faster(p) -> bool:
    """The shapes where the kernel route measured at least as fast as the reference's own layers in device time: the fp16
    up-2 layers (bench_modconv.py, CUDA-graph replay, 1x H100 80GB HBM3 at a 400 W power limit, two runs: sr256_conv0
    0.176 / 0.178 ms vs 0.283 / 0.178 ms, sr512_conv0 0.626 / 0.615 ms vs 0.647 / 0.625 ms).  Every other eval shape
    measured slower than the reference's cuDNN route (0.25x to 0.98x, DESIGN.md section 5), so it keeps that route."""
    return p.up == 2 and p.dtype == P3D_F16


def _kernel_params(layer, x, demodulate, up=1):
    """Params of a call the kernel supports, else None."""
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 4 and x.dtype in (torch.float16, torch.float32) and layer.weight.is_cuda):
        return None
    p = make_params(x, layer.weight, demodulate, up=up)
    if not supported(p):
        return None
    if demodulate:
        if layer.activation not in _ACTS or (up == 2 and _up2_padding(layer, layer.resample_filter) is None) or \
                x.shape[1:] != (layer.in_channels, layer.resolution // up, layer.resolution // up):
            return None
    elif p.kernel_size != 1:
        return None
    return p


def _eligible(layer, x, w, fused_modconv, demodulate, up=1):
    if not fused_modconv or _needs_autograd(layer, x, w):
        return None
    p = _kernel_params(layer, x, demodulate, up)
    return p if p is not None and measured_faster(p) else None


# ------------------------------------------------------------------------------------------ layer forwards
def synthesis_layer_forward(layer, x, w, noise_mode='random', fused_modconv=True, gain=1):
    """``SynthesisLayer.forward`` (networks_stylegan2.py:334-354): same arguments, return value, dtype and memory format.
    Eligible calls run synthesis_layer_kernel, every other call the original method."""
    if _eligible(layer, x, w, fused_modconv, True, layer.up) is None:
        return _reference_forward(layer)(layer, x, w, noise_mode=noise_mode, fused_modconv=fused_modconv, gain=gain)
    return synthesis_layer_kernel(layer, x, w, noise_mode=noise_mode, gain=gain)


def torgb_forward(layer, x, w, fused_modconv=True):
    """``ToRGBLayer.forward`` (networks_stylegan2.py:376-380): same arguments, return value, dtype and memory format.
    Eligible calls run torgb_kernel, every other call the original method."""
    if _eligible(layer, x, w, fused_modconv, False) is None:
        return _reference_forward(layer)(layer, x, w, fused_modconv=fused_modconv)
    return torgb_kernel(layer, x, w)


def synthesis_layer_kernel(layer, x, w, noise_mode='random', gain=1):
    """The fused_modconv branch of SynthesisLayer.forward on the kernel, for any shape p3d_modconv_supported accepts
    (raises otherwise), whatever measured_faster says."""
    p = _kernel_params(layer, x, True, layer.up)
    if p is None:
        raise RuntimeError('panic3d_b200.modconv: this SynthesisLayer call is not covered by the kernel')
    assert noise_mode in ['random', 'const', 'none']
    styles = layer.affine(w)
    noise = None
    if layer.use_noise and noise_mode == 'random':
        noise = torch.randn([x.shape[0], 1, layer.resolution, layer.resolution], device=x.device) * layer.noise_strength
    if layer.use_noise and noise_mode == 'const':
        noise = layer.noise_const * layer.noise_strength
    ws = prep(p, layer.weight, styles)
    act_gain = layer.act_gain * gain
    act_clamp = layer.conv_clamp * gain if layer.conv_clamp is not None else None
    if layer.up == 1:
        return conv(p, x, ws, bias=layer.bias, noise=noise, act=layer.activation, gain=act_gain, clamp=act_clamp)
    y = conv(p, x, ws)                                             # conv_transpose2d's tensor, rounded to the layer dtype
    y = _upfirdn2d.upfirdn2d(y, layer.resample_filter, padding=_up2_padding(layer, layer.resample_filter), gain=layer.up ** 2)
    if noise is not None:
        y = y.add_(noise)
    return _bias_act.bias_act(y, layer.bias.to(y.dtype), act=layer.activation, gain=act_gain, clamp=act_clamp)


def torgb_kernel(layer, x, w):
    """The fused_modconv branch of ToRGBLayer.forward on the kernel (raises for calls it does not cover)."""
    p = _kernel_params(layer, x, False)
    if p is None:
        raise RuntimeError('panic3d_b200.modconv: this ToRGBLayer call is not covered by the kernel')
    styles = layer.affine(w) * layer.weight_gain
    ws = prep(p, layer.weight, styles)
    return conv(p, x, ws, bias=layer.bias, act='linear', gain=1.0, clamp=layer.conv_clamp)


def flops(p) -> int:
    """Multiply-adds x 2 of one p3d_modconv_forward call (shape-computed; up 2 counts the nine taps of each input pixel)."""
    taps = p.kernel_size * p.kernel_size
    return 2 * p.batch * p.in_h * p.in_w * taps * p.in_channels * p.out_channels


