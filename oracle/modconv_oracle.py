"""Torch restatement (any device, any dtype - fp64 for the checks) of StyleGAN2's modulated convolution at inference, the
code ``panic3d_b200.modconv`` replaces.  Reference: ``_train/eg3dc/src/training/networks_stylegan2.py`` and
``torch_utils/ops/conv2d_resample.py``.

    modulated_conv2d         :40-98, the fused_modconv=True branch (with the fp16 inf-norm pre-normalisation of :60-63)
    conv2d_resample          conv2d_resample.py: the up = 1 plain-conv fast path and the up > 1 transposed-conv route
    synthesis_layer_forward  SynthesisLayer.forward, :334-354
    torgb_forward            ToRGBLayer.forward, :376-380
    SynthesisLayer / ToRGBLayer / SynthesisBlock / FullyConnectedLayer
                             minimal stand-ins with the reference's attribute names (:21-..., :304-330, :358-372, :440-486),
                             whose ``forward`` is this restatement: the GPU tests rebind them like the reference classes.

The fp16 branch (with its pre-normalisation) is pinned to the reference by the fp16 CPU fixtures, which call the
reference's layers directly with fp16 inputs (its blocks would force fp32 on CPU, networks_stylegan2.py:444-445).

``per_sample_weights`` / ``tf32_rna`` give the operands the kernel multiplies: the modulated, demodulated weights rounded
to fp16 (fp16 layers) or to tf32 with round-to-nearest, ties away from zero (fp32 layers; the kernel's cvt.rna), and the
activations rounded the same way.
"""
from __future__ import annotations

import math
import sys

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ops_oracle


# ------------------------------------------------------------------------------------------ rounding of the kernel's operands
def tf32_rna(t):
    """fp32 -> tf32 (10-bit mantissa), round to nearest, ties away from zero (PTX cvt.rna.tf32.f32); returned as fp32."""
    b = t.to(torch.float32).contiguous().view(torch.int32)
    mag = (b & 0x7FFFFFFF) + 0x1000
    r = (b & -0x80000000) | (mag & 0x7FFFE000)
    finite = torch.isfinite(t.to(torch.float32))
    return torch.where(finite, r.view(torch.float32), t.to(torch.float32))


def per_sample_weights(weight, styles, demodulate, fp16_prenorm, dtype=torch.float64):
    """w[n,o,i,ky,kx] = W * s (after the fp16 pre-normalisation when asked), times rsqrt(sum w^2 + 1e-8) when demodulating
    (networks_stylegan2.py:60-72), computed in `dtype`."""
    weight, styles = weight.to(dtype), styles.to(dtype)
    cin, kh, kw = weight.shape[1:]
    if fp16_prenorm:
        weight = weight * (1 / np.sqrt(cin * kh * kw) / weight.norm(float('inf'), dim=[1, 2, 3], keepdim=True))
        styles = styles / styles.norm(float('inf'), dim=1, keepdim=True)
    w = weight.unsqueeze(0) * styles.reshape(styles.shape[0], 1, -1, 1, 1)
    if demodulate:
        w = w * (w.square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt().reshape(styles.shape[0], -1, 1, 1, 1)
    return w


def round_operand(t, layer_dtype):
    """The rounding the kernel applies to an operand of a layer of `layer_dtype` (returned in fp64)."""
    if layer_dtype == torch.float16:
        return t.to(torch.float16).to(torch.float64)
    return tf32_rna(t.to(torch.float32)).to(torch.float64)


# ------------------------------------------------------------------------------------------ conv2d_resample
def _conv2d_wrapper(x, w, stride=1, padding=0, groups=1, transpose=False, flip_weight=True):
    """conv2d_resample.py:31-53 (without the channels_last weight detail, which does not change values)."""
    kh, kw = w.shape[2:]
    if not flip_weight and (kw > 1 or kh > 1):
        w = w.flip([2, 3])
    op = F.conv_transpose2d if transpose else F.conv2d
    return op(x, w, stride=stride, padding=padding, groups=groups)


def conv2d_resample(x, w, f=None, up=1, down=1, padding=0, groups=1, flip_weight=True, flip_filter=False):
    """conv2d_resample.py:61-143 for down = 1: the plain-conv fast path (up = 1) and the transposed-conv route (up > 1)."""
    assert down == 1
    out_channels, in_channels_per_group, kh, kw = w.shape
    fw, fh = (1, 1) if f is None else (f.shape[-1], f.shape[0])
    px0 = px1 = py0 = py1 = padding
    if up > 1:
        px0 += (fw + up - 1) // 2
        px1 += (fw - up) // 2
        py0 += (fh + up - 1) // 2
        py1 += (fh - up) // 2
        if groups == 1:
            w = w.transpose(0, 1)
        else:
            w = w.reshape(groups, out_channels // groups, in_channels_per_group, kh, kw)
            w = w.transpose(1, 2)
            w = w.reshape(groups * in_channels_per_group, out_channels // groups, kh, kw)
        px0 -= kw - 1
        px1 -= kw - up
        py0 -= kh - 1
        py1 -= kh - up
        pxt = max(min(-px0, -px1), 0)
        pyt = max(min(-py0, -py1), 0)
        x = _conv2d_wrapper(x=x, w=w, stride=up, padding=[pyt, pxt], groups=groups, transpose=True, flip_weight=(not flip_weight))
        return ops_oracle.upfirdn2d(x, f, padding=[px0 + pxt, px1 + pxt, py0 + pyt, py1 + pyt], gain=up ** 2, flip_filter=flip_filter)
    assert px0 == px1 == py0 == py1 >= 0
    return _conv2d_wrapper(x=x, w=w, padding=[py0, px0], groups=groups, flip_weight=flip_weight)


def transposed_prefilter(x, w):
    """The tensor p3d_modconv_forward writes for up = 2: conv_transpose2d(stride 2, padding 0) of the per-sample weights
    w (N, O, I, 3, 3) before the FIR (the first half of conv2d_resample's up > 1 route, groups = N)."""
    n, o, i = w.shape[:3]
    wt = w.reshape(n, o, i, 3, 3).transpose(1, 2).reshape(n * i, o, 3, 3)
    y = F.conv_transpose2d(x.reshape(1, -1, *x.shape[2:]), wt, stride=2, groups=n)
    return y.reshape(n, o, *y.shape[2:])


def oracle_conv(x, w, up, k, chunk=4096):
    """The tensor p3d_modconv_forward computes before its epilogue, for per-sample weights w (N, O, I, k, k): the grouped
    conv (up 1, padding k // 2) or transposed_prefilter (up 2).  Runs `chunk` samples per grouped call."""
    if x.shape[0] > chunk:
        return torch.cat([oracle_conv(x[i:i + chunk], w[i:i + chunk], up, k) for i in range(0, x.shape[0], chunk)])
    n = x.shape[0]
    if up == 2:
        return transposed_prefilter(x, w)
    y = F.conv2d(x.reshape(1, -1, *x.shape[2:]), w.reshape(-1, *w.shape[2:]), padding=k // 2, groups=n)
    return y.reshape(n, -1, *y.shape[2:])


def epilogue64(acc, bias=None, noise=None, act='linear', gain=1.0, clamp=None):
    """The epilogue of p3d_modconv_forward on the accumulator `acc` (N, O, H, W): clamp(act(acc + noise + bias) * gain),
    act lrelu (slope 0.2) or linear, clamp None for none.  `noise` broadcasts against acc ([N, 1, H, W] or [H, W]); `bias`
    is given in the values the kernel reads (the layer dtype)."""
    v = acc if noise is None else acc + noise.double()
    if bias is not None:
        v = v + bias.double().reshape(1, -1, 1, 1)
    if act == 'lrelu':
        v = torch.where(v > 0, v, v * 0.2)
    v = v * gain
    return v if clamp is None else v.clamp(-clamp, clamp)


# ------------------------------------------------------------------------------------------ modulated_conv2d (fused branch)
def modulated_conv2d(x, weight, styles, noise=None, up=1, down=1, padding=0, resample_filter=None, demodulate=True,
                     flip_weight=True, fused_modconv=True):
    """networks_stylegan2.py:40-98.  The fused branch is the one inference takes; the non-fused one (:75-85, training) is
    here so that the stand-ins' original method covers every call the kernel route hands back to it."""
    batch_size = x.shape[0]
    out_channels, in_channels, kh, kw = weight.shape
    if not fused_modconv:
        if x.dtype == torch.float16 and demodulate:
            weight = weight * (1 / np.sqrt(in_channels * kh * kw) / weight.norm(float('inf'), dim=[1, 2, 3], keepdim=True))
            styles = styles / styles.norm(float('inf'), dim=1, keepdim=True)
        dcoefs = per_sample_weights(weight, styles, False, False, dtype=weight.dtype).square().sum(dim=[2, 3, 4]).add(1e-8).rsqrt()
        x = x * styles.to(x.dtype).reshape(batch_size, -1, 1, 1)
        x = conv2d_resample(x=x, w=weight.to(x.dtype), f=resample_filter, up=up, down=down, padding=padding, flip_weight=flip_weight)
        if demodulate and noise is not None:
            return x * dcoefs.to(x.dtype).reshape(batch_size, -1, 1, 1) + noise.to(x.dtype)
        if demodulate:
            return x * dcoefs.to(x.dtype).reshape(batch_size, -1, 1, 1)
        return x.add_(noise.to(x.dtype)) if noise is not None else x
    w = per_sample_weights(weight, styles, demodulate, x.dtype == torch.float16 and demodulate, dtype=weight.dtype)
    x = x.reshape(1, -1, *x.shape[2:])
    w = w.reshape(-1, in_channels, kh, kw)
    x = conv2d_resample(x=x, w=w.to(x.dtype), f=resample_filter, up=up, down=down, padding=padding, groups=batch_size,
                        flip_weight=flip_weight)
    x = x.reshape(batch_size, -1, *x.shape[2:])
    if noise is not None:
        x = x.add_(noise)
    return x


# ------------------------------------------------------------------------------------------ layer forwards
def synthesis_layer_forward(layer, x, w, noise_mode='random', fused_modconv=True, gain=1):
    """SynthesisLayer.forward, networks_stylegan2.py:334-354."""
    assert noise_mode in ['random', 'const', 'none']
    styles = layer.affine(w)
    noise = None
    if layer.use_noise and noise_mode == 'random':
        noise = torch.randn([x.shape[0], 1, layer.resolution, layer.resolution], device=x.device) * layer.noise_strength
    if layer.use_noise and noise_mode == 'const':
        noise = layer.noise_const * layer.noise_strength
    flip_weight = (layer.up == 1)
    x = modulated_conv2d(x=x, weight=layer.weight, styles=styles, noise=noise, up=layer.up, padding=layer.padding,
                         resample_filter=layer.resample_filter, flip_weight=flip_weight, fused_modconv=fused_modconv)
    act_gain = layer.act_gain * gain
    act_clamp = layer.conv_clamp * gain if layer.conv_clamp is not None else None
    return ops_oracle.bias_act(x, layer.bias.to(x.dtype), act=layer.activation, gain=act_gain, clamp=act_clamp)


def torgb_forward(layer, x, w, fused_modconv=True):
    """ToRGBLayer.forward, networks_stylegan2.py:376-380."""
    styles = layer.affine(w) * layer.weight_gain
    x = modulated_conv2d(x=x, weight=layer.weight, styles=styles, demodulate=False, fused_modconv=fused_modconv)
    return ops_oracle.bias_act(x, layer.bias.to(x.dtype), clamp=layer.conv_clamp)


# ------------------------------------------------------------------------------------------ stand-ins
class FullyConnectedLayer(torch.nn.Module):
    """networks_stylegan2.py FullyConnectedLayer with activation 'linear' (the `affine` of both layers)."""

    def __init__(self, in_features, out_features, bias_init=0, lr_multiplier=1):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn([out_features, in_features]) / lr_multiplier)
        self.bias = torch.nn.Parameter(torch.full([out_features], np.float32(bias_init)))
        self.weight_gain = lr_multiplier / np.sqrt(in_features)
        self.bias_gain = lr_multiplier

    def forward(self, x):
        w = self.weight.to(x.dtype) * self.weight_gain
        b = self.bias.to(x.dtype)
        if self.bias_gain != 1:
            b = b * self.bias_gain
        return torch.addmm(b.unsqueeze(0), x, w.t())


class SynthesisLayer(torch.nn.Module):
    def __init__(self, in_channels, out_channels, w_dim, resolution, kernel_size=3, up=1, use_noise=True, activation='lrelu',
                 resample_filter=(1, 3, 3, 1), conv_clamp=None):
        super().__init__()
        self.in_channels, self.out_channels, self.w_dim, self.resolution = in_channels, out_channels, w_dim, resolution
        self.up, self.use_noise, self.activation, self.conv_clamp = up, use_noise, activation, conv_clamp
        self.register_buffer('resample_filter', ops_oracle.setup_filter(list(resample_filter)))
        self.padding = kernel_size // 2
        self.act_gain = {'lrelu': np.sqrt(2), 'linear': 1.0}[activation]
        self.affine = FullyConnectedLayer(w_dim, in_channels, bias_init=1)
        self.weight = torch.nn.Parameter(torch.randn([out_channels, in_channels, kernel_size, kernel_size]))
        if use_noise:
            self.register_buffer('noise_const', torch.randn([resolution, resolution]))
            self.noise_strength = torch.nn.Parameter(torch.zeros([]))
        self.bias = torch.nn.Parameter(torch.zeros([out_channels]))

    def forward(self, x, w, noise_mode='random', fused_modconv=True, gain=1):
        return synthesis_layer_forward(self, x, w, noise_mode=noise_mode, fused_modconv=fused_modconv, gain=gain)


class ToRGBLayer(torch.nn.Module):
    def __init__(self, in_channels, out_channels, w_dim, kernel_size=1, conv_clamp=None):
        super().__init__()
        self.in_channels, self.out_channels, self.w_dim, self.conv_clamp = in_channels, out_channels, w_dim, conv_clamp
        self.affine = FullyConnectedLayer(w_dim, in_channels, bias_init=1)
        self.weight = torch.nn.Parameter(torch.randn([out_channels, in_channels, kernel_size, kernel_size]))
        self.bias = torch.nn.Parameter(torch.zeros([out_channels]))
        self.weight_gain = 1 / np.sqrt(in_channels * (kernel_size ** 2))

    def forward(self, x, w, fused_modconv=True):
        return torgb_forward(self, x, w, fused_modconv=fused_modconv)


class SynthesisBlock(torch.nn.Module):
    """The 'skip' SynthesisBlock with in_channels > 0 (networks_stylegan2.py:440-486): conv0 (up 2), conv1, ToRGB, and the
    up-sampled image skip.  Layer calls go through the classes' current ``forward``, so an installed kernel takes them."""

    def __init__(self, in_channels, out_channels, w_dim, resolution, img_channels, use_fp16=False, conv_clamp=None,
                 channels_last=False):
        super().__init__()
        self.in_channels, self.w_dim, self.resolution, self.img_channels = in_channels, w_dim, resolution, img_channels
        self.use_fp16, self.channels_last = use_fp16, channels_last
        self.register_buffer('resample_filter', ops_oracle.setup_filter([1, 3, 3, 1]))
        self.conv0 = SynthesisLayer(in_channels, out_channels, w_dim, resolution, up=2, conv_clamp=conv_clamp)
        self.conv1 = SynthesisLayer(out_channels, out_channels, w_dim, resolution, conv_clamp=conv_clamp)
        self.torgb = ToRGBLayer(out_channels, img_channels, w_dim, conv_clamp=conv_clamp)
        self.num_conv, self.num_torgb = 2, 1

    def forward(self, x, img, ws, force_fp32=False, fused_modconv=True, upsample_image=None, **layer_kwargs):
        w_iter = iter(ws.unbind(dim=1))
        if ws.device.type != 'cuda':
            force_fp32 = True
        dtype = torch.float16 if self.use_fp16 and not force_fp32 else torch.float32
        memory_format = torch.channels_last if self.channels_last and not force_fp32 else torch.contiguous_format
        x = x.to(dtype=dtype, memory_format=memory_format)
        x = self.conv0(x, next(w_iter), fused_modconv=fused_modconv, **layer_kwargs)
        x = self.conv1(x, next(w_iter), fused_modconv=fused_modconv, **layer_kwargs)
        if img is not None:
            img = (upsample_image or _upsample2d)(img, self.resample_filter)
        y = self.torgb(x, next(w_iter), fused_modconv=fused_modconv)
        y = y.to(dtype=torch.float32, memory_format=torch.contiguous_format)
        img = img.add_(y) if img is not None else y
        return x, img


def _upsample2d(x, f, up=2):
    """upfirdn2d.upsample2d (upfirdn2d.py:300-318) for a 4-tap filter."""
    fw = f.shape[-1]
    p = [(fw + up - 1) // 2, (fw - up) // 2, (fw + up - 1) // 2, (fw - up) // 2]
    return ops_oracle.upfirdn2d(x, f, up=up, padding=p, gain=up * up)


def init_layer_(layer, seed, bias_scale=0.5, noise_strength=0.3):
    """Deterministic non-trivial parameters for a stand-in or reference layer (the reference initialises bias and
    noise_strength to zero, which would leave the epilogue untested)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, q in sorted(layer.named_parameters()):
            q.copy_(torch.randn(q.shape, generator=g) * (bias_scale if name.endswith('bias') and q.dim() == 1 and 'affine' not in name else 1.0)
                    + (1.0 if name == 'affine.bias' else 0.0))
        if getattr(layer, 'use_noise', False):
            layer.noise_strength.fill_(noise_strength)
            layer.noise_const.copy_(torch.randn(layer.noise_const.shape, generator=g))
    return layer


# ------------------------------------------------------------------------------------------ the eval generator's layer shapes
# (name, Cin, Cout, output resolution, up, kind, dtype, conv_clamp) of bench_config3.build_generator's eval generator:
# the fp32 backbone (channel_base 32768, channel_max 512, 96-channel ToRGBs, no clamp) and the fp16 8XDC SR head (clamp 256)
def _eval_shapes():
    bb = [('b4_conv1', 512, 512, 4, 1, 'layer'), ('b4_torgb', 512, 96, 4, 1, 'torgb')]
    for r in (8, 16, 32, 64, 128, 256):
        ci, co = min(32768 // (r // 2), 512), min(32768 // r, 512)
        bb += [(f'b{r}_conv0', ci, co, r, 2, 'layer'), (f'b{r}_conv1', co, co, r, 1, 'layer'), (f'b{r}_torgb', co, 96, r, 1, 'torgb')]
    sr = [('sr256_conv0', 32, 256, 256, 2, 'layer'), ('sr256_conv1', 256, 256, 256, 1, 'layer'), ('sr256_torgb', 256, 3, 256, 1, 'torgb'),
          ('sr512_conv0', 256, 128, 512, 2, 'layer'), ('sr512_conv1', 128, 128, 512, 1, 'layer'), ('sr512_torgb', 128, 3, 512, 1, 'torgb')]
    return [s + (torch.float32, None) for s in bb] + [s + (torch.float16, 256) for s in sr]


EVAL_SHAPES = _eval_shapes()


def make_layer(name, cin, cout, res, up, kind, dtype, clamp, seed=0, w_dim=64, module=None):
    """One layer of an EVAL_SHAPES row (of `module`'s classes: default these stand-ins), seeded by init_layer_."""
    module = module or sys.modules[__name__]
    if kind == 'torgb':
        layer = module.ToRGBLayer(cin, cout, w_dim, conv_clamp=clamp)
    else:
        layer = module.SynthesisLayer(cin, cout, w_dim, res, up=up, conv_clamp=clamp)
    return init_layer_(layer, seed)


def sr_head(seed=0, w_dim=64):
    """The 8XDC head's two blocks (32 -> 256 at 256^2, 256 -> 128 at 512^2, fp16, clamp 256, 3 image channels)."""
    blocks = torch.nn.ModuleList([SynthesisBlock(32, 256, w_dim, 256, 3, use_fp16=True, conv_clamp=256),
                                  SynthesisBlock(256, 128, w_dim, 512, 3, use_fp16=True, conv_clamp=256)])
    for i, b in enumerate(blocks):
        for j, layer in enumerate([b.conv0, b.conv1, b.torgb]):
            init_layer_(layer, seed + 10 * i + j)
    return blocks


def run_blocks(blocks, x, img, ws, noise_mode):
    """Blocks in sequence, three ws rows each (conv0, conv1, torgb); returns the image."""
    for i, b in enumerate(blocks):
        x, img = b(x, img, ws[:, 3 * i:3 * i + 3], noise_mode=noise_mode)
    return img


SQRT_HALF = math.sqrt(0.5)
