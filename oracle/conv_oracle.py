"""fp64 oracle of the fp32 training convolutions (panic3d_b200.conv): torch's own conv2d / conv_transpose2d and their
weight gradient in float64, the magnitude bound conv(|x|, |w|) the per-element bars scale with, and the bar's constant.

Bar (DESIGN.md 4.x): |ours - fp64| <= c(K) * conv(|x|, |w|) per element, with K the length of the element's dot product.
3xTF32 drops small * small and rounds both small parts to tf32, so each product is off by at most 3 * 2^-22 of |x||w|.
A 32-wide K chunk is summed by 12 wgmma steps, each off by at most 2^-23 of the chunk's sum of magnitudes (the tensor
cores may truncate rather than round); the ceil(K / 32) chunk sums and, for the weight gradient, up to 64 split partials
are then added with round-to-nearest fp32 adds, each off by at most 2^-24 of the running sum of magnitudes."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def bar_constant(K, splits=64):
    """c(K) of the per-element bar for dot products of length K."""
    return 3 * 2.0 ** -22 + 12 * 2.0 ** -23 + (math.ceil(K / 32) + splits) * 2.0 ** -24


def conv(x, w, stride, padding, transpose, output_padding=0):
    """conv2d / conv_transpose2d in float64 (the inputs' device)."""
    x, w = x.double(), w.double()
    if transpose:
        return F.conv_transpose2d(x, w, stride=stride, padding=padding, output_padding=output_padding)
    return F.conv2d(x, w, stride=stride, padding=padding)


def weight_grad(x, w_shape, dy, stride, padding, transpose, output_padding=0):
    """The gradient of sum(y * dy) with respect to the weight, in float64."""
    w = torch.zeros(w_shape, dtype=torch.float64, device=x.device, requires_grad=True)
    with torch.enable_grad():
        y = conv(x, w, stride, padding, transpose, output_padding)
        (g,) = torch.autograd.grad(y, w, dy.double())
    return g


def input_grad(x_shape, w, dy, stride, padding, transpose, output_padding=0):
    """The gradient of sum(y * dy) with respect to the input, in float64."""
    x = torch.zeros(x_shape, dtype=torch.float64, device=w.device, requires_grad=True)
    with torch.enable_grad():
        y = conv(x, w, stride, padding, transpose, output_padding)
        (g,) = torch.autograd.grad(y, x, dy.double())
    return g
