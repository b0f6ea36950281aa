"""panic3d_b200 - H100-native (sm_90a) implementation of panic3d's tri-plane volumetric
rendering hot path behind the reference's own Python call surface.

Layout (mirrors the reference tree under /root/reference/_train/eg3dc/src):
    csrc/                              CUDA kernels + the C ABI (include/p3d_render.h, p3d_ops.h)
    _build.py / _lib.py                nvcc build recipe / ctypes binding of lib/libp3d.so
    training/volumetric_rendering/     ImportanceRenderer, RaySampler, MipRayMarcher2, math_utils
    training/triplane.py               OSGDecoder (+ FullyConnectedLayer)
    torch_utils/ops/                   bias_act, upfirdn2d, filtered_lrelu
    cameras.py                         camera_params_to_matrix / get_rays_ortho (host-side camera helpers)
    dropin.py                          install(): makes the reference import these modules instead of its own

There is no CPU fallback anywhere in this package: ops raise if the CUDA library is
missing or a tensor is not on a CUDA device.
"""
__version__ = '0.1.0'

from . import _lib  # noqa: F401  (does not load the .so until first use)
