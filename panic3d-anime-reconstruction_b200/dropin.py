"""Plug the H100 hot path into an unmodified checkout of the reference.

The reference instantiates the renderer by import name
(`from training.volumetric_rendering.renderer import ImportanceRenderer`, triplane.py:14-15, and again when
`load_eg3dc_model` rebuilds G from current source, _train/eg3dc/util/eg3dc_v0.py:46-52) and its ops by
`from torch_utils.ops import bias_act, upfirdn2d, ...`.  `install()` registers this package's modules under
those names in `sys.modules` BEFORE the reference imports them, so `G.synthesis`, `G.f`, `G.sample_mixed`,
`_scripts.eval.generate` and the training loop call into the CUDA library with no caller edits.

    import panic3d_b200.dropin as dropin
    dropin.install()                    # before `import training.triplane` / `load_eg3dc_model(...)`
"""
from __future__ import annotations

import importlib
import sys

_RENDER = {
    'training.volumetric_rendering.renderer': '.training.volumetric_rendering.renderer',
    'training.volumetric_rendering.ray_sampler': '.training.volumetric_rendering.ray_sampler',
    'training.volumetric_rendering.ray_marcher': '.training.volumetric_rendering.ray_marcher',
    'training.volumetric_rendering.math_utils': '.training.volumetric_rendering.math_utils',
}
_OPS = {
    'torch_utils.ops.bias_act': '.torch_utils.ops.bias_act',
    'torch_utils.ops.upfirdn2d': '.torch_utils.ops.upfirdn2d',
    'torch_utils.ops.filtered_lrelu': '.torch_utils.ops.filtered_lrelu',
}


def install(renderer: bool = True, ops: bool = True, strict: bool = False):
    """Register the drop-in modules. Returns the list of reference module names now served by this package.
    `strict=True` raises if the reference already imported one of them (too late to swap by name)."""
    pkg = __name__.rsplit('.', 1)[0]
    table = {}
    if renderer:
        table.update(_RENDER)
    if ops:
        table.update(_OPS)
    done = []
    for ref_name, ours in table.items():
        try:
            mod = importlib.import_module(ours, pkg)
        except ModuleNotFoundError:
            if strict:
                raise
            continue
        prev = sys.modules.get(ref_name)
        if prev is not None and prev is not mod and strict:
            raise RuntimeError(f'{ref_name} was imported before panic3d_b200.dropin.install(); call install() first')
        sys.modules[ref_name] = mod
        parent_name, leaf = ref_name.rsplit('.', 1)
        parent = sys.modules.get(parent_name)
        if parent is not None:
            setattr(parent, leaf, mod)
        done.append(ref_name)
    return done


def install_paste(module=None, reuse_triplane=False):
    """Rebind the reference's ``paste_front`` (SURVEY 8f-3; ``training/triplane.py:608-691``) and its two render helpers
    to the fused implementation in ``panic3d_b200.paste``.  ``G.f`` looks ``paste_front`` up in its own module's globals
    at call time (triplane.py:498-502), so setting the attribute on that module is the whole plug-in: no caller edits.
    ``module``: the reference's already-imported ``training.triplane`` (default: import it by that name).
    ``reuse_triplane=True``: the occlusion render of ``paste_front`` is rendered from ``out['triplane']`` instead of a second full
    ``G.f`` (backbone + super-resolution re-run for nothing) - a documented deviation, see ``paste.REUSE_TRIPLANE``.
    Returns the names that were rebound."""
    from . import paste
    paste.REUSE_TRIPLANE = bool(reuse_triplane)
    if module is None:
        module = importlib.import_module('training.triplane')
    names = ['paste_front', 'get_front_occlusion', 'get_front_weights']
    for name in names:
        if not hasattr(module, '_p3d_reference_' + name):
            setattr(module, '_p3d_reference_' + name, getattr(module, name, None))       # keep the original reachable for A/B runs
        setattr(module, name, getattr(paste, name))
    return names


def install_modconv(module=None):
    """Rebind ``SynthesisLayer.forward`` and ``ToRGBLayer.forward`` of the reference's ``training.networks_stylegan2`` to
    ``panic3d_b200.modconv`` (the fused modulated convolution at inference).  ``superresolution.py`` imports the same
    classes, so this covers the backbone and the super-resolution head.  Calls the kernel does not cover (CPU, training,
    ``fused_modconv=False``, TF32 disallowed for fp32 layers, unsupported shapes) run the original method, which stays
    reachable as ``<class>._p3d_reference_forward``.  ``module``: the already-imported module (default: import it by that
    name).  Returns the names that were rebound."""
    from . import modconv
    if module is None:
        module = importlib.import_module('training.networks_stylegan2')
    names = []
    for cls_name, fn in (('SynthesisLayer', modconv.synthesis_layer_forward), ('ToRGBLayer', modconv.torgb_forward)):
        cls = getattr(module, cls_name)
        if '_p3d_reference_forward' not in cls.__dict__:
            cls._p3d_reference_forward = cls.forward                  # keep the original reachable for A/B runs
        cls.forward = fn
        names.append(cls_name + '.forward')
    return names


def install_conv2d(module=None):
    """Rebind ``conv2d`` and ``conv_transpose2d`` of the reference's ``torch_utils.ops.conv2d_gradfix`` to
    ``panic3d_b200.conv`` (the fp32 training convolutions in 3xTF32 on the tensor cores).  ``conv2d_resample`` looks both
    up on that module at call time, so no caller changes.  Calls the kernels do not cover, or where they did not measure
    faster than cuDNN (``conv.measured_faster``), run the originals, which stay reachable as ``_p3d_reference_conv2d`` /
    ``_p3d_reference_conv_transpose2d``.  ``module``: the already-imported module (default: import it by that name).
    Returns the names that were rebound."""
    from . import conv
    if module is None:
        module = importlib.import_module('torch_utils.ops.conv2d_gradfix')
    names = ['conv2d', 'conv_transpose2d']
    for name in names:
        if not hasattr(module, '_p3d_reference_' + name):
            setattr(module, '_p3d_reference_' + name, getattr(module, name))     # keep the original reachable for A/B runs
        setattr(module, name, getattr(conv, name))
    conv._gradfix = module
    return names


def patch_generator(G):
    """For a TriPlaneGenerator that was built BEFORE install() (e.g. unpickled): swap its two hot-path
    sub-modules in place.  Both are parameter-free, so no weights move."""
    from .training.volumetric_rendering.renderer import ImportanceRenderer
    from .training.volumetric_rendering.ray_sampler import RaySampler
    use_triplane = bool(G.rendering_kwargs.get('use_triplane', False))
    G.renderer = ImportanceRenderer(use_triplane=use_triplane)
    G.ray_sampler = RaySampler()
    return G


class _PlaneMemo:
    """Memo around ``G.backbone.synthesis`` (SURVEY 8f-1).  One subject's eval sweep calls ``G.f`` once per view - 16
    camera views plus the warm-ups - and every call re-runs the 29 M-parameter StyleGAN2 backbone on the SAME
    ``(ws, cond)`` (``triplane.py:188-196`` has ``use_cached_backbone`` / ``_last_planes`` for this, but ``G.f`` never sets
    them, and ``get_eg3d_volume`` re-runs it 168 more times, ``_util/eg3d_metrics3d.py:125-151``).  The memo returns the
    previous tri-planes when the latents and the conditioning are unchanged: compared by identity first, then by value
    (``ws`` is (N,14,512): one tiny device compare per call).  Strong references to the key tensors are held so that a
    freed-and-reallocated buffer can never alias a stale entry.  Training is untouched: calls under autograd
    (``torch.is_grad_enabled()`` with any input requiring grad), with ``update_emas=True`` or with non-'const' noise
    bypass the memo.

    Noise: ``G.f`` / ``G.synthesis`` never pass ``noise_mode``, so in the reference every call draws fresh
    ``SynthesisLayer`` noise (``networks_stylegan2.py:334-343``: default 'random') - each view of a sweep sees slightly
    different tri-planes.  Replaying one stochastic draw for all views would be neither the reference's behaviour nor
    deterministic, so the memo does one of two explicit things with a call that leaves ``noise_mode`` out:
    ``default_noise_mode='const'`` (what ``enable_plane_reuse`` sets up, a DELIBERATE, documented deviation: the whole
    sweep is rendered from the const-noise tri-planes, deterministic and cacheable) passes that mode on to the backbone;
    ``default_noise_mode=None`` leaves the call untouched and treats it as 'random' = not cacheable."""

    def __init__(self, synthesis, default_noise_mode='const'):
        self.synthesis = synthesis
        self.default_noise_mode = default_noise_mode
        self.key = None
        self.planes = None
        self.hits = self.misses = 0

    @staticmethod
    def _tensors(obj, out):
        import torch
        if isinstance(obj, torch.Tensor):
            out.append(obj)
        elif isinstance(obj, dict):
            for k in sorted(obj, key=str):
                _PlaneMemo._tensors(obj[k], out)
        elif isinstance(obj, (list, tuple)):
            for v in obj:
                _PlaneMemo._tensors(v, out)
        return out

    @staticmethod
    def _same(now, stored):
        """stored: (tensor or clone, version at store time or None for a clone)."""
        import torch
        if len(now) != len(stored):
            return False
        for x, (y, ver) in zip(now, stored):
            if ver is not None:
                if y._version != ver:
                    return False                                                  # the kept tensor was written in place: stale
                if x is y:
                    continue                                                      # same big tensor, untouched since
            if x.shape != y.shape or x.dtype != y.dtype or x.device != y.device or not torch.equal(x, y):
                return False
        return True

    def __call__(self, ws, cond=None, *args, **kwargs):
        import torch
        if 'noise_mode' not in kwargs and self.default_noise_mode is not None:
            kwargs = dict(kwargs, noise_mode=self.default_noise_mode)
        tensors = self._tensors([ws, cond, list(args), kwargs], [])
        cacheable = (not kwargs.get('update_emas', False) and kwargs.get('noise_mode', 'random') in ('const', 'none')
                     and not kwargs.get('return_more', False)
                     and not (torch.is_grad_enabled() and any(t.requires_grad for t in tensors)))
        scalars = repr(sorted((k, v) for k, v in kwargs.items() if not isinstance(v, (torch.Tensor, dict, list, tuple))))
        if cacheable and self.key is not None and self.key[1] == scalars and self._same(tensors, self.key[0]):
            self.hits += 1
            return self.planes
        planes = self.synthesis(ws, cond, *args, **kwargs)
        if cacheable:
            # small tensors (latents) are cloned; big ones (conditioning images / feature maps) are kept by reference with
            # their version counter - an in-place write bumps it and forces the value comparison
            self.key = ([(t.detach().clone(), None) if t.numel() <= 1 << 16 else (t, t._version) for t in tensors], scalars)
            self.planes = planes
            self.misses += 1
        return planes

    def clear(self):
        self.key = self.planes = None


def enable_plane_reuse(G, default_noise_mode='const'):
    """Wrap ``G.backbone.synthesis`` with a one-entry memo (see ``_PlaneMemo``); idempotent.  Returns the memo
    (``.hits`` / ``.misses`` / ``.clear()``).  With it, a 16-view sweep of one subject through unchanged ``G.f`` runs the
    backbone once, and the renderer's channels-last layout pass once (its plane cache keys on the same tensor).
    ``default_noise_mode``: the noise mode given to backbone calls that do not name one ('const': deterministic sweep,
    cacheable - differs from the reference, which redraws the layer noise for every view; None: keep the reference's
    per-call random noise, in which case only calls that explicitly ask for 'const' / 'none' are cached)."""
    import torch
    syn = G.backbone.synthesis
    if isinstance(syn, torch.nn.Module):
        # the real backbone: `synthesis` is a registered sub-module (networks_stylegan2.SynthesisNetwork), so it cannot be
        # replaced by a plain callable - the memo goes in front of its forward instead (instance attribute; Module.__call__
        # and hooks keep working, state_dict is untouched)
        memo = getattr(syn, '_p3d_plane_memo', None)
        if memo is None:
            memo = _PlaneMemo(syn.forward, default_noise_mode)
            syn.forward = memo
            syn._p3d_plane_memo = memo
        return memo
    if isinstance(syn, _PlaneMemo):
        return syn
    memo = _PlaneMemo(syn, default_noise_mode)
    G.backbone.synthesis = memo
    return memo
