"""CUDA-graph replay of the generator's launch-bound sub-networks (SURVEY.md 8f-1: the callers of the renderer).

One view of the eval sweep through the unchanged ``G.f`` is ~150 eager PyTorch launches, most of them a few microseconds long
(per-layer modulation, demodulation, noise, bias/activation, layout conversions around cuDNN), issued by one Python thread, so its
wall clock is far above its device time.  The renderer is a single launch; the StyleGAN2 backbone (``G.backbone.synthesis``) and
the super-resolution head (``G.superresolution``) are where the launches are, and for a given input signature they are static
launch sequences.  This module
captures each of them ONCE into a CUDA graph and replays it:

    ``GraphedCallable(fn)``        inference-only wrapper: the first call with a new signature (tensor shapes / dtypes, non-tensor
                                   arguments) warms up on a side stream and captures; later calls copy the inputs into the graph's
                                   static buffers, replay, and return clones of the static outputs
    ``enable_cuda_graphs(G)``      puts one in front of ``G.backbone.synthesis.forward`` and ``G.superresolution.forward``
                                   (instance attributes, like ``dropin.enable_plane_reuse``; ``state_dict`` / hooks untouched)

Nothing is traced or compiled: the captured work is exactly the kernels the eager call launches (cuDNN convolutions, the p3d ops,
PyTorch elementwise kernels), in the same order, on the same data - outputs are bit-identical to the eager call for deterministic
inputs (``noise_mode='const'`` / ``'none'``); with ``noise_mode='random'`` every replay draws fresh noise (PyTorch's CUDA generator
is graph-aware).  Calls under autograd, or whose arguments cannot be keyed (unknown types), bypass the graph.  If warm-up or capture
fails for a signature, the wrapper says so once (``RuntimeWarning``) and that signature stays on the eager path - same CUDA code, no
fallback to another implementation.
"""
from __future__ import annotations

import warnings

import torch


def _flatten(obj, tensors, path=''):
    """-> a hashable skeleton of ``obj`` with every tensor replaced by (index, shape, dtype, device); tensors collected in order."""
    if torch.is_tensor(obj):
        tensors.append(obj)
        return ('T', len(tensors) - 1, tuple(obj.shape), str(obj.dtype), str(obj.device))
    if isinstance(obj, dict):
        return ('D',) + tuple((str(k), _flatten(obj[k], tensors)) for k in sorted(obj, key=str))
    if isinstance(obj, (list, tuple)):
        return ('L' if isinstance(obj, list) else 'U',) + tuple(_flatten(v, tensors) for v in obj)
    if obj is None or isinstance(obj, (bool, int, float, str)):
        return ('C', obj)
    raise TypeError(f'unkeyable argument of type {type(obj).__name__}')


def _rebuild(obj, tensors, counter):
    """The same structure as ``obj`` with the i-th tensor replaced by ``tensors[i]``."""
    if torch.is_tensor(obj):
        counter[0] += 1
        return tensors[counter[0] - 1]
    if isinstance(obj, dict):
        out = type(obj)() if type(obj) is not dict else {}
        for k in sorted(obj, key=str):                       # same visiting order as _flatten
            out[k] = _rebuild(obj[k], tensors, counter)
        return out
    if isinstance(obj, (list, tuple)):
        return type(obj)(_rebuild(v, tensors, counter) for v in obj)
    return obj


class _Entry:
    __slots__ = ('graph', 'static_in', 'static_out', 'out_skel', 'out_obj')


class GraphedCallable:
    """See the module docstring.  ``hits`` / ``captures`` / ``bypassed`` count what happened to the calls."""

    def __init__(self, fn, name='callable', warmup=3, max_entries=8, lean_return_more=False):
        self.fn, self.name, self.warmup, self.max_entries = fn, name, warmup, max_entries
        self.lean_return_more = lean_return_more
        self.entries = {}
        self.failed = set()
        self.hits = self.captures = self.bypassed = 0

    def _capture(self, args, kwargs, tensors):
        dev = tensors[0].device
        e = _Entry()
        e.static_in = [t.detach().clone() for t in tensors]
        s_args, s_kwargs = _rebuild((list(args), kwargs), e.static_in, [0])
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():       # warm-up off the capture: cuDNN autotune, lazy inits, op caches
            for _ in range(self.warmup):
                self.fn(*s_args, **s_kwargs)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        e.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(e.graph):
            out = self.fn(*s_args, **s_kwargs)
        outs = []
        e.out_skel = _flatten(out, outs)
        e.static_out, e.out_obj = outs, out
        return e

    def __call__(self, *args, **kwargs):
        if self.lean_return_more and kwargs.get('return_more'):
            # opt-in: the reference's return_more route hands back `locals()` next to the result (networks_stylegan2.py:715-718), which
            # only debugging code reads; replay the graph of the plain call and return an empty dict in its place
            return self(*args, **{k: v for k, v in kwargs.items() if k != 'return_more'}), {}
        tensors = []
        try:
            key = _flatten((list(args), kwargs), tensors)
        except TypeError:
            key = None
        if (key is None or not tensors or not all(t.is_cuda for t in tensors) or key in self.failed
                or kwargs.get('return_more')                     # the reference returns locals() on that route: not a tensor structure
                or (torch.is_grad_enabled() and any(t.requires_grad for t in tensors))
                or torch.cuda.is_current_stream_capturing()):
            self.bypassed += 1
            return self.fn(*args, **kwargs)
        e = self.entries.get(key)
        if e is None:
            if len(self.entries) >= self.max_entries:
                self.bypassed += 1
                return self.fn(*args, **kwargs)
            try:
                with torch.cuda.device(tensors[0].device):      # capture on the tensors' device, whatever the caller's current one is
                    e = self._capture(args, kwargs, tensors)
            except Exception as err:                         # this signature stays eager; say so once
                self.failed.add(key)
                torch.cuda.synchronize()
                warnings.warn(f'panic3d_b200.graphs: capturing {self.name} failed ({type(err).__name__}: {err}); this signature stays on the '
                              'eager path', RuntimeWarning)
                self.bypassed += 1
                return self.fn(*args, **kwargs)
            self.entries[key] = e
            self.captures += 1
        with torch.no_grad(), torch.cuda.device(tensors[0].device):
            for dst, src in zip(e.static_in, tensors):
                if dst.data_ptr() != src.data_ptr():
                    dst.copy_(src)
            e.graph.replay()
            self.hits += 1
            return _rebuild(e.out_obj, [t.clone() for t in e.static_out], [0])


def enable_cuda_graphs(G, backbone=True, superresolution=True, lean_return_more=False):
    """Put a ``GraphedCallable`` in front of ``G.backbone.synthesis.forward`` and ``G.superresolution.forward``; idempotent.
    ``lean_return_more=True``: backbone calls with ``return_more=True`` (what ``G.f(x, return_more=True)`` issues, e.g.
    ``_scripts/eval/generate.py:130``) are replayed too and return ``(planes, {})`` instead of ``(planes, locals())`` - a deliberate
    deviation for callers that never look at the backbone's locals; off by default (such calls then stay eager).
    Returns {'backbone': wrapper, 'superresolution': wrapper} (``.hits`` / ``.captures`` / ``.bypassed``).  Composes with
    ``dropin.enable_plane_reuse`` in either order: the graph always ends up underneath the memo, which then skips the replay
    on repeated latents."""
    out = {}
    targets = []
    if backbone and hasattr(G, 'backbone') and isinstance(getattr(G.backbone, 'synthesis', None), torch.nn.Module):
        targets.append(('backbone', G.backbone.synthesis))
    if superresolution and isinstance(getattr(G, 'superresolution', None), torch.nn.Module):
        targets.append(('superresolution', G.superresolution))
    for name, mod in targets:
        wrapper = getattr(mod, '_p3d_graphed', None)
        if wrapper is None:
            memo = getattr(mod, '_p3d_plane_memo', None)          # dropin.enable_plane_reuse was here first: the graph goes UNDER the
            if memo is not None:                                  # memo (its value comparison of the latents is a host sync no capture allows)
                wrapper = GraphedCallable(memo.synthesis, name=name, lean_return_more=lean_return_more and name == 'backbone')
                memo.synthesis = wrapper
            else:
                wrapper = GraphedCallable(mod.forward, name=name, lean_return_more=lean_return_more and name == 'backbone')
                mod.forward = wrapper
            mod._p3d_graphed = wrapper
        out[name] = wrapper
    return out
