"""Cost of the deterministic training backward (torch.use_deterministic_algorithms(True)) against the atomic one.

Three workloads, each timed with the switch off and on, alternated in one process:
  render   config 5's training render through ImportanceRenderer: 4 views x 64^2 rays x 48+48 samples x 256^2 tri-planes,
           forward + backward of bench.py's loss
  points   the density-regularisation (Greg) point query through run_model: 4 views x 2 x 1000 points, forward + backward
  paste    paste_front_fused 'Agrad' (grad_sample=True) at the training size: 4 views, 64^2 render -> 512^2 image, backward

Per workload: ms per step (CUDA events), extra device memory at peak (torch.cuda.max_memory_allocated over the step, on minus
off), and a torch.profiler pass that splits the deterministic backward's time into the sort (CUB radix sort kernels) and the
reductions (k_texel_sum, k_pair_level / k_params_out, k_paste_dxyz_gather).  Prints one JSON line; with --out, writes it there.

    python bench_deterministic.py --steps 20 --warmup 5 [--out deterministic.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess

import torch


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'nvidia-smi unavailable'
    return {'device': torch.cuda.get_device_name(0), 'nvidia_smi': q}


def _render_step():
    from oracle import renderer_oracle as orc
    from panic3d_b200.training.triplane import OSGDecoder
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = 'cuda:0'
    N, R, S, H = 4, 64, 48, 256
    g = torch.Generator(device=dev).manual_seed(5)
    planes = torch.randn(N, 3, 32, H, H, generator=g, device=dev).requires_grad_(True)
    dec = OSGDecoder(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32}).to(dev)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=S)
    th = torch.linspace(-0.6, 0.6, N, device=dev)
    lin = (torch.arange(R, device=dev) + 0.5) / R * 0.7 - 0.35
    yy, xx = torch.meshgrid(lin, lin, indexing='ij')
    base = torch.stack([xx, yy, torch.full_like(xx, 2.0)], -1).reshape(-1, 3)
    ro = torch.stack([base @ torch.tensor([[c, 0, -s], [0, 1, 0], [s, 0, c]], device=dev) for c, s in zip(th.cos(), th.sin())])
    rd = torch.nn.functional.normalize(-ro + torch.randn_like(ro) * 0.01, dim=-1)
    r = ImportanceRenderer(use_triplane=True)

    def step():
        rgb, depth, wsum, _ = r(planes, dec, ro, rd, opts)
        loss = rgb.mean() + 0.1 * depth.mean() + 0.1 * wsum.mean()
        planes.grad = None
        dec.zero_grad(set_to_none=True)
        loss.backward()
    return step


def _points_step():
    from oracle import renderer_oracle as orc
    from panic3d_b200.training.triplane import OSGDecoder
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    dev = 'cuda:0'
    g = torch.Generator(device=dev).manual_seed(6)
    planes = torch.randn(4, 3, 32, 256, 256, generator=g, device=dev).requires_grad_(True)
    dec = OSGDecoder(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32}).to(dev)
    coords = (torch.rand(4, 2000, 3, generator=g, device=dev) * 2 - 1) * 0.3
    r = ImportanceRenderer(use_triplane=True)

    def step():
        out = r.run_model(planes, dec, coords, None, dict(orc.DEFAULT_OPTS))
        loss = out['sigma'].abs().mean()
        planes.grad = None
        dec.zero_grad(set_to_none=True)
        loss.backward()
    return step


def _paste_step():
    from oracle import paste_oracle as po
    import panic3d_b200.paste as pp
    dev = 'cuda:0'
    d = {k: v.to(dev) for k, v in po.synth_paste_inputs(42, 4, 64, 512, box_warp=0.7, reach=1.2).items() if torch.is_tensor(v)}
    image = d['image'].clone().requires_grad_(True)
    xyz = d['image_xyz'].clone().requires_grad_(True)
    kw = dict(thresh_weight=0.95, thresh_edges=0.02, thresh_occ=0.05, thresh_dxyz=0.000005)

    def step():
        img, paste, _, _ = pp.paste_front_fused(image, xyz, d['image_weights'], d['front_rgb'], d['occ'], d['ro'], d['rd'], 0.7,
                                                grad_sample=True, **kw)
        image.grad = xyz.grad = None
        (img.mean() + paste.mean()).backward()
    return step


def _time(step, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _peak(step):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


SORT = ('DeviceRadixSort',)
REDUCE = ('k_texel_sum', 'k_pair_level', 'k_params_out', 'k_paste_dxyz_gather')
BWD = ('k_sample_backward', 'k_ray_backward', 'k_paste_front_bwd')


def _kernel_ms(step, steps):
    """Device ms per step of the sort, reduction and other backward kernels, from one torch.profiler pass."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    out = {'sort': 0.0, 'reductions': 0.0, 'backward_kernels': 0.0}
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 / steps if hasattr(e, 'device_time_total') else e.cuda_time_total / 1e3 / steps
        if any(s in e.key for s in SORT):
            out['sort'] += t
        elif any(s in e.key for s in REDUCE):
            out['reductions'] += t
        elif any(s in e.key for s in BWD):
            out['backward_kernels'] += t
    return {k: round(v, 4) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_deterministic.py measures on the GPU; no CUDA device here')
    import panic3d_b200  # noqa: F401
    res = {'card': _card(), 'steps': a.steps, 'rounds': a.rounds}
    for name, make in (('render', _render_step), ('points', _points_step), ('paste', _paste_step)):
        step = make()
        row = {'off_ms': [], 'on_ms': []}
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            for _ in range(a.warmup):
                step()
        for _ in range(a.rounds):                 # off and on alternated
            for det in (False, True):
                torch.use_deterministic_algorithms(det)
                row['on_ms' if det else 'off_ms'].append(round(_time(step, a.steps), 4))
        mem = {}
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            mem[det] = _peak(step)
        row['peak_bytes_off'], row['peak_bytes_on'] = mem[False], mem[True]
        row['extra_peak_MiB'] = round((mem[True] - mem[False]) / 2 ** 20, 1)
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            row['kernels_on' if det else 'kernels_off'] = _kernel_ms(step, max(2, a.steps // 4))
        torch.use_deterministic_algorithms(False)
        row['ratio_on_off'] = round(min(row['on_ms']) / min(row['off_ms']), 3)
        res[name] = row
    res['card_after'] = _card()['nvidia_smi']
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
