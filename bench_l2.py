#!/usr/bin/env python
"""bench_l2.py - A/B of builds of libp3d.so on the fused renderer's workload, rounds alternated in one process.

    python bench_l2.py --lib NAME=PATH [--lib NAME=PATH ...] [--rounds 3] [--gather-rounds 2] [--launches 50] [--out DIR]

Each --lib is a build of the library (for example the parent commit's, and builds that differ only in the fused
renderer's L2 cache policies).  Every round runs, for each build in turn (the order rotates from round to round, so no
build always follows the same one), in a fresh process that loads that build through P3D_LIBP3D:
  * bench.py --gpus 1 --steps 100 --warmup 10 --no-e2e --no-variants --no-cpu-baseline: views/s of the flagship step;
  * bench_gather.py --rounds G --launches L: k_render_ws3 alone, the 512² fp32, 512² bf16 and 8² fp32 tri-plane arms.
The first round also passes --dump-outputs to bench.py, and the dumped .npy files of every build are compared byte for
byte with the first build's.  The card's name, power limit and maximum SM clock are read in the same run.  Prints one
JSON line: per build, the views/s of every round with their range, and the median of each bench_gather arm per round.
Nothing is written into the tree: dumps go to --out (default: a temporary directory)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       stdout=subprocess.PIPE, text=True, timeout=60, check=True).stdout.strip().splitlines()
    return q[0]


def run_json(cmd, lib):
    """Runs `cmd` from the repository root with P3D_LIBP3D=lib; returns the last line of its output that is a JSON object."""
    env = dict(os.environ, P3D_LIBP3D=lib)
    r = subprocess.run([sys.executable] + cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f'{" ".join(cmd)} with {lib} exited {r.returncode}:\n{r.stdout[-4000:]}')
    for line in reversed(r.stdout.splitlines()):
        if line.startswith('{'):
            return json.loads(line)
    raise RuntimeError(f'{" ".join(cmd)} printed no JSON line:\n{r.stdout[-4000:]}')


def same_files(a, b):
    names = sorted(os.listdir(a))
    if names != sorted(os.listdir(b)) or not names:
        return False
    for n in names:
        with open(os.path.join(a, n), 'rb') as fa, open(os.path.join(b, n), 'rb') as fb:
            if fa.read() != fb.read():
                return False
    return True


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--lib', action='append', required=True, metavar='NAME=PATH', help='a build of libp3d.so (repeat)')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--gather-rounds', type=int, default=2, help='bench_gather.py --rounds per build and round')
    ap.add_argument('--launches', type=int, default=50, help='bench_gather.py --launches')
    ap.add_argument('--out', help='directory for the --dump-outputs files (default: a temporary one)')
    args = ap.parse_args()
    libs = []
    for spec in args.lib:
        name, _, path = spec.partition('=')
        path = os.path.abspath(path)
        if not name or not os.path.isfile(path):
            raise SystemExit(f'--lib {spec}: expected NAME=PATH of an existing libp3d.so')
        libs.append((name, path))

    res = {'card': card(), 'bench': 'bench.py --gpus 1 --steps 100 --warmup 10 --no-e2e --no-variants --no-cpu-baseline',
           'builds': {name: {'views_per_s': [], 'gather': []} for name, _ in libs}}
    with tempfile.TemporaryDirectory(prefix='p3d_l2ab_') as tmp:
        out = args.out or tmp
        for rnd in range(args.rounds):
            for name, lib in libs[rnd % len(libs):] + libs[:rnd % len(libs)]:
                cmd = ['bench.py', '--gpus', '1', '--steps', '100', '--warmup', '10', '--no-e2e', '--no-variants', '--no-cpu-baseline']
                if rnd == 0:
                    cmd += ['--dump-outputs', os.path.join(out, 'dump_' + name)]
                b = res['builds'][name]
                b['views_per_s'].append(run_json(cmd, lib)['value'])
                gat = run_json(['bench_gather.py', '--rounds', str(args.gather_rounds), '--launches', str(args.launches)], lib)
                b['gather'].append({arm: v['median_ms'] for arm, v in gat['arms'].items()} | {'p512_over_p8': gat['p512_over_p8']})
                print(json.dumps({'round': rnd, 'build': name, 'views_per_s': b['views_per_s'][-1], 'gather': b['gather'][-1]}),
                      file=sys.stderr, flush=True)
        first = os.path.join(out, 'dump_' + libs[0][0])
        for name, b in res['builds'].items():
            v = b['views_per_s']
            b['views_per_s_range'] = [min(v), max(v)]
            b['dump_outputs_identical_to_' + libs[0][0]] = same_files(first, os.path.join(out, 'dump_' + name))
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
