"""Mutation check of the multiplane GPU tests (needs an H100): build libp3d.so once per single-line value mutation of the
multiplane section of csrc/render_device.cuh into a temporary directory, run tests/test_multiplane_paths_gpu.py against it
(P3D_LIBP3D), and report whether the file fails it, as it must.  The tree is not modified.

    python tests/run_mutations_multiplane.py [--files F ...] [--json out.json] [--build-only]

The mutated code is a header, so each mutant recompiles every translation unit that includes it directly (render_v1.cu,
render_backward.cu, marching_cubes.cu) from a copy next to the mutated header, where its #include "render_device.cuh"
finds the mutant first.  The fused kernels reach the header through fused_common.cuh but call none of the multiplane
functions, so their objects are the tree's.  --files runs other GPU files against the same mutants instead (to see which
of them tests/test_multiplane_gpu.py catches); the exit code then only reports that the run completed.  --build-only builds
every mutant and stops; nvcc cross-compiles, so it needs no GPU.  tests/run_mutations.py is the driver for the other kernel
files (its render_backward_multiplane target mutates the TRI lines of render_backward.cu).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from panic3d_b200 import _build  # noqa: E402

HEADER = 'render_device.cuh'
TEST_FILE = 'tests/test_multiplane_paths_gpu.py'

# Value mutations; every index they produce is still checked against its bound before it addresses memory, except the slab
# stride from W, which stays in bounds because every plane of both multiplane GPU files has H >= W.  No tap count, shared
# memory size or tap-table stride is mutated: an unwritten s_tap entry would send the backward's atomics out of bounds.
MUTATIONS = {
    'slab coordinate with align_corners=True': (
        'const float fz = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gz, 1.f), (float)g.D), 1.f), 0.5f);',
        'const float fz = __fmul_rn(__fmul_rn(__fadd_rn(gz, 1.f), (float)(g.D - 1)), 0.5f);'),
    'slab index off by one': ('t.z0 = sane ? (int)z0f : -4;', 't.z0 = sane ? (int)z0f + 1 : -4;'),
    'EG3D plane 2 normal taken as x': ('(pm ? x : y));', '(pm ? x : x));'),
    'depth axis clamped instead of zero-padded': (', zi = t.z0 + (k >> 2);', ', zi = min(max(t.z0 + (k >> 2), 0), g.D - 1);'),
    'backward scatters to one slab only': ('const int z = t.z0 + (k >> 2);', 'const int z = t.z0;'),
    'slab offset from plane_w instead of plane_h': ('const long long slab = (long long)g.H * g.stride_row;',
                                                    'const long long slab = (long long)g.W * g.stride_row;'),
    # the backward's weight of slab z0 + 1 (slab_texels; the same line in plane_taps3 is followed by `r.w[k]`)
    'backward weight of slab z0 + 1 taken as z0\'s': ('t.wz1 : t.wz0);\n        out[k]', 't.wz0 : t.wz0);\n        out[k]'),
    # the normal's zero-padding bands dropped: a point within a slab below slab 0 (or above slab D - 1) reads nothing
    'zero-padding band below slab 0 dropped': ('(fz > -2.f) &&', '(fz >= 0.f) &&'),
    'zero-padding band above slab D - 1 dropped': ('(fz < (float)g.D + 1.f)', '(fz < (float)(g.D - 1))'),
}


def including_units():
    """The .cu files that include the header directly."""
    return [s for s in _build.sources() if f'#include "{HEADER}"' in open(s).read()]


def build_mutant(nvcc, d, name):
    """Write the mutated header and copies of its including units into d, compile those, link with the tree's other
    objects; returns the library's path."""
    text = open(os.path.join(_build.CSRC, HEADER)).read()
    old, new = MUTATIONS[name]
    assert text.count(old) == 1, name
    os.makedirs(d)
    open(os.path.join(d, HEADER), 'w').write(text.replace(old, new))
    objs = {}
    for src in including_units():
        cu = os.path.join(d, os.path.basename(src))
        open(cu, 'w').write(open(src).read())
        objs[src] = cu[:-3] + '.o'
        # -I csrc: the copy finds csrc's other headers, and "../../include/..." resolves from csrc to the repository's include/
        r = subprocess.run(_build.compile_cmd(nvcc, cu, objs[src], ['-I', _build.CSRC]), stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True)
        if r.returncode:
            raise RuntimeError(f'{name}: nvcc failed on {os.path.basename(src)}\n{r.stdout}')
    lib = os.path.join(d, 'libp3d.so')
    r = subprocess.run(_build.link_cmd(nvcc, lib, [objs.get(s, _build.object_path(s)) for s in _build.sources()]),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode:
        raise RuntimeError(f'{name}: link failed\n{r.stdout}')
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--files', nargs='+')
    ap.add_argument('--json')
    ap.add_argument('--build-only', action='store_true')
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    nvcc = _build.find_nvcc()
    names = list(MUTATIONS)
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        with ThreadPoolExecutor(max_workers=max(1, min(len(names), os.cpu_count() or 1))) as ex:
            libs = list(ex.map(lambda i: build_mutant(nvcc, os.path.join(tmp, f'm{i}'), names[i]), range(len(names))))
        if args.build_only:
            print(f'built {len(libs)} mutants', flush=True)
            return
        for name, lib in zip(names, libs):
            r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-x', '-m', 'gpu', '-p', 'no:cacheprovider',
                               ] + [os.path.join(ROOT, f) for f in args.files or [TEST_FILE]], cwd=ROOT, env=dict(os.environ, P3D_LIBP3D=lib),
                               stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            failed = [ln for ln in r.stdout.splitlines() if ln.startswith('FAILED') or ln.startswith('ERROR')]
            results[name] = {'killed': r.returncode != 0, 'failures': failed, 'summary': r.stdout.strip().splitlines()[-1]}
            print(f'multiplane: {name:50s} {"killed" if r.returncode else "SURVIVED"}: {results[name]["summary"][:120]}', flush=True)
            for ln in failed[:2]:
                print(f'    {ln[:160]}', flush=True)
    if args.json:
        json.dump(results, open(args.json, 'w'), indent=1)
    sys.exit(0 if args.files or all(v['killed'] for v in results.values()) else 1)


if __name__ == '__main__':
    main()
