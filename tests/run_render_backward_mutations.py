"""Mutation check of tests/test_render_backward_paths_gpu.py (needs an H100): build libp3d.so once per single-line value
mutation of csrc/render_backward.cu into a temporary directory, run the GPU file against it (P3D_LIBP3D), and report whether
the file fails it, as it must.  The tree is not modified.  Every mutation changes a value, never an index or a bound that
guards a memory access (the tap mutation narrows the bound, so it only drops taps).

    python tests/run_render_backward_mutations.py [--json out.json] [--files tests/test_render_gpu.py ...]

--files runs other GPU files against the same mutants instead (to see which of them the rest of the suite catches);
the exit code then only reports that the run completed.

The depth gate `depth_raw >= lo_b` is not mutated: a ray's unclamped depth is a weighted mean of its interval midpoints,
which lie strictly inside [min depth, max depth] of the batch, so no case can put it on the bound and `>` equals `>=`.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]
sys.path.insert(0, ROOT)

MUTATIONS = {
    'colour factor 1.002 -> 1': ('(g.force_sigmoid ? 1.f : 1.002f)', '(g.force_sigmoid ? 1.f : 1.f)'),
    'hidden softplus derivative threshold 20 -> 5': ('(pre > 20.f ? 1.f : sigmoid_t(pre))', '(pre > 5.f ? 1.f : sigmoid_t(pre))'),
    'interval softplus derivative linear branch 1 -> 0': ('smid > 20.f ? 1.f : sigmoid_t(smid)', 'smid > 20.f ? 0.f : sigmoid_t(smid)'),
    'white background term without g_xyz': ('2.f * back * (grgb_sum + gx_sum)', '2.f * back * (grgb_sum)'),
    'suffix term not divided by 1 - alpha': ('Tr[i] * P - suffix / fc[i];', 'Tr[i] * P - suffix;'),
    'tap bound xi < W - 1': ('const bool ok = (xi >= 0) && (xi < g.W) && (yi >= 0) && (yi < g.H);\n        const float wgt = ((k & 1) ? f.wx1 : f.wx0) * ((k >> 1) ? f.wy1 : f.wy0);\n        out[k]',
                             'const bool ok = (xi >= 0) && (xi < g.W - 1) && (yi >= 0) && (yi < g.H);\n        const float wgt = ((k & 1) ? f.wx1 : f.wx0) * ((k >> 1) ? f.wy1 : f.wy0);\n        out[k]'),
    'd_w1 scaled by the bias gain': ('acc[i][j] * g.w1_gain);', 'acc[i][j] * g.b1_gain);'),
    'd_b2 scaled by the weight gain': ('atomicAdd(a.d_b2 + tid, acc * g.b2_gain);', 'atomicAdd(a.d_b2 + tid, acc * g.w2_gain);'),
    'omega without its 1/2': ('om = 0.5f * (wl + wr);', 'om = (wl + wr);'),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json')
    ap.add_argument('--files', nargs='+', default=[os.path.join('tests', 'test_render_backward_paths_gpu.py')])
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _build
    src = open(os.path.join(_build.CSRC, 'render_backward.cu')).read()
    objs = [o for o in sorted(os.listdir(os.path.join(_build.PKG, 'lib', 'obj'))) if o != 'render_backward.o']
    nvcc = '/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else 'nvcc'
    flags = [x for x in _build.NVCC_FLAGS if x != '-shared']
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        def build(i_name):
            i, name = i_name
            old, new = MUTATIONS[name]
            assert src.count(old) == 1, name
            d = os.path.join(tmp, f'm{i}')
            os.makedirs(os.path.join(d, 'a', 'b'))
            cu, obj, lib = (os.path.join(d, 'a', 'b', 'render_backward.cu'), os.path.join(d, 'render_backward.o'),
                            os.path.join(d, 'libp3d.so'))
            open(cu, 'w').write(src.replace(old, new))
            os.symlink(os.path.join(ROOT, 'include'), os.path.join(d, 'include'))      # the file's "../../include/..." includes
            for cmd in ([nvcc] + flags + ['-I', _build.CSRC, '-c', cu, '-o', obj],
                        [nvcc] + _build.ARCH + ['-shared', '-o', lib, obj] + [os.path.join(_build.PKG, 'lib', 'obj', o) for o in objs] + ['-lz']):
                r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                if r.returncode:
                    raise RuntimeError(f'{name}: nvcc failed\n{r.stdout}')
            return name, lib
        with ThreadPoolExecutor(max_workers=max(1, min(len(MUTATIONS), os.cpu_count() or 1))) as ex:
            libs = dict(ex.map(build, enumerate(MUTATIONS)))
        for name in MUTATIONS:
            r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-x', '-m', 'gpu', '-p', 'no:cacheprovider'] +
                               [os.path.join(ROOT, f) for f in args.files],
                               cwd=ROOT, env=dict(os.environ, P3D_LIBP3D=libs[name]), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                               text=True)
            failed = [ln for ln in r.stdout.splitlines() if ln.startswith('FAILED') or ln.startswith('ERROR')]
            results[name] = {'killed': r.returncode != 0, 'failures': failed, 'summary': r.stdout.strip().splitlines()[-1]}
            print(f'{name:50s} {"killed" if r.returncode else "SURVIVED"}: {results[name]["summary"][:120]}', flush=True)
            for ln in failed:
                print(f'    {ln[:160]}', flush=True)
    if args.json:
        json.dump(results, open(args.json, 'w'), indent=1)
    default = args.files == ap.get_default('files')
    sys.exit(0 if not default or all(v['killed'] for v in results.values()) else 1)


if __name__ == '__main__':
    main()
