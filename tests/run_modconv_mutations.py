"""Mutation check of tests/test_modconv_gpu.py (needs an H100): build libp3d.so once per single-line value mutation of
csrc/modconv.cu into a temporary directory, run the GPU file against it (P3D_LIBP3D), and report whether the file fails
it, as it must.  The tree is not modified.  Every mutation keeps all memory accesses in bounds.

    python tests/run_modconv_mutations.py [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MUTATIONS = {
    'demod epsilon dropped': ('block_reduce(ss, false, red) + 1e-8f', 'block_reduce(ss, false, red)'),
    'style applied per output channel': ('s = srow[ci];', 's = srow[co % a.Cin];'),
    'sub-pixel phases 1 and 2 swapped': ('    t.ntaps = s;\n',
                                         '    t.ntaps = s;\n    if (t.nphase == 4) { const int b1 = t.base[1]; t.base[1] = t.base[2]; t.base[2] = b1; }\n'),
    'last partial channel chunk skipped': ('const int ksteps = min(KCE, a.Cin - q * KCE) * ES / 32;',
                                           'const int ksteps = a.Cin - q * KCE < KCE ? 0 : KCE * ES / 32;'),
    'gain applied after the clamp': ('        v *= a.gain;\n        if (a.clamp >= 0.f) v = (v > -a.clamp && v < a.clamp) ? v : (v >= 0.f ? a.clamp : -a.clamp);\n',
                                     '        if (a.clamp >= 0.f) v = (v > -a.clamp && v < a.clamp) ? v : (v >= 0.f ? a.clamp : -a.clamp);\n        v *= a.gain;\n'),
    'noise indexed per channel': ('(long long)oy * a.snh', '(long long)(co % a.H) * a.snh'),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json')
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _build
    src = open(os.path.join(_build.CSRC, 'modconv.cu')).read()
    objs = [o for o in sorted(os.listdir(os.path.join(_build.PKG, 'lib', 'obj'))) if o != 'modconv.o']
    nvcc = '/usr/local/cuda/bin/nvcc' if os.path.exists('/usr/local/cuda/bin/nvcc') else 'nvcc'
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        os.symlink(os.path.join(ROOT, 'include'), os.path.join(tmp, 'include'))      # the file's "../../include/..." includes
        os.makedirs(os.path.join(tmp, 'a', 'b'))
        for name, (old, new) in MUTATIONS.items():
            assert src.count(old) == 1, name
            cu = os.path.join(tmp, 'a', 'b', 'modconv.cu')
            open(cu, 'w').write(src.replace(old, new))
            obj, lib = os.path.join(tmp, 'modconv.o'), os.path.join(tmp, 'libp3d.so')
            flags = [x for x in _build.NVCC_FLAGS if x != '-shared']
            subprocess.run([nvcc] + flags + ['-I', _build.CSRC, '-c', cu, '-o', obj], check=True)
            subprocess.run([nvcc] + _build.ARCH + ['-shared', '-o', lib, obj] + [os.path.join(_build.PKG, 'lib', 'obj', o) for o in objs] + ['-lz'],
                           check=True)
            r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-x', '-m', 'gpu', '-p', 'no:cacheprovider',
                                os.path.join(ROOT, 'tests', 'test_modconv_gpu.py')],
                               cwd=ROOT, env=dict(os.environ, P3D_LIBP3D=lib), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            failed = [ln for ln in r.stdout.splitlines() if ln.startswith('FAILED')]
            results[name] = {'killed': r.returncode != 0, 'first_failure': failed[0] if failed else r.stdout.strip().splitlines()[-1]}
            print(f'{name:38s} {"killed" if r.returncode else "SURVIVED"}: {results[name]["first_failure"][:150]}', flush=True)
    if args.json:
        json.dump(results, open(args.json, 'w'), indent=1)
    sys.exit(0 if all(v['killed'] for v in results.values()) else 1)


if __name__ == '__main__':
    main()
