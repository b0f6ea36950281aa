"""Mutation check of tests/test_decode_tc_depth_gpu.py (needs an H100): build libp3d.so once per single-line value mutation
of csrc/decode_tc.cu into a temporary directory, run the GPU file against it (P3D_LIBP3D), and report whether the file
fails it, as it must.  The tree is not modified.  Every mutation keeps all memory accesses in bounds and leaves the
mbarrier protocol alone (stage index, parities, arrival counts and the team stride are untouched), so none can hang.

    python tests/run_decode_tc_mutations.py [--json out.json] [--files tests/test_volume_gpu.py ...]

--files runs other GPU files against the same mutants instead (to see which of them the rest of the suite catches);
the exit code then only reports that the run completed.
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

TILE = 'const long long tile = (long long)blockIdx.x + (long long)it * gridDim.x;'
MUTATIONS = {
    # the gather computes tile it % 3 instead of tile it from the fourth tile of a CTA on
    'gather tile it % kTeams': (TILE + '\n            // ---- tap table',
                                TILE.replace('(long long)it *', '(long long)(it % kTeams) *') + '\n            // ---- tap table'),
    # the decoder writes tile it % 4's outputs from the fifth tile of a CTA on
    'decoder output tile it % kNA': (TILE + '\n#pragma unroll\n            for (int rs',
                                     TILE.replace('(long long)it *', '(long long)(it % kNA) *') + '\n#pragma unroll\n            for (int rs'),
    'tap-row view index 0': ('px, py, pz, (uint32_t)view);', 'px, py, pz, 0u);'),
    'single pass never set': ('a.single_pass = p->mlp_mode == P3D_MLP_TC_BF16;', 'a.single_pass = 0;'),
    'tiles per CTA rounded down': ('(a.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x',
                                   '(a.n_tiles - (int)blockIdx.x) / (int)gridDim.x'),
    'gather row shifted by one within the tile': ('tile * 128 + wt * 32 + lane;', 'tile * 128 + ((wt * 32 + lane + 1) & 127);'),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json')
    ap.add_argument('--files', nargs='+', default=[os.path.join('tests', 'test_decode_tc_depth_gpu.py')])
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _build
    src = open(os.path.join(_build.CSRC, 'decode_tc.cu')).read()
    objs = [o for o in sorted(os.listdir(os.path.join(_build.PKG, 'lib', 'obj'))) if o != 'decode_tc.o']
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
            cu, obj, lib = os.path.join(d, 'a', 'b', 'decode_tc.cu'), os.path.join(d, 'decode_tc.o'), os.path.join(d, 'libp3d.so')
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
            print(f'{name:42s} {"killed" if r.returncode else "SURVIVED"}: {results[name]["summary"][:120]}', flush=True)
            for ln in failed:
                print(f'    {ln[:160]}', flush=True)
    if args.json:
        json.dump(results, open(args.json, 'w'), indent=1)
    default = args.files == ap.get_default('files')
    sys.exit(0 if not default or all(v['killed'] for v in results.values()) else 1)


if __name__ == '__main__':
    main()
