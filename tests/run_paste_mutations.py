"""Mutation check of tests/test_paste_paths_gpu.py (needs an H100): build libp3d.so once per single-line value mutation
of csrc/paste_front.cu into a temporary directory, run the GPU file against it (P3D_LIBP3D), and report whether the file
fails it, as it must.  The tree is not modified.  Every mutation keeps all memory accesses in bounds (checked against the
file's shapes next to each entry) and none is equivalent at every scale the file runs.

    python tests/run_paste_mutations.py [--json out.json] [--files tests/test_paste_gpu.py ...]

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

MUTATIONS = {
    # a coordinate clipped at the lower border keeps its gradient (grid_sample's border padding gives it none)
    'lower clip keeps its gradient': ('if (ix <= 0.f) { ix = 0.f; mul = 0.f; }', 'if (ix <= 0.f) { ix = 0.f; }'),
    # the backward differentiates the front image without normalize_images' factor 2
    'backward ignores normalize_images': ('if (a.normalize) { f00 *= 2.f; f10 *= 2.f; f01 *= 2.f; f11 *= 2.f; }',
                                          'if (a.normalize) { }'),
    # eroded weights looked up at size min(R, Rf): indices stay below Rf; differs from the kernel only when R < Rf
    'eroded lookup at size min(R, Rf)': ('Tap tr = ortho_tap(vy, a.half_bw, a.inv_bw, a.Rf), tc = ortho_tap(vx, a.half_bw, a.inv_bw, a.Rf);',
                                         'Tap tr = ortho_tap(vy, a.half_bw, a.inv_bw, min(a.R, a.Rf)), tc = ortho_tap(vx, a.half_bw, a.inv_bw, min(a.R, a.Rf));'),
    # output row 0 is up-sampled from the row of output 1 (the halo row clamp starts at 1; every S here is >= 3).  At
    # scale <= 1/4 both rows clamp to source row 0, so only same_res, down and tiny_2x3 can see it
    'first image row sampled from row 1': ('min(max(ty0 + (int)threadIdx.x - 1, 0), a.S - 1)', 'min(max(ty0 + (int)threadIdx.x - 1, 1), a.S - 1)'),
    # the backward's up-sampling weights of taps (0, 1) and (1, 0) swapped
    'backward weights w01 / w10 swapped': ('w01 = by.l0 * bx.l1, w10 = by.l1 * bx.l0', 'w01 = by.l1 * bx.l0, w10 = by.l0 * bx.l1'),
    # the nearest source row rounded half up (its min(.., R - 1) keeps it in bounds); equal to the kernel at scales 1/4,
    # 1/8 and 1, different at 0.096 and 1.5
    'nearest row rounded half up': ('floorf((float)oy * a.scale)', 'floorf(((float)oy + 0.5f) * a.scale)'),
}
DEFAULT_FILES = [os.path.join('tests', 'test_paste_paths_gpu.py')]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json')
    ap.add_argument('--files', nargs='+', default=DEFAULT_FILES)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from panic3d_b200 import _build
    src = open(os.path.join(_build.CSRC, 'paste_front.cu')).read()
    objs = [o for o in sorted(os.listdir(os.path.join(_build.PKG, 'lib', 'obj'))) if o != 'paste_front.o']
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
            cu, obj, lib = os.path.join(d, 'a', 'b', 'paste_front.cu'), os.path.join(d, 'paste_front.o'), os.path.join(d, 'libp3d.so')
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
    default = args.files == DEFAULT_FILES
    sys.exit(0 if not default or all(v['killed'] for v in results.values()) else 1)


if __name__ == '__main__':
    main()
