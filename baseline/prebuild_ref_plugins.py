"""Pre-build the reference's three JIT CUDA plugins (bias_act, upfirdn2d, filtered_lrelu) for an H100 on a machine without a
GPU, into the directory layout `torch_utils/custom_ops.get_plugin` (custom_ops.py:61-157) looks for:
TORCH_EXTENSIONS_DIR/<plugin>/<md5 of sources>-<mangled GPU name>/.  Same sources (copied verbatim by install_ref.sh), same
flags (`--use_fast_math`, the only flag the reference passes) and the arch list get_plugin ends up with on a single H100:
it clears TORCH_CUDA_ARCH_LIST, so torch derives '9.0+PTX' from the device.  If ninja decides on the GPU machine that
something is stale it simply rebuilds (~40 s per plugin) - this only saves GPU minutes.

    python baseline/prebuild_ref_plugins.py baseline/_ref baseline/_ref/_torch_ext [mangled GPU name]

The GPU name defaults to custom_ops._get_mangled_gpu_name() of "NVIDIA H100 80GB HBM3"; pass the name of another card.
"""
import os, sys, time, hashlib, shutil
os.environ['TORCH_CUDA_ARCH_LIST'] = '9.0+PTX'
import torch, torch.utils.cpp_extension as ce
REF = sys.argv[1]
OUT = sys.argv[2]
GPU = sys.argv[3] if len(sys.argv) > 3 else 'nvidia-h100-80gb-hbm3'
os.environ['TORCH_EXTENSIONS_DIR'] = OUT
src_dir = os.path.join(REF, '_train/eg3dc/src/torch_utils/ops')
plugins = {
    'bias_act_plugin': (['bias_act.cpp', 'bias_act.cu'], ['bias_act.h'], ['--use_fast_math']),
    'upfirdn2d_plugin': (['upfirdn2d.cpp', 'upfirdn2d.cu'], ['upfirdn2d.h'], ['--use_fast_math']),
    'filtered_lrelu_plugin': (['filtered_lrelu.cpp', 'filtered_lrelu_wr.cu', 'filtered_lrelu_rd.cu', 'filtered_lrelu_ns.cu'], ['filtered_lrelu.h', 'filtered_lrelu.cu'], ['--use_fast_math']),
}
for name, (srcs, hdrs, flags) in plugins.items():
    t0 = time.time()
    allf = sorted(os.path.join(src_dir, f) for f in srcs + hdrs)
    h = hashlib.md5()
    for f in allf:
        h.update(open(f, 'rb').read())
    top = ce._get_build_directory(name, verbose=False)
    bdir = os.path.join(top, f'{h.hexdigest()}-{GPU}')
    os.makedirs(bdir, exist_ok=True)
    for f in allf:
        shutil.copyfile(f, os.path.join(bdir, os.path.basename(f)))
    try:
        ce.load(name=name, build_directory=bdir, verbose=False, sources=[os.path.join(bdir, s) for s in srcs], extra_cuda_cflags=flags, is_python_module=False)
        print(name, 'built in %.0fs' % (time.time() - t0), bdir)
    except Exception as e:
        print(name, 'FAILED', str(e)[-1500:])
