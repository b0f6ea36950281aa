"""Mutation check of the device PNG encoder (needs an H100): the single-line value mutations of csrc/png_deflate.cu below,
each built into its own library in a temporary directory and run against tests/test_png_device_gpu.py, which must fail on
every one.  The build, run and report are tests/run_mutations.py's: this file registers one more target with it.

    python tests/run_png_mutations.py [--json out.json] [--build-only] [--files F ...]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import run_mutations  # noqa: E402

# png_deflate.cu: every mutation changes a value, never a bound that guards an access: a chosen block never exceeds the
# stored size, so the emission buffer and the workspace slot hold every mutant's bits.
PNG_DEFLATE = {
    'distance code off by one': ('return 2 * l + (((d - 1) >> (l - 1)) & 1);', 'return 2 * l - 1 + (((d - 1) >> (l - 1)) & 1);'),
    'length code 285 with 5 extra bits': ('5, 5, 5, 5, 0};', '5, 5, 5, 5, 5};'),
    'sync-flush block omitted': ('nbytes = final_seg ? (bits + 7) / 8 : (bits + 3 + 7) / 8 + 4;', 'nbytes = (bits + 7) / 8;'),
    'Adler combine without the length term': ('B = (B + T + S * (unsigned long long)((a.len - in0 - in_n) % kAdlerMod)) % kAdlerMod;',
                                              'B = (B + T) % kAdlerMod;'),
    # equivalent for the decoded bytes (only the ratio changes): killed by the window / seam assertions
    'window does not reach into the previous segment': ('const int avail = (int)min((long long)kWin, start);', 'const int avail = 0;'),
    'CRC partial shifted by the bytes before it': ('x8pow(s_x8, total - o - bytes)', 'x8pow(s_x8, o)'),
    'fixed code: literals 144-255 of 8 bits': ('s < 256 ? 9 :', 's < 256 ? 8 :'),
    'last stored block without BFINAL': ('ob[0] = final_seg ? 1 : 0;', 'ob[0] = 0;'),
}
TARGET = ('png_deflate.cu', 'tests/test_png_device_gpu.py', PNG_DEFLATE)
run_mutations.TARGETS['png_deflate'] = TARGET

if __name__ == '__main__':
    sys.argv[1:1] = ['png_deflate']
    run_mutations.main()
