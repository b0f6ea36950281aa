"""Mutation check of the PNG kernels (needs an H100): single-line value mutations of csrc/png_deflate.cu (the device
encoder, against tests/test_png_device_gpu.py), csrc/png_inflate.cu (the device decoder, against
tests/test_png_decode_paths_gpu.py) and csrc/image_io.cu (the scan-line filter and quantisation kernels, against
tests/test_imageio_gpu.py), each built into its own library in a temporary directory and run against its GPU test
file, which must fail on every one.  The build, run and report are tests/run_mutations.py's: this file registers three
more targets with it.

    python tests/run_png_mutations.py [png_deflate] [png_inflate] [image_io] [--json out.json] [--build-only] [--files F ...]

With no target, all three run.
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

# png_inflate.cu: value mutations only.  None touches a bound that guards an access (`len > br.n - q`, `ds > 29`,
# `s > 285`, `hlit > 286`, `i + rep > hlit + hdist`, `dist > p`, `len > out_len - p`, check_job), a loop bound, a
# __syncwarp or the window mask, and every decode step still consumes bits or ends the stream, so each mutant stays in
# bounds and terminates whatever it decodes.  The reason for each is next to it.
STORED_CHECKS = 'if (len > br.n - q) return fail(P3D_PNG_ETRUNCATED);\n                    if (len > out_len - p) return fail(P3D_PNG_ELONG);'
PNG_INFLATE = {
    # a fixed block after a dynamic one decodes with the dynamic block's tables: same array sizes, symbols still checked
    'fixed tables not rebuilt after a dynamic block': ('if (t.kind != 1) fixed_tables(t);', 'if (t.kind == 0) fixed_tables(t);'),
    # length 258 reads 5 more bits (the __constant__ table only): the length is still checked against the output left
    'length symbol 285 with 5 extra bits': ('c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};',
                                            'c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 5};'),
    # a literal/length code without end-of-block is accepted; the block then ends by running out of output or input
    'no end-of-block check': ('if (t.lens[256] == 0) return P3D_PNG_ECODES;', 'if (false) return P3D_PNG_ECODES;'),
    # a single one-bit code is refused too: only more refusals
    'single one-bit code refused': ('if (left > 0 && max > 1) return false;', 'if (left > 0 && max > 0) return false;'),
    # the Adler-32 sum weighs the four bytes of a word alike: a value the status compares, nothing is indexed by it
    'Adler weight without the byte in the word': ('s2 += (n - (4 * k + c)) * x;', 's2 += (n - 4 * k) * x;'),
    # a refusal's status code swapped for a neighbour's: the refusal stays where it is
    'HLIT / HDIST refusal as ESYMBOL': ('if (hlit > 286 || hdist > 30) return P3D_PNG_ECODES;',
                                        'if (hlit > 286 || hdist > 30) return P3D_PNG_ESYMBOL;'),
    'code-length symbol outside the code as ETRUNCATED': ('if (s < 0) return P3D_PNG_ECODES;', 'if (s < 0) return P3D_PNG_ETRUNCATED;'),
    'repeat 16 first as ESYMBOL': ('if (i == 0) return P3D_PNG_ECODES;', 'if (i == 0) return P3D_PNG_ESYMBOL;'),
    'repeat past HLIT + HDIST as ETRUNCATED': ('if (i + rep > hlit + hdist) return P3D_PNG_ECODES;',
                                               'if (i + rep > hlit + hdist) return P3D_PNG_ETRUNCATED;'),
    'stored LEN past the input as ELONG': (STORED_CHECKS, STORED_CHECKS.replace('fail(P3D_PNG_ETRUNCATED)', 'fail(P3D_PNG_ELONG)')),
    'stored block past the output as ESHORT': (STORED_CHECKS, STORED_CHECKS.replace('fail(P3D_PNG_ELONG)', 'fail(P3D_PNG_ESHORT)')),
    'distance symbol 30 / 31 as EDISTANCE': ('if (ds < 0 || ds > 29) return fail(P3D_PNG_ESYMBOL);',
                                             'if (ds < 0 || ds > 29) return fail(P3D_PNG_EDISTANCE);'),
    'literal past the output as ESHORT': ('if (p >= out_len) return fail(P3D_PNG_ELONG);', 'if (p >= out_len) return fail(P3D_PNG_ESHORT);'),
    # unfilter and resample: the row above is still read only for rows r0 >= 1, the source index still checked against
    # n_in, and the 16-bit sample's other byte lies inside the same pixel
    'Average rounds up': ('type == 3 ? (a + bb) >> 1', 'type == 3 ? (a + bb + 1) >> 1'),
    # `pa <= pb` -> `pa < pb` is not here: it is equivalent.  pa = pb with a != b means c is the midpoint of a and b, so
    # the prediction a + b - c is c itself, pc = 0 < pa, and both versions pick c.  A b / c tie is not: a = 0, b = 3,
    # c = 1 gives pa = 2, pb = pc = 1
    'Paeth prefers the upper-left byte on a b / c tie': ('return pa <= pb && pa <= pc ? a : pb <= pc ? bb : c;',
                                                         'return pa <= pb && pa <= pc ? a : pb < pc ? bb : c;'),
    'band seam: rows 32-63 see a zero row above': ('if (r0 > 0 && x >= 0 && x < w) {', 'if (r0 > 32 && x >= 0 && x < w) {'),
    'nearest source index accumulated in float': ('const double scale = (double)n_in / n_out;\n    double x = scale * 0.5;',
                                                  'const float scale = (float)n_in / n_out;\n    float x = scale * 0.5f;'),
    'composite rounding constant halved': ('(0x80 << 7)', '(0x80 << 6)'),
    '16-bit samples: the low byte': ('if (c < job.channels) px[c] = q[c * bs];', 'if (c < job.channels) px[c] = q[c * bs + bs - 1];'),
}

# image_io.cu: value mutations of the quantisation and of the filter choice; no index, launch shape or shared-memory size
# changes (the row above is still read only for y >= 1).
IMAGE_IO = {
    'Up filter scored without the int8 fold': ('f = filt(2, x, l, b, ul); s2 += f < 128 ? f : 256 - f;', 'f = filt(2, x, l, b, ul); s2 += f;'),
    'Paeth wins a tie': ('if (s4 < best) { best = s4; type = 4; }', 'if (s4 <= best) { best = s4; type = 4; }'),
    'quantisation rounds to nearest': ('return (unsigned int)(int)(v * 255.f);', 'return (unsigned int)__float2int_rn(v * 255.f);'),
    'row 1 filtered against a zero row': ('prev[x * a.c + ch] = y > 0 ?', 'prev[x * a.c + ch] = y > 1 ?'),
}
# Not here: the clamp order fmaxf(fminf(v, 1), 0), which in C takes NaN to 1.  nvcc compiles either order to one
# saturating add (FADD.SAT, which takes NaN to 0) on sm_90a, so the mutant is equivalent as built;
# test_special_values_and_filter_ties holds the NaN -> 0 that both give.

TARGETS = {
    'png_deflate': ('png_deflate.cu', 'tests/test_png_device_gpu.py', PNG_DEFLATE),
    'png_inflate': ('png_inflate.cu', 'tests/test_png_decode_paths_gpu.py', PNG_INFLATE),
    'image_io': ('image_io.cu', 'tests/test_imageio_gpu.py', IMAGE_IO),
}
run_mutations.TARGETS.update(TARGETS)

if __name__ == '__main__':
    if not any(a in TARGETS for a in sys.argv[1:]):
        sys.argv[1:1] = list(TARGETS)
    run_mutations.main()
