// Tap tables and operand-tile helpers of the 3xTF32 training convolutions (conv_fp32.cu).  The table is modconv.cu's
// (same struct, same phase order, same MODE_UP2 split) plus MODE_S2; modconv.cu keeps its own copy because its mutation
// tables (tests/run_mutations.py) anchor on that text.
//
// A convolution is split into sub-pixel phases; each phase is a correlation over its own output grid.  Slots
// [base[ph], base[ph] + cnt[ph]) of the operand are phase ph's taps, row-major over (jy, jx); tap slot s reads input
// (a * sin + dy[s], b * sin + dx[s]) for output (a, b) of the phase grid (sin: the caller's input stride), with kernel tap
// w[s], and writes output (a * stride + oy0[ph], b * stride + ox0[ph]).
#pragma once
#include <stdint.h>
#include "fused_common.cuh"

namespace p3d {

struct TapTable {
    int nphase, stride, ntaps;
    int base[4], cnt[4], oh[4], ow[4], oy0[4], ox0[4];
    int w[9], dy[9], dx[9];
};

// MODE_K3: kernel 3, stride 1, padding 1.  MODE_K1: kernel 1.  MODE_UP2: conv_transpose2d with kernel 3, stride 2,
// padding 0 as four phases: output row oy = 2 a + py takes kernel rows ky = py (mod 2) at input row a + (py - ky) / 2.
// MODE_S2: kernel 3, stride 2, padding 0 (input row 2 a + ky; the caller passes sin = 2).
enum Mode { MODE_K3 = 0, MODE_K1 = 1, MODE_UP2 = 2, MODE_S2 = 3 };

// one axis: taps of phase ph (kernel index k, input offset d)
inline int ntaps_1d(int mode, int ph) { return mode == MODE_K3 || mode == MODE_S2 ? 3 : mode == MODE_K1 ? 1 : (ph == 0 ? 2 : 1); }
inline void tap_1d(int mode, int ph, int j, int& k, int& d) {
    if (mode == MODE_K3) { k = j; d = j - 1; }
    else if (mode == MODE_K1) { k = 0; d = 0; }
    else if (mode == MODE_S2) { k = j; d = j; }
    else { k = ph == 0 ? 2 * j : 1; d = -j; }
}

// The table of a kernel-`ks` layer on an in_h x in_w input; phase grids are in_h x in_w (MODE_UP2: (in_h + 1) x (in_w + 1)
// for the even phases), which a caller with another output size overrides.
inline TapTable tap_table(int mode, int in_h, int in_w, int ks) {
    TapTable t{};
    const int nph = mode == MODE_UP2 ? 2 : 1;
    t.nphase = nph * nph;
    t.stride = nph;
    int s = 0;
    for (int py = 0; py < nph; ++py)
        for (int px = 0; px < nph; ++px) {
            const int ph = py * nph + px, nty = ntaps_1d(mode, py), ntx = ntaps_1d(mode, px);
            t.base[ph] = s;
            t.cnt[ph] = nty * ntx;
            t.oh[ph] = mode == MODE_UP2 ? (py == 0 ? in_h + 1 : in_h) : in_h;
            t.ow[ph] = mode == MODE_UP2 ? (px == 0 ? in_w + 1 : in_w) : in_w;
            t.oy0[ph] = py;
            t.ox0[ph] = px;
            for (int jy = 0; jy < nty; ++jy)
                for (int jx = 0; jx < ntx; ++jx, ++s) {
                    int ky, kx, dy, dx;
                    tap_1d(mode, py, jy, ky, dy);
                    tap_1d(mode, px, jx, kx, dx);
                    t.w[s] = ky * ks + kx;
                    t.dy[s] = dy;
                    t.dx[s] = dx;
                }
        }
    t.ntaps = s;
    return t;
}

__device__ __forceinline__ uint32_t to_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}
// byte offset of (row r, K byte b) in a K-major tile with `lbo` bytes between 16-byte K columns
__device__ __forceinline__ int tile_byte(int r, int b, int lbo) { return (r >> 3) * fused::kSBO + (b >> 4) * lbo + (r & 7) * 16 + (b & 15); }

}  // namespace p3d
