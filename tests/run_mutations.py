"""Mutation check of the GPU tests (needs an H100): build libp3d.so once per single-line value mutation of a target's CUDA
source into a temporary directory, run the target's GPU test file against it (P3D_LIBP3D), and report whether the file
fails it, as it must.  The tree is not modified.

    python tests/run_mutations.py TARGET [TARGET ...] [--files F ...] [--json out.json] [--build-only]

TARGET is one of decode_tc, paste_front, render_backward, render_backward_multiplane (the TRI lines of
render_backward.cu), render_taps (the tap enumeration of render_device.cuh, against tests/test_render_backward_paths_gpu.py),
modconv, modconv_paths (more modconv.cu mutations, against tests/test_modconv_paths_gpu.py), render_fused, multiplane (the
multiplane section of the header render_device.cuh), render_simt (render_v1.cu, against tests/test_render_simt_paths_gpu.py),
render_simt_helpers (the SIMT-only helpers of render_device.cuh, against the same file), marching_cubes
(marching_cubes.cu, against tests/test_mesh_paths_gpu.py), and bias_act, upfirdn2d and filtered_lrelu (ops_bias_act.cu,
ops_upfirdn2d.cu and ops_filtered_lrelu.cu, against tests/test_ops_paths_gpu.py).  Each mutant recompiles every
translation unit that includes its source, directly or through other headers.  --files runs other GPU files against the
same mutants instead (to see which of them the rest of the suite catches); the exit code then only reports that the run
completed.  --build-only builds every mutant and stops; nvcc cross-compiles, so it needs no GPU.
--json writes {target: {mutation: result}}.
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from panic3d_b200 import _build  # noqa: E402

# decode_tc.cu: every mutation keeps all memory accesses in bounds and leaves the mbarrier protocol alone (stage index,
# parities, arrival counts and the team stride are untouched), so none can hang.
TILE = 'const long long tile = (long long)blockIdx.x + (long long)it * gridDim.x;'
DECODE_TC = {
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

# paste_front.cu: every mutation keeps all memory accesses in bounds (checked against the file's shapes next to each
# entry) and none is equivalent at every scale the file runs.
PASTE_FRONT = {
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

# render_backward.cu: every mutation changes a value, never an index or a bound that guards a memory access.
# The depth gate `depth_raw >= lo_b` is not mutated: a ray's unclamped depth is a weighted mean of its interval midpoints,
# which lie strictly inside [min depth, max depth] of the batch, so no case can put it on the bound and `>` equals `>=`.
RENDER_BACKWARD = {
    'colour factor 1.002 -> 1': ('(g.force_sigmoid ? 1.f : 1.002f)', '(g.force_sigmoid ? 1.f : 1.f)'),
    'hidden softplus derivative threshold 20 -> 5': ('(pre > 20.f ? 1.f : sigmoid_t(pre))', '(pre > 5.f ? 1.f : sigmoid_t(pre))'),
    'interval softplus derivative linear branch 1 -> 0': ('smid > 20.f ? 1.f : sigmoid_t(smid)', 'smid > 20.f ? 0.f : sigmoid_t(smid)'),
    'white background term without g_xyz': ('2.f * back * (grgb_sum + gx_sum)', '2.f * back * (grgb_sum)'),
    'suffix term not divided by 1 - alpha': ('Tr[i] * P - suffix / fc[i];', 'Tr[i] * P - suffix;'),
    'd_w1 scaled by the bias gain': ('acc[i][j] * g.w1_gain);', 'acc[i][j] * g.b1_gain);'),
    'd_b2 scaled by the weight gain': ('atomicAdd(a.d_b2 + tid, acc * g.b2_gain);', 'atomicAdd(a.d_b2 + tid, acc * g.w2_gain);'),
    'omega without its 1/2': ('om = 0.5f * (wl + wr);', 'om = (wl + wr);'),
}

# render_backward.cu, the multiplane (TRI) lines of k_sample_backward: value mutations that keep every access in bounds (the
# view offset without D only shrinks it, the scatter bound only drops taps, the normal stays bounds-checked in plane_tap).
RENDER_BACKWARD_MULTIPLANE = {
    'per-view gradient offset without D': ('(long long)3 * (TRI ? g.D : 1) * g.H', '(long long)3 * g.H'),
    'scatter stopped after the first 12 of 24 taps': ('for (int k = 0; k < NT; ++k) {', 'for (int k = 0; k < 12; ++k) {'),
    'slab taps from the next plane\'s normal': ('plane_normal(g, qd, px, py, pz), s_tap', 'plane_normal(g, (qd + 1) % 3, px, py, pz), s_tap'),
}

# modconv.cu: every mutation keeps all memory accesses in bounds.
MODCONV = {
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

# modconv.cu against tests/test_modconv_paths_gpu.py: every mutation keeps all memory accesses in bounds at every shape that
# file runs (the reason is next to each entry).
MODCONV_PATHS = {
    # the epilogue writes phase (py, 0) on a grid of in_h + 1 columns: in bounds because every up-2 shape of the file has
    # in_h <= in_w (its tall shapes run up 1 or kernel 1), so oy and ox stay inside the (2H+1) x (2W+1) output and the
    # loads stay bounds-checked; columns it no longer reaches stay NaN.  Equal to the kernel on square shapes
    'up-2 phase width from in_h': ('(px == 0 ? p->in_w + 1 : p->in_w)', '(px == 0 ? p->in_h + 1 : p->in_h)'),
    # the prep writes kernel row 2 - 2j where row 2j belongs (and columns likewise); prep only: the conv reads the tap
    # offsets, not the kernel taps, so an oracle on the weights read back through the same slots agrees with it
    'up-2 prep kernel rows reversed': ('k = ph == 0 ? 2 * j : 1;', 'k = ph == 0 ? 2 - 2 * j : 1;'),
    # an odd number of K-steps in a chunk (fp16 Cin % 64 = 16 or 48) drops its last step; fewer wgmmas on the same tiles
    'K-steps of a chunk rounded down to even': ('const int ksteps = min(KCE, a.Cin - q * KCE) * ES / 32;',
                                                'const int ksteps = min(KCE, a.Cin - q * KCE) * ES / 64 * 2;'),
    # the im2col row of output pixel pix taken from the phase height: the gathered input pixel is still checked against
    # H and W before it is read.  Equal to the kernel when the phase grid is square
    'im2col pixel from the phase height': ('const int pa = prow ? pix / owp : 0, pb = prow ? pix % owp : 0;',
                                           'const int pa = prow ? pix / tt.oh[ph] : 0, pb = prow ? pix % tt.oh[ph] : 0;'),
    # every sample reads sample 0's noise: a smaller offset into the same tensor
    'noise of sample 0 for every sample': ('(long long)n * a.snn + ', ''),
    # the N tile's padding rows get row 0's weights (wrow already points at row 0 for them); the conv never stores those
    # columns, so only the workspace check sees it
    'N-tile padding rows not zeroed': ('(live && ci < a.Cin) ?', '(ci < a.Cin) ?'),
}

# render_fused_ws3.cu: value mutations only - no stage index, parity, arrival count or transaction size changes, and every
# access stays in bounds (trow ^ 1 stays inside the 128-row tile), so none can hang.
RENDER_FUSED = {
    'colour factor 1.002 -> 1': ('const float ca = g.force_sigmoid ? om : 1.002f * om', 'const float ca = g.force_sigmoid ? om : om'),
    'colour offset also under force_sigmoid': ('cb = g.force_sigmoid ? 0.f : -0.001f * om', 'cb = -0.001f * om'),
    'neighbouring sample\'s colour': ('part += fmaf(buf[col_idx(trow, lane)], ca, cb);', 'part += fmaf(buf[col_idx(trow ^ 1, lane)], ca, cb);'),
    'omega = w_i': ('sl.om[rl * L + i] = __fmul_rn(__fadd_rn(wl, wi), 0.5f);', 'sl.om[rl * L + i] = wi;'),
    'pdf floor 0.005': ('fmaxf(w[1], w[2])), 0.5f), 0.01f), 1e-5f);', 'fmaxf(w[1], w[2])), 0.5f), 0.005f), 1e-5f);'),
    'crop flag of the coarse pass in the epilogue': ('if (st.crop[td.pass][srow]) sg = -1e3f;', 'if (st.crop[0][srow]) sg = -1e3f;'),
    'cull threshold without 1 +': ('(float)(1.0 + log(expm1(-log1p(-thr))))', '(float)(log(expm1(-log1p(-thr))))'),
    'depth from the merged depth, not the midpoint': ('acc_d = fmaf(wi, tm[c], acc_d);', 'acc_d = fmaf(wi, m_t[i], acc_d);'),
    'single pass never set': ('a.single_pass = p->mlp_mode == P3D_MLP_TC_BF16;', 'a.single_pass = 0;'),
    'fine depths stored in descending order': ('if (f < Sf) st.t_f[rl * Sf + f] = us[c];', 'if (f < Sf) st.t_f[rl * Sf + Sf - 1 - f] = us[c];'),
}

# render_device.cuh, its multiplane section: every index these mutations produce is still checked against its bound before
# it addresses memory, except the slab stride from W, which stays in bounds because every plane of both multiplane GPU files
# has H >= W.  No tap count, shared memory size or tap-table stride is mutated: an unwritten s_tap entry would send the
# backward's atomics out of bounds.
MULTIPLANE = {
    'slab coordinate with align_corners=True': (
        'const float fz = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(gz, 1.f), (float)g.D), 1.f), 0.5f);',
        'const float fz = __fmul_rn(__fmul_rn(__fadd_rn(gz, 1.f), (float)(g.D - 1)), 0.5f);'),
    'slab index off by one': ('s.z0 = sane ? (int)z0f : -4;', 's.z0 = sane ? (int)z0f + 1 : -4;'),
    'EG3D plane 2 normal taken as x': ('(pm ? x : y));', '(pm ? x : x));'),
    'depth axis clamped instead of zero-padded': ('z = TRI ? s.z0 + (k >> 2) : 0;', 'z = TRI ? min(max(s.z0 + (k >> 2), 0), g.D - 1) : 0;'),
    'taps of slab z0 + 1 taken from slab z0': ('z = TRI ? s.z0 + (k >> 2) : 0;', 'z = TRI ? s.z0 : 0;'),
    'slab offset from plane_w instead of plane_h': ('const long long slab = (long long)g.H * g.stride_row;',
                                                    'const long long slab = (long long)g.W * g.stride_row;'),
    'weight of slab z0 + 1 taken as z0\'s': ('((k >> 2) ? s.wz1 : s.wz0)', '((k >> 2) ? s.wz0 : s.wz0)'),
    # the normal's zero-padding bands dropped: a point within a slab below slab 0 (or above slab D - 1) reads nothing
    'zero-padding band below slab 0 dropped': ('(fz > -2.f) &&', '(fz >= 0.f) &&'),
    'zero-padding band above slab D - 1 dropped': ('(fz < (float)g.D + 1.f)', '(fz < (float)(g.D - 1))'),
}

# render_v1.cu against tests/test_render_simt_paths_gpu.py: value mutations only - no index, bound, shared memory size or
# launch shape changes, so every access stays in bounds and nothing can hang.  The fallback and NaN mutants act on
# auto_axis's rays (NaN limits, fallback limits), the depth one on train_cull's rays with W = 0 (k_depth_finalize is the
# clamp of both the direct and the deferred path).
RENDER_SIMT = {
    'slab test near / far faces swapped': ('const float lo = __fmul_rn(__fsub_rn(neg ? h : -h, o), inv);',
                                           'const float lo = __fmul_rn(__fsub_rn(neg ? -h : h, o), inv);'),
    # the running near limit takes the smaller of the two (max_nan's fmaxf turned into fminf)
    'near limit with fminf': ('? __int_as_float(0x7fffffff) : fmaxf(a, b); }', '? __int_as_float(0x7fffffff) : fminf(a, b); }'),
    # fmaxf / fminf drop a 0 * inf NaN that torch.maximum / torch.minimum keep
    'NaN limits dropped': ('tmin = max_nan(tmin, lo);\n            tmax = min_nan(tmax, hi);',
                           'tmin = fmaxf(tmin, lo);\n            tmax = fminf(tmax, hi);'),
    # the fallback end of a ray that misses is the largest valid end instead of the largest valid start (renderer.py:170)
    'fallback end from the largest t1': ('atomicMax(&bounds[3], float_to_ordered(tmin));', 'atomicMax(&bounds[3], float_to_ordered(tmax));'),
    'depth finalize without NaN -> inf': ('    if (isnan(d)) d = INFINITY;\n    depth[r] = fminf(fmaxf(d, lo), hi);',
                                          '    depth[r] = fminf(fmaxf(d, lo), hi);'),
    'white background not added to xyz': ('__fmul_rn(__fadd_rn(v, back), 2.f)', '__fmul_rn(v, 2.f)'),
    # fine samples per view counted as M max(S, Sf): the view index of a fine sample can only shrink, so it stays in bounds;
    # equal to the kernel when S <= Sf (s4_sf1 has S > Sf and two views)
    'fine per-view count from max(S, Sf)': ('sa.per_view = (long long)g.M * g.Sf;', 'sa.per_view = (long long)g.M * max(g.S, g.Sf);'),
}

# render_device.cuh, the helpers only the SIMT renderer runs (importance_ray, composite_weights) and the 'auto' fallback of
# coarse_sample_depth, against tests/test_render_simt_paths_gpu.py: value mutations only.  `below` stays within the cdf's
# nb + 1 entries and the depths' S.  No mutant touches the bitonic sort: an unsorted fine list breaks merge_by_rank's rank
# positions, leaving merged slots whose colour row index is never written.  The pdf threshold goes to 1e-2 because 1e-3 is
# equivalent: every bin's pdf is at least 0.01 / (2 + 0.01 nb) > 1e-3.
RENDER_SIMT_HELPERS = {
    'pdf floor 0.01 dropped': ('v = __fadd_rn(__fadd_rn(pooled, 0.01f), 1e-5f);', 'v = __fadd_rn(pooled, 1e-5f);'),
    'max-pool with fminf': ('__fadd_rn(fmaxf(wl, wc), fmaxf(wc, wr))', '__fadd_rn(fminf(wl, wc), fmaxf(wc, wr))'),
    'cdf carry not added': ('const float incl = warp_scan_add(pdf, lane) + carry;', 'const float incl = warp_scan_add(pdf, lane);'),
    'below = lo (clamped to nb)': ('const int below = max(lo - 1, 0), above = min(lo, nb);',
                                   'const int below = min(lo, nb), above = min(lo, nb);'),
    'pdf denominator threshold 1e-2': ('if (den < 1e-5f) den = 1.f;', 'if (den < 1e-2f) den = 1.f;'),
    'omega = w_i': ('v = __fmul_rn(__fadd_rn(wl, wr), 0.5f);', 'v = wr;'),
    'fallback end from the smallest valid start': ('t1 = ordered_to_float(bounds[3]);', 't1 = ordered_to_float(bounds[2]);'),
}

# render_device.cuh, the tap enumeration every SIMT gather and scatter shares (plane_tap), against
# tests/test_render_backward_paths_gpu.py: the narrowed bound only drops taps.
RENDER_TAPS = {
    'tap bound xi < W - 1': ('(x < g.W)', '(x < g.W - 1)'),
}

# marching_cubes.cu against tests/test_mesh_paths_gpu.py: every mutant keeps all accesses in bounds (vertex ids only get
# smaller, faces are written at the scanned slots), keeps the packed counts of the two passes consistent (both run the
# same cell_build / cell_walk) and leaves every cell's loops closed (they are for any decider outcome:
# tests/test_mesh_cpu.py checks all 656 configurations), so none can hang.
MARCHING_CUBES = {
    # the cell's inside bits count a node at the level as inside; node_edges and vertex_id still do not
    'cell inside test v >= level': ('ins |= (c.cv[k] > level ? 1u : 0u) << k;', 'ins |= (c.cv[k] >= level ? 1u : 0u) << k;'),
    'decider tie connects': ('const bool connected = s > level;', 'const bool connected = s >= level;'),
    'degenerate triangles kept': ('if (!same_pos(c, r, prev, nd) && !same_pos(c, prev, cur, nd) && !same_pos(c, r, cur, nd)) tri(r, prev, cur);',
                                  'tri(r, prev, cur);'),
    'vertex id without the +b edge of a +c vertex': ('    if (ax >= 2 && ob + 1 < A.d1) id += (__ldg(A.vol + o + s1) > A.level) != in0;\n', ''),
    # the two cells of a face read its corners in their own cyclic order, so they can decide differently
    'decider reads the face cycle': ('const float v00 = c.cv[kFaceCanon[f][0]], v01 = c.cv[kFaceCanon[f][1]];\n'
                                     '            const float v10 = c.cv[kFaceCanon[f][2]], v11 = c.cv[kFaceCanon[f][3]];',
                                     'const float v00 = c.cv[kFaceCyc[f][0]], v01 = c.cv[kFaceCyc[f][1]];\n'
                                     '            const float v10 = c.cv[kFaceCyc[f][2]], v11 = c.cv[kFaceCyc[f][3]];'),
    'upper-border gradient halved': ('if (i == D - 1) return __fsub_rn(__ldg(vol + n), __ldg(vol + n - stride));',
                                     'if (i == D - 1) return __fmul_rn(__fsub_rn(__ldg(vol + n), __ldg(vol + n - stride)), 0.5f);'),
}

# ops_bias_act.cu against tests/test_ops_paths_gpu.py: value mutations only.  Every bias index these mutants produce is taken
# modulo size_b (the shifted BIAS == 2 run stays a whole aligned vector because size_b and ge are multiples of VEC there), and
# no launch shape, UNROLL or vector count changes, so every access stays in bounds.
BIAS_ACT = {
    # gradient modes gate by the sign of the incoming gradient instead of the stored output
    'lrelu gradient gate reads x': (': ((yy > 0) ? x : x * alpha); }', ': ((x > 0) ? x : x * alpha); }'),
    'gradient clamp gate tests y, not yref': ('else y = (yref > -clamp && yref < clamp) ? y : (S)0;',
                                              'else y = (y > -clamp && y < clamp) ? y : (S)0;'),
    # equal to the kernel when gain == 1 (tanh's default) and for lrelu's sign gate at any positive gain
    'yy without the division by gain': ('S yy = (gain != (S)0) ? yref / gain : (S)0;', 'S yy = yref;'),
    'row-mode bias from row r + 1': ('if (BIAS == 4) brow = Elem<T>::ld(bp[r % size_b]);',
                                     'if (BIAS == 4) brow = Elem<T>::ld(bp[(r + 1) % size_b]);'),
    'per-vector bias from the next row': ('if (BIAS == 1) bshared = Elem<T>::ld(bp[(ge / step_b) % size_b]);',
                                          'if (BIAS == 1) bshared = Elem<T>::ld(bp[(ge / step_b + 1) % size_b]);'),
    'bias run shifted by one vector': ('if (BIAS == 2) bv = *reinterpret_cast<const V*>(bp + ge % size_b);',
                                       'if (BIAS == 2) bv = *reinterpret_cast<const V*>(bp + (ge + VEC) % size_b);'),
    # a vector that straddles two rows (step_b % VEC != 0) takes the first row's bias for all its elements
    'generic strided index without + k': ('((ge + k) / step_b) % size_b', '(ge / step_b) % size_b'),
    # the channel of a channels-last element counted in vectors instead of elements; equal to the kernel when VEC % C == 1
    # (fp32 on RGB)
    'generic channel run from the vector index': ('if (BIAS == 3) bi0 = (step_b == 1) ? ge % size_b : 0;',
                                                  'if (BIAS == 3) bi0 = (step_b == 1) ? vi % size_b : 0;'),
    # the tail's elements take the biases of the tensor's first elements; equal to the kernel for an unaligned caller
    # (main_n == 0) and when numel % VEC == 0 (no tail)
    'scalar tail launched with base 0': ('q.base = main_n;', 'q.base = 0;'),
}

# ops_upfirdn2d.cu against tests/test_ops_paths_gpu.py: value mutations only.  The fast kernel's shared rows are PITCH >= IN_W
# + VEC - 1 wide, so reading them without the shift a_r stays inside the row; the narrowed border test only zero-fills more
# elements of a straddling vector; the edge-clamped tiled load and the wrapped channel group index inside the image and C (a
# whole aligned group, C % VEC == 0).  No cp.async source, group count or wait, tile size, shared-memory size or launch shape
# changes.
UPF_TILED_W = 's_w[i] = p.f[sy * p.fsh + sx * p.fsw] * p.gain;\n    }\n    const int tile'
UPF_TILED_FLIP = 'const int sy = p.flip ? ky : p.fH - 1 - ky, sx = p.flip ? kx : p.fW - 1 - kx;\n        ' + UPF_TILED_W
UPFIRDN2D = {
    'fast: row flip sense swapped': ('const int sy = p.flip ? ky : F - 1 - ky;', 'const int sy = p.flip ? F - 1 - ky : ky;'),
    # equal to the kernel on rows whose base is 16-byte aligned
    'fast: shared row read without its shift a_r': ('const T* rowp = sb + (by + sr) * PITCH + s_a[b * IN_H + by + sr];',
                                                    'const T* rowp = sb + (by + sr) * PITCH;'),
    # the last image column is zero-filled where it falls inside a border-straddling vector
    'fast: straddling vector drops the last column': ('tmp[j] = (ix + j >= 0 && ix + j < p.inW) ? src[j]',
                                                      'tmp[j] = (ix + j >= 0 && ix + j < p.inW - 1) ? src[j]'),
    # equal to the kernel at gain 1
    'fast: odd-column taps without the gain': ('p.f[sy * p.fsh + sxo * p.fsw] * p.gain);', 'p.f[sy * p.fsh + sxo * p.fsw]);'),
    'tiled: gain folded in twice': (UPF_TILED_W, UPF_TILED_W.replace('* p.gain;', '* p.gain * p.gain;')),
    # equal to the kernel when flip is 0 or the filter is point-symmetric
    'tiled: flip ignored': (UPF_TILED_FLIP, UPF_TILED_FLIP.replace('p.flip ? ky : ', '').replace('p.flip ? kx : ', '')),
    # pixels outside the image read the nearest edge sample instead of zero
    'tiled: edge sample instead of zero fill': (
        'if (iy >= 0 && iy < p.inH && ix >= 0 && ix < p.inW) v = Px<T>::ld(xi[iy * p.xs[2] + ix * p.xs[3]]);',
        'v = Px<T>::ld(xi[min(max(iy, 0), p.inH - 1) * p.xs[2] + min(max(ix, 0), p.inW - 1) * p.xs[3]]);'),
    # every output column starts at tap 0; the input column (ux0 + kx) / up is still checked against [0, inW); equal to the
    # kernel at up 1
    'strided: column phase kx0 = 0': ('const int kx0 = pos_mod(-ux0, p.upx), ky0 = pos_mod(-uy0, p.upy);\n        const T* xi = xp + n * p.xs[0] + c * p.xs[1];',
                                      'const int kx0 = 0, ky0 = pos_mod(-uy0, p.upy);\n        const T* xi = xp + n * p.xs[0] + c * p.xs[1];'),
    # each thread reads channel group g + 1 (mod C / VEC) and writes group g; equal to the kernel when C == VEC
    'channels-last: reads the next channel group': ('const T* xi = xp + n * p.xs[0] + c;', 'const T* xi = xp + n * p.xs[0] + (c + VEC) % p.C;'),
}

# ops_filtered_lrelu.cu against tests/test_ops_paths_gpu.py: value mutations only.  The sign tensor is allocated with
# torch.zeros, so a byte no CTA writes reads back as code 0 every run; the shifted code position stays inside its byte and the
# offset-free sign coordinate inside the qx < sW / qy < sH check.  No tile size, shared-memory size or loop bound changes.
FILTERED_LRELU = {
    'negative code written as 0': ('if (acc < 0.f) { acc *= p.slope; sc = 1; }', 'if (acc < 0.f) { acc *= p.slope; sc = 0; }'),
    # equal to the kernel where the backward's sx = px0 - (fuW - 1) is 0
    'sign x offset ignored': ('const int qx = ux + p.sx, qy = uy + p.sy;', 'const int qx = ux, qy = uy + p.sy;'),
    'code position from qx + 1': ('>> ((qx & 3) << 1)) & 3u;', '>> (((qx + 1) & 3) << 1)) & 3u;'),
    'clamped pixels scaled by the slope in the gradient pass': ('if (sc & 2u) acc = 0.f;', 'if (sc & 2u) acc *= p.slope;'),
    # the separable vertical up-pass multiplies by up^2 * gain a second time
    'separable vertical up-pass with the gain taps': ('acc = fmaf(col[j * p.upTW], s_wu[p.fuW + ky], acc);',
                                                      'acc = fmaf(col[j * p.upTW], s_wu[ky], acc);'),
    # equal to the kernel at up 1
    'ugain without up * up': ('const float ugain = (float)p.up * (float)p.up * p.gain;', 'const float ugain = p.gain;'),
    # the bottom row of tiles stops writing sign bytes at its nominal height: the rows of the down-filter's halo below it
    # keep code 0
    'last tile row owns only its own rows': ('const int own_y1 = (tyi == p.tilesY - 1) ? p.sH : uy0 + kOutH * p.down;',
                                             'const int own_y1 = uy0 + kOutH * p.down;'),
    # a full (non-separable) filter read with its rows in the flipped order; equal to the kernel on row-symmetric filters
    'full filter rows flip sense swapped': ('const int yy = flip ? ky : fh - 1 - ky,', 'const int yy = flip ? fh - 1 - ky : ky,'),
    # the separable down filter is never flipped; equal to the kernel when flip is set or the taps are symmetric
    'separable down taps never flipped': ('s_wd[i] = p.fd[p.flip ? i : p.fdW - 1 - i];', 's_wd[i] = p.fd[i];'),
}

# target -> (source under csrc/, the GPU test file that must kill every mutant, mutations {name: (old, new)})
TARGETS = {
    'decode_tc': ('decode_tc.cu', 'tests/test_decode_tc_depth_gpu.py', DECODE_TC),
    'paste_front': ('paste_front.cu', 'tests/test_paste_paths_gpu.py', PASTE_FRONT),
    'render_backward': ('render_backward.cu', 'tests/test_render_backward_paths_gpu.py', RENDER_BACKWARD),
    'render_backward_multiplane': ('render_backward.cu', 'tests/test_multiplane_paths_gpu.py', RENDER_BACKWARD_MULTIPLANE),
    'render_taps': ('render_device.cuh', 'tests/test_render_backward_paths_gpu.py', RENDER_TAPS),
    'modconv': ('modconv.cu', 'tests/test_modconv_gpu.py', MODCONV),
    'modconv_paths': ('modconv.cu', 'tests/test_modconv_paths_gpu.py', MODCONV_PATHS),
    'render_fused': ('render_fused_ws3.cu', 'tests/test_render_fused_paths_gpu.py', RENDER_FUSED),
    'multiplane': ('render_device.cuh', 'tests/test_multiplane_paths_gpu.py', MULTIPLANE),
    'render_simt': ('render_v1.cu', 'tests/test_render_simt_paths_gpu.py', RENDER_SIMT),
    'render_simt_helpers': ('render_device.cuh', 'tests/test_render_simt_paths_gpu.py', RENDER_SIMT_HELPERS),
    'marching_cubes': ('marching_cubes.cu', 'tests/test_mesh_paths_gpu.py', MARCHING_CUBES),
    'bias_act': ('ops_bias_act.cu', 'tests/test_ops_paths_gpu.py', BIAS_ACT),
    'upfirdn2d': ('ops_upfirdn2d.cu', 'tests/test_ops_paths_gpu.py', UPFIRDN2D),
    'filtered_lrelu': ('ops_filtered_lrelu.cu', 'tests/test_ops_paths_gpu.py', FILTERED_LRELU),
}


def _include_closure(path, seen):
    """path and every file it reaches through #include "..." lines, added to seen."""
    if path not in seen and os.path.isfile(path):
        seen.add(path)
        for inc in re.findall(r'^\s*#include "([^"]+)"', open(path).read(), re.M):
            _include_closure(os.path.normpath(os.path.join(os.path.dirname(path), inc)), seen)
    return seen


def units_including(src_name):
    """The translation units under csrc/ whose #include closure contains csrc/<src_name>; for a .cu source, itself."""
    src = os.path.join(_build.CSRC, src_name)
    return [s for s in _build.sources() if src in _include_closure(s, set())]


def build_mutant(nvcc, d, target, name):
    """Copy csrc/ into d and apply the mutation there, compile every unit that includes the mutated file and link them with
    the tree's objects for the rest; returns the library's path."""
    src_name, _, mutations = TARGETS[target]
    old, new = mutations[name]
    csrc = os.path.join(d, 'csrc')
    shutil.copytree(_build.CSRC, csrc)
    path = os.path.join(csrc, src_name)
    text = open(path).read()
    assert text.count(old) == 1, f'{target}: {name}'
    open(path, 'w').write(text.replace(old, new))
    objs = {s: os.path.join(d, os.path.basename(s)[:-3] + '.o') for s in units_including(src_name)}
    lib = os.path.join(d, 'libp3d.so')
    # Each copy's includes find the copied headers first; -I csrc resolves "../../include/..." to the repository's include/.
    cmds = [_build.compile_cmd(nvcc, os.path.join(csrc, os.path.basename(s)), o, ['-I', _build.CSRC]) for s, o in objs.items()]
    for cmd in cmds + [_build.link_cmd(nvcc, lib, [objs.get(s, _build.object_path(s)) for s in _build.sources()])]:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode:
            raise RuntimeError(f'{target}: {name}: nvcc failed\n{r.stdout}')
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('targets', nargs='+', choices=sorted(TARGETS), metavar='TARGET')
    ap.add_argument('--files', nargs='+')
    ap.add_argument('--json')
    ap.add_argument('--build-only', action='store_true')
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    nvcc = _build.find_nvcc()
    mutants = [(t, name) for t in dict.fromkeys(args.targets) for name in TARGETS[t][2]]
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        with ThreadPoolExecutor(max_workers=max(1, min(len(mutants), os.cpu_count() or 1))) as ex:
            libs = list(ex.map(lambda i: build_mutant(nvcc, os.path.join(tmp, f'm{i}'), *mutants[i]), range(len(mutants))))
        if args.build_only:
            print(f'built {len(libs)} mutants', flush=True)
            return
        for (target, name), lib in zip(mutants, libs):
            files = args.files or [TARGETS[target][1]]
            r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-x', '-m', 'gpu', '-p', 'no:cacheprovider'] +
                               [os.path.join(ROOT, f) for f in files],
                               cwd=ROOT, env=dict(os.environ, P3D_LIBP3D=lib), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                               text=True)
            failed = [ln for ln in r.stdout.splitlines() if ln.startswith('FAILED') or ln.startswith('ERROR')]
            errors = [ln for ln in r.stdout.splitlines() if ln.startswith('E ')][:8]
            res = results.setdefault(target, {})[name] = {'killed': r.returncode != 0, 'failures': failed, 'errors': errors,
                                                          'summary': r.stdout.strip().splitlines()[-1]}
            print(f'{target}: {name:50s} {"killed" if r.returncode else "SURVIVED"}: {res["summary"][:120]}', flush=True)
            for ln in failed + errors[:2]:
                print(f'    {ln[:160]}', flush=True)
    if args.json:
        json.dump(results, open(args.json, 'w'), indent=1)
    sys.exit(0 if args.files or all(v['killed'] for t in results.values() for v in t.values()) else 1)


if __name__ == '__main__':
    main()
