"""GPU: the streaming tensor-core decode (k_decode_tc, csrc/decode_tc.cu) at depth, against the fp64 oracle on the device.

`p3d_decode_points` (ImportanceRenderer.run_model without grad: the sigma query of sample_mixed) and `p3d_volume_query`
(get_eg3d_volume -> get_eg3d_mesh) run this kernel whenever mlp_mode is 'auto'.  It is persistent: grid = min(n_tiles,
n_sm) CTAs, CTA b takes tiles b, b + grid, ...; twelve gather warps in three teams fill a 4-stage A1 ring that two decoder
warpgroups drain under mbarrier parities, and the gather's texel registers carry over from one tile to the next.  The
fixture-sized tests elsewhere give every CTA one tile.  Here:

  * points mode with n_tiles = k * n_sm + r (0 < r < n_sm) for k = 0, 1, 2, 3, 4, 8: CTAs run k or k + 1 tiles, which
    reaches team 0 only, teams 0-1, all three teams, all four ring stages, the first reuse of stage 0 (parity flip) and
    the second flip (`_schedule` restates the rule and each test asserts what its k reaches).  Three views with
    K % 128 != 0, so tiles straddle views on every lap, and 3K % 128 != 0, so the last tile is partial;
  * the three texel layouts of fp32 and bf16 storage at k = 8, bit-identical to NCHW of the same storage;
  * the volume query at 97^3 x 3 subjects (97^3 % 128 = 33: tiles straddle subjects ~160 laps deep) with crop and cull,
    at the eval shape 256^3 (~990 tiles per CTA) and at 257^3, whose lattice passes n = 2^24, where (float)n rounds;
  * single-pass mode (mlp_mode 2) against a bar derived from its bf16 roundings, and 10x worse than mode 1.

Every call goes through the C ABI with NaN-prefilled outputs, so an element no CTA writes fails, and NaN counts as a
failure in every error ratio.  Every call is made twice and must repeat bit for bit (the kernel has no atomics), and
must be exactly one launch in profile slot 0.

Reference: oracle/renderer_oracle.py (manual gather) and oracle/volume_oracle.py in float64 on the GPU, at most 2^19
points at a time.  test_gpu_fp64_oracle_equals_cpu_oracle pins that run to the CPU fp32 oracle that the reference
fixtures pin.  Bars: mode 1 (3-pass split bf16) 1e-4 abs, the project's bar for the decode; mode 2 per point, see
`single_pass_bars` (tests/render_abi.py).  Run with -s to see the worst error / bar of every comparison.
"""
import ctypes as C
import functools

import pytest
import torch

from oracle import renderer_oracle as orc, volume_oracle as vo
from tests import render_abi as ra
from tests.render_abi import BAR, BW, DEV, PROF_SAMPLE_DECODE, Worst, dec64, decode_points, n_sm, single_pass_bars

pytestmark = pytest.mark.gpu
N_TEAMS, N_STAGES = 3, 4          # decode_tc.cu:24 kTeams, :27 kNA
TILE = 128
CHUNK = 1 << 19                   # points per oracle call
NV, H, W = 3, 64, 80              # views; plane size (H != W, W not a power of two)
CROP, CULL = 0.1, 0.35
DEPTH_K = (0, 1, 2, 3, 4, 8)
# k -> (gather teams, ring stages, parity flips) that the deepest CTA reaches
REACH = {0: (1, 1, 0), 1: (2, 2, 0), 2: (3, 3, 0), 3: (3, 4, 0), 4: (3, 4, 1), 8: (3, 4, 2)}
LAYOUTS = ('nchw', 'channels_last', 'strided64')
FP32_PIN = 2e-6                   # fp64 device oracle vs the CPU fp32 one: the fp32 run's own rounding (measured 1.1e-6)
# share of the density points that may be excluded as within rounding of a mask threshold: single pass's sigma is ~400x
# further from the oracle than 3-pass's, so proportionally more points lie within its error of the cull threshold
BORDER_SHARE = {1: 1e-3, 2: 1e-2}
FREE_BYTES_256 = 12 << 30         # outputs of two 256^3 runs with rgb (2 x 2.5 GB) + oracle chunks, with margin


def _schedule(n_tiles, sms):
    """The persistent schedule of k_decode_tc, restated from csrc/decode_tc.cu:
    :179  grid = min(n_tiles, n_sm);
    :58   CTA b runs n_my = ceil((n_tiles - b) / grid) tiles, :82 / :124 tile b + it * grid at iteration it;
    :81   gather team j takes iterations j, j + 3, ... (three teams);
    :96   iteration it fills A1 stage it % 4; :97 / :110 wait on parity (it / 4) & 1, so stage 0 is reused (parity flips) at
          it = 4 and again at it = 8.
    Returns what the deepest CTA reaches."""
    grid = min(n_tiles, sms)
    n_my = [(n_tiles - b + grid - 1) // grid for b in range(grid)]
    deepest = max(n_my)
    return dict(grid=grid, n_my_max=deepest, n_my_min=min(n_my), teams=min(deepest, N_TEAMS), stages=min(deepest, N_STAGES),
                flips=(deepest - 1) // N_STAGES)


def _volume_dest(n, R):
    """decode_tc.cu:133 volume_dest (render_device.cuh): sample n -> element of the returned (R, R, R) volume (first axis
    flipped).  Its own inverse."""
    rr = R * R
    return (R - 1 - n // rr) * rr + n % rr


# ------------------------------------------------------------------------------------------------- inputs
def _points(seed, n, k):
    """test_plane_variants_gpu._points scaled up: random points in and around the box, 1/16 of them on each face of the box
    (grid coordinate exactly +-1) and eight far outside, shuffled so every tile and lap gets some of each."""
    g = torch.Generator().manual_seed(seed)
    h = BW / 2
    n_face = k // 16
    far = torch.tensor([[9.0, 0.0, 0.0], [-9.0, 0.1, 0.2], [0.36, 0.36, 0.36], [-0.36, -0.36, 0.0], [0.0, 9.0, 0.0],
                        [0.0, 0.0, -9.0], [1e3, 1e3, 1e3], [-0.351, 0.0, 0.351]])
    pts = [(torch.rand(n, k - 6 * n_face - len(far), 3, generator=g) * 2 - 1) * 0.45]
    for axis in range(3):
        for s in (-h, h):
            f = (torch.rand(n, n_face, 3, generator=g) * 2 - 1) * h
            f[..., axis] = s
            pts.append(f)
    pts.append(far.expand(n, -1, -1))
    x = torch.cat(pts, 1)
    return torch.stack([x[v, torch.randperm(k, generator=g)] for v in range(n)]).contiguous()


def _points_per_view(n_tiles):
    """K with ceil(3K / 128) = n_tiles, K % 128 != 0 (tiles straddle views) and 3K % 128 != 0 (the last tile is partial)."""
    for d in range(50, 128):
        K = (TILE * n_tiles - d) // NV
        if K % TILE and (NV * K) % TILE and -(-NV * K // TILE) == n_tiles:
            return K
    raise AssertionError(n_tiles)


def _layout(planes, layout, bf16):
    """The same tri-plane values as a (N,3,32,H,W) tensor in `layout` on the device (test_plane_variants_gpu._layout)."""
    dt = torch.bfloat16 if bf16 else torch.float32
    n, p, c, h, w = planes.shape
    if layout == 'nchw':
        return planes.to(DEV)
    if layout == 'channels_last':
        return planes.to(DEV, dt).reshape(n, p * c, h, w).contiguous(memory_format=torch.channels_last).view(n, p, c, h, w)
    buf = torch.full((n, p, h, w, 64), float('nan'), device=DEV, dtype=dt)
    buf[..., :c] = planes.permute(0, 1, 3, 4, 2).to(DEV, dt)
    return buf[..., :c].permute(0, 1, 4, 2, 3)


def _centre_sigma_on_cull(planes, dec):
    """Shift the sigma bias so that the median sigma of a 33^3 lattice sits at the cull threshold (the density of the
    density falls below 0.35 for sigma < ~0.52), so the cull mask both keeps and removes points."""
    pts = vo.create_samples(33, BW).to(DEV, torch.float64).expand(planes.shape[0], -1, -1)
    _, sig = orc.run_model(planes.to(DEV, torch.float64), dec64(dec), pts, orc.DEFAULT_OPTS, True)
    dec = dict(dec, b2=dec['b2'].clone())
    dec['b2'][0] += 0.52 - sig.median().item()
    return dec


# ------------------------------------------------------------------------------------------------- the kernel, through the C ABI
def _volume_query(planes, dec, R, crop, cull, mode, want_rgb=True):
    """p3d_volume_query -> sigma, rgb, density, coordinates as (N, R, R, R, c) buffers (element (a, b, c) = sample
    volume_dest(a R^2 + b R + c))."""
    from panic3d_b200 import _lib
    N = planes.shape[0]
    r = ra.renderer(False, mode)
    decoder = ra.make_decoder(dec, DEV)
    with torch.no_grad(), torch.cuda.device(DEV):
        cl = r._planes_cl(planes.to(DEV))
        p, wt = ra.decode_params(r, cl, decoder, N * R ** 3)
        sig, dens = (torch.empty((N, R, R, R, 1), device=DEV) for _ in range(2))
        rgb = torch.empty((N, R, R, R, 32), device=DEV) if want_rgb else None
        xyz = torch.empty((N, R, R, R, 3), device=DEV)
        call = lambda: _lib.check(_lib.lib().p3d_volume_query(
            C.byref(p), cl.data_ptr(), *[t.data_ptr() for t in wt], R, float(BW), -1.0 if crop is None else float(crop),
            -1.0 if cull is None else float(cull), sig.data_ptr(), _lib.ptr(rgb), dens.data_ptr(), xyz.data_ptr(),
            _lib.stream_ptr(DEV)))
        out = ra.twice(call, [sig, rgb, dens, xyz], PROF_SAMPLE_DECODE)[0]
    for t in out:
        assert t is None or not torch.isnan(t).any(), 'an output element was never written'
    return out


# ------------------------------------------------------------------------------------------------- oracle pin
def test_gpu_fp64_oracle_equals_cpu_oracle():
    """The fp64 device run of the oracle (what every test below compares with) equals the CPU fp32 oracle that the
    reference fixtures pin (tests/test_oracle_golden.py, tests/test_volume_oracle_golden.py), within the fp32 run's rounding;
    the chunked volume equals the whole one."""
    planes, dec = ra.planes_and_decoder(500, 2, H, W)
    planes = planes[:, :, :, :20, :30].contiguous()
    xyz = _points(500, 2, 600)
    p64, d64 = planes.to(DEV, torch.float64), dec64(dec)
    for a, b in zip(orc.run_model(p64, d64, xyz.to(DEV, torch.float64), orc.DEFAULT_OPTS, True),
                    orc.run_model(planes, dec, xyz, orc.DEFAULT_OPTS, True)):
        assert a.dtype == torch.float64 and a.device == p64.device
        assert (a.cpu() - b.double()).abs().max().item() <= FP32_PIN
    R = 13
    cpu = vo.volume(planes[:1], dec, orc.DEFAULT_OPTS, R, CROP)
    gpu = vo.volume(p64[:1], d64, orc.DEFAULT_OPTS, R, CROP)
    assert torch.equal(gpu['coordinates'].float().cpu(), cpu['coordinates'])
    for key in ('sigmas', 'rgbs', 'densities'):
        assert (gpu[key].cpu() - cpu[key].double()).abs().max().item() <= FP32_PIN, key
    flat = {k: v.permute(0, 2, 3, 4, 1).flip(dims=(1,)).reshape(R ** 3, -1) for k, v in gpu.items()}
    for n0, x, rgb, sigma, dens in vo.volume_chunks(p64[:1], d64, orc.DEFAULT_OPTS, R, CROP, chunk=500):
        n1 = n0 + x.shape[1]
        assert torch.equal(x[0], flat['coordinates'][n0:n1])
        for key, t in (('rgbs', rgb), ('sigmas', sigma), ('densities', dens)):
            assert (t[0] - flat[key][n0:n1]).abs().max().item() <= 1e-12, key


# ------------------------------------------------------------------------------------------------- points mode
@functools.lru_cache(maxsize=None)
def _points_case(k):
    """(planes, dec, coords, schedule) of depth k, and the fp64 oracle outputs (on the device)."""
    sms = n_sm()
    r = 5 + 7 * k
    assert 0 < r < sms
    n_tiles = k * sms + r
    K = _points_per_view(n_tiles)
    s = _schedule(n_tiles, sms)
    assert s['n_my_max'] == k + 1 and s['n_my_min'] == max(k, 1)                    # every last lap is ragged
    assert (s['teams'], s['stages'], s['flips']) == REACH[k], (k, s)
    seed = 600 + k
    planes, dec = ra.planes_and_decoder(seed, NV, H, W)
    coords = _points(seed, NV, K)
    return planes, dec, coords, s, _oracle_points(planes, dec, coords)


def _oracle_points(planes, dec, coords):
    p64, d64, x64 = planes.to(DEV, torch.float64), dec64(dec), coords.to(DEV, torch.float64)
    step = CHUNK // coords.shape[0]
    outs = [orc.run_model(p64, d64, x64[:, i:i + step], orc.DEFAULT_OPTS, True) for i in range(0, coords.shape[1], step)]
    return torch.cat([o[0] for o in outs], 1), torch.cat([o[1] for o in outs], 1)


def _check_points(got, want, bars, tag):
    worst = []
    for key, g, w, b in zip(('rgb', 'sigma'), got, want, bars):
        m = Worst()
        m.add(g, w, b)
        print(f'{tag} {key}: max abs err {m.err:.3e}, worst err / bar {m.ratio:.4f}')
        assert m.ratio <= 1.0, (tag, key, m.err, m.ratio)
        worst.append(m.err)
    return worst


@pytest.mark.parametrize('k', DEPTH_K)
def test_points_at_depth_match_fp64_oracle(k):
    planes, dec, coords, s, want = _points_case(k)
    got = decode_points(planes.to(DEV), dec, coords, 1)
    _check_points(got, want, (BAR, BAR), f'points k={k} ({coords.shape[1]} x {NV} points, {s["n_my_max"]} tiles on the '
                                         f'deepest of {s["grid"]} CTAs)')


@pytest.mark.parametrize('bf16', [False, True])
def test_points_layouts_at_depth_are_bit_identical(bf16):
    """k = 8: NCHW (layout pre-pass, SCOL = 32), (N,96,H,W) channels_last zero-copy (SCOL = 96) and a 64-channel texel
    buffer (SCOL = 0) give bit-identical outputs for one storage type; bf16 NCHW matches the oracle on the bf16-rounded
    planes."""
    planes, dec, coords, s, want = _points_case(8)
    outs = {layout: decode_points(_layout(planes, layout, bf16), dec, coords, 1, bf16=bf16) for layout in LAYOUTS}
    for layout in LAYOUTS[1:]:
        for a, b in zip(outs['nchw'], outs[layout]):
            assert torch.equal(a, b), f'{layout} differs from nchw (max {(a - b).abs().max().item()})'
    if bf16:
        want = _oracle_points(planes.bfloat16().float(), dec, coords)
    _check_points(outs['nchw'], want, (BAR, BAR), f'points k=8 {"bf16" if bf16 else "fp32"}')


def test_points_single_pass_at_depth():
    """mlp_mode 2 at k = 8 within its derived per-point bar, and at least 10x further from the oracle than mode 1."""
    planes, dec, coords, s, want = _points_case(8)
    p64, d64, x64 = planes.to(DEV, torch.float64), dec64(dec), coords.to(DEV, torch.float64)
    bars = single_pass_bars(p64, d64, x64)
    two = _check_points(decode_points(planes.to(DEV), dec, coords, 2), want, bars, 'points k=8 single pass')
    one = _check_points(decode_points(planes.to(DEV), dec, coords, 1), want, (BAR, BAR), 'points k=8 3-pass')
    for e2, e1 in zip(two, one):
        assert e2 >= 10 * e1, ('single pass is not reaching the kernel', e2, e1)


# ------------------------------------------------------------------------------------------------- volume mode
def _check_volume(out, planes, dec, R, crop, cull, mode, tag, n_lo=0, n_hi=None, cull_split=True):
    """Kernel volume `out` against the fp64 oracle on samples [n_lo, n_hi) of every subject, CHUNK at a time.

    Coordinates bit-exact; sigma / rgb within the bar.  Densities: the crop and cull masks must agree exactly except at
    points within rounding distance of a threshold, which the fp64 oracle finds: |x| or |z| within 1e-6 of the crop bound
    (the kernel compares fp32 coordinates with the bound rounded to fp32), or the twice-transformed density g(sigma)
    within |g(sigma_kernel) - g(sigma)| + 2e-6 of the cull threshold (g in fp64; 2e-6 for the kernel's fp32 expf /
    softplus): where the kernel's own sigma error, which the sigma bar bounds, carries g across the threshold.  Those are
    counted and must be under BORDER_SHARE[mode]; unmasked densities are within the sigma bar (the density's slope in
    sigma is <= 1).  Returns the worst absolute sigma / rgb errors."""
    sig_k, rgb_k, dens_k, xyz_k = out
    N = planes.shape[0]
    n_hi = R ** 3 if n_hi is None else n_hi
    p64, d64 = planes.to(DEV, torch.float64), dec64(dec)
    samples = vo.create_samples(R, BW)[:, n_lo:n_hi]
    lim = BW / 2 - crop if crop is not None else None
    ws, wr, wd = Worst(), Worst(), Worst()
    total = border = masked = cull_only = uncropped = 0
    for v in range(N):
        for n0, x, rgb, sigma, dens in vo.volume_chunks(p64[v:v + 1], d64, orc.DEFAULT_OPTS, R, crop, cull, samples=samples):
            idx = torch.arange(n_lo + n0, n_lo + n0 + x.shape[1], device=DEV)
            dest = _volume_dest(idx, R)
            assert torch.equal(xyz_k[v].reshape(-1, 3)[dest], x[0].float()), (tag, 'coordinates')
            if mode == 2:
                bar_rgb, bar_sig = (b[0] for b in single_pass_bars(p64[v:v + 1], d64, x))
            else:
                bar_rgb = bar_sig = BAR
            g_sig = sig_k[v].reshape(-1, 1)[dest]
            ws.add(g_sig, sigma[0], bar_sig)
            if rgb_k is not None:
                wr.add(rgb_k[v].reshape(-1, 32)[dest], rgb[0], bar_rgb)
            g_dens, o_dens = dens_k[v].reshape(-1)[dest], dens[0, :, 0]
            d_raw = vo.sigma2density(sigma[0, :, 0])
            near = torch.zeros_like(g_dens, dtype=torch.bool)
            cropped = torch.zeros_like(near)
            if crop is not None:
                cropped = orc.crop_mask(x, crop, BW)[0, :, 0]
                near |= ((x[0][:, [0, 2]].abs() - lim).abs() <= 1e-6).any(-1)
            if cull is not None:
                gg = vo.sigma2density(d_raw)
                moved = (vo.sigma2density(vo.sigma2density(g_sig[:, 0].double())) - gg).abs()
                near |= ~cropped & ((gg - cull).abs() <= moved + 2e-6)
            mk, mo = g_dens == -1e3, o_dens == -1e3
            assert not ((mk != mo) & ~near).any(), (tag, 'density mask differs away from the thresholds', ((mk != mo) & ~near).sum().item())
            keep = ~mk & ~mo
            if keep.any():
                wd.add(g_dens[keep], o_dens[keep], bar_sig if isinstance(bar_sig, float) else bar_sig[keep, 0])
            total += g_dens.numel()
            border += near.sum().item()
            masked += mo.sum().item()
            uncropped += (~cropped).sum().item()
            cull_only += (mo & ~cropped).sum().item()
    for key, m in (('sigma', ws), ('rgb', wr), ('density', wd)):
        if key == 'rgb' and rgb_k is None:
            continue
        print(f'{tag} {key}: max abs err {m.err:.3e}, worst err / bar {m.ratio:.4f}')
        assert m.ratio <= 1.0, (tag, key, m.err, m.ratio)
    print(f'{tag}: {masked / total:.3f} of the densities masked, cull removes {cull_only / max(uncropped, 1):.3f} of the '
          f'uncropped points; {border} of {total} ({border / total:.2e}) within rounding of a threshold, excluded')
    assert border / total < BORDER_SHARE[mode], (tag, border, total)
    if cull_split:                                                                          # the cull both keeps and removes
        assert 0.05 < cull_only / uncropped < 0.95, (tag, cull_only, uncropped)
    return ws.err, wr.err


@functools.lru_cache(maxsize=None)
def _volume97_inputs():
    planes, dec = ra.planes_and_decoder(700, NV, H, W)
    return planes, _centre_sigma_on_cull(planes, dec)


def test_volume_subjects_straddle_tiles_at_depth():
    """97^3 x 3 subjects with crop and cull: per_view % 128 = 33, so tiles straddle subjects on every lap of ~162."""
    R = 97
    planes, dec = _volume97_inputs()
    assert R ** 3 % TILE != 0
    s = _schedule(-(-NV * R ** 3 // TILE), n_sm())
    assert s['n_my_max'] >= 9 and s['flips'] >= 2, s
    out = _volume_query(planes, dec, R, CROP, CULL, 1)
    _check_volume(out, planes, dec, R, CROP, CULL, 1, f'volume 97^3 x 3 ({s["n_my_max"]} tiles per CTA)')


def test_volume_single_pass_at_depth():
    """mlp_mode 2 on the 97^3 x 3 case within its derived bar, and at least 10x further from the oracle than mode 1."""
    R = 97
    planes, dec = _volume97_inputs()
    two = _check_volume(_volume_query(planes, dec, R, CROP, CULL, 2), planes, dec, R, CROP, CULL, 2, 'volume 97^3 single pass')
    one = _check_volume(_volume_query(planes, dec, R, CROP, CULL, 1), planes, dec, R, CROP, CULL, 1, 'volume 97^3 3-pass')
    for e2, e1 in zip(two, one):
        assert e2 >= 10 * e1, ('single pass is not reaching the kernel', e2, e1)


def test_volume_eval_shape_256():
    """The eval mesh's query: 256^3 x 1 subject (131072 tiles, ~993 per CTA), crop and cull, with colours."""
    ra.skip_unless_free(FREE_BYTES_256)
    R = 256
    planes, dec = ra.planes_and_decoder(800, 1, H, W)
    dec = _centre_sigma_on_cull(planes, dec)
    s = _schedule(R ** 3 // TILE, n_sm())
    assert s['n_my_max'] >= 900, s
    torch.cuda.reset_peak_memory_stats()
    out = _volume_query(planes, dec, R, CROP, CULL, 1)
    _check_volume(out, planes, dec, R, CROP, CULL, 1, f'volume 256^3 ({s["n_my_max"]} tiles per CTA)')
    print(f'volume 256^3: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB')


def test_volume_lattice_past_2_24():
    """257^3 > 2^24 points, where (float)n in volume_point rounds: the coordinates equal volume.create_samples bit for bit
    over the whole lattice, the samples on both sides of n = 2^24 match the oracle, and the mesh's colour lookup
    (p3d_mc_lattice_coords) gives the same points for volume elements and samples on both sides of 2^24."""
    import panic3d_b200.volume as pv
    from panic3d_b200 import _lib
    R = 257
    assert R ** 3 > 2 ** 24 and (R - 1) ** 3 <= 2 ** 24
    planes, dec = ra.planes_and_decoder(900, 1, H, W)
    dec = _centre_sigma_on_cull(planes, dec)
    sig, rgb, dens, xyz = _volume_query(planes, dec, R, None, CULL, 1, want_rgb=False)
    assert rgb is None
    samples, _, _ = pv.create_samples(R, cube_length=BW)
    assert torch.equal(samples, vo.create_samples(R, BW))
    assert torch.equal(xyz.flip(dims=(1,)).reshape(1, -1, 3).cpu(), samples)
    # no crop: around n = 2^24 the x index is ~254 of 256, outside any crop bound, where the cull decides alone
    _check_volume((sig, None, dens, xyz), planes, dec, R, None, CULL, 1, 'volume 257^3 around n = 2^24',
                  n_lo=2 ** 24 - CHUNK // 2, n_hi=2 ** 24 + CHUNK // 2, cull_split=False)
    around = torch.arange(2 ** 24 - 300, 2 ** 24 + 300)
    flat = torch.cat([around, _volume_dest(around, R), torch.tensor([0, R ** 3 - 1])])
    coords = torch.full((flat.numel(), 3), float('nan'), device=DEV)
    fd = flat.to(DEV)
    _lib.check(_lib.lib().p3d_mc_lattice_coords(fd.data_ptr(), flat.numel(), R, float(BW), coords.data_ptr(), _lib.stream_ptr(DEV)))
    assert torch.equal(coords.cpu(), samples[0, _volume_dest(flat, R)])
