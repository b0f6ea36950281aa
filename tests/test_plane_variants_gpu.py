"""GPU: tri-plane storage (fp32 / bf16) x texel layout for every consumer of the tri-planes, and the fused renderer's
persistent schedule at depth.

The tensor-core kernels are compiled per plane storage and per texel stride: `stride_col` = 32 (the layout pre-pass of an
NCHW tensor), 96 (a (N,96,H,W) channels_last backbone output, read zero-copy) or anything else (SCOL = 0, the stride
comes from a register).  k_render_ws3<BF16, S, SCOL> has 2 x 2 x 3 = 12 instantiations (S = 48, 96) and
k_decode_tc<BF16, VOLUME, SCOL> another 12 (points, volume); the matrix below runs each of them, plus the SIMT renderer
in every layout.  The three layouts of one storage type load the same values and do the same arithmetic, so their
outputs must be bit-identical; bf16 storage is checked against the oracle run on the bf16-rounded planes, which are
exactly the values the kernels read.

Planes are 20 x 30 texels (W not a multiple of 4, H != W), and the rays / points reach every edge of each plane and
leave the box, so the clamped 2 x 2 footprints of the gathers are exercised in every layout."""
import pytest
import torch

from oracle import renderer_oracle as orc, volume_oracle as vo
from tests.helpers import profiled
from tests.render_abi import box_rays, make_decoder, planes_and_decoder

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
N, H, W = 2, 20, 30
LAYOUTS = ('nchw', 'channels_last', 'strided64')
TEXEL_STRIDE = {'nchw': 32, 'channels_last': 96, 'strided64': 64}
PROF_SAMPLE_DECODE, PROF_FUSED = 0, 5          # profile slots (csrc/p3d_common.cuh)


def _noise(seed, n, m, S):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, m, S, 1, generator=g), torch.rand(n * m, S, generator=g)


def _points(seed):
    """Random points in and around the box, points on all six faces of the box (grid coordinate exactly +-1: half a
    texel beyond the outer texel centres of every plane edge) and a few far outside."""
    g = torch.Generator().manual_seed(seed)
    h = 0.35                                                         # box_warp / 2
    pts = [(torch.rand(N, 700, 3, generator=g) * 2 - 1) * 0.45]
    for axis in range(3):
        for s in (-h, h):
            f = (torch.rand(N, 60, 3, generator=g) * 2 - 1) * h
            f[..., axis] = s
            pts.append(f)
    pts.append(torch.tensor([[9.0, 0.0, 0.0], [-9.0, 0.1, 0.2], [0.36, 0.36, 0.36], [-0.36, -0.36, 0.0]]).expand(N, -1, -1))
    return torch.cat(pts, 1).contiguous()


def _layout(planes, layout, bf16):
    """The same tri-plane values as a (N,3,32,H,W) tensor in `layout` on the device."""
    dt = torch.bfloat16 if bf16 else torch.float32
    n, p, c, h, w = planes.shape
    if layout == 'nchw':                      # fp32 source: the layout pre-pass writes channels-last texels (rounded to bf16)
        return planes.to(DEV)
    if layout == 'channels_last':             # (N,96,H,W) channels_last, already in the storage type: zero-copy
        return planes.to(DEV, dt).reshape(n, p * c, h, w).contiguous(memory_format=torch.channels_last).view(n, p, c, h, w)
    buf = torch.full((n, p, h, w, 64), float('nan'), device=DEV, dtype=dt)   # 64-channel texels; the unused half is NaN
    buf[..., :c] = planes.permute(0, 1, 3, 4, 2).to(DEV, dt)
    return buf[..., :c].permute(0, 1, 4, 2, 3)


def _renderer(use_triplane, bf16, mlp_mode):
    from panic3d_b200.training.volumetric_rendering.renderer import ImportanceRenderer
    r = ImportanceRenderer(use_triplane=use_triplane)
    r.planes_bf16 = bf16
    r.mlp_mode = mlp_mode
    return r


# consumer -> (S, mlp_mode) for the renderers; run_model and query_volume force the tensor-core decoder (k_decode_tc)
RENDERERS = {'fused48': (48, 1), 'fused96': (96, 1), 'simt48': (48, 0)}
CONSUMERS = tuple(RENDERERS) + ('points', 'volume')
VOL_RES, VOL_CROP, VOL_CULL = 13, 0.1, 0.35


def _centre_sigma_on_cull(planes, dec, use_triplane):
    """Shift the sigma bias so that the lattice's median sigma sits at the cull threshold (the density of the density
    falls below 0.35 for sigma < ~0.52): the cull mask then removes part of the volume and keeps part of it."""
    pts = vo.create_samples(VOL_RES, orc.DEFAULT_OPTS['box_warp']).expand(planes.shape[0], -1, -1)
    _, sig = orc.run_model(planes, dec, pts, orc.DEFAULT_OPTS, use_triplane)
    dec = dict(dec, b2=dec['b2'].clone())
    dec['b2'][0] += 0.52 - sig.median().item()
    return dec


def _consume(kind, r, x, dec, use_triplane, seed):
    """Outputs (CPU) of one consumer, and the profile counters of the call."""
    import panic3d_b200.volume as pv
    opts = dict(orc.DEFAULT_OPTS)
    decoder = make_decoder(dec, DEV)
    if kind in RENDERERS:
        S = RENDERERS[kind][0]
        opts.update(depth_resolution=S, depth_resolution_importance=S)
        ro, rd = box_rays(seed, N, 64)
        r.injected_noise = _noise(seed, N, 64, S)
        fn = lambda: r(x, decoder, ro.to(DEV), rd.to(DEV), opts)
    elif kind == 'points':
        fn = lambda: (lambda o: (o['rgb'], o['sigma']))(r.run_model(x, decoder, _points(seed).to(DEV), None, opts))
    else:
        fn = lambda: (lambda o: (o['sigmas'], o['rgbs'], o['densities'], o['coordinates']))(
            pv.query_volume(x, decoder, opts, resolution=VOL_RES, triplane_crop=VOL_CROP, cull_clouds=VOL_CULL, renderer=r))
    with torch.no_grad():
        out, prof = profiled(fn)
    return [t.cpu() for t in out], prof


def _oracle(kind, planes, dec, use_triplane, seed):
    opts = dict(orc.DEFAULT_OPTS)
    if kind in RENDERERS:
        S = RENDERERS[kind][0]
        opts.update(depth_resolution=S, depth_resolution_importance=S)
        ro, rd = box_rays(seed, N, 64)
        u_c, u_f = _noise(seed, N, 64, S)
        return list(orc.render(planes, dec, ro, rd, opts, u_c, u_f, use_triplane=use_triplane))
    if kind == 'points':
        return list(orc.run_model(planes, dec, _points(seed), opts, use_triplane))
    vols = [vo.volume(planes[i:i + 1], dec, opts, VOL_RES, VOL_CROP, VOL_CULL, use_triplane) for i in range(N)]
    return [torch.cat([v[k] for v in vols]) for k in ('sigmas', 'rgbs', 'densities', 'coordinates')]


def _assert_close(kind, got, want, tag):
    if kind == 'volume':
        sig, rgb, dens, xyz = got
        wsig, wrgb, wdens, wxyz = want
        assert torch.equal(xyz, wxyz), tag
        for key, a, b in (('sigmas', sig, wsig), ('rgbs', rgb, wrgb)):
            err = (a - b).abs().max().item()
            print(f'{tag}:{key} max abs err {err:.3e} (bar 1e-4)')
            assert err < 1e-4, (tag, key, err)
        agree = ((dens == -1e3) == (wdens == -1e3)).float().mean().item()
        keep = (dens != -1e3) & (wdens != -1e3)
        assert keep.any() and not keep.all(), tag
        err = (dens[keep] - wdens[keep]).abs().max().item()
        print(f'{tag}:densities mask agreement {agree:.5f} (bar 0.999; {1 - keep.float().mean().item():.3f} masked), '
              f'max abs err {err:.3e} (bar 1e-4)')
        assert agree > 0.999 and err < 1e-4, (tag, agree, err)
        return
    bar = 1e-3 if kind.startswith('fused') else 1e-4
    for i, (a, b) in enumerate(zip(got, want)):
        err = (a - b).abs().max().item()
        print(f'{tag}:out{i} max abs err {err:.3e} (bar {bar:.0e})')
        assert err < bar, (tag, i, err)


@pytest.mark.parametrize('use_triplane', [True, False])
@pytest.mark.parametrize('bf16', [False, True])
@pytest.mark.parametrize('kind', CONSUMERS)
def test_plane_layouts_are_bit_identical_and_match_oracle(kind, bf16, use_triplane):
    seed = 300 + CONSUMERS.index(kind) * 4 + 2 * int(bf16) + int(use_triplane)
    planes, dec = planes_and_decoder(seed, N, H, W)
    if kind == 'volume':
        dec = _centre_sigma_on_cull(planes, dec, use_triplane)
    mode = RENDERERS[kind][1] if kind in RENDERERS else 1
    outs = {}
    for layout in LAYOUTS:
        x = _layout(planes, layout, bf16)
        r = _renderer(use_triplane, bf16, mode)
        cl = r._planes_cl(x)                                  # what reaches p3d_render_params.stride_*
        assert cl.dtype == (torch.bfloat16 if bf16 else torch.float32) and cl.stride(4) == 1
        assert cl.stride(3) == TEXEL_STRIDE[layout], (layout, cl.stride())
        outs[layout], prof = _consume(kind, r, x, dec, use_triplane, seed)
        if layout == 'nchw':
            assert r._planes.buf is not None and r._planes.buf.stride(3) == 32
        else:                                                 # zero-copy: the kernels read the caller's tensor, no pre-pass
            assert cl.data_ptr() == x.data_ptr() and r._planes.buf is None
        if kind.startswith('fused'):
            assert prof[PROF_FUSED] == 1 and prof[PROF_SAMPLE_DECODE] == 0, prof
        elif kind == 'simt48':
            assert prof[PROF_FUSED] == 0 and prof[PROF_SAMPLE_DECODE] >= 1, prof
    for layout in LAYOUTS[1:]:
        for i, (a, b) in enumerate(zip(outs['nchw'], outs[layout])):
            assert torch.equal(a, b), f'{kind}: output {i} of layout {layout} differs from nchw (max {(a - b).abs().max().item()})'
    ref_planes = planes.bfloat16().float() if bf16 else planes
    _assert_close(kind, outs['nchw'], _oracle(kind, ref_planes, dec, use_triplane, seed),
                  f'{kind}/{"bf16" if bf16 else "fp32"}/{"triplane" if use_triplane else "eg3d"}')


@pytest.mark.parametrize('bf16', [False, True])
def test_texel_stride_the_fused_kernel_cannot_take(bf16):
    """A texel stride of 36 elements passes the library's 4-element alignment but not the fused renderer's 8-element one:
    mlp_mode 'auto' renders with the SIMT kernels (and still matches the oracle), a forced fused mode raises."""
    seed = 350 + int(bf16)
    planes, dec = planes_and_decoder(seed, N, H, W)
    dt = torch.bfloat16 if bf16 else torch.float32
    buf = torch.full((N, 3, H, W, 36), float('nan'), device=DEV, dtype=dt)
    buf[..., :32] = planes.permute(0, 1, 3, 4, 2).to(DEV, dt)
    x = buf[..., :32].permute(0, 1, 4, 2, 3)
    r = _renderer(True, bf16, 'auto')
    assert r._planes_cl(x).stride(3) == 36
    got, prof = _consume('fused48', r, x, dec, True, seed)
    assert prof[PROF_FUSED] == 0 and prof[PROF_SAMPLE_DECODE] >= 1, prof
    _assert_close('simt48', got, _oracle('fused48', planes.bfloat16().float() if bf16 else planes, dec, True, seed), 'stride36')
    with pytest.raises(RuntimeError, match='fused'):
        _consume('fused48', _renderer(True, bf16, 1), x, dec, True, seed)


# ---------------------------------------------------------------------------------------------
# the fused renderer's persistent schedule at depth: a CTA of the grid (min(groups, SMs) CTAs) runs n_my ray groups
# through a 4-deep state ring and a 2-deep omega slot whose mbarrier parities flip once per lap
# ---------------------------------------------------------------------------------------------
DEPTH_LAPS = (0, 2, 4, 6, 8)         # k in n_groups = k * n_sm + r: CTAs run k or k + 1 groups (1 when k = 0)


def _depth_check(S, k, bf16=False, layout='nchw'):
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    GR = 384 // S                                         # rays per group
    r_ = 10 + 2 * k                                       # even and non-zero: two views of whole groups, ragged last lap
    assert r_ < n_sm
    groups = k * n_sm + r_
    M = groups * GR // N
    n_my = (groups + n_sm - 1) // n_sm
    assert n_my == k + 1 and (k == 0 or groups % n_sm != 0)
    seed = 400 + S + k + int(bf16)
    planes, dec = planes_and_decoder(seed, N, 64, 64)
    ro, rd = box_rays(seed, N, M)
    u_c, u_f = _noise(seed, N, M, S)
    opts = dict(orc.DEFAULT_OPTS, depth_resolution=S, depth_resolution_importance=S)
    x = _layout(planes, layout, bf16)
    runs = []
    for _ in range(2):
        r = _renderer(True, bf16, 1)
        r.injected_noise = (u_c, u_f)
        with torch.no_grad():
            out, prof = profiled(lambda: r(x, make_decoder(dec, DEV), ro.to(DEV), rd.to(DEV), opts))
        assert prof[PROF_FUSED] == 1 and prof[PROF_SAMPLE_DECODE] == 0, prof
        runs.append([t.cpu() for t in out])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    ref = orc.render(planes.bfloat16().float() if bf16 else planes, dec, ro, rd, opts, u_c, u_f, use_triplane=True)
    for got, want, key in zip(runs[0], ref, ('rgb', 'depth', 'wsum', 'xyz')):
        err = (got - want).abs().max().item()
        print(f'depth S={S} {"bf16" if bf16 else "fp32"} {layout}: {groups} groups (up to {n_my} per CTA on {n_sm} SMs) '
              f'{key} max abs err {err:.3e} (bar 1e-3)')
        assert err < 1e-3, (S, k, key, err)


@pytest.mark.parametrize('k', DEPTH_LAPS)
@pytest.mark.parametrize('S', [48, 96])
def test_fused_schedule_at_depth_matches_oracle(S, k):
    _depth_check(S, k)


def test_fused_schedule_at_depth_with_bf16_zero_copy_planes():
    _depth_check(48, 8, bf16=True, layout='channels_last')
