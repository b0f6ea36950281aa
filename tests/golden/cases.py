"""Case table shared by the golden generator (make_golden.py), the oracle tests
and the GPU parity tests.  A case fully determines its inputs through
``oracle.renderer_oracle.synth_inputs`` (numpy PCG64), so fixtures hold only
reference outputs."""
from __future__ import annotations

import copy

from oracle import renderer_oracle as orc


def _opts(**over):
    o = copy.deepcopy(orc.DEFAULT_OPTS)
    o.update(over)
    return o


_SMALL = dict(N=1, R=16, P=64, opts=_opts(depth_resolution=12, depth_resolution_importance=12),
              cameras=[(10.0, 30.0, 1.0, 30.0)])


def _small(seed, **over):
    c = copy.deepcopy(_SMALL)
    c['seed'] = seed
    opts_over = over.pop('opts', {})
    c.update(over)
    c['opts'].update(opts_over)
    return c


RENDER_CASES = {
    # BASELINE.json configs[0]: 64x64 rays, 48(+48) samples, 32-ch 256^2 tri-plane, N=1
    'config1': dict(seed=1, N=1, R=64, P=256, opts=_opts(depth_resolution=48, depth_resolution_importance=48),
                    cameras=[(0.0, 30.0, 1.0, 30.0)]),
    'small_plain': _small(11),
    # the eval script's flags (generate.py:53-57): force_sigmoid, crop 0.1, cull 0.5
    'small_eval_flags': _small(12, triplane_crop=0.1, cull_clouds=0.5, force_sigmoid=True),
    'small_eval_flags_dense': _small(25, triplane_crop=0.1, cull_clouds=0.5, force_sigmoid=True, sigma_bias=2.0),
    'small_binarize': _small(13, binarize_clouds=0.5, triplane_crop=0.05, sigma_bias=1.0),
    'small_ortho': _small(14, ortho=True, cameras=[(0.0, 0.0, 1.0, -1.0)]),
    'small_ortho_side': _small(15, ortho=True, cameras=[(20.0, -135.0, 1.0, -1.0)], triplane_crop=0.1, cull_clouds=0.5),
    'small_black_eg3dplanes': _small(16, use_triplane=False, opts=dict(white_back=False)),
    'small_disparity': _small(17, opts=dict(disparity_space_sampling=True)),
    'small_auto_limits': _small(18, opts=dict(ray_start='auto', ray_end='auto')),
    'small_no_importance': _small(19, opts=dict(depth_resolution=24, depth_resolution_importance=0)),
    'small_batch3': _small(20, N=3, cameras=[(0.0, -180.0, 1.0, 30.0), (0.0, 90.0, 1.0, 30.0), (60.0, -45.0, 1.2, 45.0)]),
    'small_lrmul_uneven': _small(21, lr_mul=0.5, R=12, opts=dict(depth_resolution=20, depth_resolution_importance=9)),
    'small_shared_planes': _small(22, N=2, share_planes=True, cameras=[(0.0, 0.0, 1.0, 30.0), (0.0, 150.0, 1.0, 30.0)]),
    # training-time sampling (train_eclustrousC.py:436-437) on a mid-size plane, 2 views
    'mid_train48': dict(seed=23, N=2, R=32, P=128, opts=_opts(depth_resolution=48, depth_resolution_importance=48),
                        cameras=[(0.0, -60.0, 1.0, 30.0), (-20.0, 120.0, 1.0, 30.0)]),
    # eval sampling 96+96 (eg3dc_v0.py:30-31) on a small image
    'mid_eval96': dict(seed=24, N=1, R=24, P=128, opts=_opts(), cameras=[(0.0, 0.0, 1.0, 30.0)],
                       triplane_crop=0.1, cull_clouds=0.5, force_sigmoid=True, sigma_bias=2.0),
    # ---- fused tensor-core kernel coverage (it exists for S = Sf in {48, 96} only): the option matrix of the small_* cases at 48+48
    'fused48_ortho': _small(51, ortho=True, cameras=[(20.0, -135.0, 1.0, -1.0)], opts=dict(depth_resolution=48, depth_resolution_importance=48)),
    'fused48_auto_limits': _small(52, opts=dict(ray_start='auto', ray_end='auto', depth_resolution=48, depth_resolution_importance=48)),
    'fused48_disparity': _small(53, opts=dict(disparity_space_sampling=True, depth_resolution=48, depth_resolution_importance=48)),
    'fused48_black_eg3dplanes': _small(54, use_triplane=False, opts=dict(white_back=False, depth_resolution=48, depth_resolution_importance=48)),
    'fused48_shared_planes': _small(55, N=2, share_planes=True, cameras=[(0.0, 0.0, 1.0, 30.0), (0.0, 150.0, 1.0, 30.0)],
                                    opts=dict(depth_resolution=48, depth_resolution_importance=48)),
    'fused48_binarize': _small(56, binarize_clouds=0.5, triplane_crop=0.05, sigma_bias=1.0, opts=dict(depth_resolution=48, depth_resolution_importance=48)),
    'fused96_lrmul_black': _small(57, lr_mul=0.5, opts=dict(white_back=False, depth_resolution=96, depth_resolution_importance=96)),
    # BASELINE.json configs[1] (the benchmarked workload) at N=2: 128x128 rays, 96+96 samples, 512^2 planes, no cull ->
    # strict tolerance.  The fixture keeps every 8th ray of the reference output (store_stride) to stay under 1 MB.
    'headline96': dict(seed=58, N=2, R=128, P=512, opts=_opts(), cameras=[(0.0, -150.0, 1.0, 30.0), (0.0, 60.0, 1.0, 30.0)], store_stride=8),
}

POINT_CASES = {
    'pts_small': dict(seed=31, N=2, P=64, K=1000, R=1, opts=_opts(depth_resolution=2, depth_resolution_importance=0), cameras=None),
    'pts_eg3dplanes': dict(seed=32, N=1, P=32, K=513, R=1, use_triplane=False, force_sigmoid=True,
                           opts=_opts(depth_resolution=2, depth_resolution_importance=0), cameras=None),
}

# dense volume query (get_eg3d_volume, _util/eg3d_metrics3d.py:94-183): odd sides exercise the un-floored float indices
VOLUME_CASES = {
    'vol_plain13': dict(seed=41, N=1, P=64, R=1, res=13, opts=_opts(depth_resolution=2, depth_resolution_importance=0), cameras=None),
    'vol_crop_cull16': dict(seed=42, N=1, P=64, R=1, res=16, triplane_crop=0.1, cull_clouds=0.35, sigma_bias=1.5,
                            opts=_opts(depth_resolution=2, depth_resolution_importance=0), cameras=None),
    'vol_crop0_eg3dplanes10': dict(seed=43, N=1, P=32, R=1, res=10, triplane_crop=0.0, use_triplane=False, force_sigmoid=True,
                                   opts=_opts(depth_resolution=2, depth_resolution_importance=0), cameras=None),
}


def build_case_inputs(case):
    o = case['opts']
    planes, dec, c2w, K, u_c, u_f = orc.synth_inputs(
        case['seed'], case['N'], case['R'], int(o['depth_resolution']), int(o['depth_resolution_importance']),
        case['P'], cameras=case.get('cameras'), share_planes=case.get('share_planes', False))
    dec['lr_mul'] = case.get('lr_mul', 1.0)
    dec['force_sigmoid'] = case.get('force_sigmoid', False)
    if case.get('sigma_bias'):
        dec['b2'] = dec['b2'].clone()
        dec['b2'][0] += case['sigma_bias']
    return planes, dec, c2w, K, u_c, u_f, copy.deepcopy(o)
