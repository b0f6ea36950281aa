"""GPU: the fused modulated convolution (panic3d_b200.modconv, csrc/modconv.cu) against the fp64 oracle.

Reference: ``oracle/modconv_oracle.py``.  Every layer shape of the eval generator (the fp32 backbone 4^2 -> 256^2 with its
96-channel ToRGBs, the fp16 8XDC super-resolution head with its 3-channel ToRGBs) runs at N = 1 and N = 3, on NCHW and
channels_last inputs, and is compared with the fp64 conv of the kernel's OWN rounded operands (the prepared weights read
back from the workspace, the activations rounded to fp16 / tf32-rna), followed by the epilogue in fp64:

    bar = |gain| * K * 2^-23 * S  +  u(ref)

S = the oracle run on |x| and |w| (so K 2^-23 S bounds any fp32 accumulation order over the K = taps x Cin products) and
u(ref) one ulp of the output dtype at the reference value.  Tests print the worst error as a fraction of the bar (-rA).
The fp64 oracle runs on the GPU for the big shapes; ``test_gpu_oracle_equals_cpu_oracle`` pins it to the CPU run.
"""
import ctypes as C
import math

import pytest
import torch

from oracle.modconv_oracle import EVAL_SHAPES, epilogue64, oracle_conv

pytestmark = pytest.mark.gpu

SQRT_HALF = math.sqrt(0.5)
U16, U32 = 2.0 ** -10, 2.0 ** -23

SHAPES = EVAL_SHAPES
SRHEAD = [s[:6] for s in SHAPES if s[0].startswith('sr')]

@pytest.fixture(scope='module')
def env():
    import __graft_entry__ as g
    g.build()
    import panic3d_b200.modconv as mc
    from panic3d_b200 import _lib
    from oracle import modconv_oracle as mo
    torch.backends.cudnn.allow_tf32 = True
    return mc, _lib, mo


def _make(mo, *shape, **kw):
    return mo.make_layer(*shape, **kw).cuda().requires_grad_(False)


def _inputs(layer, n, res_in, dtype, channels_last, seed=1, w_dim=64):
    g = torch.Generator(device='cuda').manual_seed(seed)
    x = torch.randn(n, layer.in_channels, res_in, res_in, device='cuda', generator=g).to(dtype)
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    w = torch.randn(n, w_dim, device='cuda', generator=g)
    return x, w


class _Slot7:
    """Launches counted under profile slot 7 (the modulated convolution) inside the block."""

    def __init__(self, lib):
        self.L = lib.lib()

    def __enter__(self):
        self.L.p3d_profile_enable(1)
        self.L.p3d_profile_read(None, None, 0, 1)
        return self

    def __exit__(self, *a):
        torch.cuda.synchronize()
        ms, cnt = (C.c_double * 8)(), (C.c_uint64 * 8)()
        self.L.p3d_profile_read(ms, cnt, 8, 1)
        self.L.p3d_profile_enable(0)
        self.count = int(cnt[7])


def _check_layer(env, shape, n, channels_last, noise_mode='none', gain=1.0):
    mc, lib, mo = env
    name, cin, cout, res, up, kind, dtype, clamp = shape
    layer = _make(mo, *shape)
    x, w = _inputs(layer, n, res // up, dtype, channels_last)
    with torch.no_grad():
        p = mc.make_params(x, layer.weight, kind == 'layer', up=up)
        assert mc.supported(p), name
        styles = layer.affine(w) * (layer.weight_gain if kind == 'torgb' else 1)
        ws = mc.prep(p, layer.weight, styles)
        noise = layer.noise_const * layer.noise_strength if (kind == 'layer' and noise_mode == 'const') else None
        if kind == 'torgb':
            y = mc.conv(p, x, ws, bias=layer.bias, act='linear', clamp=clamp)
            g_eff = 1.0
        elif up == 1:
            y = mc.conv(p, x, ws, bias=layer.bias, noise=noise, act='lrelu', gain=layer.act_gain * gain,
                        clamp=None if clamp is None else clamp * gain)
            g_eff = layer.act_gain * gain
        else:
            y = mc.conv(p, x, ws)                                  # the pre-filter tensor
            g_eff = 1.0
        wk = mc.unpack_workspace(p, ws).double()
        x64 = mo.round_operand(x, dtype)
        acc = oracle_conv(x64, wk, up, layer.weight.shape[-1])
        s_abs = oracle_conv(x64.abs(), wk.abs(), up, layer.weight.shape[-1])
        bias = layer.bias.to(dtype)
        if kind == 'torgb':
            ref = epilogue64(acc, bias, clamp=layer.conv_clamp)
        elif up == 1:
            ref = epilogue64(acc, bias, noise, 'lrelu', layer.act_gain * gain,
                             None if layer.conv_clamp is None else layer.conv_clamp * gain)
        else:
            ref = acc
        K = wk.shape[2] * wk.shape[3] * wk.shape[4]
        bar = abs(g_eff) * K * U32 * s_abs + (U16 if dtype == torch.float16 else U32) * ref.abs() + 2.0 ** -24
        err = (y.double() - ref).abs()
        frac = float((err / bar).max())
    assert y.shape == ref.shape and y.dtype == dtype
    assert y.is_contiguous(memory_format=mc._out_format(x))
    print(f'{name} N={n} cl={channels_last}: max err {float(err.max()):.3e}, {frac:.3f} of the bar')
    assert frac <= 1.0, (name, frac)
    return layer, x, w, y


@pytest.mark.parametrize('shape', SHAPES, ids=[s[0] for s in SHAPES])
@pytest.mark.parametrize('n', [1, 3])
@pytest.mark.parametrize('channels_last', [False, True], ids=['nchw', 'cl'])
def test_every_eval_layer_shape_against_the_oracle(env, shape, n, channels_last):
    _check_layer(env, shape, n, channels_last)


def test_epilogue_noise_gain_clamp(env):
    """const noise, gain sqrt(0.5) and gain 0.5 (layer gain sqrt(2) * 0.5: an effective gain of sqrt(0.5), so gain before and
    after the clamp differ), with a clamp that binds on a fair share of the outputs."""
    for gain in (SQRT_HALF, 0.5):
        _, _, _, y = _check_layer(env, ('b16_conv1_clamped', 512, 512, 16, 1, 'layer', torch.float32, 0.5), 3, False, noise_mode='const', gain=gain)
        assert float((y.abs() == torch.tensor(0.5 * gain, dtype=y.dtype, device=y.device)).double().mean()) > 0.05   # the clamp binds
        _check_layer(env, ('sr_conv1_clamped', 96, 128, 32, 1, 'layer', torch.float16, 0.5), 3, True, noise_mode='const', gain=gain)
    _check_layer(env, ('torgb_clamped', 96, 3, 32, 1, 'torgb', torch.float16, 0.05), 3, False)


def test_gpu_oracle_equals_cpu_oracle(env):
    mc, lib, mo = env
    torch.manual_seed(0)
    x = torch.randn(2, 32, 6, 6, dtype=torch.float64)
    w = torch.randn(2, 24, 32, 3, 3, dtype=torch.float64)
    for up in (1, 2):
        a = oracle_conv(x, w, up, 3)
        b = oracle_conv(x.cuda(), w.cuda(), up, 3).cpu()
        assert float((a - b).abs().max()) <= 1e-12 * float(a.abs().max())


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32])
def test_prep_weights_equal_the_oracle(env, dtype):
    """The prepared per-sample weights are the oracle's rounded to the compute type, except where the fp32 demodulation
    sum order flips a rounding: then 1 ulp of the compute type, on a small share."""
    mc, lib, mo = env
    layer = _make(mo, 'p', 256, 128, 32, 1, 'layer', dtype, None)
    x, w = _inputs(layer, 3, 32, dtype, False)
    with torch.no_grad():
        layer.weight[:4] *= 1e-6                                  # sum w^2 ~ 1e-9 on these rows: the 1e-8 of dcoefs decides them
        p = mc.make_params(x, layer.weight, True)
        styles = layer.affine(w)
        got = mc.unpack_workspace(p, mc.prep(p, layer.weight, styles)).double()
        want = mo.round_operand(mo.per_sample_weights(layer.weight, styles, True, dtype == torch.float16), dtype)
    ulp = (U16 if dtype == torch.float16 else 2.0 ** -10) * want.abs().clamp_min(2.0 ** -14)
    diff = (got - want).abs()
    share = float((diff > 0).double().mean())
    print(f'{dtype}: {share:.2e} of the weights one rounding away from the oracle')
    assert bool((diff <= ulp * 1.0001).all()) and share < 0.01


def test_fp16_layers_stay_within_two_ulps_of_the_reference_order(env):
    """The reference rounds the fp16 conv before bias_act; the kernel rounds once after its epilogue."""
    mc, lib, mo = env
    for shape in [s + (torch.float16, 256) for s in SRHEAD if s[5] == 'layer' and s[4] == 1]:
        layer = _make(mo, *shape)
        x, w = _inputs(layer, 1, shape[3], torch.float16, False)
        with torch.no_grad():
            got = mc.synthesis_layer_kernel(layer, x, w, noise_mode='none')
            ref = mo.synthesis_layer_forward(layer, x, w, noise_mode='none')
            # the fp64 reference-order value, to size the accumulation slack of the two routes
            p = mc.make_params(x, layer.weight, True)
            wk = mc.unpack_workspace(p, mc.prep(p, layer.weight, layer.affine(w))).double()
            s_abs = oracle_conv(x.double().abs(), wk.abs(), 1, 3) * layer.act_gain
        K = wk[0, 0].numel()
        bar = 2 * U16 * ref.double().abs() + 2 * K * U32 * s_abs + 2.0 ** -24
        frac = float(((got.double() - ref.double()).abs() / bar).max())
        print(f'{shape[0]}: {frac:.3f} of the 2-ulp bar')
        assert frac <= 1.0


@pytest.mark.parametrize('noise_mode', ['random', 'const', 'none'])
def test_noise_draws_like_the_original_method(env, noise_mode):
    mc, lib, mo = env
    layer = _make(mo, 'n', 128, 128, 64, 1, 'layer', torch.float32, None)
    layer.noise_strength.fill_(5.0)                                # a different draw would move every output far
    x, w = _inputs(layer, 3, 64, torch.float32, False)
    with torch.no_grad():
        torch.manual_seed(123)
        got = mc.synthesis_layer_kernel(layer, x, w, noise_mode=noise_mode)
        torch.manual_seed(123)
        ref = mo.SynthesisLayer.forward(layer, x, w, noise_mode=noise_mode)
        p = mc.make_params(x, layer.weight, True)
        wk = mc.unpack_workspace(p, mc.prep(p, layer.weight, layer.affine(w))).double()
        s_abs = oracle_conv(x.double().abs(), wk.abs(), 1, 3) * layer.act_gain
    err = (got.double() - ref.double()).abs()
    assert float((err / (s_abs * 2.0 ** -9 + 1e-5)).max()) <= 1.0          # TF32 on both routes


def test_up2_layer_equals_the_original_method(env):
    mc, lib, mo = env
    for dtype, clamp in ((torch.float32, None), (torch.float16, 256)):
        layer = _make(mo, 'u', 64, 128, 32, 2, 'layer', dtype, clamp)
        x, w = _inputs(layer, 3, 16, dtype, True)
        with torch.no_grad():
            torch.manual_seed(5)
            got = mc.synthesis_layer_kernel(layer, x, w, noise_mode='random', gain=SQRT_HALF)
            torch.manual_seed(5)
            ref = mo.SynthesisLayer.forward(layer, x, w, noise_mode='random', gain=SQRT_HALF)
        assert got.shape == ref.shape and got.dtype == ref.dtype
        tol = 2e-2 if dtype == torch.float16 else 3e-3
        assert float((got.double() - ref.double()).abs().max()) <= tol * float(ref.double().abs().max())


def _sr_head(mo, seed=0):
    return mo.sr_head(seed).cuda().requires_grad_(False)


def _run_blocks(blocks, x, img, ws, noise_mode):
    from oracle.modconv_oracle import run_blocks
    return run_blocks(blocks, x, img, ws, noise_mode)


def _installed(mo):
    import panic3d_b200.dropin as dropin
    return dropin.install_modconv(mo)


def _uninstall(mo):
    for cls in (mo.SynthesisLayer, mo.ToRGBLayer):
        cls.forward = cls._p3d_reference_forward


def _kernel_everywhere(mo, mc):
    """Bind the stand-ins to the kernel route for every layer, whatever measured_faster says."""
    mo.SynthesisLayer.forward = lambda self, x, w, noise_mode='random', fused_modconv=True, gain=1: mc.synthesis_layer_kernel(self, x, w, noise_mode, gain)
    mo.ToRGBLayer.forward = lambda self, x, w, fused_modconv=True: mc.torgb_kernel(self, x, w)


def test_whole_modules_with_and_without_install(env):
    mc, lib, mo = env
    torch.manual_seed(0)
    sr = _sr_head(mo)
    x = torch.randn(1, 32, 128, 128, device='cuda')
    img = torch.randn(1, 3, 128, 128, device='cuda')
    ws = torch.randn(1, 6, 64, device='cuda')
    bb = torch.nn.ModuleList([mo.SynthesisBlock(512 if r <= 128 else 256, min(32768 // r, 512), 64, r, 96) for r in (8, 16, 32, 64, 128, 256)])
    for i, b in enumerate(bb):
        for j, l in enumerate([b.conv0, b.conv1, b.torgb]):
            mo.init_layer_(l, 100 + 10 * i + j)
    bb = bb.cuda().requires_grad_(False)
    xb = torch.randn(1, 512, 4, 4, device='cuda')
    wsb = torch.randn(1, 18, 64, device='cuda')
    with torch.no_grad():
        ref_sr = _run_blocks(sr, x, img.clone(), ws, 'none')
        ref_bb = _run_blocks(bb, xb, None, wsb, 'const')
        assert _installed(mo) == ['SynthesisLayer.forward', 'ToRGBLayer.forward']
        try:
            with _Slot7(lib) as c:                                # installed: the eligible layers (the SR head's two conv0)
                got_sr = _run_blocks(sr, x, img.clone(), ws, 'none')
                got_bb = _run_blocks(bb, xb, None, wsb, 'const')
            _kernel_everywhere(mo, mc)
            with _Slot7(lib) as ck:                               # every layer on the kernel
                all_sr = _run_blocks(sr, x, img.clone(), ws, 'none')
                all_bb = _run_blocks(bb, xb, None, wsb, 'const')
        finally:
            _uninstall(mo)
    assert c.count == 2 * 2 and ck.count == 2 * (6 + 18)
    assert torch.equal(got_bb, ref_bb)                           # no backbone shape is eligible
    for tag, a, b in (('installed SR head', got_sr, ref_sr), ('kernel SR head', all_sr, ref_sr), ('kernel backbone', all_bb, ref_bb)):
        d = float((a - b).abs().max()) / float(b.abs().max())
        print(f'{tag}: max |diff| / max |img| = {d:.2e}')
        assert d <= 1e-2


class _Synthesis(torch.nn.Module):
    """A backbone synthesis stand-in: blocks from a constant 4^2 input, called as G.backbone.synthesis(ws, cond, ...)."""

    def __init__(self, blocks, x0):
        super().__init__()
        self.blocks = blocks
        self.register_buffer('x0', x0)

    def forward(self, ws, cond=None, noise_mode='const'):
        return _run_blocks(self.blocks, self.x0.expand(ws.shape[0], -1, -1, -1), None, ws, noise_mode)


class _Superres(torch.nn.Module):
    def __init__(self, blocks):
        super().__init__()
        self.blocks = blocks

    def forward(self, x, img, ws):
        return _run_blocks(self.blocks, x, img, ws, 'none')


def test_capture_replays_bit_identical_and_eager_is_deterministic(env):
    """graphs.enable_cuda_graphs on the installed modules, under the plane memo as bench_config3 --graphs --reuse_triplane
    --modconv arranges them: the replays equal eager bit for bit, and two eager calls are bit-identical."""
    mc, lib, mo = env
    import panic3d_b200.dropin as dropin
    from panic3d_b200 import graphs
    torch.manual_seed(3)
    bb = torch.nn.ModuleList([mo.SynthesisBlock(512, 512, 64, r, 96) for r in (8, 16, 32)])
    for i, b in enumerate(bb):
        for j, layer in enumerate([b.conv0, b.conv1, b.torgb]):
            mo.init_layer_(layer, 200 + 10 * i + j)
    G = torch.nn.Module()
    G.backbone = torch.nn.Module()
    G.backbone.synthesis = _Synthesis(bb, torch.randn(1, 512, 4, 4))
    G.superresolution = _Superres(_sr_head(mo, seed=3))
    G = G.cuda().requires_grad_(False)
    ws = torch.randn(1, 9, 64, device='cuda')
    x = torch.randn(1, 32, 128, 128, device='cuda')
    img = torch.randn(1, 3, 128, 128, device='cuda')
    wsr = torch.randn(1, 6, 64, device='cuda')
    _installed(mo)
    try:
        with torch.no_grad():
            e_bb = [G.backbone.synthesis(ws) for _ in range(2)]
            with _Slot7(lib) as c:
                e_sr = [G.superresolution(x, img.clone(), wsr) for _ in range(2)]
            memo = dropin.enable_plane_reuse(G)
            gr = graphs.enable_cuda_graphs(G)
            r_bb = [G.backbone.synthesis(ws.clone()) for _ in range(2)]
            r_sr = [G.superresolution(x, img.clone(), wsr) for _ in range(3)]
    finally:
        _uninstall(mo)
    assert torch.equal(e_bb[0], e_bb[1]) and torch.equal(e_sr[0], e_sr[1])
    assert all(torch.equal(r, e_bb[0]) for r in r_bb) and all(torch.equal(r, e_sr[0]) for r in r_sr)
    assert gr['backbone'].captures == 1 and gr['superresolution'].captures == 1 and gr['superresolution'].hits >= 2
    assert memo.hits >= 1 and c.count == 2 * 2 * 2              # eager: the two eligible conv0 layers, prep + conv, two calls


def test_eligibility(env):
    """The kernel runs for eligible calls (fp16 up-2 layers, measured_faster) and not under autograd, with
    fused_modconv=False, for unsupported shapes, for shapes measured slower than cuDNN, or for fp32 layers with TF32
    disallowed; those calls equal the original method."""
    mc, lib, mo = env
    layer = _make(mo, 'e', 64, 64, 32, 2, 'layer', torch.float16, 256)
    x, w = _inputs(layer, 2, 16, torch.float16, False)
    with torch.no_grad(), _Slot7(lib) as c:
        mc.synthesis_layer_forward(layer, x, w, noise_mode='none')
    assert c.count == 2                                           # prep + conv

    def same_as_original(lay, xx, **kw):
        det = torch.backends.cudnn.deterministic
        torch.backends.cudnn.deterministic = True                 # the original route's own cuDNN algorithms, run twice
        try:
            with _Slot7(lib) as c:
                torch.manual_seed(9)
                a = mc.synthesis_layer_forward(lay, xx, w, **kw)
                torch.manual_seed(9)
                b = mo.SynthesisLayer.forward(lay, xx, w, **kw)
        finally:
            torch.backends.cudnn.deterministic = det
        assert c.count == 0 and torch.equal(a, b)

    with torch.no_grad():
        same_as_original(layer, x, noise_mode='none', fused_modconv=False)
        l32 = _make(mo, 'e32', 64, 64, 16, 1, 'layer', torch.float32, None)           # measured slower than cuDNN
        x32, _ = _inputs(l32, 2, 16, torch.float32, False)
        same_as_original(l32, x32, noise_mode='none')
        torch.backends.cudnn.allow_tf32 = False
        try:
            same_as_original(_make(mo, 'e32u', 64, 64, 32, 2, 'layer', torch.float32, None), x.float(), noise_mode='none')
        finally:
            torch.backends.cudnn.allow_tf32 = True
        l24 = _make(mo, 'e24', 24, 64, 32, 2, 'layer', torch.float16, 256)           # Cin not a multiple of 16
        x24, _ = _inputs(l24, 2, 16, torch.float16, False)
        same_as_original(l24, x24, noise_mode='none')
    layer.requires_grad_(True)
    same_as_original(layer, x, noise_mode='none')                 # autograd
