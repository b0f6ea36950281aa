"""Hand-written backward of the renderer oracle, and its magnitude twin, for the training-path gradient tests.

TEST INFRASTRUCTURE ONLY (see renderer_oracle.py).  ``render_backward`` restates, in the dtype of the planes (float64 in the
tests), the gradient of ``renderer_oracle.render`` with injected depths and masks with respect to the tri-planes and the four
decoder tensors, in the order csrc/render_backward.cu computes it: per ray dL/dw_i, dL/dalpha_i through the suffix sum
``total - prefix``, dL/dsigma_j and omega_j; per sample the decoder backward; the feature gradient scattered to the bilinear
taps.  With ``mag=True`` every product and partial sum is taken in absolute value (the magnitude adjoint A), plus the floors
listed at ``_floors``: the bar of an element whose kernel value is an n-step fp32 computation is (n + c) u A.
tests/test_render_backward_oracle_cpu.py checks the signed run against torch autograd of renderer_oracle.render.

Positions are taken as the kernel makes them: ``ro + t rd`` and the tap footprint in fp32 (``taps``).  They are constants of
the reference graph, so this fixes which texels a sample reads without changing any derivative.

``depth`` > 1 is multiplane tri-planes (dev::slab_footprint / dev::plane_tap<true>): planes (N, 3, C*depth, H, W) in the
reference's indexing (channel c*depth + d is feature c of slab d, as multiplane_oracle.sample_multiplane reads them), 8 taps
per plane, and the plane gradient comes back in the same indexing.  At depth 1 every function computes what it did before
the argument existed, bit for bit.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import renderer_oracle as orc

Tensor = torch.Tensor
COL_FACTOR = 1.002          # d(rgb) / d(sigmoid): decode's rgb * (1 + 2 * 0.001) - 0.001
SOFTPLUS_THRESH = 20.0      # F.softplus's linear branch (and the kernels' softplus_t / its derivative)
U = 2.0 ** -24
CHUNK = 1 << 16             # samples per step of the (K, taps, C) intermediates: 0.8 GB in fp64 at 48 taps


def taps(xyz: Tensor, H: int, W: int, box_warp: float, use_triplane: bool, depth: int = 1, *, normal_triplane=None,
         slab_align_corners: bool = False):
    """Taps of points xyz (K,3), in the kernel's fp32.  depth 1: bilinear (dev::bilinear_footprint, dev::plane_tap<false>), texel
    index p*H*W + y*W + x (-1 outside the plane) and weight wx*wy, each (K,12) in plane-major, then row, then column order.
    depth D > 1: trilinear (dev::slab_footprint, dev::plane_tap<true>), texel index ((p*D + z)*H + y)*W + x and weight
    (wx*wy)*wz, each (K,24): per plane, k & 1 the column, (k >> 1) & 1 the row, k >> 2 the slab (z0, then z0 + 1).
    normal_triplane (plane 2's normal from that plane order) and slab_align_corners exist for negative controls."""
    assert xyz.dtype == torch.float32
    grid = orc.plane_coords((2.0 / box_warp) * xyz[None], use_triplane)[0]          # 3,K,2
    fx = ((grid[..., 0] + 1) * W - 1) * 0.5
    fy = ((grid[..., 1] + 1) * H - 1) * 0.5
    x0f, y0f = torch.floor(fx), torch.floor(fy)
    wx1, wy1 = fx - x0f, fy - y0f
    x0, y0 = x0f.long(), y0f.long()
    idx, wgt = [], []
    if depth > 1:
        D = depth
        scaled = (2.0 / box_warp) * xyz
        third = use_triplane if normal_triplane is None else normal_triplane
        gz = torch.stack([scaled[:, 2], scaled[:, 1], scaled[:, 0 if third else 1]])          # dev::plane_normal
        fz = (gz + 1) * (D - 1) * 0.5 if slab_align_corners else ((gz + 1) * D - 1) * 0.5
        z0f = torch.floor(fz)
        wz1 = fz - z0f
        z0 = torch.where((fz > -2) & (fz < D + 1), z0f, torch.full_like(z0f, -4)).long()   # slab_footprint's `sane`
        for p in range(3):
            for dz, wz in ((0, 1 - wz1[p]), (1, wz1[p])):
                for dy, wy in ((0, 1 - wy1[p]), (1, wy1[p])):
                    for dx, wx in ((0, 1 - wx1[p]), (1, wx1[p])):
                        xi, yi, zi = x0[p] + dx, y0[p] + dy, z0[p] + dz
                        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H) & (zi >= 0) & (zi < D)
                        idx.append(torch.where(ok, ((p * D + zi) * H + yi) * W + xi, -1))
                        wgt.append(torch.where(ok, (wx * wy) * wz, 0.0))
        return torch.stack(idx, 1), torch.stack(wgt, 1)
    for p in range(3):
        for dy, wy in ((0, 1 - wy1[p]), (1, wy1[p])):
            for dx, wx in ((0, 1 - wx1[p]), (1, wx1[p])):
                xi, yi = x0[p] + dx, y0[p] + dy
                ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
                idx.append(torch.where(ok, (p * H + yi) * W + xi, -1))
                wgt.append(torch.where(ok, wx * wy, 0.0))
    return torch.stack(idx, 1), torch.stack(wgt, 1)


def gather(flat: Tensor, idx: Tensor, wgt: Tensor) -> Tensor:
    """Per-plane sums of texels flat (3[D]HW, C) at taps (K,12) or (K,24) -> (K,3,C), CHUNK samples at a time."""
    out = []
    for i in range(0, idx.shape[0], CHUNK):
        v = flat[idx[i:i + CHUNK].clamp_min(0)] * wgt[i:i + CHUNK].to(flat.dtype)[..., None]
        out.append(v.reshape(v.shape[0], 3, idx.shape[1] // 3, -1).sum(2))
    return torch.cat(out) if len(out) != 1 else out[0]


def texels(planes_n: Tensor, depth: int = 1) -> Tensor:
    """The texels of one view's planes (3, C*depth, H, W) as rows of the taps' index: (3*depth*H*W, C)."""
    if depth > 1:
        CD, H, W = planes_n.shape[1:]
        return planes_n.reshape(3, CD // depth, depth, H, W).permute(0, 2, 3, 4, 1).reshape(3 * depth * H * W, CD // depth)
    C, H, W = planes_n.shape[1:]
    return planes_n.permute(0, 2, 3, 1).reshape(3 * H * W, C)


def _plane_grad(g: Tensor, H: int, W: int, depth: int) -> Tensor:
    """(N, 3*depth*H*W, C) texel gradients -> the planes' (N, 3, C*depth, H, W) indexing."""
    N, _, C = g.shape
    if depth > 1:
        return g.reshape(N, 3, depth, H, W, C).permute(0, 1, 5, 2, 3, 4).reshape(N, 3, C * depth, H, W)
    return g.reshape(N, 3, H, W, C).permute(0, 1, 4, 2, 3)


def texel_counts(ro, rd, depths, H, W, box_warp, use_triplane=True, depth: int = 1) -> Tensor:
    """How many tap contributions each texel (N,3,H,W), or (N,3,D,H,W) for depth D > 1, receives from the samples at
    `depths`: the number of atomic adds k_sample_backward makes into it."""
    N = ro.shape[0]
    out = torch.zeros(N, 3 * depth * H * W, dtype=torch.int64, device=ro.device)
    for n in range(N):
        for d in depths:
            if d is None:
                continue
            xyz = (ro[n, :, None] + d[n, ..., 0, None] * rd[n, :, None]).reshape(-1, 3)
            idx, _ = taps(xyz, H, W, box_warp, use_triplane, depth)
            idx = idx[idx >= 0]
            out[n] += torch.bincount(idx, minlength=3 * depth * H * W)
    return out.reshape(N, 3, depth, H, W) if depth > 1 else out.reshape(N, 3, H, W)


def _floors(c: float, C: int, Hd: int):
    """Absolute errors of the kernel that are not a relative error of its own value, written as magnitudes in units of
    (c u), so that (k + c) u A covers them:
      alpha = 1 - expf(-x) and 1 - alpha: absolute error <= 3u each (expf to 2 ulp, one subtraction), so alpha and
        exp(-x) enter A as value + 3/c;
      s (1 - s) of a colour: 1 - sigmoid_t(o) is off by <= 2u absolute -> + 2/c; and the fp32 logit o is off by
        (Hd + 1) u m2 (m2 = |h| |W2| + |b2|), a relative (Hd + 1) m2 u change of s (1 - s) -> factor 1 + (Hd + 1) m2 / c;
      the pre-activation is off by (C + 1) u m1 (m1 = |x| |W1| + |b1|): sigmoid(pre) by a relative (C + 1) m1 u and
        softplus(pre) by sigmoid(pre) (C + 1) m1 u absolute."""
    return 3.0 / c, 2.0 / c, (Hd + 1) / c, (C + 1) / c


def _decoder_backward(out, n, flat, idx, wgt, x, pre, hs, s, dsig, dcol, mats, gains, mag, floors, sp_thresh, plane_mean):
    """k_sample_backward's part for the samples of view n: dlog = (dsig, dcol s (1 - s)) back through the decoder into
    out['w1' / 'b1' / 'w2' / 'b2'] and, scattered to the taps (idx, wgt), into out['planes'][n] ((3[D]HW, C))."""
    W1, B1, W2, B2 = mats
    g1, g2, lr = gains
    fs, fo, fp = floors
    st = s * (1 - s)
    if mag:
        x_a = gather(flat.abs(), idx, wgt).sum(1) / 3
        m1 = x_a @ W1.abs().t() + B1.abs()
        sgp = torch.sigmoid(pre)
        hs_a = hs.abs() + sgp * fp * m1
        m2 = hs_a @ W2.abs().t() + B2.abs()
        st = st * (1 + fo * m2[:, 1:]) + fs
        dpre_f = torch.where(pre > sp_thresh, torch.ones_like(pre), sgp) * (1 + fp * m1)
        x_use, hs_use, W1u, W2u = x_a, hs_a, W1.abs(), W2.abs()
    else:
        dpre_f = torch.where(pre > sp_thresh, torch.ones_like(pre), torch.sigmoid(pre))
        x_use, hs_use, W1u, W2u = x, hs, W1, W2
    dlog = torch.cat([dsig[:, None], dcol * st], 1)
    dpre = (dlog @ W2u) * dpre_f
    dx = (dpre @ W1u) * plane_mean
    out['w2'] += g2 * (dlog.t() @ hs_use)
    out['b2'] += lr * dlog.sum(0)
    out['w1'] += g1 * (dpre.t() @ x_use)
    out['b1'] += lr * dpre.sum(0)
    for i in range(0, idx.shape[0], CHUNK):
        contrib = dx[i:i + CHUNK, None, :] * wgt[i:i + CHUNK].to(dx.dtype)[..., None]        # (K,12|24,C)
        ok = idx[i:i + CHUNK] >= 0
        out['planes'][n].index_add_(0, idx[i:i + CHUNK][ok], contrib[ok])


def _decoder_forward(planes_n, dec, xyz, box_warp, use_triplane, depth: int = 1):
    """Taps, texels (3[D]HW, C), features, pre-activations, softplus and logits of points xyz (K,3) fp32 on view planes_n
    ((3, C*depth, H, W))."""
    H, W = planes_n.shape[2:]
    lr = dec.get('lr_mul', 1.0)
    g1, g2 = lr / math.sqrt(dec['w1'].shape[1]), lr / math.sqrt(dec['w2'].shape[1])
    idx, wgt = taps(xyz, H, W, box_warp, use_triplane, depth)
    flat = texels(planes_n, depth)
    x = gather(flat, idx, wgt).sum(1) / 3
    pre = x @ (dec['w1'] * g1).t() + dec['b1'] * lr
    hs = F.softplus(pre)
    o = hs @ (dec['w2'] * g2).t() + dec['b2'] * lr
    return idx, wgt, flat, x, pre, hs, o


def points_backward(planes: Tensor, dec: Dict, xyz: Tensor, g_sigma: Tensor, box_warp: float, use_triplane: bool = True,
                    mag: bool = False, c: float = 1.0, sp_thresh: float = SOFTPLUS_THRESH, depth: int = 1):
    """Gradients {planes, w1, b1, w2, b2} of sum(sigma * g_sigma) over run_model's sigma at points xyz (N,K,3) fp32 (the
    density-regularisation backward, k_sample_backward in point mode), or with mag=True its magnitude adjoint."""
    dt = planes.dtype
    N, _, CD, H, W = planes.shape
    C = CD // depth
    lr = dec.get('lr_mul', 1.0)
    g1, g2 = lr / math.sqrt(dec['w1'].shape[1]), lr / math.sqrt(dec['w2'].shape[1])
    mats = (dec['w1'] * g1, dec['b1'] * lr, dec['w2'] * g2, dec['b2'] * lr)
    _, fs, fo, fp = _floors(c, C, mats[0].shape[0])
    out = dict(planes=torch.zeros(N, 3 * depth * H * W, C, dtype=dt, device=planes.device),
               w1=torch.zeros_like(mats[0]), b1=torch.zeros_like(mats[1]), w2=torch.zeros_like(mats[2]),
               b2=torch.zeros_like(mats[3]))
    for n in range(N):
        idx, wgt, flat, x, pre, hs, o = _decoder_forward(planes[n], dec, xyz[n], box_warp, use_triplane, depth)
        g = g_sigma[n].reshape(-1).to(dt)
        dcol = torch.zeros(x.shape[0], mats[2].shape[0] - 1, dtype=dt, device=planes.device)
        _decoder_backward(out, n, flat, idx, wgt, x, pre, hs, torch.sigmoid(o[:, 1:]), g.abs() if mag else g, dcol, mats,
                          (g1, g2, lr), mag, (fs, fo, fp), sp_thresh, 1.0 / 3.0)
    out['planes'] = _plane_grad(out['planes'], H, W, depth)
    return out


def sigma_error_bound(planes_n: Tensor, dec: Dict, xyz: Tensor, box_warp: float, use_triplane: bool = True,
                      depth: int = 1) -> Tensor:
    """Per point (K,), a bound on the fp32 SIMT decode's sigma error (render_v1.cu): the gather, the pre-activation's
    C + 1 fmas, softplus_t to 4 ulp and the logit's Hd + 1 fmas, each taken over the magnitudes of its operands.  The
    gather: one slab, 12 fmas, two adds and a division by 3 (16u of the features' magnitude); depth > 1, 24 fmas
    (gather_features<*, true>: 8 per plane), the two roundings of the weight (wx wy) wz, two adds and the division (29u)."""
    idx, wgt, flat, x, pre, hs, o = _decoder_forward(planes_n, dec, xyz, box_warp, use_triplane, depth)
    lr = dec.get('lr_mul', 1.0)
    C = dec['w1'].shape[1]
    W1a = (dec['w1'] * (lr / math.sqrt(C))).abs()
    w20 = (dec['w2'][0] * (lr / math.sqrt(dec['w2'].shape[1]))).abs()
    x_a = gather(flat.abs(), idx, wgt).sum(1) / 3
    m1 = x_a @ W1a.t() + (dec['b1'] * lr).abs()
    d_hs = torch.sigmoid(pre) * (C + (17 if depth == 1 else 30)) * U * m1 + 4 * U * hs.abs()
    return (w20.shape[0] + 1) * U * ((hs.abs() + d_hs) @ w20 + abs(float(dec['b2'][0]) * lr)) + d_hs @ w20


def render_backward(planes: Tensor, dec: Dict, ro: Tensor, rd: Tensor, opts: Dict, depths, masks, grads,
                    triplane_crop=None, cull_clouds=None, binarize_clouds=None, use_triplane: bool = True,
                    bounds=None, fwd=None, dead=None, mag: bool = False, c: float = 1.0,
                    col_factor: float = COL_FACTOR, sp_thresh: float = SOFTPLUS_THRESH, plane_mean: float = 1.0 / 3.0,
                    depth: int = 1):
    """Gradients {planes (N,3,C*depth,H,W), w1, b1, w2, b2} of sum(out * grad) over render's outputs (rgb, depth, wsum,
    xyz).

    planes / dec in the compute dtype; ro, rd (N,M,3) and depths (coarse (N,M,S,1), fine (N,M,Sf,1) or None) fp32;
    masks as renderer_oracle.render takes them (ignored without a mask flag); grads = (g_rgb (N,M,32), g_depth, g_wsum
    (N,M,1), g_xyz (N,M,3)).  bounds: the depth clamp (lo, hi), default min / max of all depths.  fwd: per view
    (sigma_c (M,S), rgb_c (M,S,32), sigma_f, rgb_f) to composite with instead of this run's own (the kernel's fp32
    forward values, post-mask).  dead: (N,M) bool, rays whose depth gradient is gated off as the kernel's W == 0 gates it
    (W = sum w is ill-conditioned near 0: an fp32 alpha = 1 - expf(-x) is exactly 0 for x below u).  mag: the magnitude
    adjoint with the floors of `_floors` for the constant c.
    col_factor / sp_thresh / plane_mean: the colour factor, the softplus-derivative threshold and the plane mean of dx,
    changeable for negative controls."""
    dt = planes.dtype
    N, _, CD, H, W = planes.shape
    C = CD // depth
    d_c, d_f = depths
    S, Sf = d_c.shape[2], (0 if d_f is None else d_f.shape[2])
    bw = opts['box_warp']
    back = 1.0 if opts.get('white_back', False) else 0.0
    lr = dec.get('lr_mul', 1.0)
    force = bool(dec.get('force_sigmoid', False))
    g1, g2 = lr / math.sqrt(dec['w1'].shape[1]), lr / math.sqrt(dec['w2'].shape[1])
    W1, B1, W2, B2 = dec['w1'] * g1, dec['b1'] * lr, dec['w2'] * g2, dec['b2'] * lr
    Hd = W1.shape[0]
    if bounds is None:
        every = torch.cat([d_c.reshape(N, -1)] + ([] if d_f is None else [d_f.reshape(N, -1)]), 1)
        bounds = (every.min(), every.max())
    lo, hi = (float(b) for b in bounds)
    fa, fs, fo, fp = _floors(c, C, Hd)
    ab = (lambda t: t.abs()) if mag else (lambda t: t)
    cf = 1.0 if force else col_factor
    masked_any = bool(triplane_crop or cull_clouds or binarize_clouds)
    out = dict(planes=torch.zeros(N, 3 * depth * H * W, C, dtype=dt, device=planes.device),
               w1=torch.zeros_like(W1), b1=torch.zeros_like(B1), w2=torch.zeros_like(W2), b2=torch.zeros_like(B2))
    g_rgb_all, g_dep_all, g_w_all, g_xyz_all = grads
    for n in range(N):
        tc, tf = d_c[n, ..., 0], (None if d_f is None else d_f[n, ..., 0])            # (M,S), (M,Sf) fp32
        M = tc.shape[0]
        t_src = tc if tf is None else torch.cat([tc, tf], 1)                             # (M,L) in sample order
        L = t_src.shape[1]
        xyz = (ro[n, :, None] + t_src[..., None] * rd[n, :, None])                       # (M,L,3) fp32, as the kernel
        xyz_flat = torch.cat([xyz[:, :S].reshape(-1, 3), xyz[:, S:].reshape(-1, 3)])    # coarse samples, then fine
        idx, wgt = taps(xyz_flat, H, W, bw, use_triplane, depth)
        flat = texels(planes[n], depth)
        x = gather(flat, idx, wgt).sum(1) / 3
        pre = x @ W1.t() + B1
        hs = F.softplus(pre)
        o = hs @ W2.t() + B2
        s = torch.sigmoid(o[:, 1:])
        rgb = s if force else s * (1 + 2 * 0.001) - 0.001
        sig = o[:, 0]
        if masked_any:
            mk = torch.cat([masks[0][n].reshape(-1)] + ([] if tf is None else [masks[1][n].reshape(-1)]))
            sig = torch.where(mk, torch.full_like(sig, -1e3), sig)
            if binarize_clouds:
                sig = torch.where(mk, sig, torch.full_like(sig, 1e3))
        if fwd is not None:       # composite the kernel's values (the decoder backward recomputes s itself: see _floors)
            sig = torch.cat([fwd[n][0].reshape(-1)] + ([] if tf is None else [fwd[n][2].reshape(-1)])).to(dt)
            rgb = torch.cat([fwd[n][1].reshape(-1, 32)] + ([] if tf is None else [fwd[n][3].reshape(-1, 32)])).to(dt)

        def per_ray(v):                                   # (K, ...) in coarse-then-fine sample order -> (M, L, ...)
            a = v[:M * S].reshape(M, S, *v.shape[1:])
            return a if tf is None else torch.cat([a, v[M * S:].reshape(M, Sf, *v.shape[1:])], 1)

        order = torch.sort(t_src, dim=1, stable=True)[1]
        t = torch.gather(t_src, 1, order)
        sg = torch.gather(per_ray(sig), 1, order)
        col = torch.cat([per_ray(rgb), xyz.to(dt)], -1)
        col = torch.gather(col, 1, order[..., None].expand(-1, -1, col.shape[-1]))
        delta = (t[:, 1:] - t[:, :-1]).to(dt)
        tmid = ((t[:, :-1] + t[:, 1:]) / 2).to(dt)
        smid = (sg[:, :-1] + sg[:, 1:]) / 2 - 1
        xd = F.softplus(smid) * delta
        e = torch.exp(-xd)
        alpha = 1 - e
        fc = 1 - alpha + 1e-10
        T = torch.cumprod(torch.cat([torch.ones_like(fc[:, :1]), fc[:, :-1]], 1), 1)
        w = alpha * T
        Wsum = w.sum(1)
        depth_raw = (w * tmid).sum(1) / Wsum
        live = (Wsum != 0) & torch.isfinite(depth_raw) & (depth_raw >= lo) & (depth_raw <= hi)
        if dead is not None:
            live &= ~dead[n]
        g_col = torch.cat([g_rgb_all[n], g_xyz_all[n]], -1).to(dt)                        # (M,35)
        g_dep = torch.where(live, g_dep_all[n, :, 0].to(dt), torch.zeros_like(Wsum))
        g_w = g_w_all[n, :, 0].to(dt)
        q = (ab(col) * ab(g_col)[:, None]).sum(-1)
        common = ab(g_w) + (2 * back * ab(g_col).sum(-1) if mag else -2 * back * g_col.sum(-1))
        Wsafe = torch.where(live, Wsum, torch.ones_like(Wsum))
        dr = torch.where(live, depth_raw, torch.zeros_like(depth_raw))
        if mag:     # W and D are sums of w = alpha T, each off by 3u T absolute: W by 3u sum(T) (see _floors), D by up to 2x that
            wrel = 1 + 3 * fa * T.sum(1) / Wsafe
            dep_term = ab(g_dep)[:, None] * (tmid.abs() + dr.abs()[:, None]) * wrel[:, None] / Wsafe[:, None]
        else:
            dep_term = g_dep[:, None] * (tmid - dr[:, None]) / Wsafe[:, None]
        P = q[:, :-1] + q[:, 1:] + common[:, None] + dep_term
        wk = (alpha + fa) * T if mag else w
        wP = wk * P
        incl = torch.cumsum(wP, 1)
        total = incl[:, -1:]
        suffix = total + incl if mag else total - incl
        dalpha = T * P + suffix / fc if mag else T * P - suffix / fc
        dsp = torch.where(smid > sp_thresh, torch.ones_like(smid), torch.sigmoid(smid))
        dsb = dalpha * ((e + fa) if mag else e) * delta * dsp
        zero = torch.zeros_like(dsb[:, :1])
        dsig_sorted = 0.5 * (torch.cat([zero, dsb], 1) + torch.cat([dsb, zero], 1))
        om_sorted = 0.5 * (torch.cat([zero, wk], 1) + torch.cat([wk, zero], 1))
        dsig_r = torch.zeros_like(dsig_sorted).scatter_(1, order, dsig_sorted)
        om_r = torch.zeros_like(om_sorted).scatter_(1, order, om_sorted)

        def flat_samples(v):                              # (M, L) -> (K,) coarse then fine
            return torch.cat([v[:, :S].reshape(-1), v[:, S:].reshape(-1)])

        dsig = flat_samples(dsig_r)
        if binarize_clouds:
            dsig = torch.zeros_like(dsig)
        elif masked_any:
            dsig = torch.where(mk, torch.zeros_like(dsig), dsig)
        omega = flat_samples(om_r)
        ray_of = torch.cat([torch.arange(M, device=ro.device).repeat_interleave(S),
                            torch.arange(M, device=ro.device).repeat_interleave(Sf)])
        dcol = 2 * omega[:, None] * ab(g_rgb_all[n].to(dt))[ray_of]
        _decoder_backward(out, n, flat, idx, wgt, x, pre, hs, s, dsig, dcol * cf, (W1, B1, W2, B2),
                          (g1, g2, lr), mag, (fs, fo, fp), sp_thresh, plane_mean)
    out['planes'] = _plane_grad(out['planes'], H, W, depth)
    return out
