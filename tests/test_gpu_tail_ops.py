"""The kernels around the convs of the benchmarked training step, at production shape and at their edges, against fp64.

Each op has a reference here (fp64, on the device in the GPU tests) and an fp32 emulation of what its kernel computes
(csrc/nlt_ops.cu), so that the CPU tests can show that each reference passes the fp32 computation and flags the
mistakes a kernel could make: a wrong step count or a rounded (1 - beta) in AMSGrad, two resampler taps swapped, a
missing factor 2 in the L2 gradient, a K-mean divided by K - 1, image inputs left in [0, 255].

Metric: r = |got - ref| / (abs_ref + tiny), as in tests/test_gpu_census.py (max_rel).  The ops here sum at most a
handful of terms per element (the K-mean: K), so fp32 stays within a few 2^-24 of abs_ref and their bar is ELEM_BAR
(2^-20, 16 ulps).  The reductions (the L2 loss over 3 * 1024^2 values) and the fixed-point UV scatter keep the
census's TAU; the scatter's floor follows from its fixed-point quantum (scatter_floor).  AMSGrad has its own bars (see amsgrad_r).
"""
import math
import time

import pytest
import torch

from oracle import nlt_oracle as O
from tests.test_gpu_census import TAIL_FLOOR, TAU, TINY, _record, max_rel

ELEM_BAR = 2.0 ** -20
# AMSGrad: m, v and vhat are one fused multiply-add from their fp32 operands (a few roundings: 4 ulps of the operand
# magnitudes); p is one rounding of p plus the step, and the step (lr_t * m / (sqrt(vhat) + eps)) is a few more
# roundings on top of those of m and vhat
ADAM_STATE_BAR = 2.0 ** -22
ADAM_STEP_BAR = 2.0 ** -20
LR, B1, B2, EPS = 1e-3, 0.9, 0.999, 1e-7          # trainvali.Adam defaults, as bench.TrainRun builds it


def f32(x):
    """The float32 value of a Python float, as a Python float (what the kernel receives)."""
    return float(torch.tensor(x, dtype=torch.float32))


def worst(got, ref, abs_ref, tiny=TINY):
    """(r, index of the worst element, got there, ref there) for failure messages."""
    got = got.to(ref.device, torch.float64)
    r = (got - ref).abs() / (abs_ref + tiny)
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))
    i = int(r.reshape(-1).argmax())
    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape))
    return float(r.reshape(-1)[i]), idx, float(got.reshape(-1)[i]), float(ref.reshape(-1)[i])


def check(name, got, ref, abs_ref, bar, tiny=TINY, out=None):
    r, idx, g, w = worst(got, ref, abs_ref, tiny)
    if out is not None:
        out[name] = r
    assert r <= bar, '%s: r = %.3g > %.3g at %s (got %r, want %r)' % (name, r, bar, idx, g, w)
    return r


# ----------------------------------------------------------------------------------------------------------------
# references (fp64) and fp32 emulations of the kernels
# ----------------------------------------------------------------------------------------------------------------
def sample_points(warp, H, W):
    """The kernel's sample points: warp * (W, H) formed in fp32, then exact in fp64."""
    return torch.stack((warp[..., 0] * float(W), warp[..., 1] * float(H)), dim=3).double()


def corner0(x):
    return O.set_left_top_corner(x, 0)


def uv2cam_ref(pred_uv, base, warp, rgb_camspc):
    """fp64 (ref, |.|) of the camera outputs of nlt_uv2cam_fwd from the product's own fp32 pred_uv (corner zeroed):
    {'pred': ..., 'base': ..., 'fg': ..., 'gt': ...}."""
    B, H, W, _ = pred_uv.shape
    w = sample_points(warp, H, W)
    p, b = pred_uv.double(), corner0(base.double())
    fg = O.resampler(corner0(torch.ones_like(p)), w)
    out = {'pred': (O.resampler(p, w), O.resampler(p.abs(), w)),
           'base': (O.resampler(b, w), O.resampler(b.abs(), w)),
           'fg': (fg, fg)}
    if rgb_camspc is not None:
        rgb = rgb_camspc.double()
        out['gt'] = (rgb * fg, rgb.abs() * fg)
    return out


def taps32(warp, H, W, swap=None):
    """fp32 tap weights and flat texel indices of the kernel's resampler_taps (order (fx,fy), (cx,cy), (fx,cy),
    (cx,fy)); index -1 where the tap contributes zero.  swap=(i, j) exchanges two weights (a control)."""
    x, y = warp[..., 0] * float(W), warp[..., 1] * float(H)
    inside = (x > -1) & (y > -1) & (x < W) & (y < H)
    fx, fy = torch.floor(x), torch.floor(y)
    cx, cy = fx + 1, fy + 1
    dx, dy = cx - x, cy - y
    ws = [dx * dy, (1 - dx) * (1 - dy), dx * (1 - dy), (1 - dx) * dy]
    if swap is not None:
        ws[swap[0]], ws[swap[1]] = ws[swap[1]], ws[swap[0]]
    idx = []
    for ix, iy in ((fx, fy), (cx, cy), (fx, cy), (cx, fy)):
        ok = inside & (ix >= 0) & (ix <= W - 1) & (iy >= 0) & (iy <= H - 1)
        idx.append(torch.where(ok, iy * W + ix, torch.full_like(ix, -1)).long())
    return ws, idx


def resample32(data, warp, swap=None):
    """fp32 emulation of the kernel's four-tap sum (texel (0,0) read as zero)."""
    B, H, W, C = data.shape
    ws, idx = taps32(warp, H, W, swap)
    flat = data.reshape(B, H * W, C)
    out = torch.zeros(warp.shape[:3] + (C,), dtype=torch.float32, device=data.device)
    for w, i in zip(ws, idx):
        live = i > 0
        v = torch.gather(flat, 1, i.clamp(min=0).reshape(B, -1, 1).expand(-1, -1, C)).reshape(out.shape)
        out = out + w.unsqueeze(-1) * torch.where(live.unsqueeze(-1), v, torch.zeros_like(v))
    return out


def uv2cam_bwd_ref(d, warp, H, W):
    """fp64 (ref, |.|) of d(net_out): d pulled back through the resampler, zero at texel (0,0)."""
    B = d.shape[0]
    w = sample_points(warp, H, W)
    p = torch.zeros(B, H, W, d.shape[3], dtype=torch.float64, device=d.device, requires_grad=True)
    pc = O.resampler(p, w)
    ref = torch.autograd.grad(pc, p, d.double(), retain_graph=True)[0]
    absr = torch.autograd.grad(pc, p, d.double().abs())[0]
    ref[:, 0, 0, :] = 0
    absr[:, 0, 0, :] = 0
    return ref, absr


def scatter_floor(gmax):
    """Floor of r for nlt_uv2cam_bwd_det.  Its precision is absolute: half a quantum 2^(e - 37) per contribution
    (e = floor(log2 max|d|)), about four contributions per texel at 1:1 magnification, so the floor is the one at which
    that error reads as r = TAU: 2^(e - 36) / TAU.  The census's TAIL_FLOOR * max|d| is 2^9 finer; over all 32 images
    of a batch a texel fed only by small values reads 1.006 TAU with it.  Texels of a value 2^20 below gmax keep ~18
    of fp32's 24 bits.  Below the smallest normal the fp32 products w * g are themselves quantised: the floor stays
    above TINY.  The fixed-point sum itself is checked bit for bit against uv2cam_bwd_fixed32."""
    e = (int(torch.tensor(gmax, dtype=torch.float32).view(torch.int32)) >> 23 & 0xff) - 127
    return 2.0 ** (e - 36) / TAU + TINY


def uv2cam_bwd_fixed32(d, warp, H, W, swap=None):
    """Emulation of nlt_uv2cam_bwd_det: fp32 products w * g, rounded to 64-bit fixed point at 2^(37 - e) with
    e = floor(log2 max|d|), summed as integers, converted back."""
    B, ih, iw, C = d.shape
    gmax = float(d.abs().max())
    e = (int(torch.tensor(gmax, dtype=torch.float32).view(torch.int32)) >> 23 & 0xff) - 127
    scale = 2.0 ** (37 - e)
    ws, idx = taps32(warp, H, W, swap)
    acc = torch.zeros(B * H * W, C, dtype=torch.int64, device=d.device)
    boff = (torch.arange(B, device=d.device) * H * W).view(B, 1, 1)
    for w, i in zip(ws, idx):
        live = i > 0
        q = torch.round((w.unsqueeze(-1) * d).double() * scale).long()
        q = torch.where(live.unsqueeze(-1), q, torch.zeros_like(q))
        acc.index_add_(0, (i.clamp(min=0) + boff).reshape(-1), q.reshape(-1, C))
    return (acc.double() / scale).float().reshape(B, H, W, C)


def l2_ref(pred, gt, scale):
    """fp64 (loss_b, |.|) and (d_pred, |.|) of nlt_l2_loss: loss_b = mean((pred - gt)^2) over a sample,
    d_pred = 2 (pred - gt) scale / per_sample."""
    B = pred.shape[0]
    p, g = pred.double().reshape(B, -1), gt.double().reshape(B, -1)
    n = p.shape[1]
    dif = p - g
    loss = (dif * dif).mean(1)
    d = 2.0 * dif * scale / n
    dabs = 2.0 * (p.abs() + g.abs()) * scale / n
    return (loss, loss), (d.reshape(pred.shape), dabs.reshape(pred.shape))


def l2_fp32(pred, gt, scale, factor=2.0):
    B = pred.shape[0]
    dif = (pred - gt).reshape(B, -1)
    n = dif.shape[1]
    return (dif * dif).sum(1) * f32(1.0 / n), (dif * f32(factor * scale / n)).reshape(pred.shape)


def kmean_ref(x, K, w=None):
    """fp64 (mean, |.|) over the K k-major stacked observations of x [K*B, ...] (weights w [B, K])."""
    xk = x.double().reshape((K, -1) + tuple(x.shape[1:]))
    if w is not None:
        wk = w.double().t().reshape((K, -1) + (1,) * (x.dim() - 1))
        return (xk * wk).sum(0) / K, (xk * wk).abs().sum(0) / K
    return xk.sum(0) / K, xk.abs().sum(0) / K


def kmean_fp32(x, K, divisor=None):
    xk = x.reshape((K, -1) + tuple(x.shape[1:]))
    s = xk[0].clone()
    for k in range(1, K):
        s = s + xk[k]
    return s * f32(1.0 / (divisor or K))


def amsgrad_ref(p, g, m, v, vh, t, b1=B1, b2=B2, lr=LR, eps=EPS):
    """O.amsgrad_step in fp64 with the hyper-parameters as the kernel receives them (float32 values): 1 - beta is then
    the same exact number in fp64 as the kernel's 1.f - b."""
    return O.amsgrad_step(p.double(), g.double(), m.double(), v.double(), vh.double(), t, f32(lr), f32(b1), f32(b2),
                          f32(eps))


def amsgrad_fp32(p, g, m, v, vh, t, lr=LR, b1=B1, b2=B2, eps=EPS):
    """The kernel's fp32 arithmetic (nvcc contracts a + b * c into one fused multiply-add)."""
    fma = lambda a, b, c: (a.double() * b.double() + c.double()).float()
    c1, c2 = torch.tensor(1.0 - f32(b1)).float(), torch.tensor(1.0 - f32(b2)).float()
    lr_t = f32(f32(lr) * math.sqrt(1.0 - f32(b2) ** t) / (1.0 - f32(b1) ** t))
    mi = fma(g - m, c1, m)
    vi = fma(fma(g, g, -v), c2, v)
    vhi = torch.maximum(vh, vi)
    pi = p - (lr_t * mi) / (torch.sqrt(vhi) + f32(eps))
    return pi, mi, vi, vhi


def amsgrad_r(got, p0, g, m0, v0, vh0, t, **ref_kw):
    """{'m', 'v', 'vhat': r against 4-ulp bars of the operand magnitudes; 'p': r of the step part}.
    m = m0 + (g - m0) c1: magnitude |m0| + (|g| + |m0|) c1, likewise v with g^2.  p: |p - p_ref| less one rounding of
    p, over the magnitude of the step, lr_t (|m0| + (|g| + |m0|) c1) / (sqrt(vhat_ref) + eps)."""
    pr, mr, vr, vhr = amsgrad_ref(p0, g, m0, v0, vh0, t, **ref_kw)
    c1, c2 = 1.0 - f32(B1), 1.0 - f32(B2)
    gd, m0d, v0d = g.double(), m0.double(), v0.double()
    mabs = m0d.abs() + (gd.abs() + m0d.abs()) * c1
    vabs = v0d + (gd * gd + v0d) * c2
    vhabs = torch.maximum(vh0.double(), vabs)
    lr_t = f32(LR) * math.sqrt(1 - f32(B2) ** t) / (1 - f32(B1) ** t)
    sabs = lr_t * mabs / (vhr.sqrt() + f32(EPS))
    pg, mg, vg, vhg = (x.to(pr.device, torch.float64) for x in got)
    dp = ((pg - pr).abs() - pr.abs() * 2.0 ** -24).clamp(min=0)
    rp = dp / (sabs + TINY)
    rp = torch.where(torch.isfinite(pg), rp, torch.full_like(rp, math.inf))
    return {'p': float(rp.max()), 'm': max_rel(mg, mr, mabs), 'v': max_rel(vg, vr, vabs),
            'vhat': max_rel(vhg, vhr, vhabs)}


def amsgrad_ok(r):
    return r['p'] <= ADAM_STEP_BAR and all(r[k] <= ADAM_STATE_BAR for k in ('m', 'v', 'vhat'))


# ----------------------------------------------------------------------------------------------------------------
# CPU: each reference passes its fp32 computation and flags the controls
# ----------------------------------------------------------------------------------------------------------------
def _cpu_tail(seed=3, B=2, H=24, ih=20):
    from util import synth
    bt = synth.make_batch(B, H, ih, seed=seed)
    g = torch.Generator().manual_seed(seed)
    net = torch.randn(B, H, H, 3, generator=g)
    pred_uv = corner0(net + bt[1])
    return pred_uv, bt[1], bt[4], bt[6]


def test_uv2cam_reference_passes_fp32_and_flags_swapped_taps():
    pred_uv, base, warp, rgb = _cpu_tail()
    ref, absr = uv2cam_ref(pred_uv, base, warp, rgb)['pred']
    assert max_rel(resample32(pred_uv, warp), ref, absr) <= ELEM_BAR / 4
    for swap in ((0, 1), (2, 3), (0, 3)):
        assert max_rel(resample32(pred_uv, warp, swap), ref, absr) >= 1e3 * ELEM_BAR, swap
    ref, absr = uv2cam_ref(pred_uv, base, warp, rgb)['base']
    assert max_rel(resample32(corner0(base), warp), ref, absr) <= ELEM_BAR / 4
    # image inputs 255 times too large (uint8 samples never divided by 255)
    assert max_rel(resample32(corner0(base * 255), warp), ref, absr) >= 1e3 * ELEM_BAR


def test_uv2cam_bwd_reference_passes_fixed_point_emulation_and_flags_swapped_taps():
    pred_uv, base, warp, _ = _cpu_tail()
    B, H = pred_uv.shape[:2]
    d = torch.randn(B, warp.shape[1], warp.shape[2], 3, generator=torch.Generator().manual_seed(4))
    ref, absr = uv2cam_bwd_ref(d, warp, H, H)
    tiny = scatter_floor(float(d.abs().max()))
    assert max_rel(uv2cam_bwd_fixed32(d, warp, H, H), ref, absr, tiny) <= TAU / 4
    assert max_rel(uv2cam_bwd_fixed32(d, warp, H, H, swap=(0, 1)), ref, absr, tiny) >= 1e3 * TAU
    # one value 2^20 above the rest: the census floor is too fine for the absolute quantum; the quantum's floor passes
    d[:] *= 2.0 ** -20
    d[1, 5, 5, 1] = 1.5
    ref, absr = uv2cam_bwd_ref(d, warp, H, H)
    emu = uv2cam_bwd_fixed32(d, warp, H, H)
    assert max_rel(emu, ref, absr, TAIL_FLOOR * 1.5 + TINY) > TAU
    assert max_rel(emu, ref, absr, scatter_floor(1.5)) <= TAU


def test_l2_reference_passes_fp32_and_flags_missing_factor_2():
    g = torch.Generator().manual_seed(5)
    pred, gt = torch.rand(3, 16, 20, 3, generator=g), torch.rand(3, 16, 20, 3, generator=g)
    (loss, labs), (d, dabs) = l2_ref(pred, gt, 0.125)
    l32, d32 = l2_fp32(pred, gt, 0.125)
    assert max_rel(l32, loss, labs) <= TAU / 4 and max_rel(d32, d, dabs) <= ELEM_BAR / 4
    assert max_rel(l2_fp32(pred, gt, 0.125, factor=1.0)[1], d, dabs) >= 0.1
    # inputs 255 times too large
    assert max_rel(l2_fp32(pred * 255, gt * 255, 0.125)[0], loss, labs) >= 1e3


def test_kmean_reference_passes_fp32_and_flags_k_minus_1():
    K = 6
    x = torch.randn(K * 2, 5, 7, 16, generator=torch.Generator().manual_seed(6))
    ref, absr = kmean_ref(x, K)
    assert max_rel(kmean_fp32(x, K), ref, absr) <= ELEM_BAR / 4
    assert max_rel(kmean_fp32(x, K, divisor=K - 1), ref, absr) >= 0.1
    # the last observation skipped
    assert max_rel(kmean_fp32(x[:(K - 1) * 2], K - 1) * f32((K - 1) / K), ref, absr) >= 1e-3


def _adam_state(n=4096, seed=7):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g) * 0.1
    return p, torch.zeros(n), torch.zeros(n), torch.zeros(n), g


def test_amsgrad_reference_passes_fp32_and_flags_wrong_step_and_rounded_betas():
    p, m, v, vh, gen = _adam_state()
    for t in (1, 2, 3):
        g = torch.randn(p.shape, generator=gen) * (1e-2 if t == 3 else 1.0)
        got = amsgrad_fp32(p, g, m, v, vh, t)
        r = amsgrad_r(got, p, g, m, v, vh, t)
        assert amsgrad_ok(r) and r['p'] <= ADAM_STEP_BAR / 4, (t, r)
        if t >= 2:       # step t - 1 / t + 1 (t - 1 = 0 gives lr_t = inf / nan)
            for tt in (t - 1, t + 1):
                assert amsgrad_r(amsgrad_fp32(p, g, m, v, vh, tt), p, g, m, v, vh, t)['p'] >= 1e3 * ADAM_STEP_BAR
        # (1 - beta) formed in fp64 from the exact decimals instead of the kernel's 1.f - b: v is off by
        # 2.1e-5 relative (1 - 0.999f vs 0.001) and flagged; m's 2.4e-7 is at its own bar and is not separable
        r64 = amsgrad_r(O.amsgrad_step(p.double(), g.double(), m.double(), v.double(), vh.double(), t, f32(LR)),
                        p, g, m, v, vh, t)
        assert r64['v'] >= 20 * ADAM_STATE_BAR and r64['m'] <= 2 * ADAM_STATE_BAR
        p, m, v, vh = got
    # both branches of max(vhat, v) were taken by step 3 (smaller gradients leave vhat > v)
    assert bool((vh > v).any()) and bool((vh == v).any())


def test_amsgrad_reference_at_a_large_step_count_and_tiny_gradients():
    p, m, v, vh, gen = _adam_state()
    m, v = torch.randn(p.shape, generator=gen) * 1e-3, torch.rand(p.shape, generator=gen) * 1e-6
    vh = v * 2
    g = torch.randn(p.shape, generator=gen)
    g[:64] = 0
    g[64:128] = 1e-30          # g * g underflows
    got = amsgrad_fp32(p, g, m, v, vh, 10 ** 5)
    assert amsgrad_ok(amsgrad_r(got, p, g, m, v, vh, 10 ** 5))


def test_u8_reference_flags_values_left_in_0_255():
    v = torch.arange(256, dtype=torch.uint8)
    ref = torch.tensor([f32(i / 255.0) for i in range(256)], dtype=torch.float32)
    assert torch.equal(v.double().div(255.0).float(), ref)
    assert not torch.equal(v.float(), ref)


# ----------------------------------------------------------------------------------------------------------------
# GPU: nlt_uv2cam_fwd
# ----------------------------------------------------------------------------------------------------------------
def _lib():
    import nlt_native as nat
    return nat, nat.lib()


def edge_warp(warp, W, H):
    """Overwrites rows 0-1 of image 0 with edge sample points, in pixels / (W, H) (exact in fp32 when W, H are powers
    of two; otherwise the reference reads the same fp32 products as the kernel)."""
    pts = [(0, 0), (1, 0), (0, 1), (5, 7), (W - 1, H - 1),                # exact integer texel coordinates
           (-0.5, 3), (3, -0.25), (-0.999, -0.5),                         # in (-1, 0)
           (W - 0.5, 3), (3, H - 0.125), (W - 0.001, H - 0.75),           # in (W - 1, W)
           (-1, 3), (3, -1), (W, 3), (3, H), (-1, -1), (W, H),            # exactly -1 / W: zero
           (-5, 3), (3, 1e6), (-1e30, 2), (W * 3, H * 3),                  # far outside
           (0.25, 0.25), (0.5, 0), (0, 0.5), (-0.5, -0.5), (0.999, 0.001), (1, 1), (-0.25, 0.75)]   # around (0,0)
    w = warp.clone()
    row = torch.tensor([[x / W, y / H] for x, y in pts], dtype=torch.float32)
    w[0, 0, :len(pts)] = row
    w[0, 1, :len(pts)] = row.flip(0)
    return w


def synth_tail(B, uv, cam, seed):
    """(base, warp, rgb_camspc) of bench's synthetic batch on the device; past 8 images the first 8 repeat (the host
    generator is slow at batch 32)."""
    from util import synth
    bt = synth.make_batch(min(B, 8), uv, cam, seed=seed)
    rep = lambda t: t.cuda().repeat((B + 7) // 8, 1, 1, 1)[:B].contiguous()
    return rep(bt[1]), rep(bt[4]), rep(bt[6])


def run_uv2cam_fwd(net, base, warp, rgb, skip=1):
    nat, lib = _lib()
    B, H, W, _ = net.shape
    ih, iw = warp.shape[1:3]
    dev = net.device
    pred_uv = torch.full((B, H, W, 3), float('nan'), device=dev)
    out = {k: torch.full((B, ih, iw, 3), float('nan'), device=dev) for k in ('pred', 'base', 'fg', 'gt')}
    nat.check(lib.nlt_uv2cam_fwd(nat.ptr(net), nat.ptr(base), nat.ptr(warp), nat.ptr(rgb), B, H, W, ih, iw, skip,
                                 nat.ptr(pred_uv), nat.ptr(out['pred']), nat.ptr(out['base']), nat.ptr(out['fg']),
                                 nat.ptr(out['gt']), nat.stream()))
    return pred_uv, out


FWD_CASES = [(8, 1024, 1024), (32, 1024, 1024), (2, 1024, 768), (2, 512, 1000)]


@pytest.mark.gpu
@pytest.mark.parametrize('B,uv,cam', FWD_CASES, ids=['b%d_uv%d_cam%d' % c for c in FWD_CASES])
def test_uv2cam_fwd_at_production_shape_and_edges(B, uv, cam):
    dev = torch.device('cuda')
    t0 = time.perf_counter()
    base, warp, rgb = synth_tail(B, uv, cam, 21)
    warp = edge_warp(warp, uv, uv)
    net = torch.randn(B, uv, uv, 3, device=dev, generator=torch.Generator(dev).manual_seed(22))
    stats = {}
    for skip in (1, 0):
        pred_uv, out = run_uv2cam_fwd(net, base, warp, rgb, skip)
        want = corner0(net + base if skip else net)            # fp32 sum, texel (0,0) multiplied by 0
        assert torch.equal(pred_uv, want), 'pred_uv (skip %d) differs from net_out + base at %s' % (
            skip, (pred_uv != want).nonzero()[:4].tolist())
        ref = uv2cam_ref(pred_uv, base, warp, rgb)
        for k in ('pred', 'base', 'fg', 'gt'):
            check('%s_skip%d' % (k, skip), out[k], ref[k][0], ref[k][1], ELEM_BAR, out=stats)
    # the edge rows: exactly -1 / W and far-outside points give exact zeros, through the same metric (tiny = TINY)
    n_zero = int((ref['fg'][0][0, :2] == 0).all(-1).sum())
    assert n_zero >= 2 * 13, n_zero
    _record('tail_uv2cam_fwd_b%d_uv%d_cam%d' % (B, uv, cam), {'r': stats, 'bar': ELEM_BAR, 'exact_zero_points': n_zero,
                                                              'seconds': time.perf_counter() - t0})


# ----------------------------------------------------------------------------------------------------------------
# GPU: nlt_uv2cam_bwd_det
# ----------------------------------------------------------------------------------------------------------------
def run_bwd_det(d, warp, H, W, ws=None):
    nat, lib = _lib()
    B, ih, iw, _ = d.shape
    need = lib.nlt_uv2cam_bwd_workspace_bytes(B, H, W)
    if ws is None:
        ws = torch.zeros((need + 7) // 8, dtype=torch.int64, device=d.device)
    g = torch.full((B, H, W, 3), float('nan'), device=d.device)
    nat.check(lib.nlt_uv2cam_bwd_det(nat.ptr(d), nat.ptr(warp), B, H, W, ih, iw, nat.ptr(g), ws.data_ptr(),
                                     nat.stream()))
    return g, ws


def _bwd_case(case, dev):
    """(d, warp, uv) of one named case."""
    from util import synth
    gen = torch.Generator(dev).manual_seed(31)
    if case in ('synth_b8', 'synth_b32'):
        B = 8 if case == 'synth_b8' else 32
        return torch.randn(B, 1024, 1024, 3, device=dev, generator=gen), synth_tail(B, 1024, 1024, 1235)[1], 1024
    if case == 'magnify4':           # 256^2 UV from a 1024^2 camera: lanes hand over both right taps
        bt = synth.make_batch(2, 256, 1024, seed=32, device='cuda')
        return torch.randn(2, 1024, 1024, 3, device=dev, generator=gen), bt[4], 256
    if case == 'one_texel':          # every pixel of image 0 on one interior texel: 2^20 contributions per tap
        bt = synth.make_batch(2, 1024, 1024, seed=33, device='cuda')
        warp = bt[4].clone()
        warp[0] = torch.tensor([100.25 / 1024, 200.5 / 1024], device=dev)
        d = torch.randn(2, 1024, 1024, 3, device=dev, generator=gen)
        d[0] = d[0].abs()              # one sign: the texel's sum grows to ~2^19 max|d|
        return d, warp, 1024
    if case == 'odd_33':             # B * ih * iw = 3 * 1089: image boundaries inside a warp, a partial last warp
        bt = synth.make_batch(3, 64, 33, seed=34, device='cuda')
        return torch.randn(3, 33, 33, 3, device=dev, generator=gen), bt[4], 64
    bt = synth.make_batch(2, 256, 256, seed=35, device='cuda')
    d = torch.randn(2, 256, 256, 3, device=dev, generator=gen)
    if case == 'one_huge':
        d *= 2.0 ** -20
        d[1, 100, 100, 1] = 1.5
    elif case == 'gmax_pow2':
        d = d / d.abs().max() * 0.5
        d[0, 7, 9, 2] = -0.5
        d[1, 50, 60, 0] = 0.5
    elif case == 'gmax_subnormal':
        d = (d / d.abs().max() * 2.0 ** -130).float()
        assert float(d.abs().max()) < 2.0 ** -126 and float(d.abs().max()) > 0
    elif case == 'zeros':
        d.zero_()
    return d, bt[4], 256


BWD_CASES = ['synth_b8', 'synth_b32', 'magnify4', 'one_texel', 'odd_33', 'one_huge', 'gmax_pow2', 'gmax_subnormal',
             'zeros']


@pytest.mark.gpu
@pytest.mark.parametrize('case', BWD_CASES)
def test_uv2cam_bwd_det_against_fp64_pullback(case):
    dev = torch.device('cuda')
    t0 = time.perf_counter()
    d, warp, uv = _bwd_case(case, dev)
    g1, ws = run_bwd_det(d, warp, uv, uv)
    torch.cuda.synchronize()
    acc = ws[32:]                   # behind the 256-byte max slot: the fixed-point accumulator
    assert int(acc.count_nonzero()) == 0, 'accumulator not re-zeroed: %d words left' % int(acc.count_nonzero())
    g2, _ = run_bwd_det(d, warp, uv, uv, ws)
    assert torch.equal(g1, g2), 'two calls differ at %s' % (g1 != g2).nonzero()[:4].tolist()
    if case == 'zeros':
        assert int(g1.count_nonzero()) == 0 and not bool(g1.isnan().any())
        _record('tail_uv2cam_bwd_%s' % case, {'r': 0.0})
        return
    # the fixed-point sum is exact integer arithmetic on the fp32 products: the emulation reproduces it bit for bit
    emu = uv2cam_bwd_fixed32(d, warp, uv, uv)
    assert torch.equal(g1, emu), 'differs from the fixed-point emulation at %s' % (g1 != emu).nonzero()[:4].tolist()
    del emu
    gmax = float(d.abs().max())
    tiny = scatter_floor(gmax)
    rec = {}
    for i0 in range(0, d.shape[0], 8):            # fp64 pullbacks in slices of 8 images
        sl = slice(i0, i0 + 8)
        ref, absr = uv2cam_bwd_ref(d[sl], warp[sl], uv, uv)
        r = check('d_net_out[%d:]' % i0, g1[sl], ref, absr, TAU, tiny)
        rec['r'] = max(rec.get('r', 0.0), r)
        del ref, absr
    rec.update({'bar': TAU, 'tiny': tiny, 'gmax': gmax, 'seconds': time.perf_counter() - t0})
    _record('tail_uv2cam_bwd_%s' % case, rec)


# ----------------------------------------------------------------------------------------------------------------
# GPU: nlt_l2_loss
# ----------------------------------------------------------------------------------------------------------------
def run_l2(pred, gt, B, per, scale):
    nat, lib = _lib()
    ws = torch.full(((lib.nlt_l2_loss_workspace_bytes(B, per) + 3) // 4,), float('nan'), device=pred.device)
    loss = torch.full((B,), float('nan'), device=pred.device)
    d = torch.full((B * per,), float('nan'), device=pred.device)
    nat.check(lib.nlt_l2_loss(nat.ptr(pred), nat.ptr(gt), B, per, scale, nat.ptr(loss), nat.ptr(d), nat.ptr(ws),
                              nat.stream()))
    return loss, d


L2_CASES = [(8, 3 << 20, 0), (32, 3 << 20, 0), (8, 3 << 20, 1), (8, (3 << 20) - 3, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize('B,per,off', L2_CASES, ids=['b8', 'b32', 'b8_offset1', 'b8_odd'])
def test_l2_loss_at_production_shape(B, per, off):
    """per-sample loss and d_pred at 3 * 1024^2 values per sample; pointers one float off 16 bytes and an odd
    per_sample run the scalar path at size."""
    dev = torch.device('cuda')
    gen = torch.Generator(dev).manual_seed(41)
    buf_p = torch.rand(B * per + 4, device=dev, generator=gen)
    buf_g = torch.rand(B * per + 4, device=dev, generator=gen)
    pred, gt = buf_p[off:off + B * per], buf_g[off:off + B * per]
    scale = 1.0 / B
    loss, d = run_l2(pred, gt, B, per, scale)
    (lr, la), (dr, da) = l2_ref(pred.view(B, per), gt.view(B, per), f32(scale))
    st = {}
    check('loss', loss, lr, la, TAU, out=st)
    check('d_pred', d.view(B, per), dr, da, ELEM_BAR, out=st)
    _record('tail_l2_b%d_per%d_off%d' % (B, per, off), {'r': st})


# ----------------------------------------------------------------------------------------------------------------
# GPU: nlt_kmean_fwd / nlt_kmean_bwd at cfg3's level-0 observation shape (K = 6, B = 16, 1024^2 x 16: 6.4 GB)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_kmean_at_cfg3_level0_shape():
    nat, lib = _lib()
    dev = torch.device('cuda')
    K, B, H, C = 6, 16, 1024, 16
    per = H * H * C
    gen = torch.Generator(dev).manual_seed(51)
    x = torch.randn(K * B, H, H, C, device=dev, generator=gen)
    assert x.numel() * 4 > 2 ** 32
    w = torch.rand(B, K, device=dev, generator=gen) + 0.5
    imgs = [0, B - 1]
    st = {}
    for wt in (None, w):
        out = torch.full((B, H, H, C), float('nan'), device=dev)
        nat.check(lib.nlt_kmean_fwd(nat.ptr(x), nat.ptr(wt), K, B, per, nat.ptr(out), nat.stream()))
        ref, absr = kmean_ref(x.view(K, B, H, H, C)[:, imgs].reshape(K * 2, H, H, C), K,
                              None if wt is None else wt[imgs])
        check('fwd' + ('_w' if wt is not None else ''), out[imgs], ref, absr, ELEM_BAR, out=st)
        del out
    # backward: d_in = mask(y) * (beta * d_in + d_out * w / K), images {0, B-1} of every k
    d_out = torch.randn(B, H, H, C, device=dev, generator=gen)
    prev = torch.randn(K * B, H, H, C, device=dev, generator=gen)
    y = x                          # LeakyReLU mask from the observation activations
    for wt in (None, w):
        d_in = prev.clone()
        nat.check(lib.nlt_kmean_bwd(nat.ptr(d_out), nat.ptr(wt), K, B, per, 1.0, nat.ptr(y), nat.ACT_CODES['leakyrelu'], nat.ptr(d_in),
                                    nat.stream()))
        sel = [k * B + i for k in range(K) for i in imgs]
        wk = torch.ones(len(sel), device=dev, dtype=torch.float64) if wt is None else \
            torch.stack([wt[i, k] for k in range(K) for i in imgs]).double()
        g = d_out[imgs].double().repeat(K, 1, 1, 1) * wk.view(-1, 1, 1, 1) / K
        mask = torch.where(y[sel] > 0, 1.0, 0.3).double()
        ref = (g + prev[sel].double()) * mask
        absr = (g.abs() + prev[sel].double().abs()) * mask
        check('bwd_beta1_mask' + ('_w' if wt is not None else ''), d_in[sel], ref, absr, ELEM_BAR, out=st)
        del d_in
    _record('tail_kmean_cfg3_level0', {'r': st, 'bar': ELEM_BAR})


# ----------------------------------------------------------------------------------------------------------------
# GPU: nlt_amsgrad_step_dev
# ----------------------------------------------------------------------------------------------------------------
def amsgrad_param_count():
    """The largest flat parameter count among the benchmarked training arms (cfg3: depth 1024)."""
    import bench
    best = 0
    for name in ('cfg4', 'cfg2', 'cfg4k3', 'cfg3'):
        wl = bench.WORKLOADS[name]
        chans = O.model_channels(bench.oracle_cfg(wl), 5 + wl['c_extra'], 3)
        n = sum(k * k * cin * cout + cout for net in chans.values() for layer in net for _, cin, cout, k, _ in layer)
        best = max(best, n)
    return best


def run_amsgrad_dev(st, g, step_dev):
    nat, lib = _lib()
    p, m, v, vh = st
    nat.check(lib.nlt_amsgrad_step_dev(nat.ptr(p), nat.ptr(g), nat.ptr(m), nat.ptr(v), nat.ptr(vh), p.numel(),
                                       step_dev.data_ptr(), LR, B1, B2, EPS, 1.0, nat.stream()))


def _adam_grads(n, t, dev, gen):
    g = torch.randn(n, device=dev, generator=gen) * (1e-2 if t == 3 else 1e-1)
    g[:4096] = 0                                  # exactly zero
    g[4096:8192] = 1e-25                          # g * g underflows to zero in fp32
    return g


@pytest.mark.gpu
def test_amsgrad_dev_at_model_size_and_in_a_graph():
    dev = torch.device('cuda')
    n = amsgrad_param_count()
    gen = torch.Generator(dev).manual_seed(61)
    rec = {'n': n}
    for mode in ('eager', 'graph', 'step1e5'):
        p = torch.randn(n, device=dev, generator=gen) * 0.05
        if mode == 'step1e5':
            m = torch.randn(n, device=dev, generator=gen) * 1e-3
            v = torch.rand(n, device=dev, generator=gen) * 1e-4
            vh = v * torch.where(torch.rand(n, device=dev, generator=gen) < 0.5, 2.0, 1.0)
        else:
            m, v, vh = (torch.zeros(n, device=dev) for _ in range(3))
        state = [p, m, v, vh]
        t0 = 10 ** 5 if mode == 'step1e5' else 0
        step_dev = torch.full((1,), t0, dtype=torch.int32, device=dev)
        gbuf = torch.zeros(n, device=dev)
        graph = None
        if mode == 'graph':
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                run_amsgrad_dev(state, gbuf, step_dev)
        branches = None
        for t in range(t0 + 1, t0 + 4):
            gbuf.copy_(_adam_grads(n, t - t0, dev, gen))
            before = [x.clone() for x in state]
            if graph is not None:
                graph.replay()
            else:
                run_amsgrad_dev(state, gbuf, step_dev)
            torch.cuda.synchronize()
            assert int(step_dev) == t, (mode, int(step_dev), t)
            r = amsgrad_r(state, before[0], gbuf, before[1], before[2], before[3], t)
            rec['%s_t%d' % (mode, t)] = r
            assert amsgrad_ok(r), (mode, t, r)
            vi = before[2].double() + (gbuf.double() ** 2 - before[2].double()) * (1 - f32(B2))
            branches = {'vhat_kept': int((before[3].double() > vi).sum()), 'v_taken': int((before[3].double() <= vi).sum())}
        rec[mode + '_branches'] = branches
        assert branches['vhat_kept'] > 0 and branches['v_taken'] > 0, (mode, branches)
        del state, p, m, v, vh, gbuf
    _record('tail_amsgrad_dev', rec)


# ----------------------------------------------------------------------------------------------------------------
# GPU: nlt_u8_to_f32
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('base_len', [0, 4096, 1 << 22])
def test_u8_to_f32_all_values_and_tails(base_len):
    nat, lib = _lib()
    dev = torch.device('cuda')
    want_tab = torch.tensor([f32(i / 255.0) for i in range(256)], dtype=torch.float32, device=dev)
    for r in range(1, 18):           # lengths 1 .. 17 modulo 16 on top of base_len
        n = base_len + r + 256
        src = (torch.arange(n, device=dev) * 7 + r).remainder(256).to(torch.uint8)
        out = torch.full((n,), float('nan'), device=dev)
        nat.check(lib.nlt_u8_to_f32(src.data_ptr(), n, nat.ptr(out), nat.stream()))
        want = want_tab[src.long()]
        assert torch.equal(out, want), (n, (out != want).nonzero()[:4].tolist())
