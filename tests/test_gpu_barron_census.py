"""The Barron training loss (`loss = barron`, csrc/nlt_barron.cu) against fp64, element by element, at the shapes the
shipped configs and the benchmarked workloads train at, on the data a model produces, and at the edges of the wavelet
pyramid.  tests/test_gpu_barron.py stays as it is: it is the comparison with the pinned oracle at its own tolerance.

Metric: r = |got - ref| / (abs_ref + tiny) per element, as in tests/test_gpu_census.py (max_rel); the worst element is
reported.  ref is oracle/barron_oracle.py in float64 on the kernel's own fp32 inputs, one sample at a time.
 * d_pred: ref by autograd through the oracle; abs_ref = |alpha| |M|^T |W|^T |g| (BO.image_nll_abs_grad): the chain
   with every filter tap, matrix entry and per-coefficient Charbonnier gradient g in magnitude.  Bar GRAD_BAR.
 * loss: the data term D_b = mean over the coefficients of sqrt(z^2 + 1) - 1, z = w / scale.  The reported loss is
   D_b + log(scale) + log Z, and at scale 0.01 the constant (-3.42) holds every bit of an fp32 loss that a converged
   model's D_b (~1e-5 .. 1e-4) would need: one rounding of the loss is 2.4e-7 absolute.  So D_b is read from a second
   call with log_z = -logf(scale), which makes the kernel's constant exactly 0; the regular call must equal that
   value plus the constant as one fp32 addition, bit for bit.  r = |D_got - D_ref| / D_ref, bar DATA_BAR.

Bars come from fp32 controls on the CPU, not from the GPU: tests/barron_host_check.cpp (the kernels' per-element code,
nlt_barron_core.h, run in host loops with a double-precision loss sum) meets them at 2 x 512^2, at odd sizes and at every
level count, and the seeded mistakes below (fp32 variants of the oracle arithmetic) fail them.
 * DATA_BAR = 2^-20.  Each term is a handful of roundings; a block adds 512 of them in fp32 (log2 512 = 9 levels of
   shuffles) and everything after that is double.  The naive form sqrtf(z^2 + 1) - 1 loses 5e-4 of D on the converged
   family; a random-order fp32 sum of the per-block partials (what float atomics did) loses ~1e-6 at 1024^2.
 * GRAD_BAR = 2^-16.  Ten filter passes forward and ten adjoint passes back at five levels, each a 7- or 9-tap fp32
   sum, around one Charbonnier gradient.
The host checker's worst over its cases is 1.5e-7 for the data term and 1.8e-6 for d_pred (the linear regime, where
every coefficient's gradient is near +-1 / scale and the adjoint sums do not shrink), 6x and 8x below the bars; the
seeded mistakes that break d_pred do so by 0.4 or more.
"""
import ctypes
import ctypes.util
import math
import os
import subprocess
import time

import numpy as np
import pytest
import torch

from oracle import barron_oracle as BO
from tests.test_gpu_census import CSRC, ROOT, _record, max_rel
from tests.test_gpu_tail_ops import check

LOG_Z = 1.185495232349193            # losses.Barron.LOG_Z_ALPHA1
SCALE = 0.01
DATA_BAR = 2.0 ** -20
GRAD_BAR = 2.0 ** -16
NAN = float('nan')
BT = 256                             # threads per block of the kernels; a block adds 2 * BT terms at most

_LIBM = ctypes.CDLL(ctypes.util.find_library('m'))
_LIBM.logf.restype, _LIBM.logf.argtypes = ctypes.c_float, [ctypes.c_float]
LOGF_SCALE = _LIBM.logf(SCALE)                                 # logf(scale), as the entry point forms it
CONSTANT = float(np.float32(LOGF_SCALE) + np.float32(LOG_Z))   # logf(scale) + log_z in fp32: the loss of pred == gt
DATA_LOG_Z = -LOGF_SCALE                                       # makes that constant exactly 0


# ----------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------
FAMILIES = ['noisy', 'converged', 'large', 'zero', 'camera', 'mask', 'frac']


def islands(N, H, W, gen, device):
    """[N, H, W, 1] 0/1 foreground: two or three discs per sample, the rest exactly 0 (what uv2cam leaves outside
    the object)."""
    yy = torch.arange(H, device=device, dtype=torch.float32).view(H, 1)
    xx = torch.arange(W, device=device, dtype=torch.float32).view(1, W)
    out = torch.zeros(N, H, W, 1, device=device)
    for n in range(N):
        c = torch.rand(3, 3, generator=gen, device=device)
        for k in range(2 + n % 2):
            cy, cx, r = float(c[k, 0]) * H, float(c[k, 1]) * W, (0.15 + 0.2 * float(c[k, 2])) * min(H, W)
            out[n, ..., 0] += (((yy - cy) ** 2 + (xx - cx) ** 2) < r * r).float()
    return out.clamp(max=1)


def make_case(family, N, H, W, seed, device='cpu'):
    """fp32 (pred, gt, alpha or None) of one data family.
    noisy: pred = gt + 0.03 N(0, 1) (|z| ~ 3, the middle of the Charbonnier curve);  converged: + 1e-4 N(0, 1) (|z| ~ 1e-2,
    the quadratic regime);  large: + N(0, 1) (|z| ~ 100, the linear regime);  zero: pred == gt;  camera: noisy inside
    foreground islands, both images exactly 0 outside;  mask: noisy, alpha a 0/1 island mask;  frac: noisy, alpha a
    fractional map with exact 0s and 1s."""
    gen = torch.Generator(device).manual_seed(seed)
    gt = torch.rand(N, H, W, 3, generator=gen, device=device)
    noise = torch.randn(N, H, W, 3, generator=gen, device=device)
    alpha = None
    sigma = {'converged': 1e-4, 'large': 1.0, 'zero': 0.0}.get(family, 0.03)
    pred = gt + sigma * noise
    if family == 'zero':
        pred = gt.clone()
    elif family == 'camera':
        fg = islands(N, H, W, gen, device)
        gt, pred = gt * fg, pred * fg
    elif family == 'mask':
        alpha = islands(N, H, W, gen, device)
    elif family == 'frac':
        alpha = (1.5 * torch.rand(N, H, W, 1, generator=gen, device=device) - 0.25).clamp(0, 1)
    return pred.contiguous(), gt.contiguous(), None if alpha is None else alpha.contiguous()


def make_mixed(H, W, seed, device='cpu'):
    """One sample of every family in one batch (alpha 1 for the families without one)."""
    parts = [make_case(f, 1, H, W, seed + i, device) for i, f in enumerate(FAMILIES)]
    pred = torch.cat([p for p, _, _ in parts]).contiguous()
    gt = torch.cat([g for _, g, _ in parts]).contiguous()
    alpha = torch.cat([a if a is not None else torch.ones(1, H, W, 1, device=device) for _, _, a in parts]).contiguous()
    return pred, gt, alpha


# ----------------------------------------------------------------------------------------------------------------
# fp64 reference
# ----------------------------------------------------------------------------------------------------------------
def reference(pred, gt, alpha, levels, loss_scale):
    """fp32 inputs -> fp64 (D [N] data term, d_pred, abs_ref) on the inputs' device, one sample at a time (a whole
    16 x 1024^2 fp64 graph would take several GB)."""
    N, H, W, _ = pred.shape
    count = H * W * 3
    D = torch.empty(N, dtype=torch.float64, device=pred.device)
    dp = torch.empty(pred.shape, dtype=torch.float64, device=pred.device)
    ab = torch.empty_like(dp)
    for b in range(N):
        p = pred[b:b + 1].double().requires_grad_(True)
        res = gt[b:b + 1].double() - p
        a = None if alpha is None else alpha[b:b + 1].double()
        if a is not None:
            res = res * a
        x = BO.rgb_to_syuv(res).permute(0, 3, 1, 2).reshape(3, H, W)
        d = BO.charbonnier(BO.wavelet_flatten(BO.wavelet_construct(x, levels)), SCALE).sum() / count
        g, = torch.autograd.grad(d * loss_scale, p)
        D[b], dp[b] = d.detach(), g[0]
        absr = BO.image_nll_abs_grad(res.detach(), SCALE, levels, loss_scale / count)
        ab[b] = (absr if a is None else absr * a.abs())[0]
    return D, dp, ab


def data_r(got, D):
    """Relative error of the data term per sample (an exact 0 is asked of D = 0)."""
    return max_rel(got, D, D)


def max_levels(H, W):
    return BO.max_num_levels((1, H, W))


# ----------------------------------------------------------------------------------------------------------------
# fp32 emulations with seeded mistakes
# ----------------------------------------------------------------------------------------------------------------
def _decimate32(x, f, axis, shift, edge_repeat=False):
    """BO._filter_decimate in fp32; edge_repeat pads symmetrically (... x1 x0 | x0 x1 ...) instead of reflecting."""
    dim = axis + 1
    n = x.shape[dim]
    below, above = (len(f) - 1) // 2, len(f) // 2
    if edge_repeat:
        r = torch.remainder(torch.arange(-below, n + above), 2 * n)
        idx = torch.where(r < n, r, 2 * n - 1 - r)
    else:
        idx = BO.reflect_indices(n, below, above)
    xp = x.index_select(dim, idx)
    xp = xp.narrow(dim, shift, xp.shape[dim] - shift)
    return (xp.unfold(dim, len(f), 2) * f).sum(-1)


MISTAKES = ['hi_unshifted', 'edge_repeat', 'yuv_untransposed', 'alpha_dropped', 'naive_charbonnier']


def barron_f32(pred, gt, alpha, levels, loss_scale, mistake=None):
    """The kernels' computation in fp32 (the adjoint by fp32 autograd) -> (data term [N] as the kernel forms it,
    d_pred).  `mistake` switches in one of MISTAKES."""
    N, H, W, _ = pred.shape
    one = lambda v: torch.tensor(v, dtype=torch.float32)
    inv_scale = one(1.0) / one(SCALE)
    inv_count = one(1.0) / one(float(H * W * 3))
    res = gt - pred
    if alpha is not None:
        res = res * alpha
    x = BO.rgb_to_syuv(res).permute(0, 3, 1, 2).reshape(N * 3, H, W).detach().requires_grad_(True)
    lo, hi = BO.cdf97_analysis_filters(torch.float32)
    sh, er = (0 if mistake == 'hi_unshifted' else 1), mistake == 'edge_repeat'
    im, pyr = x, []
    for _ in range(levels):
        h, l = _decimate32(im, hi, 0, sh, er), _decimate32(im, lo, 0, 0, er)
        pyr.append((_decimate32(h, hi, 1, sh, er), _decimate32(l, hi, 1, sh, er), _decimate32(h, lo, 1, 0, er)))
        im = _decimate32(l, lo, 1, 0, er)
    pyr.append(im)
    flat = BO.wavelet_flatten(tuple(pyr))
    z = flat.detach() * inv_scale
    z2 = z * z
    ch = torch.sqrt(z2 + 1) - 1 if mistake == 'naive_charbonnier' else z2 / (torch.sqrt(z2 + 1) + 1)
    data = (ch.reshape(N, -1).double().sum(1) * float(inv_count)).float()
    g = (one(loss_scale) * inv_count) * (z * inv_scale / torch.sqrt(z2 + 1))
    gx, = torch.autograd.grad(flat, x, g)
    gy = gx.reshape(N, 3, H, W).permute(0, 2, 3, 1)
    m = torch.tensor(BO._YUV_FROM_RGB, dtype=torch.float32)
    d_rgb = one(BO.SYUV_SCALE) * (gy @ (m if mistake == 'yuv_untransposed' else m.t()))
    if alpha is not None and mistake != 'alpha_dropped':
        d_rgb = alpha * d_rgb
    return data, -d_rgb


def block_partials32(pred, gt, levels):
    """Per-block fp32 partials of sample 0's Charbonnier terms, 2 * BT consecutive terms each, as the loss-producing
    launches form them (stable form)."""
    _, H, W, _ = pred.shape
    x = BO.rgb_to_syuv(gt[:1].double() - pred[:1].double()).permute(0, 3, 1, 2).reshape(3, H, W)
    w = BO.wavelet_flatten(BO.wavelet_construct(x, levels)).float().reshape(-1)
    z = w * (torch.tensor(1.0) / torch.tensor(SCALE))
    ch = (z * z / (torch.sqrt(z * z + 1) + 1)).numpy()
    pad = (-ch.size) % (2 * BT)
    return np.concatenate([ch, np.zeros(pad, np.float32)]).reshape(-1, 2 * BT).astype(np.float64).sum(1)


def atomic_order_sum(partials, seed):
    """fp32 running sum of the partials in a random order: what one float atomic per block gives."""
    p = partials.astype(np.float32)[np.random.default_rng(seed).permutation(partials.size)]
    return float(np.add.accumulate(p, dtype=np.float32)[-1])


# ----------------------------------------------------------------------------------------------------------------
# CPU: the host checker meets the bars; the seeded mistakes fail them
# ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp('barron_census') / 'barron_host_check.so')
    subprocess.check_call(['g++', '-O2', '-shared', '-fPIC', '-std=c++17', '-I', CSRC, '-o', so,
                           os.path.join(ROOT, 'tests', 'barron_host_check.cpp')])
    lib = ctypes.CDLL(so)
    fp = ctypes.POINTER(ctypes.c_float)
    lib.barron_host.restype = ctypes.c_int
    lib.barron_host.argtypes = [fp, fp, fp] + [ctypes.c_int32] * 4 + [ctypes.c_float] * 3 + [fp, fp]
    return lib


def run_host(lib, pred, gt, alpha, levels, loss_scale, log_z):
    P = lambda t: None if t is None else t.numpy().ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    N, H, W, _ = pred.shape
    loss = torch.full((N,), NAN)
    d = torch.full_like(pred, NAN)
    assert lib.barron_host(P(pred), P(gt), P(alpha), N, H, W, levels, SCALE, log_z, loss_scale, P(loss), P(d)) == 0
    return loss, d


def host_r(lib, pred, gt, alpha, levels, loss_scale=0.25):
    """(r of the data term, r of d_pred) of the host checker; also its loss = data term + constant in one fp32 add."""
    loss_d, d = run_host(lib, pred, gt, alpha, levels, loss_scale, DATA_LOG_Z)
    loss_f, _ = run_host(lib, pred, gt, alpha, levels, loss_scale, LOG_Z)
    assert torch.equal(loss_f, loss_d + torch.tensor(CONSTANT))
    D, ref, absr = reference(pred, gt, alpha, levels, loss_scale)
    return data_r(loss_d, D), max_rel(d, ref, absr)


HOST_CASES = ([(2, 512, 512, 5, f) for f in ('noisy', 'converged', 'large', 'camera', 'frac')]
              + [(s[0], s[1], s[2], 5, f) for s in ((3, 33, 17), (5, 83, 71)) for f in FAMILIES]
              + [(3, h, w, lv, f) for h, w in ((17, 40), (33, 17), (5, 7), (2, 2))
                 for lv in range(1, max_levels(h, w) + 1) for f in ('noisy', 'converged')])


def _case_id(c):
    return '%dx%dx%d_l%d_%s' % c


@pytest.mark.parametrize('case', HOST_CASES, ids=_case_id)
def test_host_checker_meets_the_bars(host, case):
    N, H, W, levels, family = case
    pred, gt, alpha = make_case(family, N, H, W, seed=H * 7 + W + levels)
    rd, rg = host_r(host, pred, gt, alpha, levels)
    assert rd <= DATA_BAR and rg <= GRAD_BAR, (rd, rg)


def test_host_checker_on_a_mixed_batch(host):
    pred, gt, alpha = make_mixed(33, 17, seed=5)
    rd, rg = host_r(host, pred, gt, alpha, 5)
    assert rd <= DATA_BAR and rg <= GRAD_BAR, (rd, rg)


@pytest.mark.parametrize('family', ['noisy', 'converged', 'frac'])
def test_fp32_emulation_meets_the_bars(family):
    """The emulation the mistakes are seeded into is itself within the bars when nothing is wrong."""
    pred, gt, alpha = make_case(family, 2, 64, 48, seed=3)
    D, ref, absr = reference(pred, gt, alpha, 5, 0.25)
    data, d = barron_f32(pred, gt, alpha, 5, 0.25)
    assert data_r(data, D) <= DATA_BAR and max_rel(d, ref, absr) <= GRAD_BAR


@pytest.mark.parametrize('mistake', MISTAKES)
def test_seeded_mistakes_fail_the_bars(mistake):
    family = {'alpha_dropped': 'frac', 'naive_charbonnier': 'converged'}.get(mistake, 'noisy')
    pred, gt, alpha = make_case(family, 2, 64, 64, seed=4)
    D, ref, absr = reference(pred, gt, alpha, 5, 0.25)
    data, d = barron_f32(pred, gt, alpha, 5, 0.25, mistake)
    rd, rg = data_r(data, D), max_rel(d, ref, absr)
    if mistake == 'naive_charbonnier':
        assert rd >= 100 * DATA_BAR, rd             # the gradient does not cancel and stays within its bar
        assert rg <= GRAD_BAR, rg
    else:
        assert rg >= 100 * GRAD_BAR, rg


def test_naive_charbonnier_loses_the_converged_data_term_at_production_size():
    pred, gt, _ = make_case('converged', 1, 512, 512, seed=6)
    D = reference(pred, gt, None, 5, 1.0)[0]
    data, _ = barron_f32(pred, gt, None, 5, 1.0, 'naive_charbonnier')
    assert data_r(data, D) >= 100 * DATA_BAR
    data, _ = barron_f32(pred, gt, None, 5, 1.0)
    assert data_r(data, D) <= DATA_BAR / 4


def test_random_order_fp32_sum_of_block_partials_fails_the_data_bar_at_1024():
    """The per-sample sum the kernel made with one float atomic per block: at 1024^2 its order-dependent error is about
    the size of DATA_BAR; the worst of eight orders fails it, the fixed-order double sum passes with room."""
    pred, gt, _ = make_case('noisy', 1, 1024, 1024, seed=8)
    inv_count = float(np.float32(1.0) / np.float32(3 * 1024 * 1024))
    parts = block_partials32(pred, gt, 5)
    assert parts.size >= 6000
    D = float(reference(pred, gt, None, 5, 1.0)[0][0])
    fixed = abs(float(np.float32(parts.sum() * inv_count)) - D) / D
    orders = [abs(float(np.float32(atomic_order_sum(parts, s)) * np.float32(inv_count)) - D) / D for s in range(8)]
    assert fixed <= DATA_BAR / 4, fixed
    assert max(orders) >= DATA_BAR, orders


def test_workspace_query_refuses_what_the_entry_point_refuses():
    import nlt_native as nat
    lib = nat.lib()
    for args in ((1, 32, 32, 0), (1, 32, 32, 13), (1, 32, 32, 6), (0, 32, 32, 5), (65536, 32, 32, 1), (1, 1, 32, 1),
                 (1, 2, 2, 2), (-1, 32, 32, 5)):
        assert lib.nlt_barron_loss_workspace_bytes(*args) < 0, args
    for args in ((1, 2, 2, 1), (65535, 2, 2, 1), (16, 1024, 1024, 5), (3, 5, 7, 3)):
        need = lib.nlt_barron_loss_workspace_bytes(*args)
        B, H, W = args[:3]
        assert need > 4 * 3 * B * H * W * 2 and need % 8 == 0, (args, need)


# ----------------------------------------------------------------------------------------------------------------
# GPU: direct C-ABI calls
# ----------------------------------------------------------------------------------------------------------------
GUARD = 4096                          # floats behind the workspace that no kernel may touch
GUARD_VALUE = 12345.0
RECORD = {'bars': {'data': DATA_BAR, 'd_pred': GRAD_BAR}}


def note(key, rec):
    RECORD[key] = rec
    _record('barron', RECORD)


def _lib():
    import nlt_native as nat
    return nat, nat.lib()


def guarded_workspace(N, H, W, levels, device, fill=NAN):
    _, lib = _lib()
    need = lib.nlt_barron_loss_workspace_bytes(N, H, W, levels)
    assert need > 0 and need % 4 == 0, need
    buf = torch.full((need // 4 + GUARD,), fill, device=device)
    buf[need // 4:] = GUARD_VALUE
    return buf, need // 4


def run_kernel(pred, gt, alpha, levels, loss_scale, log_z=LOG_Z, grad=True, ws=None):
    nat, lib = _lib()
    N, H, W, _ = pred.shape
    buf, n = guarded_workspace(N, H, W, levels, pred.device) if ws is None else ws
    loss = torch.full((N,), NAN, device=pred.device)
    d = torch.full_like(pred, NAN) if grad else None
    nat.check(lib.nlt_barron_loss(nat.ptr(pred), nat.ptr(gt), nat.ptr(alpha), N, H, W, levels, SCALE, log_z,
                                  loss_scale, nat.ptr(loss), nat.ptr(d), nat.ptr(buf), nat.stream()))
    torch.cuda.synchronize()
    assert bool((buf[n:] == GUARD_VALUE).all()), 'nlt_barron_loss wrote behind its workspace'
    return loss, d


def gpu_case(pred, gt, alpha, levels, loss_scale, families=None):
    """Both calls (constant 0 and the regular one) against fp64 -> record {'data': r, 'd_pred': r, ...}; asserts."""
    loss_d, d = run_kernel(pred, gt, alpha, levels, loss_scale, DATA_LOG_Z)
    loss, d2 = run_kernel(pred, gt, alpha, levels, loss_scale)
    assert torch.equal(d, d2), 'd_pred depends on log_z'
    assert torch.equal(loss, loss_d + CONSTANT), 'loss != data term + constant in one fp32 addition'
    D, ref, absr = reference(pred, gt, alpha, levels, loss_scale)
    N = pred.shape[0]
    rec = {'data': 0.0, 'd_pred': 0.0, 'D': [float(v) for v in D]}
    errors = []
    for b in range(N):
        tag = '' if families is None else ' (%s)' % families[b]
        rd = data_r(loss_d[b:b + 1], D[b:b + 1])
        rec['data'] = max(rec['data'], rd)
        if rd > DATA_BAR:
            errors.append('data term[%d]%s: r = %.3g (got %r, want %r)' % (b, tag, rd, float(loss_d[b]), float(D[b])))
        try:
            rec['d_pred'] = max(rec['d_pred'], check('d_pred[%d]%s' % (b, tag), d[b], ref[b], absr[b], GRAD_BAR))
        except AssertionError as e:
            rec['d_pred'] = max(rec['d_pred'], max_rel(d[b], ref[b], absr[b]))
            errors.append(str(e))
    if alpha is not None:
        dead = (alpha == 0).expand_as(d)
        rec['alpha0_elems'] = int(dead.sum())
        if not bool((d[dead] == 0).all()):
            errors.append('d_pred not exactly 0 where alpha == 0')
    for b in range(N):
        if float(D[b]) == 0.0:          # pred == gt (or masked out): the constant, and no gradient at all
            if not (float(loss[b]) == CONSTANT and int(d[b].count_nonzero()) == 0):
                errors.append('sample %d: zero residual gave loss %r, %d nonzero d_pred' % (
                    b, float(loss[b]), int(d[b].count_nonzero())))
    return rec, errors


SHAPES = {(4, 512, 512): FAMILIES,                               # dragon_specular / dragon_sss: batch 4, 512^2
          (8, 1024, 1024): ['noisy', 'converged', 'camera'],     # cfg2 / cfg4 camera images
          (16, 1024, 1024): ['noisy', 'converged'],              # cfg3
          (2, 512, 384): FAMILIES, (2, 384, 512): FAMILIES,
          (3, 33, 17): FAMILIES, (5, 83, 71): FAMILIES}
CASES = [(s, f) for s, fams in SHAPES.items() for f in fams]


@pytest.mark.gpu
@pytest.mark.parametrize('shape,family', CASES, ids=lambda v: 'x'.join(map(str, v)) if isinstance(v, tuple) else v)
def test_barron_at_shape(shape, family):
    N, H, W = shape
    dev = torch.device('cuda')
    t0 = time.perf_counter()
    pred, gt, alpha = make_case(family, N, H, W, seed=N * 1000 + H + W, device=dev)
    if family == 'zero':
        assert torch.equal(pred, gt)
    rec, errors = gpu_case(pred, gt, alpha, 5, 1.0 / N)
    rec['seconds'] = time.perf_counter() - t0
    note('%dx%dx%d %s' % (N, H, W, family), rec)
    assert not errors, '\n'.join(errors)


LEVEL_CASES = [(h, w, lv, f) for h, w in ((17, 40), (33, 17), (5, 7), (2, 2))
               for lv in range(1, max_levels(h, w) + 1) for f in ('noisy', 'converged', 'frac')]


@pytest.mark.gpu
@pytest.mark.parametrize('H,W,levels,family', LEVEL_CASES)
def test_barron_at_every_level_count(H, W, levels, family):
    """The deepest levels run on axes of length 2 and 3, where the reflecting boundary wraps more than once."""
    pred, gt, alpha = make_case(family, 3, H, W, seed=H * 50 + W + levels, device=torch.device('cuda'))
    rec, errors = gpu_case(pred, gt, alpha, levels, 0.5)
    note('%dx%d levels %d %s' % (H, W, levels, family), rec)
    assert not errors, '\n'.join(errors)


@pytest.mark.gpu
@pytest.mark.parametrize('H,W', [(33, 17), (83, 71), (512, 384)])
def test_barron_on_a_mixed_batch(H, W):
    """One sample per family in one launch: no sample's sum may pick up another's coefficients across a warp or
    block boundary (the zero sample must give the constant exactly)."""
    pred, gt, alpha = make_mixed(H, W, seed=H + W, device=torch.device('cuda'))
    rec, errors = gpu_case(pred, gt, alpha, 5, 0.125, families=FAMILIES)
    note('mixed %dx%d' % (H, W), rec)
    assert not errors, '\n'.join(errors)


@pytest.mark.gpu
@pytest.mark.parametrize('shape,family', [((3, 83, 71), 'frac'), ((4, 512, 512), 'noisy'),
                                          ((8, 1024, 1024), 'noisy')], ids=str)
def test_entry_point_contract(shape, family):
    """NaN-filled outputs and workspace, a canary behind the workspace (run_kernel), two identical calls bit-identical,
    a zeroed workspace bit-identical to a NaN-filled one, and d_pred = NULL leaves the loss bit-identical."""
    N, H, W = shape
    dev = torch.device('cuda')
    pred, gt, alpha = make_case(family, N, H, W, seed=11, device=dev)
    ws = guarded_workspace(N, H, W, 5, dev)
    loss1, d1 = run_kernel(pred, gt, alpha, 5, 0.25, ws=ws)
    loss2, d2 = run_kernel(pred, gt, alpha, 5, 0.25, ws=ws)                  # the workspace now holds the last call
    loss3, d3 = run_kernel(pred, gt, alpha, 5, 0.25, ws=guarded_workspace(N, H, W, 5, dev, fill=0.0))
    loss4, _ = run_kernel(pred, gt, alpha, 5, 0.0, grad=False)
    rec = {'loss_two_calls_equal': bool(torch.equal(loss1, loss2)),
           'loss_two_calls_max_abs_diff': float((loss1 - loss2).abs().max()),
           'd_pred_two_calls_equal': bool(torch.equal(d1, d2)),
           'zeroed_workspace_equal': bool(torch.equal(loss1, loss3) and torch.equal(d1, d3)),
           'no_grad_loss_equal': bool(torch.equal(loss1, loss4))}
    note('contract %dx%dx%d' % shape, rec)
    assert bool(torch.isfinite(loss1).all()) and bool(torch.isfinite(d1).all())
    assert all(v for k, v in rec.items() if k.endswith('equal')), rec


@pytest.mark.gpu
def test_refused_arguments_leave_the_outputs_untouched():
    nat, lib = _lib()
    dev = torch.device('cuda')
    pred, gt, _ = make_case('noisy', 2, 32, 32, seed=1, device=dev)
    ws = torch.full((1 << 20,), NAN, device=dev)
    loss, d = torch.full((2,), NAN, device=dev), torch.full_like(pred, NAN)
    P = nat.ptr

    def call(B=2, levels=5, scale=SCALE, p=pred, g=gt, lo=loss, w=ws):
        return lib.nlt_barron_loss(P(p), P(g), None, B, 32, 32, levels, scale, LOG_Z, 1.0, P(lo), P(d), P(w),
                                   nat.stream())

    for kw in (dict(levels=0), dict(levels=13), dict(levels=6), dict(B=0), dict(scale=0.0), dict(scale=-0.01),
               dict(scale=NAN), dict(p=None), dict(g=None), dict(lo=None), dict(w=None)):
        rc = call(**kw)
        assert rc < 0, (kw, rc)
        assert lib.nlt_last_error()
    torch.cuda.synchronize()
    assert bool(loss.isnan().all()) and bool(d.isnan().all()) and bool(ws.isnan().all())


# ----------------------------------------------------------------------------------------------------------------
# GPU: in the model
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_barron_in_a_training_step_at_the_shipped_shape():
    """One eager training step with `loss = barron` at dragon_specular's shape (UV and camera 512^2, batch 4, depth
    256): the model's own pred_camspc / gt_camspc (foreground islands on an exact-zero background) and the d_pred that
    losses.Barron produced, with the model's grad_scale = 1 / B (keep_batch), against fp64."""
    import models
    from oracle import nlt_oracle as O
    from util import io as ioutil, synth
    B, S = 4, 512
    dev = torch.device('cuda')
    cfg = ioutil.make_config(uvh=S, uvw=S, imh=S, imw=S, loss='barron', depth0=16, depth=256, kernel=2, stride=2)
    oc = dict(depth0=16, depth=256, kernel=2, stride=2, norm='None', act='leakyrelu', pool='None', use_obs=True,
              skip_connect_base=True, imh=S, imw=S, uvh=S, uvw=S)
    model = models.get_model_class('nlt')(cfg)
    model.register_trainable()
    model.build(5, 3)
    model.load_params(O.init_params(oc, seed=7, dtype=torch.float64))
    bt = synth.make_batch(B, S, S, seed=21)
    pred, gt, kw, _ = model(bt, mode='train')
    kw['keep_batch'] = True
    model.set_loss_grad_scale(1.0 / B)
    per = model.compute_loss(pred, gt, **kw)
    (_, barron), = model.wloss
    assert type(barron).__name__ == 'Barron' and barron.grad_scale == 1.0 / B
    d = barron.d_pred.clone()
    model.backward()
    torch.cuda.synchronize()
    D, ref, absr = reference(pred.to(dev), gt.to(dev), None, 5, 1.0 / B)
    rg = check('model d_pred', d, ref, absr, GRAD_BAR)
    c64 = math.log(SCALE) + LOG_Z
    # the reported loss: the fp32 constant plus D, rounded once more at |loss| ~ 3.4
    rl = float(((per.double() - (CONSTANT + D)).abs() / (D + 2.0 ** -22 * abs(c64))).max())
    fg = float((gt == 0).all(-1).double().mean())
    note('model dragon_specular', {'batch': B, 'd_pred': rg, 'loss_r': rl, 'D': [float(v) for v in D],
                                   'background_fraction': fg})
    assert rl <= 1.0, rl
    assert 0.0 < fg < 1.0, fg
