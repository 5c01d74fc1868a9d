"""`norm = pixel | instance` (csrc/nlt_norm.cu, engine.NormLayer) against fp64: the ops at the shapes a norm layer sees
in the benchmarked workloads and at their edges, the layers in place during one training step, and the graphed step.

Metric: r = |got - ref| / (abs_ref + tiny) per element, as in tests/test_gpu_census.py (max_rel): ref is the fp64 op on
the kernel's own fp32 operands, abs_ref the same expression with every term replaced by its magnitude, so a bar counts
fp32 roundings.

What is compared with what.
 * pixel norm, forward: y = act(x * rsqrt(mean_c x^2 + 1e-8)), abs_ref = |y| (a sum of squares does not cancel).
   Backward: dx_c = r dz_c - x_c r^3 <dz, x> / C, abs_ref = r |dz_c| + |x_c| r^3 <|dz|, |x|> / C.  Bar ELEM_BAR: a lane
   adds at most C / 4 / 32 * 4 = 192 squares at C = 6144, the butterfly five more, then one rsqrt and one product.
 * instance norm, statistics: `mean` and `rstd` (the side outputs of nlt_instnorm_fwd) against the fp64 two-pass mean and
   biased variance.  mean: abs_ref = mean |x|, ELEM_BAR.  rstd: abs_ref = rstd, RSTD_BAR (below).
 * instance norm, y and the backward pass are functions of (x, mean, rstd) as fp32 arguments -- nlt_instnorm_bwd takes
   them as such -- so their references are the fp64 formulas on those fp32 values: z = gamma (x - mean) rstd + beta with
   abs_ref = |gamma| |x - mean| rstd + |beta| (x - mean of two fp32 numbers is one rounding of its own magnitude; every
   activation is 1-Lipschitz, so abs_ref carries through it), ELEM_BAR;
   dx = gamma rstd (dz - mean dz - xhat mean(dz xhat)), abs_ref term by term, INST_DX_BAR; dgamma = sum dz xhat and
   dbeta = sum dz over up to 8 * 2^20 terms, TAU.  With the statistics held to their own bars this pins y end to end;
   y is also held against the all-fp64 formula with abs_ref = |gamma| (|x| + |mean|) rstd + |beta| at RSTD_BAR, which is
   what the fp32 `mean` (half an ulp of |mean|, not of std) allows.

RSTD_BAR.  The kernel centres every 1024-pixel chunk on the chunk's own fp32 mean and merges (count, mean, centred second
moment) over the chunks in double.  The centred squares are non-negative, so the second moment is a plain fp32 sum: a
thread adds ceil(1024 / rows) of them serially (rows = max(256 / C, 1): 64 terms at C = 16, 1024 at C >= 256) and `rows`
partials are added on top: expected error sqrt(1024) / 2 roundings = 2^-20 of the variance at the longest serial run,
half of that in rstd.  RSTD_BAR = 2^-18 leaves 8x, and holds at every mean / std: the shift removes the
(mean / std)^2 * 2^-24 that E[x^2] - mean^2 on raw fp32 sums loses (onepass_stats below emulates that form, in its
summation order, and fails the bar from mean / std = 30 on; it is the record of why the kernel changed).
INST_DX_BAR = 2^-18 for the same reason: dx contains two per-(sample, channel) means summed the same way.

The activation's derivative is applied by the consumer from the saved output; dz here is d(loss) / d(norm output)
already multiplied by it.
"""
import time

import pytest
import torch

from tests.test_gpu_census import TAU, _bias_init, _record, max_rel, poison_workspaces, poisoned_allocations
from tests.test_gpu_tail_ops import ELEM_BAR, check

RSTD_BAR = 2.0 ** -18
INST_DX_BAR = 2.0 ** -18
EPS_PIXEL, EPS_INSTANCE = 1e-8, 1e-6
IN_CHUNK = 1024                      # pixels per partial of the instance-norm reductions (nlt_norm.cu)
ACT_CODE = {None: 0, 'relu': 1, 'leakyrelu': 2, 'elu': 3}
NAN = float('nan')


# ----------------------------------------------------------------------------------------------------------------
# fp64 references
# ----------------------------------------------------------------------------------------------------------------
def act_of(z, act, slope=0.3):
    if act is None:
        return z
    if act == 'relu':
        return z.clamp(min=0)
    if act == 'leakyrelu':
        return torch.where(z > 0, z, slope * z)
    return torch.where(z > 0, z, torch.expm1(z))


def pixel_fwd_ref(x, act):
    """x [..., C] fp32 -> (y, |y|) in fp64."""
    xd = x.double()
    r = torch.rsqrt((xd * xd).mean(-1, keepdim=True) + EPS_PIXEL)
    y = act_of(xd * r, act)
    return y, y.abs()


def pixel_bwd_ref(x, dz):
    xd, dd = x.double(), dz.double()
    C = x.shape[-1]
    r = torch.rsqrt((xd * xd).mean(-1, keepdim=True) + EPS_PIXEL)
    s = (dd * xd).sum(-1, keepdim=True)
    sa = (dd.abs() * xd.abs()).sum(-1, keepdim=True)
    return r * dd - xd * r ** 3 * s / C, r * dd.abs() + xd.abs() * r ** 3 * sa / C


def inst_stats_ref(x):
    """x [HW, C] fp32 of one sample -> fp64 (mean, rstd, mean |x|, std), two-pass."""
    xd = x.double()
    mean = xd.mean(0)
    var = ((xd - mean) ** 2).mean(0)
    return mean, torch.rsqrt(var + EPS_INSTANCE), xd.abs().mean(0), var.sqrt()


def inst_apply_ref(x, gamma, beta, mean, rstd, act):
    """(y, abs_ref) of one sample x [HW, C] from the statistics as given (any dtype; taken exactly)."""
    g, b, m, rs = gamma.double(), beta.double(), mean.double(), rstd.double()
    d = x.double() - m
    return act_of(g * d * rs + b, act), g.abs() * d.abs() * rs + b.abs()


def inst_apply_ref_loose(x, gamma, beta, mean64, rstd64, act):
    g, b = gamma.double(), beta.double()
    xd = x.double()
    return (act_of(g * (xd - mean64) * rstd64 + b, act),
            g.abs() * (xd.abs() + mean64.abs()) * rstd64 + b.abs())


def inst_bwd_ref(x, dz, gamma, mean, rstd):
    """One sample: (dx, |.|), and this sample's terms (sum dz xhat, |.|), (sum dz, |.|) of dgamma / dbeta."""
    g, m, rs = gamma.double(), mean.double(), rstd.double()
    dd = dz.double()
    xh = (x.double() - m) * rs
    mdz, mdzx = dd.mean(0), (dd * xh).mean(0)
    dx = g * rs * (dd - mdz - xh * mdzx)
    dxa = g.abs() * rs * (dd.abs() + dd.abs().mean(0) + xh.abs() * (dd.abs() * xh.abs()).mean(0))
    return (dx, dxa), ((dd * xh).sum(0), (dd.abs() * xh.abs()).sum(0)), (dd.sum(0), dd.abs().sum(0))


# ----------------------------------------------------------------------------------------------------------------
# fp32 emulations of the kernels (with the mistakes a kernel could make as switches)
# ----------------------------------------------------------------------------------------------------------------
def lanes_per_pixel(C):
    g = 1
    while g < 32 and g * 4 < C:
        g <<= 1
    return g


def pixel_fwd_f32(x, act, eps=EPS_PIXEL, div=None, share_only=False, slope=0.3):
    C = x.shape[-1]
    sq = x * x
    if share_only:                    # the butterfly left out: each lane normalises by its own float4 groups' sum
        lane = (torch.arange(C) // 4) % lanes_per_pixel(C)
        ss = torch.stack([sq[..., lane == l].sum(-1) for l in range(lanes_per_pixel(C))], -1)[..., lane]
    else:
        ss = sq.sum(-1, keepdim=True)
    return act_of(x * torch.rsqrt(ss * torch.tensor(1.0 / (div or C)).float() + torch.tensor(eps).float()), act, slope)


def pixel_bwd_f32(x, dz, eps=EPS_PIXEL, drop_term=False):
    C = x.shape[-1]
    invc = torch.tensor(1.0 / C).float()
    r = torch.rsqrt((x * x).sum(-1, keepdim=True) * invc + torch.tensor(eps).float())
    k = r * r * r * (x * dz).sum(-1, keepdim=True) * invc
    return r * dz if drop_term else r * dz - x * k


def chunk_sums(v):
    """v [HW, C] fp32 -> [nchunk, C] fp32 sums in the kernels' order: per chunk, rows = max(256 / C, 1) threads per
    channel each add every rows-th pixel serially, then the rows are added in order."""
    HW, C = v.shape
    rows = max(256 // C, 1)
    out = []
    for p0 in range(0, HW, IN_CHUNK):
        ch = v[p0:p0 + IN_CHUNK]
        acc = torch.zeros(rows, C, dtype=torch.float32)
        for t in range(0, ch.shape[0], rows):
            blk = ch[t:t + rows]
            acc[:blk.shape[0]] += blk
        s = torch.zeros(C, dtype=torch.float32)
        for r in range(rows):
            s = s + acc[r]
        out.append(s)
    return torch.stack(out)


def chunk_counts(HW):
    return torch.tensor([min(HW, p0 + IN_CHUNK) - p0 for p0 in range(0, HW, IN_CHUNK)], dtype=torch.float64)


def shifted_stats(x, eps=EPS_INSTANCE, unbiased=False, drop_chunk=None):
    """The kernel's statistics of one sample x [HW, C]: per chunk the fp32 mean a, then sum (x - a) and sum (x - a)^2
    in fp32, merged in double in chunk order (Chan).  -> fp32 (mean, rstd)."""
    HW, C = x.shape
    cnt = chunk_counts(HW)
    a = torch.stack([chunk_sums(x[p0:p0 + IN_CHUNK])[0] * torch.tensor(1.0 / int(n)).float()
                     for p0, n in zip(range(0, HW, IN_CHUNK), cnt)])
    d = torch.cat([x[p0:p0 + IN_CHUNK] - a[k] for k, p0 in enumerate(range(0, HW, IN_CHUNK))])
    r, q = chunk_sums(d).double(), chunk_sums(d * d).double()
    n_tot, m, m2 = 0.0, torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64)
    for k in range(len(cnt)):
        if k == drop_chunk:
            continue
        nk = float(cnt[k])
        mk = a[k].double() + r[k] / nk
        m2k = (q[k] - r[k] * r[k] / nk).clamp(min=0)
        dlt, tot = mk - m, n_tot + nk
        m = m + dlt * nk / tot
        m2 = m2 + m2k + dlt * dlt * n_tot * nk / tot
        n_tot = tot
    var = m2 / ((HW - 1) if unbiased else HW)
    return m.float(), (1.0 / torch.sqrt(var + float(torch.tensor(eps).float()))).float()


def onepass_stats(x, eps=EPS_INSTANCE):
    """The form this kernel used before: fp32 chunk sums of x and x^2, var = E[x^2] - mean^2 in double."""
    HW = x.shape[0]
    s, s2 = chunk_sums(x).double().sum(0), chunk_sums(x * x).double().sum(0)
    m = s / HW
    var = (s2 / HW - m * m).clamp(min=0)
    return m.float(), (1.0 / torch.sqrt(var + float(torch.tensor(eps).float()))).float()


def inst_fwd_f32(x, gamma, beta, mean, rstd, act, slope=0.3):
    return act_of(gamma * ((x - mean) * rstd) + beta, act, slope)


def inst_bwd_f32(x, dz, gamma, mean, rstd, prior=None, accumulate=0, drop_term=False, swap=False):
    """x, dz [N, HW, C]; mean, rstd [N, C] fp32 -> fp32 (dx, dgamma, dbeta) as the kernels form them."""
    N, HW, C = x.shape
    dx = torch.empty_like(x)
    gs, bs = torch.zeros(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64)
    for n in range(N):
        xh = (x[n] - mean[n]) * rstd[n]
        a, b = chunk_sums(dz[n]).double().sum(0), chunk_sums(dz[n] * xh).double().sum(0)
        mdz, mdzx = (a / HW).float(), (b / HW).float()
        dx[n] = gamma * rstd[n] * (dz[n] - mdz - (0 if drop_term else xh * mdzx))
        bs, gs = bs + a, gs + b
    if swap:
        gs, bs = bs, gs
    base = prior if accumulate else (torch.zeros(C), torch.zeros(C))
    return dx, base[0] + gs.float(), base[1] + bs.float()


# ----------------------------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------------------------
DATA = ['centred', 'offset3', 'offset30', 'offset300', 'const_channel', 'scale_1e-4', 'scale_1e+4', 'zero_pixel']


def make_x(kind, N, HW, C, seed, device='cpu'):
    """[N, HW, C] fp32.  Every sample has its own scale and shift, so statistics shared across the batch show.
    centred: 2 randn + 0.3 (mean / std 0.15).  offsetR: per channel std in [0.05, 2], mean = +-R std.
    const_channel: channel 1 of sample 0 constant 3 and channel 2 of the last sample constant 0 (variance exactly 0).
    zero_pixel: the first and last pixel of every sample all zero."""
    gen = torch.Generator(device).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device=device, generator=gen)
    ru = lambda *s: torch.rand(*s, device=device, generator=gen)
    per = 1 + 0.5 * torch.arange(N, device=device, dtype=torch.float32).view(N, 1, 1)
    if kind.startswith('offset'):
        ratio = float(kind[6:])
        std = 0.05 + 1.95 * ru(1, 1, C)
        sign = torch.where(ru(1, 1, C) < 0.5, -1.0, 1.0)
        return ((std * rn(N, HW, C) + sign * ratio * std) * per).contiguous()
    x = (2 * rn(N, HW, C) + 0.3) * per + 0.1 * (per - 1)
    if kind == 'const_channel':
        x[0, :, 1] = 3.0
        x[N - 1, :, 2] = 0.0
    elif kind.startswith('scale_'):
        x = x * float(kind[6:])
    elif kind == 'zero_pixel':
        x[:, 0] = 0
        x[:, HW - 1] = 0
    return x.contiguous()


def make_affine(C, seed, device='cpu'):
    gen = torch.Generator(device).manual_seed(seed)
    gamma = 1 + 0.3 * torch.randn(C, device=device, generator=gen)
    beta = 0.3 * torch.randn(C, device=device, generator=gen)
    return gamma, beta


def make_dz(y, act, seed):
    """d(loss) / d(norm output), already multiplied by act'(y) as the consumer does; correlated with y so that
    mean(dz xhat) is not small."""
    gen = torch.Generator(y.device).manual_seed(seed)
    gy = torch.randn(y.shape, device=y.device, generator=gen) + 0.25 * y.clamp(-4, 4)
    if act == 'leakyrelu':
        gy = gy * torch.where(y > 0, 1.0, 0.3)
    elif act == 'relu':
        gy = gy * (y > 0)
    elif act == 'elu':
        gy = gy * torch.where(y > 0, torch.ones_like(y), y + 1)
    return gy.float().contiguous()


# ----------------------------------------------------------------------------------------------------------------
# CPU: each reference passes its fp32 emulation and flags the seeded mistakes
# ----------------------------------------------------------------------------------------------------------------
CPU_SHAPE = (2, 2304, 16)            # three chunks, the last partial; 16 thread rows of 64 serial terms


def _r_pixel_fwd(got, x, act):
    ref, absr = pixel_fwd_ref(x, act)
    return max_rel(got, ref, absr)


@pytest.mark.parametrize('kind', ['centred', 'offset30', 'scale_1e-4', 'scale_1e+4', 'zero_pixel'])
@pytest.mark.parametrize('C', [16, 12, 260])
def test_pixel_references_pass_fp32_and_flag_mistakes(kind, C):
    x = make_x(kind, 2, 300, C, seed=5)
    for act in ACT_CODE:
        assert _r_pixel_fwd(pixel_fwd_f32(x, act), x, act) <= ELEM_BAR / 2, act
    assert _r_pixel_fwd(pixel_fwd_f32(x, None, div=C - 1), x, None) >= 100 * ELEM_BAR
    assert _r_pixel_fwd(pixel_fwd_f32(x, None, share_only=True), x, None) >= 100 * ELEM_BAR
    assert _r_pixel_fwd(pixel_fwd_f32(x, 'leakyrelu', slope=0.2), x, 'leakyrelu') >= 0.1
    dz = make_dz(pixel_fwd_f32(x, 'leakyrelu'), 'leakyrelu', 6)
    ref, absr = pixel_bwd_ref(x, dz)
    assert max_rel(pixel_bwd_f32(x, dz), ref, absr) <= ELEM_BAR / 2
    assert max_rel(pixel_bwd_f32(x, dz, drop_term=True), ref, absr) >= 100 * ELEM_BAR
    if kind in ('scale_1e-4', 'zero_pixel'):          # where eps counts: 1e-6 instead of 1e-8
        if kind == 'scale_1e-4':                      # a zero pixel gives y = 0 under any eps; its dx = dz / sqrt(eps)
            assert _r_pixel_fwd(pixel_fwd_f32(x, None, eps=1e-6), x, None) >= 100 * ELEM_BAR
        assert max_rel(pixel_bwd_f32(x, dz, eps=1e-6), ref, absr) >= 100 * ELEM_BAR
    if kind == 'zero_pixel':
        assert float(ref[:, 0].abs().max()) > 0 and max_rel(ref[:, 0], 1e4 * dz[:, 0].double(), absr[:, 0]) <= 1e-12


def _r_stats(fn, x, **kw):
    """(r of mean, r of rstd) of an fp32 statistics function over the samples of x."""
    rm = rr = 0.0
    for n in range(x.shape[0]):
        mean, rstd, mabs, _ = inst_stats_ref(x[n])
        m32, r32 = fn(x[n], **kw)
        rm, rr = max(rm, max_rel(m32, mean, mabs)), max(rr, max_rel(r32, rstd, rstd))
    return rm, rr


@pytest.mark.parametrize('kind', [k for k in DATA if k != 'zero_pixel'])
def test_instance_statistics_reference_passes_the_shifted_form_at_every_offset(kind):
    x = make_x(kind, *CPU_SHAPE, seed=7)
    rm, rr = _r_stats(shifted_stats, x)
    assert rm <= ELEM_BAR / 2 and rr <= RSTD_BAR / 2, (rm, rr)
    if kind == 'const_channel':
        m32, r32 = shifted_stats(x[0])
        assert float(m32[1]) == 3.0 and abs(float(r32[1]) - 1000.0) <= 1e-3


def test_one_pass_variance_fails_on_offset_inputs_and_passes_on_centred_ones():
    """E[x^2] - mean^2 from fp32 chunk sums, in the summation order of the kernel that used it: the relative error of
    rstd grows with (mean / std)^2.  This is why the kernel centres each chunk first."""
    r = {k: _r_stats(onepass_stats, make_x(k, *CPU_SHAPE, seed=7))[1] for k in ('centred', 'offset30', 'offset300')}
    assert r['centred'] <= RSTD_BAR / 2, r
    assert r['offset30'] >= 2 * RSTD_BAR and r['offset300'] >= 100 * RSTD_BAR, r


def test_instance_statistics_reference_flags_mistakes():
    x = make_x('centred', *CPU_SHAPE, seed=7)
    assert _r_stats(shifted_stats, x, unbiased=True)[1] >= 10 * RSTD_BAR         # HW - 1: 1 / (2 HW) = 2.2e-4
    for k in range(3):
        rm, rr = _r_stats(shifted_stats, x, drop_chunk=k)
        assert rm >= 100 * ELEM_BAR and rr >= 10 * RSTD_BAR, (k, rm, rr)
    # statistics over the whole batch instead of per sample
    shared = lambda xn: shifted_stats(x.reshape(-1, x.shape[2]))
    rm, rr = _r_stats(shared, x)
    assert rm >= 1e3 * ELEM_BAR and rr >= 1e3 * RSTD_BAR
    # eps matters where the variance is small: 1e-5 / 1e-8 instead of 1e-6
    for kind in ('scale_1e-4', 'const_channel'):
        xs = make_x(kind, *CPU_SHAPE, seed=7)
        for eps in (1e-5, 1e-8):
            assert _r_stats(shifted_stats, xs, eps=eps)[1] >= 1e3 * RSTD_BAR, (kind, eps)


def _cpu_instance(kind, act='leakyrelu'):
    x = make_x(kind, *CPU_SHAPE, seed=9)
    N, HW, C = x.shape
    gamma, beta = make_affine(C, 10)
    st = [shifted_stats(x[n]) for n in range(N)]
    mean, rstd = torch.stack([s[0] for s in st]), torch.stack([s[1] for s in st])
    y = torch.stack([inst_fwd_f32(x[n], gamma, beta, mean[n], rstd[n], act) for n in range(N)])
    return x, gamma, beta, mean, rstd, y, make_dz(y, act, 11)


def _r_inst_bwd(got, x, dz, gamma, mean, rstd, prior=None):
    dx, dg, db = got
    N, C = mean.shape
    r = {'dx': 0.0}
    gs, ga, bs, ba = (torch.zeros(C, dtype=torch.float64, device=x.device) for _ in range(4))
    if prior is not None:
        gs, ga, bs, ba = prior[0].double(), prior[0].double().abs(), prior[1].double(), prior[1].double().abs()
    for n in range(N):
        (ref, absr), (g, gabs), (b, babs) = inst_bwd_ref(x[n], dz[n], gamma, mean[n], rstd[n])
        r['dx'] = max(r['dx'], max_rel(dx[n], ref, absr))
        gs, ga, bs, ba = gs + g, ga + gabs, bs + b, ba + babs
    if dg is not None:
        r['dgamma'] = max_rel(dg, gs, ga)
    if db is not None:
        r['dbeta'] = max_rel(db, bs, ba)
    return r


def _inst_bwd_ok(r):
    return r['dx'] <= INST_DX_BAR and r.get('dgamma', 0) <= TAU and r.get('dbeta', 0) <= TAU


@pytest.mark.parametrize('kind', ['centred', 'offset30', 'offset300', 'const_channel', 'scale_1e-4', 'scale_1e+4'])
def test_instance_references_pass_fp32_and_flag_mistakes(kind):
    x, gamma, beta, mean, rstd, y, dz = _cpu_instance(kind)
    N = x.shape[0]
    for act in ACT_CODE:
        for n in range(N):
            ref, absr = inst_apply_ref(x[n], gamma, beta, mean[n], rstd[n], act)
            assert max_rel(inst_fwd_f32(x[n], gamma, beta, mean[n], rstd[n], act), ref, absr) <= ELEM_BAR / 2
            m64, r64 = inst_stats_ref(x[n])[:2]
            ref, absr = inst_apply_ref_loose(x[n], gamma, beta, m64, r64, act)
            assert max_rel(inst_fwd_f32(x[n], gamma, beta, mean[n], rstd[n], act), ref, absr) <= RSTD_BAR / 2
    ref, absr = inst_apply_ref(x[0], gamma, beta, mean[0], rstd[0], 'leakyrelu')
    assert max_rel(inst_fwd_f32(x[0], gamma, beta, mean[0], rstd[0], 'leakyrelu', slope=0.2), ref, absr) >= 0.05
    assert max_rel(inst_fwd_f32(x[0], gamma, beta, mean[1], rstd[1], 'leakyrelu'), ref, absr) >= 1e3 * ELEM_BAR
    assert max_rel(inst_fwd_f32(x[0], beta, gamma, mean[0], rstd[0], 'leakyrelu'), ref, absr) >= 1e3 * ELEM_BAR
    # backward
    r = _r_inst_bwd(inst_bwd_f32(x, dz, gamma, mean, rstd), x, dz, gamma, mean, rstd)
    assert r['dx'] <= INST_DX_BAR / 2 and r['dgamma'] <= TAU / 4 and r['dbeta'] <= TAU / 4, r
    assert torch.isfinite(inst_bwd_f32(x, dz, gamma, mean, rstd)[0]).all()
    bad = _r_inst_bwd(inst_bwd_f32(x, dz, gamma, mean, rstd, drop_term=True), x, dz, gamma, mean, rstd)
    assert bad['dx'] >= 100 * INST_DX_BAR, bad
    bad = _r_inst_bwd(inst_bwd_f32(x, dz, gamma, mean, rstd, swap=True), x, dz, gamma, mean, rstd)
    assert bad['dgamma'] >= 100 * TAU and bad['dbeta'] >= 100 * TAU, bad
    prior = (torch.randn(x.shape[2], generator=torch.Generator().manual_seed(12)) * 50,
             torch.randn(x.shape[2], generator=torch.Generator().manual_seed(13)) * 50)
    ok = _r_inst_bwd(inst_bwd_f32(x, dz, gamma, mean, rstd, prior, accumulate=1), x, dz, gamma, mean, rstd, prior)
    assert _inst_bwd_ok(ok), ok
    bad = _r_inst_bwd(inst_bwd_f32(x, dz, gamma, mean, rstd, prior, accumulate=0), x, dz, gamma, mean, rstd, prior)
    assert bad['dgamma'] >= 100 * TAU and bad['dbeta'] >= 100 * TAU, bad


# ----------------------------------------------------------------------------------------------------------------
# the shapes a norm layer sees in the benchmarked workloads
# ----------------------------------------------------------------------------------------------------------------
def norm_layer_shapes(wl_name, uv=None):
    """[(H, C)] of the input of every NormLayer of one U-Net of a workload built with norm != None, read off the
    network's own layer list (the model test below holds the shapes it meets on the device against this)."""
    import bench
    from networks.convnet import Network
    wl = bench.WORKLOADS[wl_name]
    cfg = bench.make_config(wl)['DEFAULT']
    net = Network(int(cfg['depth0']), int(cfg['depth']), int(cfg['kernel']), int(cfg['stride']), norm_type='instance',
                  act_type=cfg['act'], pool_type=cfg['pool'])
    size, out = uv or wl['uv'], []
    for blk in net.layers:
        for c, nm in zip(blk.convs, blk.norms):
            size = size // c.s if c.kind == 'conv' else size * c.s
            if nm is not None:
                out.append((size, c.cout))
    return out


def production_shapes():
    """Distinct (N, HW, C): cfg4 (batch 8, depth 256) whole, cfg3 (batch 16, depth 1024) where it goes deeper, and the
    level-0 feature map 8 x 1024^2 x 16, the largest tensor of the model."""
    import bench
    shapes = {(bench.WORKLOADS['cfg4']['batch'], h * h, c) for h, c in norm_layer_shapes('cfg4')}
    shapes |= {(bench.WORKLOADS['cfg3']['batch'], h * h, c) for h, c in norm_layer_shapes('cfg3') if c >= 512}
    shapes.add((8, 1024 * 1024, 16))
    return sorted(shapes, key=lambda s: (-s[0] * s[1] * s[2], s))


def test_production_shapes_cover_the_large_maps_and_the_deep_levels():
    shapes = production_shapes()
    assert (8, 1024 * 1024, 4) in shapes and (8, 512 * 512, 16) in shapes and (16, 16, 1024) in shapes
    assert len(norm_layer_shapes('cfg4')) == 24 and len(norm_layer_shapes('cfg3')) == 32


# ----------------------------------------------------------------------------------------------------------------
# GPU: direct C-ABI calls
# ----------------------------------------------------------------------------------------------------------------
GUARD = 4096                          # floats behind the workspace that no kernel may touch
GUARD_VALUE = 12345.0


RECORD = {'bars': {'elem': ELEM_BAR, 'rstd': RSTD_BAR, 'instance_dx': INST_DX_BAR, 'tau': TAU}}


def note(key, rec):
    """Worst r per op, shape and data kind of this session, rewritten whole after every test
    (parity_census_norm.json)."""
    RECORD[key] = rec
    _record('norm', RECORD)


def _lib():
    import nlt_native as nat
    return nat, nat.lib()


def nan_like(t):
    return torch.full_like(t, NAN)


def run_pixel(x, act=None, dz=None):
    nat, lib = _lib()
    C = x.shape[-1]
    out = nan_like(x)
    if dz is None:
        nat.check(lib.nlt_pixelnorm_fwd(nat.ptr(x), x.numel() // C, C, ACT_CODE[act], nat.ptr(out), nat.stream()))
    else:
        nat.check(lib.nlt_pixelnorm_bwd(nat.ptr(x), nat.ptr(dz), x.numel() // C, C, nat.ptr(out), nat.stream()))
    return out


def guarded_workspace(N, HW, C, device):
    """Exactly nlt_instnorm_workspace_bytes bytes, NaN-filled, followed by the guard."""
    _, lib = _lib()
    need = lib.nlt_instnorm_workspace_bytes(N, HW, C)
    assert need > 0 and need % 4 == 0, need
    buf = torch.full((need // 4 + GUARD,), NAN, device=device)
    buf[need // 4:] = GUARD_VALUE
    return buf, need // 4


def guard_intact(buf, n):
    return bool((buf[n:] == GUARD_VALUE).all())


def run_inst_fwd(x, gamma, beta, act, ws=None):
    nat, lib = _lib()
    N, HW, C = x.shape
    ws, n = guarded_workspace(N, HW, C, x.device) if ws is None else ws
    y, mean, rstd = nan_like(x), torch.full((N, C), NAN, device=x.device), torch.full((N, C), NAN, device=x.device)
    nat.check(lib.nlt_instnorm_fwd(nat.ptr(x), nat.ptr(gamma), nat.ptr(beta), N, HW, C, ACT_CODE[act], EPS_INSTANCE,
                                   nat.ptr(y), nat.ptr(mean), nat.ptr(rstd), nat.ptr(ws), nat.stream()))
    assert guard_intact(ws, n), 'nlt_instnorm_fwd wrote behind its workspace'
    return y, mean, rstd


def run_inst_bwd(x, dz, gamma, mean, rstd, dgamma, dbeta, accumulate):
    nat, lib = _lib()
    N, HW, C = x.shape
    ws, n = guarded_workspace(N, HW, C, x.device)
    dx = nan_like(x)
    nat.check(lib.nlt_instnorm_bwd(nat.ptr(x), nat.ptr(dz), nat.ptr(gamma), nat.ptr(mean), nat.ptr(rstd), N, HW, C,
                                   nat.ptr(dx), nat.ptr(dgamma), nat.ptr(dbeta), accumulate, nat.ptr(ws), nat.stream()))
    assert guard_intact(ws, n), 'nlt_instnorm_bwd wrote behind its workspace'
    return dx


def pixel_case(x, act, seed, st):
    """Forward with `act` and backward of one input against fp64, in slices of samples; r into st."""
    y = run_pixel(x, act)
    dz = make_dz(y, act, seed)
    dx = run_pixel(x, dz=dz)
    for n in range(x.shape[0]):
        ref, absr = pixel_fwd_ref(x[n], act)
        st['y'] = max(st.get('y', 0.0), check('pixel y[%d]' % n, y[n], ref, absr, ELEM_BAR))
        ref, absr = pixel_bwd_ref(x[n], dz[n])
        st['dx'] = max(st.get('dx', 0.0), check('pixel dx[%d]' % n, dx[n], ref, absr, ELEM_BAR))
    return y, dx


def instance_forward_case(x, gamma, beta, act, st, errors):
    """nlt_instnorm_fwd against fp64; failures are collected so that the backward pass is still measured."""
    y, mean, rstd = run_inst_fwd(x, gamma, beta, act)
    ratio = 0.0
    for n in range(x.shape[0]):
        m64, r64, mabs, std = inst_stats_ref(x[n])
        ratio = max(ratio, float((m64.abs() / std.clamp(min=1e-30)).max()))
        refs = [('mean', mean[n], m64, mabs, ELEM_BAR), ('rstd', rstd[n], r64, r64, RSTD_BAR)]
        ref, absr = inst_apply_ref(x[n], gamma, beta, mean[n], rstd[n], act)
        refs.append(('y', y[n], ref, absr, ELEM_BAR))
        ref, absr = inst_apply_ref_loose(x[n], gamma, beta, m64, r64, act)
        refs.append(('y_fp64_stats', y[n], ref, absr, RSTD_BAR))
        for name, got, ref, absr, bar in refs:
            try:
                st[name] = max(st.get(name, 0.0), check('instance %s[%d]' % (name, n), got, ref, absr, bar, out={}))
            except AssertionError as e:
                st[name] = max(st.get(name, 0.0), max_rel(got, ref, absr))
                errors.append(str(e))
    st['max_mean_over_std'] = ratio
    return y, mean, rstd


def instance_backward_case(x, dz, gamma, mean, rstd, st, seed):
    """nlt_instnorm_bwd as a function of its fp32 arguments: overwrite over NaN, twice (bit-identical), accumulate on
    known values, NULL dgamma, NULL dbeta."""
    C = x.shape[2]
    dev = x.device
    outs = []
    for _ in range(2):
        dg, db = torch.full((C,), NAN, device=dev), torch.full((C,), NAN, device=dev)
        outs.append((run_inst_bwd(x, dz, gamma, mean, rstd, dg, db, 0), dg, db))
    for a, b, what in zip(outs[0], outs[1], ('dx', 'dgamma', 'dbeta')):
        assert torch.equal(a, b), 'two calls differ in %s at %s' % (what, (a != b).nonzero()[:4].tolist())
    r = _r_inst_bwd(outs[0], x, dz, gamma, mean, rstd)
    st.update({k: max(st.get(k, 0.0), v) for k, v in r.items()})
    assert _inst_bwd_ok(r), r
    gen = torch.Generator(dev).manual_seed(seed)
    prior = (torch.randn(C, device=dev, generator=gen) * 50, torch.randn(C, device=dev, generator=gen) * 50)
    dg, db = prior[0].clone(), prior[1].clone()
    dx = run_inst_bwd(x, dz, gamma, mean, rstd, dg, db, 1)
    assert torch.equal(dx, outs[0][0])
    r = _r_inst_bwd((dx, dg, db), x, dz, gamma, mean, rstd, prior)
    st['dgamma_acc'], st['dbeta_acc'] = r['dgamma'], r['dbeta']
    assert _inst_bwd_ok(r), r
    for null in ('dgamma', 'dbeta'):
        dg = None if null == 'dgamma' else torch.full((C,), NAN, device=dev)
        db = None if null == 'dbeta' else torch.full((C,), NAN, device=dev)
        dx = run_inst_bwd(x, dz, gamma, mean, rstd, dg, db, 0)
        assert torch.equal(dx, outs[0][0]), 'dx changes with a NULL %s' % null
        if dg is not None:
            assert torch.equal(dg, outs[0][1])
        if db is not None:
            assert torch.equal(db, outs[0][2])
    return outs[0][0]


def instance_case(x, act, seed, st):
    C = x.shape[2]
    gamma, beta = make_affine(C, seed, x.device)
    errors = []
    y, mean, rstd = instance_forward_case(x, gamma, beta, act, st, errors)
    dz = make_dz(y, act, seed + 1)
    dx = instance_backward_case(x, dz, gamma, mean, rstd, st, seed + 2)
    assert not errors, '\n'.join(errors)
    return y, mean, rstd, dx, gamma, beta


def _shape_id(s):
    return 'n%d_hw%d_c%d' % s


PROD = production_shapes()
PROD_DATA = {PROD[0]: ['centred', 'offset30'], (8, 512 * 512, 16): ['centred', 'offset30', 'offset300'],
             (16, 16, 1024): ['centred', 'offset30']}


@pytest.mark.gpu
@pytest.mark.parametrize('shape', PROD, ids=_shape_id)
def test_ops_at_production_shape(shape):
    """Both norms, forward and backward, on the tensors of the benchmarked workloads (1024 chunks per sample at
    1024^2: the grid-stride loops wrap, the double-precision merge runs over all of them)."""
    N, HW, C = shape
    dev = torch.device('cuda')
    t0 = time.perf_counter()
    rec = {}
    try:
        for kind in PROD_DATA.get(shape, ['centred']):
            x = make_x(kind, N, HW, C, seed=100 + C, device=dev)
            st = rec.setdefault(kind, {'pixel': {}, 'instance': {}})
            pixel_case(x, 'leakyrelu', 101, st['pixel'])
            instance_case(x, 'leakyrelu', 102, st['instance'])
            del x
    finally:                          # a failing case leaves its numbers too
        rec['seconds'] = time.perf_counter() - t0
        note('prod_' + _shape_id(shape), rec)


HWS = [1, 2, 1023, 1024, 1025, 2049]
CS = [4, 12, 20, 36, 48, 96, 260, 1024, 6144]
EDGES = ([(3, hw, 12) for hw in HWS] + [(1, hw, 260) for hw in HWS] + [(3, hw, 16) for hw in HWS]
         + [(1 if c >= 1024 else 3, 1025, c) for c in CS] + [(5, 33, c) for c in CS])


@pytest.mark.gpu
@pytest.mark.parametrize('shape', EDGES, ids=_shape_id)
def test_ops_at_edge_shapes(shape):
    """Chunk boundaries of the instance reductions (HW around 1024 and 2048, the single-pixel sample with var = 0 and
    rstd = 1000), channel counts whose lane groups get uneven shares of the float4 groups (12, 20, 36), whose thread
    rows do not fill the block (12, 20, 36, 48, 96), beyond the block (260, 1024) and the last that fits shared
    memory (6144); N = 1 and odd N; pixel counts that leave dead lane groups in the last warp."""
    N, HW, C = shape
    dev = torch.device('cuda')
    acts = list(ACT_CODE)
    act = acts[(HW + C // 4) % 4]
    x = make_x('centred', N, HW, C, seed=HW + C, device=dev)
    rec = {'act': str(act), 'pixel': {}, 'instance': {}}
    pixel_case(x, act, 201, rec['pixel'])
    y, mean, rstd, dx, gamma, beta = instance_case(x, act, 202, rec['instance'])
    if HW == 1:
        assert torch.equal(mean, x[:, 0]) and float((rstd - 1000).abs().max()) <= 1e-3
        want = act_of(beta.double(), act).expand(N, C)
        assert max_rel(y[:, 0], want, want.abs()) <= ELEM_BAR
        assert int(dx.count_nonzero()) == 0
    note('edge_' + _shape_id(shape), rec)


DATA_SHAPES = [(3, 1025, 12), (2, 2049, 48), (1, 1024, 260), (2, 65536, 16)]


@pytest.mark.gpu
@pytest.mark.parametrize('shape', DATA_SHAPES, ids=_shape_id)
@pytest.mark.parametrize('kind', DATA)
def test_ops_on_offset_constant_scaled_and_zero_inputs(kind, shape):
    N, HW, C = shape
    dev = torch.device('cuda')
    x = make_x(kind, N, HW, C, seed=300 + C, device=dev)
    rec = {'pixel': {}, 'instance': {}}
    try:
        _, pdx = pixel_case(x, 'leakyrelu', 301, rec['pixel'])
        y, mean, rstd, dx, gamma, beta = instance_case(x, 'leakyrelu', 302, rec['instance'])
    finally:
        note('data_%s_%s' % (kind, _shape_id(shape)), rec)
    assert bool(torch.isfinite(dx).all()) and bool(torch.isfinite(pdx).all())
    if kind == 'const_channel':
        # variance exactly 0: eps alone under the root, the mean exact, the output the activation of beta
        assert float(mean[0, 1]) == 3.0 and float(mean[N - 1, 2]) == 0.0
        assert abs(float(rstd[0, 1]) - 1000.0) <= 1e-3 and abs(float(rstd[N - 1, 2]) - 1000.0) <= 1e-3
        want = act_of(beta.double(), 'leakyrelu')
        for n, c in ((0, 1), (N - 1, 2)):
            assert max_rel(y[n, :, c], want[c].expand(HW), want[c].abs().expand(HW)) <= ELEM_BAR
    if kind == 'zero_pixel':
        py = run_pixel(x, 'leakyrelu')
        assert int(py[:, 0].count_nonzero()) == 0 and int(py[:, HW - 1].count_nonzero()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize('act', list(ACT_CODE), ids=str)
@pytest.mark.parametrize('shape', [(3, 1025, 12), (2, 33, 96)], ids=_shape_id)
def test_every_fused_activation(act, shape):
    x = make_x('centred', *shape, seed=400, device=torch.device('cuda'))
    rec = {'pixel': {}, 'instance': {}}
    y, _ = pixel_case(x, act, 401, rec['pixel'])
    yi = instance_case(x, act, 402, rec['instance'])[0]
    for out in (y, yi):
        neg = out < 0
        if act == 'relu':
            assert not bool(neg.any()) and bool((out == 0).any())
        elif act == 'elu':
            assert bool(neg.any()) and float(out.min()) > -1.0
        else:
            assert bool(neg.any())
    note('act_%s_%s' % (act, _shape_id(shape)), rec)


@pytest.mark.gpu
def test_workspace_size_and_refused_arguments():
    """The host-side checks return NLT_ERR_INVALID before any launch: outputs stay NaN."""
    nat, lib = _lib()
    dev = torch.device('cuda')
    for N, HW, C in ((0, 4, 4), (2, 0, 4), (2, 4, 0), (-1, 4, 4), (2, -5, 4), (2, 4, -4)):
        assert lib.nlt_instnorm_workspace_bytes(N, HW, C) < 0, (N, HW, C)
    for N, HW, C in ((1, 1, 4), (8, 1 << 20, 16), (3, 1025, 12), (16, 16, 1024)):
        nchunk = (HW + IN_CHUNK - 1) // IN_CHUNK
        assert lib.nlt_instnorm_workspace_bytes(N, HW, C) == 4 * (N * nchunk * 3 * C + 2 * N * C)

    def refused(rc):
        assert rc == -1, rc          # NLT_ERR_INVALID
        assert lib.nlt_last_error()

    for C in (6, 6148, 6150):
        x = torch.ones(2, 3, C, device=dev)
        g, b = torch.ones(C, device=dev), torch.zeros(C, device=dev)
        out, mean, rstd = nan_like(x), torch.full((2, C), NAN, device=dev), torch.full((2, C), NAN, device=dev)
        ws = torch.full((1 << 16,), NAN, device=dev)
        refused(lib.nlt_instnorm_fwd(nat.ptr(x), nat.ptr(g), nat.ptr(b), 2, 3, C, 0, EPS_INSTANCE, nat.ptr(out),
                                     nat.ptr(mean), nat.ptr(rstd), nat.ptr(ws), nat.stream()))
        refused(lib.nlt_instnorm_bwd(nat.ptr(x), nat.ptr(x), nat.ptr(g), nat.ptr(b), nat.ptr(g), 1, 6, C, nat.ptr(out),
                                     None, None, 0, nat.ptr(ws), nat.stream()))
        if C % 4:
            refused(lib.nlt_pixelnorm_fwd(nat.ptr(x), 6, C, 0, nat.ptr(out), nat.stream()))
            refused(lib.nlt_pixelnorm_bwd(nat.ptr(x), nat.ptr(x), 6, C, nat.ptr(out), nat.stream()))
        torch.cuda.synchronize()
        assert bool(out.isnan().all()) and bool(mean.isnan().all()) and bool(ws.isnan().all()), C
    x = torch.ones(2, 3, 8, device=dev)
    g = torch.ones(8, device=dev)
    out = nan_like(x)
    for act in (-1, 4):
        refused(lib.nlt_pixelnorm_fwd(nat.ptr(x), 6, 8, act, nat.ptr(out), nat.stream()))
        refused(lib.nlt_instnorm_fwd(nat.ptr(x), nat.ptr(g), nat.ptr(g), 2, 3, 8, act, EPS_INSTANCE, nat.ptr(out),
                                     nat.ptr(g), nat.ptr(g), nat.ptr(x), nat.stream()))
    refused(lib.nlt_pixelnorm_fwd(nat.ptr(x), 0, 8, 0, nat.ptr(out), nat.stream()))
    refused(lib.nlt_pixelnorm_fwd(None, 6, 8, 0, nat.ptr(out), nat.stream()))
    refused(lib.nlt_instnorm_fwd(nat.ptr(x), nat.ptr(g), nat.ptr(g), 2, 3, 8, 0, EPS_INSTANCE, nat.ptr(out),
                                 nat.ptr(g), nat.ptr(g), None, nat.stream()))
    torch.cuda.synchronize()
    assert bool(out.isnan().all())


# ----------------------------------------------------------------------------------------------------------------
# GPU: the layers in place, and the graphed step
# ----------------------------------------------------------------------------------------------------------------
MODEL_WL = 'cfg4'                     # UV 1024^2, batch 8, 64-channel query stack, default options (tensor cores on)
FIT = 0.9


def norm_config(kind):
    import bench
    cfg = bench.make_config(bench.WORKLOADS[MODEL_WL])
    cfg['DEFAULT']['norm'] = kind
    return cfg


def norm_layers(model):
    return [(('%s.%d.%d.norm' % (net, li, ci)), nm) for net in ('query', 'obs')
            for li, blk in enumerate(model.net[net].layers) for ci, nm in enumerate(blk.norms) if nm is not None]


def poison_norm_workspaces(mp):
    """NormLayer._ws is the layer's own buffer, outside the engine's workspace pools: NaN-filled before every use
    (inside a capture the fill is recorded, so every replay starts from NaN too)."""
    import engine
    real = engine.NormLayer._workspace

    def workspace(self, *a):
        ws = real(self, *a)
        ws.fill_(NAN)
        return ws
    mp.setattr(engine.NormLayer, '_workspace', workspace)


def _build_model(kind):
    import bench
    import models
    wl = bench.WORKLOADS[MODEL_WL]
    model = models.get_model_class('nlt')(norm_config(kind))
    model.register_trainable()
    model.build(5 + wl['c_extra'], 3)
    _bias_init(model)
    if kind == 'instance':
        g = torch.Generator().manual_seed(12)
        for _, nm in norm_layers(model):
            nm.kernel.copy_(1 + 0.3 * torch.randn(nm.kernel.shape, generator=g))
    return model, wl


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['pixel', 'instance'])
def test_norm_layers_in_a_training_step(kind, monkeypatch):
    """One eager training step of the cfg4 model with `norm = kind` at batch 8, default options: every NormLayer's
    actual input, dz and outputs against the fp64 references above, right where the layer runs (the convs around them
    are the census's).  This is the data the kernels see in a model: conv outputs with a bias, not centred."""
    import engine
    from util import synth
    dev = torch.device('cuda')
    t0 = time.perf_counter()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    model, wl = _build_model(kind)
    B = wl['batch'] if free >= 60e9 else (4 if free >= 30e9 else 2)
    names = {id(nm): name for name, nm in norm_layers(model)}
    assert len(names) == 24 + 12
    bt = synth.make_batch(B, wl['uv'], wl['uv'], seed=1235, c_extra=wl['c_extra'], k_obs=wl['k_obs'])
    bt = tuple(t.to(dev) if torch.is_tensor(t) else t for t in bt)
    rec, errors, seen = {}, [], []
    real_backward = engine.NormLayer._backward

    def backward(self, x, out, saved):
        engine.settle(out)
        dz = out.grad
        real_backward(self, x, out, saved)
        if dz is None or not x.needs_grad:
            return
        name = names[id(self)]
        N, H, W, C = x.t.shape
        seen.append((H, C))
        xs, ys, dzs, dxs = (t.reshape(N, H * W, C) for t in (x.t, out.t, dz, x.grad))
        st = rec.setdefault(name, {'shape': [N, H, W, C]})
        try:
            if kind == 'pixel':
                for n in range(N):
                    ref, absr = pixel_fwd_ref(xs[n], self.act)
                    st['y'] = max(st.get('y', 0.0), check(name + ' y', ys[n], ref, absr, ELEM_BAR))
                    ref, absr = pixel_bwd_ref(xs[n], dzs[n])
                    st['dx'] = max(st.get('dx', 0.0), check(name + ' dx', dxs[n], ref, absr, ELEM_BAR))
            else:
                mean, rstd = (s.reshape(N, C) for s in saved)
                ratio = 0.0
                for n in range(N):
                    m64, r64, mabs, std = inst_stats_ref(xs[n])
                    ratio = max(ratio, float((m64.abs() / std.clamp(min=1e-30)).max()))
                    st['mean'] = max(st.get('mean', 0.0), max_rel(mean[n], m64, mabs))
                    st['rstd'] = max(st.get('rstd', 0.0), max_rel(rstd[n], r64, r64))
                    ref, absr = inst_apply_ref(xs[n], self.kernel, self.bias, mean[n], rstd[n], self.act)
                    st['y'] = max(st.get('y', 0.0), max_rel(ys[n], ref, absr))
                st['max_mean_over_std'] = ratio
                st.update(_r_inst_bwd((dxs, self.gkernel, self.gbias), xs, dzs, self.kernel, mean, rstd))
                assert st['mean'] <= ELEM_BAR and st['rstd'] <= RSTD_BAR and st['y'] <= ELEM_BAR and _inst_bwd_ok(st), st
        except AssertionError as e:
            errors.append('%s: %s' % (name, e))

    poison_workspaces()
    model.flat_grads.fill_(NAN)
    with monkeypatch.context() as mp:
        poisoned_allocations(mp)
        poison_norm_workspaces(mp)
        mp.setattr(engine.NormLayer, '_backward', backward)
        pred, gt, kw, _ = model(bt, mode='train')
        kw['keep_batch'] = True
        model.set_loss_grad_scale(1.0 / B)
        model.compute_loss(pred, gt, **kw)
        model.backward()
    torch.cuda.synchronize()
    note('model_' + kind, {'batch': B, 'layers': rec, 'seconds': time.perf_counter() - t0,
                                   'peak_mem_GB': torch.cuda.max_memory_allocated() / 1e9})
    assert not errors, '\n'.join(errors)
    assert len(rec) == len(names), sorted(set(names.values()) - set(rec))
    # the shapes met on the device are the ones the op tests derive from the layer list
    assert sorted(set(seen)) == sorted(set(norm_layer_shapes(MODEL_WL)))
    # every layer's gradient was written (the alignment padding between them stays as filled)
    assert all(bool(torch.isfinite(g).all()) for g in model.gradients)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['pixel', 'instance'])
def test_graph_replays_of_a_norm_step_equal_eager_and_fp64(kind, monkeypatch):
    """Three replays (b0, b1, b0) of trainvali.GraphedTrainStep with `norm = kind` at cfg4's shape: bit-identical to
    the graph's body run eagerly from the restored state, and within the bars of tests/test_gpu_graph_step.py.
    NormLayer.forward allocates mean, rstd and its workspace inside the captured region."""
    import tests.test_gpu_graph_step as G
    import trainvali
    from util import synth

    class _NormArm(G._Arm):
        def __init__(self, B):
            self.model, wl = _build_model(kind)
            self.B, self.uv = B, wl['uv']
            self.opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
            self.host = [synth.make_batch(B, self.uv, self.uv, seed=1235 + i, c_extra=wl['c_extra'], pin=True,
                                          k_obs=wl['k_obs']) for i in range(2)]
            dev = self.model.device
            self.dev = [tuple(t.to(dev) if torch.is_tensor(t) else t for t in b) for b in self.host]
            self.step = trainvali.GraphedTrainStep(trainvali.Strategy(), self.model, self.opt, B)

    tried = []
    for B in (8, 4, 2):
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base_alloc = torch.cuda.memory_allocated()
        a = _NormArm(B)
        with monkeypatch.context() as mp:
            G._poison(mp)
            poison_norm_workspaces(mp)
            a.step._capture(a.dev[0])
        assert a.step.full_step_in_graph
        ok, peak = G._fits(base_alloc)
        tried.append({'batch': B, 'peak_after_capture_GB': peak / 1e9})
        if ok or B == 2:
            break
        del a
    layers = norm_layers(a.model)
    if kind == 'instance':
        flat = a.model.flat_grads
        lo, hi = flat.data_ptr(), flat.data_ptr() + 4 * flat.numel()
        for name, nm in layers:
            for t in (nm.gkernel, nm.gbias):
                assert lo <= t.data_ptr() and t.data_ptr() + 4 * t.numel() <= hi, name + ' gradient outside flat_grads'
        start = [(nm.kernel.clone(), nm.bias.clone()) for _, nm in layers]
    init = a.state()
    seq = [0, 1, 0]
    graph_out, stats = [], []
    for t, bi in enumerate(seq, 1):
        before = a.state()
        loss, to_vis = a.step(a.step.static_batch if t == 1 else a.dev[bi])
        torch.cuda.synchronize()
        out = a.outputs(loss, to_vis)
        assert bool(torch.isfinite(out['flat_grads']).all()) and bool(torch.isfinite(out['loss']).all())
        stats.append(G.fp64_checks(out, before, a.dev[bi], t, B))
        graph_out.append(out)
    if kind == 'instance':
        for (name, nm), (k0, b0) in zip(layers, start):
            assert int((nm.kernel != k0).sum()) > 0 and int((nm.bias != b0).sum()) > 0, name + ' did not move'
    a.restore(init)
    with monkeypatch.context() as mp:
        G._poison(mp)
        poison_norm_workspaces(mp)
        for t, bi in enumerate(seq, 1):
            poison_workspaces()
            loss, to_vis = a.step._body(a.dev[bi], with_update=True)
            torch.cuda.synchronize()
            G._equal(graph_out[t - 1], a.outputs(loss, to_vis), '%s-norm replay %d vs eager' % (kind, t))
    note('graph_' + kind, {'batch': B, 'tried': tried,
                                   'max_r': {k: max(s[k] for s in stats) for k in stats[0]},
                                   'peak_mem_GB': torch.cuda.max_memory_allocated() / 1e9})
    del a, graph_out
    torch.cuda.empty_cache()
