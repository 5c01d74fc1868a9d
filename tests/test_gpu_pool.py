"""`pool = max | avg` on the GPU: the 2x2 pool and the bilinear x2 upsample (csrc/nlt_pool.cu) against fp64, whole
pooling U-Nets against the fp64 oracle (oracle/pool_oracle.py), one eager production-shape step checked launch by launch,
the graphed step, and test mode with a broadcast observation override.

Metric of the op checks: r = |got - ref| / (the fp64 op on |operands|), as in tests/test_gpu_census.py.
"""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nlt_oracle as O           # noqa: E402
from oracle import pool_oracle as P          # noqa: E402
from tests.test_gpu_census import (TAU, TAU_TC_WGRAD, Census, _bias_init, _imgs, _record, controls,  # noqa: E402
                                   poison_workspaces, poisoned_allocations, vjp_input)
from tests.test_gpu_model import make_model, ocfg, rel_fro   # noqa: E402

OP_BAR = 2.0 ** -22
TINY = 2.0 ** -126
MAX, AVG = 0, 1


def _lib():
    import nlt_native as nat
    return nat


def r_of(got, ref, absr):
    got, ref, absr = got.double(), ref.double(), absr.double()
    err = (got - ref).abs()
    err = torch.where(got.isnan(), torch.full_like(err, float('inf')), err)
    return float((err / absr.clamp(min=TINY)).max())


# ---- fp64 references (device tensors) ----
def up_ref(x):
    """UpSampling2D(2, 'bilinear') in fp64 on the device: the clamped .25 / .75 stencil along H, then along W."""
    def along(a, dim):
        n = a.shape[dim]
        lo = torch.cat((a.narrow(dim, 0, 1), a.narrow(dim, 0, n - 1)), dim)
        hi = torch.cat((a.narrow(dim, 1, n - 1), a.narrow(dim, n - 1, 1)), dim)
        ev, od = 0.25 * lo + 0.75 * a, 0.75 * a + 0.25 * hi
        out = torch.stack((ev, od), dim + 1)
        shape = list(a.shape)
        shape[dim] = 2 * n
        return out.reshape(shape)
    return along(along(x, 1), 2)


def adjoint(fn, x_shape, g, dtype=torch.float64):
    x = torch.zeros(x_shape, dtype=dtype, device=g.device, requires_grad=True)
    (d,) = torch.autograd.grad(fn(x), x, g)
    return d


def _mask_of(y):
    return torch.where(y > 0, 1.0, 0.3)


def run_pool(x, kind, d_y=None, beta=0.0, mask=None, d_x=None):
    nat = _lib()
    N, H, W, C = x.shape
    lib = nat.lib()
    if d_y is None:
        y = torch.full((N, (H + 1) // 2, (W + 1) // 2, C), float('nan'), device=x.device)
        nat.check(lib.nlt_pool2x2_fwd(nat.ptr(x), N, H, W, C, kind, nat.ptr(y), nat.stream()))
        return y
    nat.check(lib.nlt_pool2x2_bwd(nat.ptr(x), nat.ptr(d_y), N, H, W, C, kind, beta, nat.ptr(mask),
                                  2 if mask is not None else 0, nat.ptr(d_x), nat.stream()))
    return d_x


def run_up(x, d_y=None, beta=0.0, mask=None, d_x=None):
    nat = _lib()
    lib = nat.lib()
    if d_y is None:
        N, H, W, C = x.shape
        y = torch.full((N, 2 * H, 2 * W, C), float('nan'), device=x.device)
        nat.check(lib.nlt_upsample2x_bilinear_fwd(nat.ptr(x), N, H, W, C, nat.ptr(y), nat.stream()))
        return y
    N, H, W, C = d_x.shape
    nat.check(lib.nlt_upsample2x_bilinear_bwd(nat.ptr(d_y), N, H, W, C, beta, nat.ptr(mask),
                                              2 if mask is not None else 0, nat.ptr(d_x), nat.stream()))
    return d_x


def max_bwd_emulation(x, d_y, beta, mask, old):
    """fp32 emulation of the max-pool adjoint: d_y to the first maximum, (g + beta * old) * act'(mask)."""
    N, H, W, C = x.shape
    arg = P.first_argmax(x)
    g = torch.zeros((4,) + tuple(arg.shape), dtype=torch.float32, device=x.device)
    g.scatter_(0, arg.unsqueeze(0), d_y.unsqueeze(0))
    Ho, Wo = arg.shape[1], arg.shape[2]
    full = torch.zeros((N, 2 * Ho, 2 * Wo, C), dtype=torch.float32, device=x.device)
    for t in range(4):
        full[:, t >> 1::2, t & 1::2] = g[t]
    v = full[:, :H, :W]
    if beta:
        v = v + beta * old
    if mask is not None:
        v = v * _mask_of(mask)
    return v


SHAPES = [(2, 8, 8, 16), (3, 7, 5, 3), (1, 9, 10, 40), (2, 5, 6, 1024), (1, 1, 1, 4), (2, 33, 17, 16)]


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('epilogue', ['plain', 'beta_mask'])
def test_ops_against_fp64(shape, epilogue):
    dev = torch.device('cuda')
    g0 = torch.Generator(device='cpu').manual_seed(sum(shape))
    x = (torch.randn(shape, generator=g0) + 0.2).to(dev)
    x[..., 0] = torch.round(x[..., 0] * 2)           # exact ties in one channel
    if shape[3] > 1:
        x[0, :2, :2, 1] = 0.5                         # an all-equal window
    beta = 1.0 if epilogue == 'beta_mask' else 0.0
    stats = {}
    N, H, W, C = shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    x64 = x.double()
    # ---- pools, forward ----
    y = run_pool(x, MAX)
    assert torch.equal(y, P.max_pool_same(x)), 'max pool forward is not the fp32 maximum'
    y = run_pool(x, AVG)
    stats['avg_fwd'] = r_of(y, P.avg_pool_same(x64), P.avg_pool_same(x64.abs()))
    # ---- pools, backward ----
    d_y = torch.randn((N, Ho, Wo, C), generator=g0).to(dev)
    old = torch.randn(shape, generator=g0).to(dev) if beta else None
    mask = x if beta else None
    d_x = old.clone() if beta else torch.full(shape, float('nan'), device=dev)
    got = run_pool(x, MAX, d_y, beta, mask, d_x)
    want = max_bwd_emulation(x, d_y, beta, mask, old)
    assert torch.equal(got, want), 'max pool backward (beta %g) differs from the fp32 emulation' % beta
    d_x = old.clone() if beta else torch.full(shape, float('nan'), device=dev)
    got = run_pool(x, AVG, d_y, beta, mask, d_x)
    m64 = _mask_of(x).double() if beta else 1.0
    ref = adjoint(P.avg_pool_same, shape, d_y.double())
    absr = adjoint(P.avg_pool_same, shape, d_y.double().abs())
    if beta:
        ref, absr = ref + old.double(), absr + old.double().abs()
    stats['avg_bwd'] = r_of(got, ref * m64, absr * m64)
    # ---- upsample ----
    y = run_up(x)
    stats['up_fwd'] = r_of(y, up_ref(x64), up_ref(x64.abs()))
    d_y = torch.randn((N, 2 * H, 2 * W, C), generator=g0).to(dev)
    d_x = old.clone() if beta else torch.full(shape, float('nan'), device=dev)
    got = run_up(None, d_y, beta, mask, d_x)
    ref = adjoint(up_ref, shape, d_y.double())
    absr = adjoint(up_ref, shape, d_y.double().abs())
    if beta:
        ref, absr = ref + old.double(), absr + old.double().abs()
    stats['up_bwd'] = r_of(got, ref * m64, absr * m64)
    # ---- two runs are bit-identical ----
    d_x2 = old.clone() if beta else torch.full(shape, float('nan'), device=dev)
    assert torch.equal(run_up(None, d_y, beta, mask, d_x2), got)
    assert all(v <= OP_BAR for v in stats.values()), stats


def test_ops_at_production_size_past_32bit_offsets():
    """C = 160 at 1024 x 1024, batch 8: 5.4 GB of input, byte offsets far past 2^32."""
    dev = torch.device('cuda')
    N, H, W, C = 8, 1024, 1024, 160
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.randn((N, H, W, C), generator=g, device=dev)
    stats = {}
    y = run_pool(x, MAX)
    for n in (0, N - 1):
        assert torch.equal(y[n], P.max_pool_same(x[n:n + 1])[0])
    d_y = torch.randn(y.shape, generator=g, device=dev)
    d_x = torch.full_like(x, float('nan'))
    run_pool(x, MAX, d_y, 0.0, None, d_x)
    for n in (0, N - 1):
        assert torch.equal(d_x[n:n + 1], max_bwd_emulation(x[n:n + 1], d_y[n:n + 1], 0.0, None, None))
    y = run_pool(x, AVG)
    stats['avg_fwd'] = max(r_of(y[n:n + 1], P.avg_pool_same(x[n:n + 1].double()),
                                P.avg_pool_same(x[n:n + 1].double().abs())) for n in (0, N - 1))
    del y, d_y, d_x
    xs = x[:, :512, :512].contiguous()              # the upsample writes 4x its input
    del x
    torch.cuda.empty_cache()
    y = run_up(xs)
    stats['up_fwd'] = max(r_of(y[n:n + 1], up_ref(xs[n:n + 1].double()), up_ref(xs[n:n + 1].double().abs()))
                          for n in (0, N - 1))
    d_y = torch.randn(y.shape, generator=g, device=dev)
    del y
    mask = torch.randn(xs.shape, generator=g, device=dev)
    old = torch.randn(xs.shape, generator=g, device=dev)
    d_x = old.clone()
    run_up(None, d_y, 1.0, mask, d_x)
    for n in (0, N - 1):
        ref = adjoint(up_ref, (1, 512, 512, C), d_y[n:n + 1].double()) + old[n:n + 1].double()
        absr = adjoint(up_ref, (1, 512, 512, C), d_y[n:n + 1].double().abs()) + old[n:n + 1].double().abs()
        m = _mask_of(mask[n:n + 1]).double()
        stats['up_bwd_%d' % n] = r_of(d_x[n:n + 1], ref * m, absr * m)
    _record('pool_ops_large', stats)
    assert all(v <= OP_BAR for v in stats.values()), stats


def test_ops_reject_bad_arguments():
    nat = _lib()
    x = torch.zeros(1, 4, 4, 4, device='cuda')
    y = torch.zeros(1, 2, 2, 4, device='cuda')
    assert nat.lib().nlt_pool2x2_fwd(nat.ptr(x), 1, 4, 4, 4, 7, nat.ptr(y), nat.stream()) != 0
    assert nat.lib().nlt_upsample2x_bilinear_fwd(nat.ptr(x), 1, 0, 4, 4, nat.ptr(y), nat.stream()) != 0


# ------------------------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------------------------
class _MaskedAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask):
        ctx.save_for_backward(mask)
        return torch.where(x > 0, x, 0.3 * x)

    @staticmethod
    def backward(ctx, g):
        (mask,) = ctx.saved_tensors
        return g * torch.where(mask, 1.0, 0.3).to(g.dtype), None


def _product(monkeypatch, over, B, seed, tc):
    """Runs one train step of a pooling model; returns it with the product's LeakyReLU branch masks (per conv / norm)
    and the argmax of every max pool, taken from the pre-pool tensor the pool read."""
    import engine
    import nlt_native as nat
    from util import synth
    with nat.options(tc=tc):
        m, cfg = make_model(**over)
        oc = ocfg(cfg)
        bt = synth.make_batch(B, oc['uvh'], oc['imh'], seed=seed)
        params = P.init_params(oc, seed=7, dtype=torch.float64)
        m.build(5, 3)
        m.load_params(params)
        masks, args = {}, {}
        conv_fwd, norm_fwd, pool_fwd = engine.ConvLayer.forward, engine.NormLayer.forward, engine.PoolLayer.forward

        def tap(layer, out):
            if layer.act is not None:
                masks[layer.name.split(' ')[0].replace('.norm', '')] = (out.t > 0).cpu()
            return out
        monkeypatch.setattr(engine.ConvLayer, 'forward', lambda self, segs, tape=None: tap(self, conv_fwd(self, segs, tape)))
        monkeypatch.setattr(engine.NormLayer, 'forward', lambda self, x, tape=None: tap(self, norm_fwd(self, x, tape)))

        def pool_forward(self, x, tape=None):
            if self.kind == 'max':
                args[self.name.split(' ')[0]] = P.first_argmax(x.t).cpu()
            return pool_fwd(self, x, tape)
        monkeypatch.setattr(engine.PoolLayer, 'forward', pool_forward)
        try:
            pred, gt, kw, _ = m(bt, mode='train')
            kw['keep_batch'] = True
            m.set_loss_grad_scale(1.0 / B)
            m.compute_loss(pred, gt, **kw)
            m.backward()
            torch.cuda.synchronize()
        finally:
            monkeypatch.undo()
    return m, oc, bt, params, masks, args, pred


def _oracle(params, oc, bt, B, masks=None, args=None, monkeypatch=None):
    ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    bt64 = tuple(t.double() if torch.is_tensor(t) else t for t in bt)
    flips = {'act_flipped': 0, 'act_total': 0, 'argmax_flipped': 0, 'argmax_total': 0}
    if masks is not None:
        def act(x, type_, key):
            mk = masks[key]
            flips['act_flipped'] += int(((x.detach() > 0) != mk).sum())
            flips['act_total'] += mk.numel()
            return _MaskedAct.apply(x, mk)

        def pool(x, kind, key):
            if kind != 'max':
                return P.avg_pool_same(x)
            a = args[key]
            flips['argmax_flipped'] += int((P.first_argmax(x) != a).sum())
            flips['argmax_total'] += a.numel()
            return P.max_pool_same(x, a)
        monkeypatch.setattr(P, '_act', act)
        monkeypatch.setattr(P, '_pool', pool)
    try:
        pred, gt = P.model_call(ps, oc, bt64, 'train')
        (O.l2_loss(gt, pred, keep_batch=True).sum() / B).backward()
    finally:
        if monkeypatch is not None:
            monkeypatch.undo()
    return pred.detach(), {k: v.grad for k, v in ps.items()}, flips


@pytest.mark.parametrize('pool', ['max', 'avg'])
@pytest.mark.parametrize('norm', ['None', 'pixel'])
@pytest.mark.parametrize('tc', [0, 1])
def test_pool_model_against_the_oracle(pool, norm, tc, monkeypatch):
    B = 2
    over = dict(uvh=64, uvw=64, imh=64, imw=64, stride=1, pool=pool, norm=norm)
    m, oc, bt, params, masks, args, pred = _product(monkeypatch, over, B, 1234, tc)
    p64, g_masked, flips = _oracle(params, oc, bt, B, masks, args, monkeypatch)
    _, g_plain, _ = _oracle(params, oc, bt, B)
    grads = m.export_grads()
    assert set(grads) == set(params)
    fwd = float((pred.double().cpu() - p64).abs().max())
    worst_masked = max((rel_fro(grads[k], g_masked[k]), k) for k in params)
    worst_plain = max((rel_fro(grads[k], g_plain[k]), k) for k in params)
    _record('pool_model_%s_%s_tc%d' % (pool, norm, tc), {
        'pred_max_abs': fwd, 'worst_rel_fro_masked': worst_masked, 'worst_rel_fro_plain': worst_plain, **flips})
    if tc == 0:
        assert fwd <= 5e-5, fwd
    else:
        assert fwd <= 2e-4, fwd
    assert worst_masked[0] <= 1e-4, (worst_masked, flips)
    assert worst_plain[0] <= 3e-3, (worst_plain, flips)


def test_infer_with_broadcast_override_equals_the_tiled_override():
    """Test mode (nlt_test.py): a batch-1 observation override is upsampled once as a broadcast segment (batch 1, bit
    for bit the upsample of each image of the tiled override), and the prediction equals the run with the override
    tiled to the batch.  The convs may pick a different kernel for a broadcast segment than for a full one, so the two
    predictions are compared at fp32 round-off rather than bit for bit."""
    import nlt_test
    from util import synth
    m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64, stride=1, pool='max')
    m.build(5, 3)
    _bias_init(m)
    bt = synth.make_batch(3, 64, 64, seed=21)
    bt = tuple(t.cuda() if torch.is_tensor(t) else t for t in bt)
    feat = nlt_test.extract_feat(m, [bt], 1)
    assert all(f.shape[0] == 1 for f in feat)
    for f in feat[1:]:
        up1 = run_up(f.contiguous())
        up3 = run_up(f.expand(3, -1, -1, -1).contiguous())
        assert up1.shape[0] == 1 and all(torch.equal(up1[0], up3[i]) for i in range(3))
    a = m.call(bt, 'test', obs_override=feat)[0]
    b = m.call(bt, 'test', obs_override=[f.expand(3, -1, -1, -1).contiguous() for f in feat])[0]
    torch.cuda.synchronize()
    assert float((a - b).abs().max()) <= 1e-6 * max(1.0, float(b.abs().max()))


# ------------------------------------------------------------------------------------------------------------------
# production shape: one eager step, every launch against fp64
# ------------------------------------------------------------------------------------------------------------------
POOL_WL = dict(uv=1024, c_extra=0, depth=256, kernel=2, k_obs=1, batch=8, train=True)


def pool_config(wl, pool):
    from util import io as ioutil
    uv = wl['uv']
    return ioutil.make_config(uvh=uv, uvw=uv, imh=uv, imw=uv, loss='l2', depth0=16, depth=wl['depth'],
                              kernel=wl['kernel'], stride=1, pool=pool)


class PoolCensus(Census):
    """The census of tests/test_gpu_census.py with the pool and the upsample as gradient consumers: a conv output that
    feeds a pool receives the pool's adjoint of the pooled tensor's gradient; a tensor that feeds an upsample receives
    the upsample's adjoint of the upsampled tensor's gradient.  The forward of both ops is checked element by element."""

    def __init__(self, monkeypatch):
        import engine
        from networks import convnet
        super().__init__(monkeypatch)
        self.ops = {}
        census = self
        orig_pool, orig_up = engine.PoolLayer.forward, engine.upsample2x

        def pool_forward(layer, x, tape=None):
            y = orig_pool(layer, x, tape)
            name = layer.name.split(' ')[0]
            idx = _imgs(x.t.shape[0])
            xi = x.t[idx]
            if layer.kind == 'max':
                ok = torch.equal(y.t[idx], P.max_pool_same(xi))
                census.ops['fwd ' + name] = {'r': 0.0 if ok else float('inf')}
                arg = P.first_argmax(x.t)
            else:
                census.ops['fwd ' + name] = {'r': r_of(y.t[idx], P.avg_pool_same(xi.double()),
                                                       P.avg_pool_same(xi.double().abs()))}
                arg = None
            census.consumers[id(x)].append(('pool', layer.kind, arg, y))
            census.keep += [x, y]
            return y

        def upsample(a, tape=None):
            y = orig_up(a, tape)
            idx = _imgs(a.t.shape[0])
            ai = a.t[idx].double()
            n = sum(1 for k in census.ops if k.startswith('fwd upsample'))
            census.ops['fwd upsample%d %s' % (n, tuple(a.t.shape))] = {
                'r': r_of(y.t[idx], up_ref(ai), up_ref(ai.abs()))}
            census.consumers[id(a)].append(('up', y))
            census.keep += [a, y]
            return y
        monkeypatch.setattr(engine.PoolLayer, 'forward', pool_forward)
        monkeypatch.setattr(convnet, 'upsample2x', upsample)

    def adjoint(self, a, idx):
        """fp64 (ref, |.|, 1xTF32, 3xTF32 - a_lo b_hi) of the gradient every consumer sends to Act `a`, images idx."""
        N, Hin, Win, C = a.t.shape
        shape = (len(idx), Hin, Win, C)
        out = None
        for c in self.consumers[id(a)]:
            if c[0] == 'conv':
                _, L, coff, Cs = c
                dz = torch.cat([self.dz[id(L)][i] for i in idx], 0)
                f = lambda d, w, L=L, coff=coff, Cs=Cs: vjp_input(L.kind, L.s, d, w, Hin, Win, L.cin)[..., coff:coff + Cs]
                terms = [f(dz.double(), L.kernel.double()), f(dz.double().abs(), L.kernel.double().abs())]
                terms += list(controls(f, dz, L.kernel))
            elif c[0] == 'kmean':
                _, K, agg = c
                terms = [t / K for t in self.adjoint(agg, [i % agg.t.shape[0] for i in idx])]
            elif c[0] == 'pool':
                _, kind, arg, y = c
                if kind == 'max':
                    ai = arg[idx]
                    op = lambda z, ai=ai: P.max_pool_same(z, ai)
                else:
                    op = P.avg_pool_same
                terms = [adjoint(op, shape, t) for t in self.adjoint(y, idx)]
            else:
                terms = [adjoint(up_ref, shape, t) for t in self.adjoint(c[1], idx)]
            out = terms if out is None else [o + t for o, t in zip(out, terms)]
        return out


def test_census_of_a_pool_training_step(monkeypatch):
    """One eager step of the dragon_specular network with stride 1 and `pool = max` at UV 1024^2, batch 8 (5 / 3 input
    channels), allocations NaN-poisoned: every conv launch against fp64 at the census bars, and the pool / upsample
    forward at 2^-22.  The pool and upsample adjoints are checked through the input gradients of the convs in front of
    them.  Records the kernel routes the library picks for the stride-1 convs."""
    import models
    from util import synth
    t0 = time.perf_counter()
    B, uv = POOL_WL['batch'], POOL_WL['uv']
    model = models.get_model_class('nlt')(pool_config(POOL_WL, 'max'))
    model.register_trainable()
    model.build(5, 3)
    _bias_init(model)
    bt = synth.make_batch(B, uv, uv, seed=1235)
    bt = tuple(t.to(model.device) if torch.is_tensor(t) else t for t in bt)
    torch.cuda.synchronize()
    census = PoolCensus(monkeypatch)
    poison_workspaces()
    model.flat_grads.fill_(float('nan'))
    with monkeypatch.context() as mp:
        poisoned_allocations(mp)
        pred, gt, kw, to_vis = model(bt, mode='train')
        kw['keep_batch'] = True
        model.set_loss_grad_scale(1.0 / B)
        model.compute_loss(pred, gt, **kw)
        census.set_tail_reference(to_vis['pred'], gt, bt[4], uv, model._d_pred, 1.0 / B)
        model.backward()
    torch.cuda.synchronize()
    census.finish_wgrad()
    torch.cuda.synchronize()
    routes = census.route_table()
    rec = {'uv': uv, 'batch': B, 'pool': 'max', 'stride': 1, 'seconds': time.perf_counter() - t0,
           'fwd': census.fwd, 'dgrad': census.dgrad, 'wgrad': census.wgrad, 'ops': census.ops, 'tail': census.tail,
           'routes': routes, 'peak_mem_GB': torch.cuda.max_memory_allocated() / 1e9}
    _record('census_pool_max', rec)
    bad = []
    for kind, table in (('fwd', rec['fwd']), ('dgrad', rec['dgrad']), ('wgrad', rec['wgrad'])):
        for layer, st in table.items():
            bar = TAU_TC_WGRAD if kind == 'wgrad' and 'tc_wgrad_kernel' in routes[layer].get('wgrad', {}) else TAU
            for key in ('r', 'r_bias'):
                if key in st and not st[key] <= bar:
                    bad.append('%s %s %s = %.3g (bar %.3g)' % (kind, layer, key, st[key], bar))
    for name, st in rec['ops'].items():
        if not st['r'] <= OP_BAR:
            bad.append('%s r = %.3g' % (name, st['r']))
    assert rec['tail'] is not None and rec['tail']['r'] <= TAU, rec['tail']
    assert not bad, '\n'.join(bad)
    n_conv = len(rec['fwd'])
    assert n_conv == len(rec['wgrad']) == len(model.named_convs()), (n_conv, len(rec['wgrad']))
    # the input gradient of every conv in front of a pool or an upsample went through those adjoints
    assert 'query.1.1' in rec['dgrad'] and 'query.6.1' in rec['dgrad'] and 'query.7.0' in rec['dgrad']
    # 12 pools (6 query + 6 observation blocks); 17 upsamples: the first up block upsamples its two distinct sources,
    # the other five three each
    assert len([k for k in rec['ops'] if 'pool' in k]) == 12 and len(rec['ops']) == 12 + 17, sorted(rec['ops'])


# ------------------------------------------------------------------------------------------------------------------
# the graphed step
# ------------------------------------------------------------------------------------------------------------------
def test_graph_replays_of_a_pool_step_equal_eager_and_fp64(monkeypatch):
    """Three replays (b0, b1, b0) of trainvali.GraphedTrainStep for `pool = max` at UV 1024^2, batch 8: bit-identical
    to the graph's body run eagerly from the restored state, and within the bars of tests/test_gpu_graph_step.py."""
    import tests.test_gpu_graph_step as G
    import trainvali
    from util import synth

    class _PoolArm(G._Arm):
        def __init__(self, B):
            import models
            self.B, self.uv = B, POOL_WL['uv']
            self.model = models.get_model_class('nlt')(pool_config(POOL_WL, 'max'))
            self.model.register_trainable()
            self.model.build(5, 3)
            _bias_init(self.model)
            self.opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
            self.host = [synth.make_batch(B, self.uv, self.uv, seed=1235 + i, pin=True) for i in range(2)]
            dev = self.model.device
            self.dev = [tuple(t.to(dev) if torch.is_tensor(t) else t for t in b) for b in self.host]
            self.step = trainvali.GraphedTrainStep(trainvali.Strategy(), self.model, self.opt, B)

    B = POOL_WL['batch']
    a = _PoolArm(B)
    with monkeypatch.context() as mp:
        G._poison(mp)
        a.step._capture(a.dev[0])
    assert a.step.full_step_in_graph
    init = a.state()
    seq = [0, 1, 0]
    graph_out, stats = [], []
    for t, bi in enumerate(seq, 1):
        before = a.state()
        loss, to_vis = a.step(a.step.static_batch if t == 1 else a.dev[bi])
        torch.cuda.synchronize()
        out = a.outputs(loss, to_vis)
        stats.append(G.fp64_checks(out, before, a.dev[bi], t, B))
        graph_out.append(out)
    a.restore(init)
    with monkeypatch.context() as mp:
        G._poison(mp)
        for t, bi in enumerate(seq, 1):
            poison_workspaces()
            loss, to_vis = a.step._body(a.dev[bi], with_update=True)
            torch.cuda.synchronize()
            G._equal(graph_out[t - 1], a.outputs(loss, to_vis), 'pool replay %d vs eager' % t)
    _record('graph_pool_max', {'batch': B, 'max_r': {k: max(s[k] for s in stats) for k in stats[0]},
                               'peak_mem_GB': torch.cuda.max_memory_allocated() / 1e9})
