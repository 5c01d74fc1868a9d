"""Census of the benchmarked training step: every conv launch of one eager step, at the shapes bench.py times, checked
element by element against fp64, with a pinned record of which kernels serve each layer.

Metric.  For an output element, r = |got - ref| / (abs_ref + tiny), where ref is the fp64 op applied to the product's
own fp32 operands and abs_ref the same op applied to their magnitudes (|x|, |w|, |dz|), summed over every term that
reaches the element.  fp32 accumulation stays within a few 2^-24 * sqrt(K) of abs_ref; a 3xTF32 product that drops
one of its cross terms, or a 1xTF32 product, is off by ~2^-12 per product.  The bar is on max r per op (TAU).

What a step is checked for (one eager `model(bt, 'train')`, `compute_loss`, `backward()` per arm):
 * forward: every conv output (after its activation) for images {0, N-1};
 * input gradient: the final, accumulated gradient of every conv output (the `dz` its producer reads) against
   mask(y) * sum over consumers of the adjoint of the consumer's own `dz` (conv consumers and the K-mean), images
   {0, N-1} -- this covers beta = 1 accumulation, the activation mask and the fused / parked final-conv term;
 * weight and bias gradient: the whole tensor, reference accumulated over all images;
 * the tail once: the final conv's `dz` against the fp64 L2 gradient of the product's own UV prediction pulled back
   through the resampler.
Every float32 CUDA allocation made by the engine during the step comes back filled with NaN, and so do the weight
gradient buffer and the scratch workspaces, so an element no kernel writes fails the check.

Routes: per (layer, op) the library kernels that launched, as `nlt_kernel_launch_count` deltas, against the tables in
tests/census_routes/<arm>.json.  `NLT_UPDATE_ROUTES=1` rewrites the tables.
"""
import collections
import glob
import json
import math
import os
import re
import sys
import time

import pytest
import torch

from oracle import nlt_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'neural-light-transport_b200', 'csrc')
ROUTES_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'census_routes')

TAU = 2.0 ** -15          # bar on max r for the forward, input-gradient and weight-gradient ops
TINY = 2.0 ** -126        # smallest normal fp32: only an exact zero reference asks for an exact zero
PERTURB = 1e-3            # size of the single-element perturbation control, in units of rms(ref)
# The UV-space tail scatters through 64-bit fixed point whose quantum is 2^-37 of the batch's largest |d pred|
# (nlt_ops.cu fixed_scale); its error is absolute, so its floor is that quantum with 2^7 to spare.
TAIL_FLOOR = 2.0 ** -30
# Weight gradients served by the wgmma kernel (tc_wgrad_kernel) measure up to 3.7 * TAU on an H100 (cfg4k3's 3x3
# stride-1 convs; 0.6-0.8 * TAU at the 2x2 shapes), more than a 1xTF32 emulation of the same op (0.1-1.4 * TAU) and
# 70x the fp32 route (<= 0.011 * TAU).  Until that kernel is brought back to 3xTF32 accuracy its bar is 16 * TAU:
# 4x over the worst measurement, still 2x below the single-element perturbation control there (>= 22 * TAU).
TAU_TC_WGRAD = 2.0 ** -11


# ----------------------------------------------------------------------------------------------------------------
# the metric and its controls (device-agnostic)
# ----------------------------------------------------------------------------------------------------------------
def max_rel(got, ref, abs_ref, tiny=TINY):
    """max over elements of |got - ref| / (abs_ref + tiny); a non-finite element of `got` counts as infinity."""
    if ref.numel() == 0:
        return 0.0
    got = got.to(ref.device, torch.float64)
    r = (got - ref).abs() / (abs_ref + tiny)
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))
    return float(r.max())


def tf32_round(x):
    """fp32 -> nearest TF32 (10 explicit mantissa bits, ties away from zero) by bit operations, as the kernels'
    tf32_round (nlt_common.cuh)."""
    b = x.to(torch.float32).contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def controls(f, a, b):
    """Negative controls of the bilinear op f(a, b) (a: the activation / gradient operand, b: the other one), products
    in fp64: (1xTF32: both operands rounded to TF32, 3xTF32 without its a_lo * b_hi term: a_hi (b_hi + b_lo))."""
    a_hi, b_hi = tf32_round(a), tf32_round(b)
    b_lo = tf32_round(b - b_hi)
    return (f(a_hi.double(), b_hi.double()),
            f(a_hi.double(), b_hi.double() + b_lo.double()))


def three_tf32(f, a, b):
    """The full 3xTF32 product a_hi b_hi + a_hi b_lo + a_lo b_hi (fp64 sums)."""
    a_hi, b_hi = tf32_round(a), tf32_round(b)
    a_lo, b_lo = tf32_round(a - a_hi), tf32_round(b - b_hi)
    a_hi, b_hi, a_lo, b_lo = (t.double() for t in (a_hi, b_hi, a_lo, b_lo))
    return f(a_hi, b_hi) + f(a_hi, b_lo) + f(a_lo, b_hi)


def perturbed_r(ref, abs_ref, tiny=TINY):
    """r of the reference with ONE element moved by PERTURB * rms(ref): the element of median abs_ref."""
    if ref.numel() == 0:
        return math.inf
    flat = abs_ref.reshape(-1)
    med = float(flat.kthvalue(max(1, (flat.numel() + 1) // 2)).values)
    rms = float(ref.pow(2).mean().sqrt())
    return PERTURB * rms / (med + tiny)


def conv_fn(kind):
    return O.conv2d_same if kind == 'conv' else O.conv2d_transpose_same


def vjp_input(kind, s, dz, w, Hin, Win, cin):
    """Adjoint of the SAME conv / transposed conv with respect to its input (bilinear in dz, w)."""
    x0 = torch.zeros(dz.shape[0], Hin, Win, cin, dtype=dz.dtype, device=dz.device, requires_grad=True)
    return torch.autograd.grad(conv_fn(kind)(x0, w, None, s), x0, dz)[0]


def vjp_weight(kind, s, x, dz, wshape):
    """Gradient of the SAME conv / transposed conv with respect to its kernel (bilinear in x, dz)."""
    w0 = torch.zeros(wshape, dtype=x.dtype, device=x.device, requires_grad=True)
    return torch.autograd.grad(conv_fn(kind)(x, w0, None, s), w0, dz)[0]


def op_stats(got, ref, abs_ref, ctl, tiny=TINY):
    """{'r', 'r_1xtf32', 'r_3xtf32_no_lohi', 'r_perturbed'} of one checked op."""
    out = {'r': max_rel(got, ref, abs_ref, tiny), 'r_perturbed': perturbed_r(ref, abs_ref, tiny)}
    if ctl is not None:
        out['r_1xtf32'] = max_rel(ctl[0], ref, abs_ref, tiny)
        out['r_3xtf32_no_lohi'] = max_rel(ctl[1], ref, abs_ref, tiny)
    return out


# ----------------------------------------------------------------------------------------------------------------
# CPU: the metric separates fp32 / full 3xTF32 from the three controls
# ----------------------------------------------------------------------------------------------------------------
def _cpu_case(op):
    """(f, a, b) of a small 2x2 / stride-2 conv and its two adjoints, seeded; a, b fp32."""
    g = torch.Generator().manual_seed({'fwd': 1, 'dgrad': 2, 'wgrad': 3}[op])
    N, H, W, ci, co = 2, 10, 12, 16, 16
    x = torch.rand(N, H, W, ci, generator=g) * 2 - 1
    w = (torch.rand(2, 2, ci, co, generator=g) * 2 - 1) * math.sqrt(6.0 / (4 * (ci + co)))
    dz = torch.randn(N, H // 2, W // 2, co, generator=g) * 1e-3
    if op == 'fwd':
        return (lambda a, b: O.conv2d_same(a, b, None, 2)), x, w
    if op == 'dgrad':
        return (lambda a, b: vjp_input('conv', 2, a, b, H, W, ci)), dz, w
    return (lambda a, b: vjp_weight('conv', 2, a, b, (2, 2, ci, co))), x, dz


@pytest.mark.parametrize('op', ['fwd', 'dgrad', 'wgrad'])
def test_metric_passes_fp32_and_full_3xtf32(op):
    f, a, b = _cpu_case(op)
    ref, absr = f(a.double(), b.double()), f(a.double().abs(), b.double().abs())
    assert max_rel(f(a, b), ref, absr) <= TAU / 4          # plain fp32 (torch CPU)
    assert max_rel(three_tf32(f, a, b), ref, absr) <= TAU / 4


@pytest.mark.parametrize('op', ['fwd', 'dgrad', 'wgrad'])
def test_metric_flags_tf32_controls(op):
    f, a, b = _cpu_case(op)
    ref, absr = f(a.double(), b.double()), f(a.double().abs(), b.double().abs())
    one, no_lohi = controls(f, a, b)
    assert max_rel(one, ref, absr) >= 2 * TAU
    assert max_rel(no_lohi, ref, absr) >= 2 * TAU


@pytest.mark.parametrize('op', ['fwd', 'dgrad', 'wgrad'])
def test_metric_flags_one_perturbed_element_that_frobenius_misses(op):
    f, a, b = _cpu_case(op)
    ref, absr = f(a.double(), b.double()), f(a.double().abs(), b.double().abs())
    flat = absr.reshape(-1)
    i = int(flat.kthvalue(max(1, (flat.numel() + 1) // 2)).indices)
    bad = ref.clone().reshape(-1)
    bad[i] += PERTURB * float(ref.pow(2).mean().sqrt())
    bad = bad.reshape(ref.shape)
    assert float((bad - ref).norm() / ref.norm()) < 1e-4      # invisible to a 1e-4 relative Frobenius bar
    assert max_rel(bad, ref, absr) >= 2 * TAU
    assert max_rel(bad, ref, absr) == pytest.approx(perturbed_r(ref, absr), rel=1e-9)


def test_metric_counts_unwritten_elements():
    f, a, b = _cpu_case('fwd')
    ref, absr = f(a.double(), b.double()), f(a.double().abs(), b.double().abs())
    got = f(a, b)
    got[-1, -1, -1, -1] = float('nan')
    assert max_rel(got, ref, absr) == math.inf


def test_tf32_round_matches_the_kernels_bit_trick():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -11, -3.0000002, 2 ** -20 * 1.37], dtype=torch.float32)
    r = tf32_round(x)
    assert (r.view(torch.int32) & 0x1FFF).eq(0).all()
    assert ((r - x).abs() <= x.abs() * 2 ** -11).all()
    assert float(r[1]) == 1.0 + 2 ** -10                   # ties away from zero


# ----------------------------------------------------------------------------------------------------------------
# GPU census
# ----------------------------------------------------------------------------------------------------------------
def kernel_labels():
    """Every kernel label the library counts (NLT_CUDA_LAUNCH_CHECK("...") in csrc/)."""
    labels = set()
    for path in glob.glob(os.path.join(CSRC, '*.cu')) + glob.glob(os.path.join(CSRC, '*.cuh')):
        with open(path) as f:
            labels.update(re.findall(r'NLT_CUDA_LAUNCH_CHECK\("([^"]+)"\)', f.read()))
    return sorted(labels)


def _record(name, obj):
    """Writes the per-op table next to the parity records (tests/test_gpu_parity.py), as parity_census_<name>.json."""
    from tests.test_gpu_parity import _record as parity_record
    parity_record('census_' + name, obj)


def _imgs(n):
    return sorted({0, n - 1})


def _short(layer):
    return layer.name.split(' ')[0]


def _materialize(segs, idx):
    """The virtual concat of `segs` for images idx: (exact fp64 input, the fp32 values a kernel reads, fp64 |input|).
    A `sub` segment is a - sub (fp32 difference in the kernel, exact here); a broadcast segment repeats image 0."""
    ex, f32, mag = [], [], []
    for sg in segs:
        t = sg.a.t
        sel = t[[0] * len(idx)] if sg.bcast else t[idx]
        if sg.sub is not None:
            s = sg.sub[idx]
            ex.append(sel.double() - s.double())
            f32.append(sel - s)
            mag.append(sel.double().abs() + s.double().abs())
        else:
            ex.append(sel.double())
            f32.append(sel)
            mag.append(sel.double().abs())
    return torch.cat(ex, 3), torch.cat(f32, 3), torch.cat(mag, 3)


def _mask(y, act):
    if act is None:
        return None
    assert act == 'leakyrelu', act
    return torch.where(y > 0, 1.0, 0.3).double()


def _act(z, act):
    return z if act is None else O.act(z, act)


def forward_check(layer, segs, y, idx):
    x, x32, xm = _materialize(segs, idx)
    w, b = layer.kernel, layer.bias
    f = lambda a, bb: conv_fn(layer.kind)(a, bb, None, layer.s)
    bias = b.double().view(1, 1, 1, -1)
    ref = f(x, w.double()) + bias
    absr = f(xm, w.double().abs()) + bias.abs()       # |act(u) - act(v)| <= |u - v|: the pre-activation scale bounds
    ctl = controls(f, x32, w)
    return op_stats(y.t[idx], _act(ref, layer.act), absr, [_act(c + bias, layer.act) for c in ctl])


def wgrad_terms(layer, segs, dz, chunk_bytes=1 << 30):
    """fp64 (ref, |.|, 1xTF32, 3xTF32 - a_lo b_hi) of the kernel gradient and (ref, |.|) of the bias gradient,
    accumulated over all images in chunks."""
    N = dz.shape[0]
    Hin, Win = next(sg.a.t for sg in segs if not sg.bcast).shape[1:3]
    per = max(1, chunk_bytes // (8 * Hin * Win * layer.cin))
    f = lambda a, d: vjp_weight(layer.kind, layer.s, a, d, tuple(layer.kernel.shape))
    acc = [torch.zeros(layer.kernel.shape, dtype=torch.float64, device=dz.device) for _ in range(4)]
    for i0 in range(0, N, per):
        idx = list(range(i0, min(N, i0 + per)))
        x, x32, xm = _materialize(segs, idx)
        d = dz[idx]
        acc[0] += f(x, d.double())
        acc[1] += f(xm, d.double().abs())
        c1, c3 = controls(lambda a, dd: f(a, dd), x32, d)
        acc[2] += c1
        acc[3] += c3
        del x, x32, xm
    dzd = dz.double()
    return acc, (dzd.sum(dim=(0, 1, 2)), dzd.abs().sum(dim=(0, 1, 2)))


class Census:
    """Hooks around ConvLayer.forward / ._backward, engine.contribute / settle and kmean (installed by monkeypatch)."""

    def __init__(self, monkeypatch, forward_only=False):
        import engine
        import nlt_native as nat
        self.engine, self.nat = engine, nat
        self.labels = kernel_labels()
        self.forward_only = forward_only
        self.fwd, self.dgrad, self.wgrad, self.tail = {}, {}, {}, None
        self.routes = collections.defaultdict(lambda: collections.defaultdict(collections.Counter))
        self.consumers = collections.defaultdict(list)   # id(Act) -> [('conv', layer, coff, C) | ('kmean', K, agg)]
        self.keep = []                                   # the Acts whose ids key the tables above
        self.dz = {}                                     # id(layer) -> {image: fp32 dz [1, H, W, Cout]}
        self.pending_w = []                              # (layer, terms) compared after the tape
        self.parked_by = {}
        self.ctx = None                                  # [layer name, Counter of dgrad launches inside its backward]
        self.last_conv = None
        self.tail_ref = None
        orig_fwd, orig_bwd = engine.ConvLayer.forward, engine.ConvLayer._backward
        orig_contrib, orig_settle, orig_kmean = engine.contribute, engine.settle, engine.kmean
        census = self

        def forward(layer, segs, tape=None):
            n0 = census.counts()
            y = orig_fwd(layer, segs, tape)
            census.routes[_short(layer)]['fwd'].update(census.delta(n0))
            census.on_forward(layer, segs, y)
            return y

        def _backward(layer, segs, y, N, Hin, Win):
            n0 = census.counts()
            outer, census.ctx = census.ctx, [_short(layer), collections.Counter()]
            try:
                engine.settle(y)
                if y.grad is not None:
                    census.on_backward(layer, segs, y)
                orig_bwd(layer, segs, y, N, Hin, Win)
                total = census.delta(n0)
                total.subtract(census.ctx[1])
                census.routes[_short(layer)]['wgrad'].update(+total)
            finally:
                census.ctx = outer

        def contribute(target, write_fn, offer=None, can_fuse=None):
            n0 = census.counts()
            was = target.pending
            orig_contrib(target, write_fn, offer, can_fuse)
            if was is None and target.pending is not None and census.ctx is not None:
                census.parked_by[id(target)] = census.ctx[0]
            census.attribute(census.ctx[0] if census.ctx is not None else None, census.delta(n0))

        def settle(a):
            owner = census.parked_by.get(id(a)) if a.pending is not None else None
            n0 = census.counts()
            orig_settle(a)
            census.attribute(owner, census.delta(n0))

        def kmean(obs_y, K, tape=None, weights=None):
            agg = orig_kmean(obs_y, K, tape, weights)
            if agg is not obs_y:
                assert weights is None
                census.consumers[id(obs_y)].append(('kmean', K, agg))
                census.keep.append(agg)
            return agg

        monkeypatch.setattr(engine.ConvLayer, 'forward', forward)
        monkeypatch.setattr(engine.ConvLayer, '_backward', _backward)
        monkeypatch.setattr(engine, 'contribute', contribute)
        monkeypatch.setattr(engine, 'settle', settle)
        monkeypatch.setattr(engine, 'kmean', kmean)
        monkeypatch.setattr(sys.modules['models.nlt'], 'kmean', kmean)

    # ---- launch counting ----
    def counts(self):
        return collections.Counter({k: self.nat.kernel_launch_count(k) for k in self.labels})

    def delta(self, n0):
        d = self.counts()
        d.subtract(n0)
        return +d

    def attribute(self, owner, d):
        if owner is None or not d:
            return
        self.routes[owner]['dgrad'].update(d)
        if self.ctx is not None:
            self.ctx[1].update(d)

    def route_table(self):
        return {layer: {op: dict(sorted(c.items())) for op, c in sorted(ops.items()) if c}
                for layer, ops in sorted(self.routes.items())}

    # ---- forward ----
    def on_forward(self, layer, segs, y):
        name = _short(layer)
        N = y.t.shape[0]
        self.fwd[name] = forward_check(layer, segs, y, _imgs(N))
        self.last_conv = layer
        coff = 0
        for sg in segs:
            if sg.a.needs_grad:
                self.consumers[id(sg.a)].append(('conv', layer, coff, sg.C))
            self.keep.append(sg.a)
            coff += sg.C
        self.keep.append(y)

    # ---- backward ----
    def adjoint(self, a, idx):
        """fp64 (ref, |.|, 1xTF32, 3xTF32 - a_lo b_hi) of the gradient every consumer sends to Act `a`, images idx."""
        N, Hin, Win, C = a.t.shape
        out = None
        for c in self.consumers[id(a)]:
            if c[0] == 'conv':
                _, L, coff, Cs = c
                dz = torch.cat([self.dz[id(L)][i] for i in idx], 0)
                f = lambda d, w, L=L, coff=coff, Cs=Cs: vjp_input(L.kind, L.s, d, w, Hin, Win, L.cin)[..., coff:coff + Cs]
                terms = [f(dz.double(), L.kernel.double()), f(dz.double().abs(), L.kernel.double().abs())]
                terms += list(controls(f, dz, L.kernel))
            else:
                _, K, agg = c
                B = agg.t.shape[0]
                terms = [t / K for t in self.adjoint(agg, [i % B for i in idx])]
            out = terms if out is None else [o + t for o, t in zip(out, terms)]
        return out

    def on_backward(self, layer, segs, y):
        name = _short(layer)
        dz = y.grad
        N = dz.shape[0]
        idx = _imgs(N)
        if layer is self.last_conv and self.tail_ref is not None:
            ref, absr, tiny = self.tail_ref
            self.tail = op_stats(dz[idx], ref, absr, None, tiny)
        elif self.consumers.get(id(y)):
            ref, absr, c1, c3 = self.adjoint(y, idx)
            m = _mask(y.t[idx], layer.act)
            if m is not None:
                ref, absr, c1, c3 = ref * m, absr * m, c1 * m, c3 * m
            st = op_stats(dz[idx], ref, absr, (c1, c3))
            st['consumers'] = [_short(c[1]) if c[0] == 'conv' else 'kmean' for c in self.consumers[id(y)]]
            self.dgrad[name] = st
        if any(sg.a.needs_grad for sg in segs):
            self.dz[id(layer)] = {i: dz[i:i + 1].clone() for i in idx}
        self.pending_w.append((layer, wgrad_terms(layer, segs, dz)))

    def finish_wgrad(self):
        for layer, (w, b) in self.pending_w:
            st = op_stats(layer.gkernel, w[0], w[1], (w[2], w[3]))
            st['r_bias'] = max_rel(layer.gbias, b[0], b[1])
            self.wgrad[_short(layer)] = st
        self.pending_w = []

    def set_tail_reference(self, pred_uv, gt_c, warp, uv, d_pred, scale):
        """fp64 d(net_out) of images {0, B-1}: L2 gradient at the resampled product prediction, pulled back through
        the resampler (the corner texel is multiplied by 0 in the forward)."""
        B = pred_uv.shape[0]
        idx = _imgs(B)
        p = pred_uv[idx].double().requires_grad_(True)
        wp = warp[idx].double()
        wp = torch.stack((wp[..., 0] * uv, wp[..., 1] * uv), dim=3)
        pc = O.resampler(p, wp)
        gt = gt_c[idx].double()
        n = pc[0].numel()
        d = 2.0 * (pc.detach() - gt) * scale / n
        dm = 2.0 * (pc.detach().abs() + gt.abs()) * scale / n
        ref = torch.autograd.grad(pc, p, d, retain_graph=True)[0]
        absr = torch.autograd.grad(pc, p, dm)[0]
        ref[:, 0, 0, :] = 0
        absr[:, 0, 0, :] = 0
        self.tail_ref = (ref, absr, TAIL_FLOOR * float(d_pred.abs().max()))


class poisoned_allocations:
    """float32 CUDA tensors from torch.empty / torch.empty_like come back NaN-filled while active."""

    def __init__(self, monkeypatch):
        real_empty, real_like = torch.empty, torch.empty_like

        def fill(t):
            if isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.is_cuda:
                t.fill_(float('nan'))
            return t
        monkeypatch.setattr(torch, 'empty', lambda *a, **k: fill(real_empty(*a, **k)))
        monkeypatch.setattr(torch, 'empty_like', lambda *a, **k: fill(real_like(*a, **k)))


def poison_workspaces():
    import engine
    todo = [engine._WS, engine._WS_SIDE]
    while todo:
        ws = todo.pop()
        if ws.buf is not None:
            ws.buf.fill_(float('nan'))
        for ch in ws.arena.chunks:
            ch.fill_(float('nan'))
        todo += list(ws.subs.values())


def check_routes(arm, got):
    path = os.path.join(ROUTES_DIR, '%s.json' % arm)
    if os.environ.get('NLT_UPDATE_ROUTES') == '1':
        os.makedirs(ROUTES_DIR, exist_ok=True)
        with open(path, 'w') as f:
            json.dump(got, f, indent=1, sort_keys=True)
            f.write('\n')
        return
    assert os.path.exists(path), 'no route table %s (NLT_UPDATE_ROUTES=1 writes it)' % path
    with open(path) as f:
        want = json.load(f)
    diff = []
    for layer in sorted(set(want) | set(got)):
        for op in sorted(set(want.get(layer, {})) | set(got.get(layer, {}))):
            w, g = want.get(layer, {}).get(op, {}), got.get(layer, {}).get(op, {})
            if w != g:
                diff.append('  %-11s %-5s expected %s\n  %-11s %-5s      got %s' % (layer, op, w, '', '', g))
    assert not diff, 'kernel routes of %s changed (NLT_UPDATE_ROUTES=1 rewrites %s):\n%s' % (
        arm, os.path.relpath(path, ROOT), '\n'.join(diff))


def _summary(c):
    out = {}
    for kind, table in (('fwd', c.fwd), ('dgrad', c.dgrad), ('wgrad', c.wgrad)):
        if not table:
            continue
        worst = max(table.items(), key=lambda kv: kv[1]['r'])
        out[kind] = {'max_r': worst[1]['r'], 'layer': worst[0], 'headroom_vs_tau': TAU / max(worst[1]['r'], 1e-300)}
        for ctl in ('r_1xtf32', 'r_3xtf32_no_lohi', 'r_perturbed'):
            low = min(table.items(), key=lambda kv: kv[1][ctl])
            out[kind]['min_' + ctl] = low[1][ctl]
            out[kind]['min_%s_layer' % ctl] = low[0]
            out[kind]['min_%s_over_max_r' % ctl] = low[1][ctl] / max(worst[1]['r'], 1e-300)
    if c.tail is not None:
        out['tail'] = {'max_r': c.tail['r']}
    return out


# arm -> (workload, batch, options).  The training arms run at bench.py's batch 8 where the step fits comfortably
# (a cfg4 step at batch 8 was estimated at ~15 GB from the 57 GB of batch 32; not measured): routes depend on the
# shape, so the measured batch is what pins the benchmarked routes.  cfg3 runs at batch 2 (bench: 16) -- with K = 6
# its observation stream already carries 12 full-resolution images, and its deep 1024-channel levels keep their
# shapes; cfg1 runs at batch 2 (bench: 1) so that the observation override is a broadcast segment.
ARMS = {
    'cfg4': ('cfg4', 8, {}),
    'cfg2': ('cfg2', 8, {}),
    'cfg4_tc0': ('cfg4', 8, {'tc': 0}),
    'cfg4k3': ('cfg4k3', 8, {}),
    'cfg3_b2': ('cfg3', 2, {}),
    'cfg1_b2': ('cfg1', 2, {}),
}


def _bias_init(model):
    """Keras starts biases at zero; small seeded biases make the bias paths count."""
    g = torch.Generator().manual_seed(11)
    for _, c in model.named_convs():
        c.bias.copy_((torch.rand(c.bias.shape, generator=g) * 2 - 1) * 0.1)


@pytest.mark.gpu
@pytest.mark.parametrize('arm', list(ARMS))
def test_census_of_the_benchmarked_step(arm, monkeypatch):
    import bench
    import models
    import nlt_native as nat
    import nlt_test
    from util import synth
    wl_name, B, opts = ARMS[arm]
    wl = bench.WORKLOADS[wl_name]
    uv = wl['uv']
    t0 = time.perf_counter()
    with nat.options(**opts):
        model = models.get_model_class('nlt')(bench.make_config(wl))
        model.register_trainable()
        model.build(5 + wl['c_extra'], 3)
        _bias_init(model)
        bt = synth.make_batch(B, uv, uv, seed=1235, c_extra=wl['c_extra'], k_obs=wl['k_obs'])
        dev = model.device
        bt = tuple(t.to(dev) if torch.is_tensor(t) else t for t in bt)
        feat = nlt_test.extract_feat(model, [bt], 1) if not wl['train'] else None
        torch.cuda.synchronize()
        census = Census(monkeypatch, forward_only=not wl['train'])
        poison_workspaces()
        model.flat_grads.fill_(float('nan'))
        with monkeypatch.context() as mp:
            poisoned_allocations(mp)
            if not wl['train']:
                model.call(bt, 'test', obs_override=feat)
            else:
                pred, gt, kw, to_vis = model(bt, mode='train')
                kw['keep_batch'] = True
                model.set_loss_grad_scale(1.0 / B)
                model.compute_loss(pred, gt, **kw)
                census.set_tail_reference(to_vis['pred'], gt, bt[4], uv, model._d_pred, 1.0 / B)
                model.backward()
        torch.cuda.synchronize()
        census.finish_wgrad()
        torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    routes = census.route_table()
    rec = {'arm': arm, 'workload': wl_name, 'batch': B, 'options': opts, 'tau': TAU, 'census_seconds': seconds,
           'summary': _summary(census), 'fwd': census.fwd, 'dgrad': census.dgrad, 'wgrad': census.wgrad,
           'tail': census.tail, 'routes': routes, 'peak_mem_GB': torch.cuda.max_memory_allocated() / 1e9}
    _record(arm, rec)
    del census, model
    torch.cuda.empty_cache()

    bad = []
    for kind, table in (('fwd', rec['fwd']), ('dgrad', rec['dgrad']), ('wgrad', rec['wgrad'])):
        for layer, st in table.items():
            bar = TAU_TC_WGRAD if kind == 'wgrad' and 'tc_wgrad_kernel' in routes[layer].get('wgrad', {}) else TAU
            for key in ('r', 'r_bias'):
                if key in st and not st[key] <= bar:
                    bad.append('%s %s %s = %.3g (bar %.3g)%s' % (kind, layer, key, st[key], bar,
                                                                  ' consumers %s' % st['consumers']
                                                                  if 'consumers' in st else ''))
    if wl['train']:
        assert rec['tail'] is not None, 'the final conv was never reached by the backward pass'
        if not rec['tail']['r'] <= TAU:
            bad.append('tail d(net_out) r = %.3g' % rec['tail']['r'])
    assert not bad, '%s: %d checks over the bar:\n%s' % (arm, len(bad), '\n'.join(bad))
    n_conv = len(rec['fwd'])
    assert n_conv >= 14 and (not wl['train'] or len(rec['wgrad']) == n_conv), (n_conv, len(rec['wgrad']))
    check_routes(arm, routes)
    if arm == 'cfg4':
        # what profiles/README.md says the benchmarked step runs
        assert 'pwx_fwd_kernel' in routes['query.0.0']['fwd']
        for layer in ('query.1.0', 'obs.1.0', 'query.2.0', 'obs.2.0'):
            assert 'pwd2s_mma_kernel' in routes[layer]['dgrad'], (layer, routes[layer])


# ----------------------------------------------------------------------------------------------------------------
# cfg4 at batch 32, one layer at a time: byte offsets past 2^32
# ----------------------------------------------------------------------------------------------------------------
# (layer, kind, k, s, source channels, cout, activation, input gradient): the level-0 query conv reads 64 channels
# (8 GB at batch 32); the level-1 down-convs run forward, input gradient (two consumers: beta = 1 and the mask on the
# second) and weight gradient
LARGE = [('query.0.0', 'conv', 1, 1, [3, 60, 1], 16, None, False),
         ('query.1.0', 'conv', 2, 2, [16, 16], 16, 'leakyrelu', True),
         ('obs.1.0', 'conv', 2, 2, [16], 16, 'leakyrelu', True)]


@pytest.mark.gpu
@pytest.mark.parametrize('name,kind,k,s,segc,cout,act,dgrad', LARGE, ids=[r[0] for r in LARGE])
def test_batch32_layer_past_32bit_offsets(name, kind, k, s, segc, cout, act, dgrad, monkeypatch):
    import engine
    import nlt_native as nat
    B, uv, idx = 32, 1024, [0, 15, 31]
    dev = torch.device('cuda')
    g = torch.Generator(dev).manual_seed(5)
    xs = [torch.rand(B, uv, uv, c, device=dev, generator=g) * 2 - 1 for c in segc]
    L = engine.ConvLayer(kind, k, s, cout, act)
    L.name = name
    L.build(sum(segc), dev, torch.Generator().manual_seed(1))
    L.bias.copy_((torch.rand(cout, device=dev, generator=g) * 2 - 1) * 0.1)
    L.gkernel.fill_(float('nan'))
    L.gbias.fill_(float('nan'))
    poison_workspaces()
    stats = {}
    try:
        with monkeypatch.context() as mp:
            poisoned_allocations(mp)
            acts = [engine.Act(x, act='leakyrelu' if dgrad else None, needs_grad=dgrad) for x in xs]
            tape = engine.Tape()
            n_cons = 2 if dgrad else 1
            ys = [L.forward([engine.Seg(a) for a in acts], tape) for _ in range(n_cons)]
            segs = [engine.Seg(a) for a in acts]
            stats['fwd'] = forward_check(L, segs, ys[0], idx)
            dzs = [torch.randn(y.t.shape, device=dev, generator=g) * 1e-3 for y in ys]
            dz_sum = dzs[0] if n_cons == 1 else dzs[0] + dzs[1]
            w_terms = wgrad_terms(L, segs, dzs[0]) if n_cons == 1 else None
            for y, d in zip(ys, dzs):
                y.grad = d.clone()
            tape.backward()
            torch.cuda.synchronize()
    except nat.NativeError as e:          # a clean refusal is an acceptable outcome; wrong numbers are not
        _record('b32_' + name, {'layer': name, 'native_error': str(e)})
        return
    if w_terms is None:
        # two consumers: the weight gradient accumulates both, the input gradient sums both adjoints
        w_terms = wgrad_terms(L, segs, dzs[0])
        w2 = wgrad_terms(L, segs, dzs[1])
        w_terms = ([a + b for a, b in zip(w_terms[0], w2[0])], tuple(a + b for a, b in zip(w_terms[1], w2[1])))
        Hin, Win = uv, uv
        coff = 0
        for si, a in enumerate(acts):
            C = a.t.shape[3]
            f = lambda d, w, coff=coff, C=C: vjp_input(kind, s, d, w, Hin, Win, L.cin)[..., coff:coff + C]
            ref = absr = c1 = c3 = 0
            for d in dzs:
                d = d[idx]
                ref = ref + f(d.double(), L.kernel.double())
                absr = absr + f(d.double().abs(), L.kernel.double().abs())
                k1, k3 = controls(f, d, L.kernel)
                c1, c3 = c1 + k1, c3 + k3
            m = _mask(a.t[idx], 'leakyrelu')
            stats['dgrad_seg%d' % si] = op_stats(a.grad[idx], ref * m, absr * m, (c1 * m, c3 * m))
            coff += C
    w, b = w_terms
    stats['wgrad'] = op_stats(L.gkernel, w[0], w[1], (w[2], w[3]))
    stats['wgrad']['r_bias'] = max_rel(L.gbias, b[0], b[1])
    _record('b32_' + name, {'layer': name, 'batch': B, 'images': idx, 'tau': TAU, 'ops': stats})
    bad = ['%s %s = %.3g' % (op, key, st[key]) for op, st in stats.items() for key in ('r', 'r_bias')
           if key in st and not st[key] <= TAU]
    assert not bad, '%s at batch 32: %s' % (name, bad)
