"""Which kernels each route-selecting option value sends a conv to.

For every option setting the GPU tests use (plus switching each on-by-default route off), forward, input gradient and
weight gradient of a set of shapes from tests/test_gpu_ops.py run through the engine, and the launches of every kernel
label (`nlt_kernel_launch_count` deltas) are compared with tests/census_routes/options.json.  The oracle tests of those
options compare an option's value against the default; this table is what shows that each value still selects its
kernels.  `NLT_UPDATE_ROUTES=1` rewrites the table.
"""
import ctypes as C

import pytest
import torch

from tests.test_gpu_census import check_routes, kernel_labels

pytestmark = pytest.mark.gpu

# kind, k, s, H, W, seg channels, cout (test_gpu_ops.GEOMS, and the shapes of its wide-stencil tests)
SHAPES = [
    ('conv', 1, 1, 32, 32, [64], 16),            # pointwise into 16 channels
    ('conv', 1, 1, 160, 144, [4, 16, 16], 3),    # final 1x1 conv: coalesced weight gradient
    ('conv', 2, 2, 8, 512, [16, 16], 32),        # depth-to-space input gradient K = 32 -> 16
    ('conv', 2, 2, 16, 256, [32], 64),           # ... K = 64 -> 32 (pwd2s_first)
    ('conv', 2, 2, 16, 256, [16, 16], 16),       # staged-patch weight gradient
    ('conv', 2, 2, 4, 512, [16], 32),            # staged-patch forward
    ('conv', 2, 1, 256, 256, [16], 16),          # 16 -> 16 stride-1 stencil
    ('conv', 2, 1, 16, 16, [16], 16),
    ('deconv', 2, 1, 12, 200, [4], 4),           # row-stream stencils
    ('conv', 2, 1, 7, 130, [8], 8),
    ('deconv', 2, 2, 4, 64, [32, 64, 64], 16),   # outer-product weight gradient
    ('deconv', 2, 2, 5, 48, [16], 16),
    ('deconv', 2, 2, 3, 128, [8, 32], 4),        # depth-to-space forward into 4 channels
    ('deconv', 2, 2, 16, 16, [64, 64], 32),      # tensor-core shapes
    ('conv', 2, 2, 32, 32, [32, 32], 64),
    ('conv', 2, 2, 64, 256, [32], 128),
    ('conv', 3, 2, 8, 8, [8, 4], 32),            # phase-decomposed general kernels
    ('deconv', 3, 2, 5, 6, [16, 3], 8),
    ('deconv', 2, 2, 4, 4, [8], 3),              # k == s transposed, Cout % 4 != 0: phases
    ('conv', 2, 1, 16, 24, [32], 32),            # wide stencil shapes
    ('conv', 2, 2, 16, 24, [4], 16),
    ('conv', 2, 1, 9, 16, [8], 8),
    ('deconv', 2, 1, 12, 20, [8], 8),
]

# (H, W, c_skip, c_other, down_cout, dk) of test_gpu_ops.test_final_conv_input_gradient_rides_on_down_conv_dgrad: the
# final 1x1 conv's input gradient fused into the down-conv's
FUSED = [(8, 512, 16, 4, 16, 2), (16, 16, 16, 4, 16, 2), (8, 8, 16, 4, 16, 1)]

ARMS = [
    {},
    {'tc': 0}, {'tc': 2}, {'tc': 2, 'tc_rawhi': 0}, {'tcs': 0}, {'tc_wgrad': 0},
    {'pwx': 0}, {'tiny': 0}, {'wop': 0}, {'wop': 2}, {'pwmma': 0}, {'pwmma': 1, 'tc': 0},
    {'pf': 1}, {'pf': 1, 'tiny': 0}, {'pf': 1, 'pwx': 0}, {'pf': 1, 'pf_s1': 1}, {'pf': 1, 'pwd2s_first': 1}, {'pf': 1, 'pf_ns': 2, 'pwx_ns': 2},
    {'tc': 0, 'wgrad_rows': 0},
    {'tc': 0, 'dconv_wide32': 1}, {'tc': 0, 'dconv_wide32': 2}, {'tc': 0, 'dconv_wide_first': 0},
    {'tc': 0, 'dconv_wide8': 0, 'dconv_wide32': 0, 'dconv_wide_first': 0},
    {'dconv_wide': 0}, {'tc': 0, 'dconv_wide': 0}, {'dconv_cw': 0}, {'tc': 0, 'dconv_cw': 0},
]


def _arm_name(opts):
    return ','.join('%s=%d' % kv for kv in opts.items()) or 'default'


def _shape_name(kind, k, s, H, W, segc, cout):
    return '%s%dx%d/s%d %dx%d %s->%d' % (kind, k, k, s, H, W, '+'.join(map(str, segc)), cout)


def _fused_name(H, W, c_skip, c_other, down_cout, dk):
    return '%dx%d skip %d other %d down %dx%d->%d' % (H, W, c_skip, c_other, dk, dk, down_cout)


class Counts:
    def __init__(self, nat):
        self.nat, self.labels = nat, kernel_labels()
        self.last = self.now()

    def now(self):
        return {k: self.nat.kernel_launch_count(k) for k in self.labels}

    def take(self):
        """Launches per kernel label since the previous take()."""
        n = self.now()
        d = {k: n[k] - self.last[k] for k in self.labels if n[k] != self.last[k]}
        self.last = n
        return dict(sorted(d.items()))


def _layer_routes(engine, nat, counts, kind, k, s, H, W, segc, cout):
    dev = torch.device('cuda')
    torch.manual_seed(7)
    xs = [torch.randn(2, H, W, c, device=dev) for c in segc]
    L = engine.ConvLayer(kind, k, s, cout, 'leakyrelu')
    L.build(sum(segc), dev, torch.Generator().manual_seed(1))
    acts = [engine.Act(x, act='leakyrelu', needs_grad=True) for x in xs]
    tape = engine.Tape()
    out = {}
    counts.take()
    y = L.forward([engine.Seg(a) for a in acts], tape)
    out['fwd'] = counts.take()
    y.grad = torch.randn_like(y.t)
    engine.WGRAD_HOOK = lambda layer: out.setdefault('wgrad', counts.take())
    try:
        tape.backward()
    finally:
        engine.WGRAD_HOOK = None
    out['dgrad'] = counts.take()
    # the same forward without a workspace (nlt_gconv_fwd, the fp32 path)
    d = L._fwd_desc([engine.Seg(a) for a in acts], 2, H, W)
    nat.check(nat.lib().nlt_gconv_fwd(C.byref(d), nat.ptr(L.bias), nat.ACT_CODES['leakyrelu'], 0.0, None, 0,
                                      nat.ptr(torch.empty_like(y.t)), nat.stream()))
    out['fwd_nows'] = counts.take()
    return out


def _fused_routes(engine, nat, counts, H, W, c_skip, c_other, down_cout, dk):
    dev = torch.device('cuda')
    torch.manual_seed(21)
    gen = lambda: torch.Generator().manual_seed(4)
    down = engine.ConvLayer('conv', dk, dk, down_cout, 'leakyrelu')
    down.build(c_skip, dev, gen())
    final = engine.ConvLayer('conv', 1, 1, 3, None)
    final.build(c_other + c_skip, dev, gen())
    a_skip = engine.Act(torch.randn(2, H, W, c_skip, device=dev), act='leakyrelu', needs_grad=True)
    a_other = engine.Act(torch.randn(2, H, W, c_other, device=dev), act='leakyrelu', needs_grad=True)
    tape = engine.Tape()
    y_down = down.forward([engine.Seg(a_skip)], tape)
    y_fin = final.forward([engine.Seg(a_other), engine.Seg(a_skip)], tape)
    y_down.grad = torch.randn_like(y_down.t)
    y_fin.grad = torch.randn_like(y_fin.t)
    counts.take()
    tape.backward()
    return {'bwd': counts.take()}


def test_option_routes():
    import engine
    import nlt_native as nat
    counts = Counts(nat)
    table = {}
    for opts in ARMS:
        arm = _arm_name(opts)
        with nat.options(**opts):
            for g in SHAPES:
                table['%s | %s' % (arm, _shape_name(*g))] = _layer_routes(engine, nat, counts, *g)
            for f in FUSED:
                table['%s | fused %s' % (arm, _fused_name(*f))] = _fused_routes(engine, nat, counts, *f)
        torch.cuda.synchronize()
    check_routes('options', table)
