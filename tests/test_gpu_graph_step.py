"""The step bench.py times -- trainvali.GraphedTrainStep, one CUDA graph holding forward, L2 loss, backward and the
device-step AMSGrad update -- replay by replay at the benchmarked shapes.

Per arm (the model built as bench.TrainRun builds it, with the census's seeded biases):
 * three replays on bench's rotating batches b0, b1, b0: the first on the static input buffers, the others through the
   copy-in path;
 * the same three steps run eagerly through the graph's own body (`_body(batch, with_update=True)`) from the restored
   initial state must match bit for bit: loss, predictions, gradients, parameters, the AMSGrad moments and the step
   counter.  Every kernel of the step is deterministic (fixed-order reductions, a fixed-point UV scatter), so the
   census's fp64 verdict on the eager step (tests/test_gpu_census.py) carries over to what bench times;
 * each replay's own outputs against fp64: the camera-space resampling of its UV prediction, the loss, and every
   element of the AMSGrad update from the pre-replay state and the replay's gradients;
 * the same replays fed uint8 batches (datasets `uint8_inputs`), from host and from device memory, must equal the
   float32 replays: the graph's inputs are normalised by v / 255 as in the eager step.
During capture and in the eager twin, float32 allocations and every layer's gradient are NaN-filled (the fills are recorded
into the graph, so every replay starts from NaN), and so are the scratch workspaces, so an element no kernel writes
fails.
"""
import time

import pytest
import torch

from tests.test_gpu_census import TAU, _bias_init, _record, poison_workspaces, poisoned_allocations
from tests.test_gpu_tail_ops import (ADAM_STATE_BAR, ADAM_STEP_BAR, B2, ELEM_BAR, amsgrad_ok, amsgrad_r, check, f32,
                                     uv2cam_ref)

# arm -> (workload, batches to try): bench's batch first; cfg3 falls back to a smaller batch when the graph and its
# eager twin would not fit together
ARMS = {'cfg4': ('cfg4', [8]), 'cfg2': ('cfg2', [8]), 'cfg4k3': ('cfg4k3', [8]), 'cfg3': ('cfg3', [16, 8, 4])}
FIT = 0.9                 # of the device memory, for the graph's step plus an eager step of the same size
KEYS = ('loss', 'pred', 'pred_camspc', 'base_camspc', 'gt_camspc', 'flat_grads', 'flat_params', 'm', 'v', 'vhat')


class _Arm:
    def __init__(self, wl_name, B):
        import bench
        import models
        import trainvali
        from util import synth
        wl = bench.WORKLOADS[wl_name]
        self.B, self.uv = B, wl['uv']
        self.model = models.get_model_class('nlt')(bench.make_config(wl))
        self.model.register_trainable()
        self.model.build(5 + wl['c_extra'], 3)
        _bias_init(self.model)
        self.opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
        self.host = [synth.make_batch(B, self.uv, self.uv, seed=1235 + i, c_extra=wl['c_extra'], pin=True,
                                      k_obs=wl['k_obs']) for i in range(2)]
        dev = self.model.device
        self.dev = [tuple(t.to(dev) if torch.is_tensor(t) else t for t in b) for b in self.host]
        self.step = trainvali.GraphedTrainStep(trainvali.Strategy(), self.model, self.opt, B)

    def state(self):
        o = self.opt
        return [t.clone() for t in (self.model.flat_params, o.m, o.v, o.vhat, o.step_dev)]

    def restore(self, st):
        o = self.opt
        for dst, src in zip((self.model.flat_params, o.m, o.v, o.vhat, o.step_dev), st):
            dst.copy_(src)
        o.iterations = int(st[4])

    def outputs(self, loss, to_vis):
        o = self.opt
        out = {'loss': loss, 'pred': to_vis['pred'], 'pred_camspc': to_vis['pred_camspc'],
               'base_camspc': to_vis['base_camspc'], 'gt_camspc': to_vis['gt_camspc'],
               'flat_grads': self.model.flat_grads, 'flat_params': self.model.flat_params, 'm': o.m, 'v': o.v,
               'vhat': o.vhat}
        out = {k: v.clone() for k, v in out.items()}
        out['step'] = int(o.step_dev)
        return out


def _poison(mp):
    """NaN-filled float32 allocations, gradient buffer at the start of every step, and scratch workspaces (the graph's
    own, which _capture sets up right before it returns the warm-up's cached blocks)."""
    import engine
    poisoned_allocations(mp)
    begin = engine.ParamBucket.begin_step

    def begin_step(bucket):
        for L in bucket.layers:          # the layers' gradients (not the alignment padding between them)
            L.gkernel.fill_(float('nan'))
            L.gbias.fill_(float('nan'))
        begin(bucket)
    mp.setattr(engine.ParamBucket, 'begin_step', begin_step)
    empty = torch.cuda.empty_cache

    def empty_cache():
        empty()
        poison_workspaces()
    mp.setattr(torch.cuda, 'empty_cache', empty_cache)


def _diff(a, b):
    if a.shape != b.shape:
        return 'shape %s vs %s' % (tuple(a.shape), tuple(b.shape))
    ne = (a != b) & ~(a.isnan() & b.isnan())
    idx = ne.nonzero()[:3].tolist()
    return '%d elements differ, first %s: %s vs %s' % (int(ne.sum()), idx, [float(a[tuple(i)]) for i in idx],
                                                       [float(b[tuple(i)]) for i in idx])


def _equal(got, want, what):
    bad = [(k, _diff(got[k], want[k])) for k in KEYS if not torch.equal(got[k], want[k])]
    assert got['step'] == want['step'], '%s: step counter %d vs %d' % (what, got['step'], want['step'])
    assert not bad, '%s:\n%s' % (what, '\n'.join('  %s: %s' % kv for kv in bad))


def fp64_checks(out, before, batch, t, B):
    """r of one replay's own outputs against fp64 (asserts the bars; returns the table)."""
    st = {}
    ref = uv2cam_ref(out['pred'], batch[1], batch[4], batch[6])
    for k in ('pred', 'base', 'gt'):
        check(k + '_camspc', out[k + '_camspc'], ref[k][0], ref[k][1], ELEM_BAR, out=st)
    del ref
    pc, gt = out['pred_camspc'].double(), out['gt_camspc'].double()
    loss = ((pc - gt) ** 2).reshape(B, -1).mean(1).sum() / B
    check('loss', out['loss'].reshape(1), loss.reshape(1), loss.reshape(1), TAU, out=st)
    p0, m0, v0, vh0 = before[:4]
    r = amsgrad_r((out['flat_params'], out['m'], out['v'], out['vhat']), p0, out['flat_grads'], m0, v0, vh0, t)
    st.update({'amsgrad_' + k: x for k, x in r.items()})
    assert amsgrad_ok(r), 'AMSGrad at step %d over its bars (m/v/vhat %.3g, p %.3g): %s' % (
        t, ADAM_STATE_BAR, ADAM_STEP_BAR, r)
    assert out['step'] == t, (out['step'], t)
    return st


def _fits(base_alloc):
    """Whether an eager step of the same size fits beside the captured graph (estimated from the warm-up peak)."""
    peak = torch.cuda.max_memory_allocated()
    total = torch.cuda.get_device_properties(0).total_memory
    return base_alloc + 2 * (peak - base_alloc) <= FIT * total, peak


@pytest.mark.gpu
@pytest.mark.parametrize('arm', list(ARMS))
def test_graph_replays_equal_eager_and_fp64(arm, monkeypatch):
    from util import synth
    wl_name, batches = ARMS[arm]
    t0 = time.perf_counter()
    tried = []
    for B in batches:
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base_alloc = torch.cuda.memory_allocated()
        a = _Arm(wl_name, B)
        with monkeypatch.context() as mp:
            _poison(mp)
            a.step._capture(a.dev[0])
        assert a.step.full_step_in_graph
        ok, peak = _fits(base_alloc)
        tried.append({'batch': B, 'peak_after_capture_GB': peak / 1e9})
        if ok or B == batches[-1]:
            break
        del a
    init = a.state()
    seq = [0, 1, 0]

    # ---- three replays: static buffers, then the copy-in path ----
    graph_out, stats, branches = [], [], None
    for t, bi in enumerate(seq, 1):
        before = a.state()
        loss, to_vis = a.step(a.step.static_batch if t == 1 else a.dev[bi])
        torch.cuda.synchronize()
        out = a.outputs(loss, to_vis)
        stats.append(fp64_checks(out, before, a.dev[bi], t, B))
        if t == 3:
            g = out['flat_grads'].double()
            v_new = before[2].double() + (g * g - before[2].double()) * (1 - f32(B2))
            kept = before[3].double() > v_new
            branches = {'vhat_kept': int(kept.sum()), 'v_taken': int((~kept).sum())}
        graph_out.append(out)
        del before
    assert branches['vhat_kept'] > 0 and branches['v_taken'] > 0, branches

    # ---- the eager twin: the graph's own body, from the restored initial state ----
    a.restore(init)
    with monkeypatch.context() as mp:
        _poison(mp)
        for t, bi in enumerate(seq, 1):
            poison_workspaces()
            loss, to_vis = a.step._body(a.dev[bi], with_update=True)
            torch.cuda.synchronize()
            _equal(graph_out[t - 1], a.outputs(loss, to_vis), '%s replay %d vs eager' % (arm, t))
            del loss, to_vis
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()

    # ---- uint8 batches through the graph, from host and from device memory ----
    for where in ('host', 'device'):
        a.restore(init)
        for t, bi in enumerate(seq, 1):
            u8 = synth.as_uint8(a.host[bi])
            if where == 'device':
                u8 = tuple(x.cuda() if torch.is_tensor(x) else x for x in u8)
            loss, to_vis = a.step(u8)
            torch.cuda.synchronize()
            _equal(a.outputs(loss, to_vis), graph_out[t - 1], '%s uint8 (%s) replay %d vs float32' % (arm, where, t))

    rec = {'arm': arm, 'workload': wl_name, 'batch': B, 'tried': tried, 'seconds': time.perf_counter() - t0,
           'peak_mem_GB': peak / 1e9, 'bars': {'elem': ELEM_BAR, 'tau': TAU, 'amsgrad_state': ADAM_STATE_BAR,
                                               'amsgrad_step': ADAM_STEP_BAR},
           'max_r': {k: max(s[k] for s in stats) for k in stats[0]}, 'per_replay': stats,
           'amsgrad_branches_replay3': branches, 'n_params': int(a.model.flat_params.numel())}
    _record('graph_' + arm, rec)
    del a, graph_out
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_graph_captured_from_a_uint8_batch():
    """A graph whose first (capturing) call gets uint8 images computes what one captured from float32 images does."""
    import trainvali
    from tests.test_gpu_model import make_model
    from util import synth
    bts = [synth.make_batch(2, 64, 64, seed=400 + i) for i in range(2)]
    res = {}
    for kind in ('f32', 'u8'):
        m, _ = make_model(uvh=64, uvw=64, imh=64, imw=64)
        m.seed = 5
        m.build(5, 3)
        opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
        step = trainvali.GraphedTrainStep(trainvali.Strategy(), m, opt, 2)
        losses = []
        for bt in bts:
            loss, _ = step(synth.as_uint8(bt) if kind == 'u8' else bt)
            losses.append(loss.clone())
        torch.cuda.synchronize()
        res[kind] = (torch.stack(losses), m.flat_params.clone(), opt.vhat.clone())
    for a, b in zip(res['u8'], res['f32']):
        assert torch.equal(a, b), _diff(a, b)
