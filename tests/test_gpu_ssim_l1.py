"""The CUDA L1 and SSIM losses (nlt_l1_loss, nlt_ssim_loss) against their fp64 oracles, at the model level and inside
the graphed training step.

SSIM bars: the per-sample loss error and the d_pred relative Frobenius error must each be within 2x of what fp32 costs
TF's own formulation on the same input family (tests/test_oracle_losses.py: EMUL_ERR at 256^2, or the emulation at
the test's own shape where that is larger, as it is for small images), and never above 1e-5 / 1e-3."""
import pytest
import torch

from oracle import loss_oracle as LO
from oracle import nlt_oracle as O
from tests.test_oracle_losses import EMUL_ERR, emul_errors, make_images, ssim_ref64

pytestmark = pytest.mark.gpu

LOSS_CEIL, DPRED_CEIL = 1e-5, 1e-3
SHAPES = [(1, 11, 11), (2, 11, 37), (3, 33, 17), (2, 83, 71), (8, 256, 256), (8, 1024, 1024), (32, 1024, 1024)]
RECORD = {}


def _record():
    """Writes the measured errors beside the parity records (tests/test_gpu_parity.py), as parity_ssim_l1.json."""
    from tests.test_gpu_parity import _record as parity_record
    parity_record('ssim_l1', RECORD)


def _nan(n):
    return torch.full((n,), float('nan'), device='cuda')


def run_ssim(pred, gt, loss_scale, grad=True, max_val=1.0):
    import nlt_native as nat
    lib = nat.lib()
    B, H, W, _ = pred.shape
    ws = _nan((lib.nlt_ssim_loss_workspace_bytes(B, H, W) + 3) // 4)
    loss = _nan(B)
    d = torch.full_like(pred, float('nan')) if grad else None
    nat.check(lib.nlt_ssim_loss(nat.ptr(pred), nat.ptr(gt), B, H, W, max_val, loss_scale, nat.ptr(loss), nat.ptr(d),
                                nat.ptr(ws), nat.stream()))
    torch.cuda.synchronize()
    return loss, d


def run_l1(pred, gt, loss_scale, grad=True):
    import nlt_native as nat
    lib = nat.lib()
    B = pred.shape[0]
    per = pred.numel() // B
    ws = _nan((lib.nlt_l1_loss_workspace_bytes(B, per) + 3) // 4)
    loss = _nan(B)
    d = torch.full_like(pred, float('nan')) if grad else None
    nat.check(lib.nlt_l1_loss(nat.ptr(pred), nat.ptr(gt), B, per, loss_scale, nat.ptr(loss), nat.ptr(d), nat.ptr(ws),
                              nat.stream()))
    torch.cuda.synchronize()
    return loss, d


def _rel_fro(got, want):
    return float((got.double() - want).norm() / want.norm())


@pytest.mark.parametrize('family', ['noisy', 'saturated'])
@pytest.mark.parametrize('shape', SHAPES, ids=['x'.join(map(str, s)) for s in SHAPES])
def test_ssim_against_fp64(shape, family):
    B, H, W = shape
    gt_np, pred_np = make_images(family, B, H, W, seed=B + H + W)
    bar_l, bar_d = EMUL_ERR[family]['loss'], EMUL_ERR[family]['d_pred']
    if H * W <= 256 * 256:
        el, ed = emul_errors(gt_np, pred_np)
        bar_l, bar_d = max(bar_l, el), max(bar_d, ed)
    bar_l, bar_d = min(2 * bar_l, LOSS_CEIL), min(2 * bar_d, DPRED_CEIL)
    gt, pred = torch.from_numpy(gt_np).cuda(), torch.from_numpy(pred_np).cuda()
    del gt_np, pred_np
    scale = 1.0 / B
    loss, d = run_ssim(pred, gt, scale)
    assert not loss.isnan().any() and not d.isnan().any()
    # reference in fp64 on the device (a few samples at a time for the big shapes)
    errs_l, num, den = [], 0.0, 0.0
    for b0 in range(0, B, 4):
        l64, d64 = ssim_ref64(gt[b0:b0 + 4], pred[b0:b0 + 4], scale, device='cuda')
        errs_l.append(float((loss[b0:b0 + 4].double() - l64).abs().max()))
        num += float((d[b0:b0 + 4].double() - d64).norm() ** 2)
        den += float(d64.norm() ** 2)
        del l64, d64
    el, ed = max(errs_l), (num / den) ** 0.5
    key = 'ssim %s %s' % (family, shape)
    RECORD[key] = {'loss_err': el, 'loss_bar': bar_l, 'd_pred_rel_fro': ed, 'd_pred_bar': bar_d}
    _record()
    assert el <= bar_l and ed <= bar_d, RECORD[key]
    # no gradient requested: bit-identical losses; and a second call is bit-identical
    loss_v, _ = run_ssim(pred, gt, scale, grad=False)
    loss2, d2 = run_ssim(pred, gt, scale)
    assert torch.equal(loss_v, loss) and torch.equal(loss2, loss) and torch.equal(d2, d)


def test_ssim_bad_arguments_return_negative():
    import nlt_native as nat
    lib = nat.lib()
    x = torch.zeros(2, 16, 16, 3, device='cuda')
    ws = torch.zeros(1024, device='cuda')
    loss = torch.zeros(2, device='cuda')
    p = lambda t: nat.ptr(t)
    ok = (p(x), p(x), 2, 16, 16, 1.0, 1.0, p(loss), None, p(ws), nat.stream())
    assert lib.nlt_ssim_loss(*ok) == 0
    for i, bad in [(0, None), (1, None), (7, None), (9, None), (2, 0), (3, 10), (4, 10), (5, 0.0)]:
        args = list(ok)
        args[i] = bad
        assert lib.nlt_ssim_loss(*args) < 0, i
    torch.cuda.synchronize()


L1_SHAPES = [(2, 33, 17), (8, 1024, 1024), (32, 1024, 1024)]


@pytest.mark.parametrize('shape', L1_SHAPES, ids=['x'.join(map(str, s)) for s in L1_SHAPES])
def test_l1_against_fp64(shape):
    B, H, W = shape
    g = torch.Generator(device='cuda').manual_seed(H + B)
    gt = torch.randint(0, 256, (B, H, W, 3), generator=g, device='cuda').float() / 255
    pred = gt + 0.05 * torch.randn(B, H, W, 3, generator=g, device='cuda')
    tie = torch.rand(B, H, W, 3, generator=g, device='cuda') < 0.1
    pred = torch.where(tie, gt, pred).contiguous()
    scale = 1.0 / B
    loss, d = run_l1(pred, gt, scale)
    g64, p64 = gt.double(), pred.double().requires_grad_(True)
    l64 = LO.l1_loss(g64, p64, keep_batch=True)
    (l64.sum() * scale).backward()
    el = float(((loss.double() - l64.detach()) / l64.detach()).abs().max())
    ed = _rel_fro(d, p64.grad)
    RECORD['l1 %s' % (shape,)] = {'loss_rel_err': el, 'd_pred_rel_fro': ed}
    _record()
    assert el <= 1e-6 and ed <= 1e-6, RECORD['l1 %s' % (shape,)]
    assert int(tie.sum()) > 0 and bool((d[tie] == 0).all())        # ties: an exact 0 gradient
    loss_v, _ = run_l1(pred, gt, scale, grad=False)
    assert torch.equal(loss_v, loss)


# ---------------------------------------------------------------------------
# model level: one train step on the default route, 64^2, depth 256
# ---------------------------------------------------------------------------
LOG_Z = 1.185495232349193


def _oracle_objective(loss):
    from oracle import barron_oracle as BO
    terms = {'ssim': lambda gt, pred: LO.ssim_loss(gt, pred, keep_batch=True),
             'l1': lambda gt, pred: LO.l1_loss(gt, pred, keep_batch=True),
             'barron': lambda gt, pred: BO.barron_loss(gt, pred, LOG_Z, keep_batch=True)}
    from models.base import Model
    parts = [Model._parse_loss_and_weight(s) for s in loss.split(',')]
    return lambda gt, pred, keep_batch=True: sum(w * terms[n](gt, pred) for n, w in parts)


@pytest.mark.parametrize('loss', ['ssim', 'l1', 'barron,1e+0ssim'])
def test_model_train_step(loss, monkeypatch):
    import nlt_native as nat
    from tests.test_gpu_model import rel_fro
    from tests.test_gpu_parity import _oracle_grads, _product_and_masks
    with nat.options(tc=1):
        B = 2
        m, oc, bt, params, masks, pred, per = _product_and_masks(dict(uvh=64, uvw=64, imh=64, imw=64, loss=loss), B,
                                                                 seed=77)
        objective = _oracle_objective(loss)
        monkeypatch.setattr(O, 'l2_loss', objective)          # _oracle_grads differentiates sum_b O.l2_loss(...) / B
        p64, g_masked, flips = _oracle_grads(params, oc, bt, B, masks)
        bt64 = tuple(t.double() if torch.is_tensor(t) else t for t in bt)
        with torch.no_grad():
            pr, gt, _, _ = O.model_call(params, oc, bt64, 'train')
            want = objective(gt, pr)
        loss_err = float(((per.double().cpu() - want) / want).abs().max())
        grads = m.export_grads()
        worst = max(rel_fro(grads[k], g_masked[k]) for k in params)
        RECORD['model %s' % loss] = {'loss_rel_err': loss_err, 'worst_wgrad_rel_fro_masked': worst,
                                     'flipped_bits': flips['flipped']}
        _record()
        assert loss_err <= 1e-4 and worst <= 1e-4, RECORD['model %s' % loss]


# ---------------------------------------------------------------------------
# the graphed cfg4 step with `loss = ssim`, `barron` and `barron,1e+0ssim`
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('objective', ['ssim', 'barron', 'barron,1e+0ssim'])
def test_graph_step_replays_equal_eager(objective, monkeypatch):
    """GraphedTrainStep at the cfg4 shape, batch 8: three replays (b0, b1, b0) equal the graph's body run eagerly from
    the restored state, bit for bit, the loss value included (every loss sums its per-sample partials in a fixed
    order)."""
    import bench
    import trainvali
    from tests.test_gpu_census import poison_workspaces
    from tests.test_gpu_graph_step import _Arm, _equal, _poison
    from util import io as ioutil

    wl = bench.WORKLOADS['cfg4']
    cfg = ioutil.make_config(uvh=wl['uv'], uvw=wl['uv'], imh=wl['uv'], imw=wl['uv'], loss=objective, depth0=16,
                             depth=wl['depth'], kernel=wl['kernel'], stride=2)
    real_make_config = bench.make_config
    monkeypatch.setattr(bench, 'make_config', lambda w: cfg if w is wl else real_make_config(w))
    a = _Arm('cfg4', 8)
    want_terms = {'ssim': ['SSIM'], 'barron': ['Barron'], 'barron,1e+0ssim': ['Barron', 'SSIM']}[objective]
    assert [type(f).__name__ for _, f in a.model.wloss] == want_terms
    with monkeypatch.context() as mp:
        _poison(mp)
        a.step._capture(a.dev[0])
    assert a.step.full_step_in_graph
    init = a.state()
    seq = [0, 1, 0]
    graph_out = []
    for t, bi in enumerate(seq, 1):
        loss, to_vis = a.step(a.step.static_batch if t == 1 else a.dev[bi])
        torch.cuda.synchronize()
        graph_out.append(a.outputs(loss, to_vis))
    assert all(bool(torch.isfinite(o['loss']).all()) for o in graph_out)
    assert not torch.equal(graph_out[0]['loss'], graph_out[2]['loss'])      # same batch, updated parameters
    a.restore(init)
    # one validation call (no gradient) at the initial parameters: the loss the first replay trained on
    vloss, _ = trainvali.distributed_vali_step(trainvali.Strategy(), a.model, a.dev[0], 8)
    torch.cuda.synchronize()
    torch.testing.assert_close(vloss.reshape(1), graph_out[0]['loss'].reshape(1), rtol=1e-6, atol=0)
    with monkeypatch.context() as mp:
        _poison(mp)
        for t, bi in enumerate(seq, 1):
            poison_workspaces()
            loss, to_vis = a.step._body(a.dev[bi], with_update=True)
            torch.cuda.synchronize()
            _equal(graph_out[t - 1], a.outputs(loss, to_vis), '%s replay %d vs eager' % (objective, t))
            del loss, to_vis
    RECORD['graph cfg4 ' + objective] = {'losses': [float(o['loss']) for o in graph_out], 'vali_loss': float(vloss)}
    _record()
    del a, graph_out
    torch.cuda.empty_cache()
