"""Model-level parity: Model.call / backward / train step on the GPU against
the fp64 oracle and the committed golden vectors.

Stated tolerances (fp32 SIMT path vs fp64 oracle): pred_camspc max-abs <= 2e-5,
weight-gradient relative Frobenius error <= 1e-4 (SURVEY.md 8d)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nlt_oracle as O   # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), 'golden')


def make_model(**over):
    import models
    from util import io as ioutil
    cfg = ioutil.make_config(**over)
    Model = models.get_model_class('nlt')
    m = Model(cfg)
    m.register_trainable()
    return m, cfg


def ocfg(cfg):
    g = lambda k: cfg.get('DEFAULT', k)
    return dict(depth0=int(g('depth0')), depth=int(g('depth')), kernel=int(g('kernel')), stride=int(g('stride')),
                norm=g('norm'), act=g('act'), pool=g('pool'), use_obs=cfg.getboolean('DEFAULT', 'use_obs'),
                skip_connect_base=cfg.getboolean('DEFAULT', 'skip_connect_base'), imh=int(g('imh')),
                imw=int(g('imw')), uvh=int(g('uvh')), uvw=int(g('uvw')))


def rel_fro(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def run_pair(over, B=2, seed=1234, c_extra=0, im=None):
    from util import synth
    m, cfg = make_model(**over)
    oc = ocfg(cfg)
    bt = synth.make_batch(B, oc['uvh'], im or oc['imh'], seed=seed, c_extra=c_extra)
    if im and im != oc['imh']:
        # the dataset resizes rgb_camspc to (imh, imw) but leaves the warp at its native
        # resolution (nlt/datasets/nlt.py:141-147): "always warp first and then resize"
        small = synth.make_batch(B, oc['uvh'], oc['imh'], seed=seed + 1)
        bt = bt[:6] + (small[6],) + bt[7:10] + (small[10],)
    params = O.init_params(oc, c_query=5 + c_extra, c_obs=3, seed=7, dtype=torch.float64)
    m.build(5 + c_extra, 3)
    m.load_params(params)
    for v in params.values():
        v.requires_grad_(True)
    bt64 = tuple(t.double() if torch.is_tensor(t) else t for t in bt)
    pred64, gt64, _, vis64 = O.model_call(params, oc, bt64, 'train')
    per64 = O.l2_loss(gt64, pred64, keep_batch=True)
    (per64.sum() / B).backward()
    pred, gt, kw, vis = m(bt, mode='train')
    kw['keep_batch'] = True
    m.set_loss_grad_scale(1.0 / B)
    per = m.compute_loss(pred, gt, **kw)
    m.backward()
    return m, params, (pred, gt, per, vis), (pred64, gt64, per64, vis64)


@pytest.fixture(params=['fp32', 'tc'])
def path(request):
    """Runs a test on both execution paths of the library: 'fp32' = fp32-FMA kernels only (strict parity
    bar), 'tc' = wgmma 3xTF32 kernels wherever a shape is eligible (the default, performance path)."""
    import nlt_native as nat
    with nat.options(tc=1 if request.param == 'tc' else 0):
        yield request.param


CASES = [
    dict(uvh=64, uvw=64, imh=64, imw=64),                                   # shipped family, bottleneck 1x1
    dict(uvh=128, uvw=128, imh=128, imw=128, depth=64),                     # shallower
    dict(uvh=64, uvw=64, imh=64, imw=64, kernel=3),                         # north-star 3x3
    dict(uvh=64, uvw=64, imh=64, imw=64, use_obs=False, skip_connect_base=False, act='relu'),
    dict(uvh=64, uvw=64, imh=48, imw=48),                                   # warp res != (imh, imw): resize path
]


@pytest.mark.parametrize('over', CASES)
def test_train_forward_backward_matches_oracle(over, path):
    im = 64 if over.get('imh') == 48 else None
    m, params, got, want = run_pair(over, im=im)
    pred, gt, per, vis = got
    pred64, gt64, per64, vis64 = want
    assert float((pred.double().cpu() - pred64.detach()).abs().max()) <= 2e-5
    assert float((gt.double().cpu() - gt64.detach()).abs().max()) <= 5e-6
    assert float((vis['pred'].double().cpu() - vis64['pred'].detach()).abs().max()) <= 2e-5
    np.testing.assert_allclose(per.double().cpu().numpy(), per64.detach().numpy(), rtol=1e-4)
    grads = m.export_grads()
    for name, p in params.items():
        if p.grad is None:     # obs stream unused (use_obs=False)
            assert float(grads[name].abs().max()) == 0.0
            continue
        # ReLU's derivative is discontinuous: a pre-activation within fp32 round-off of 0 flips a
        # mask bit against the fp64 oracle and moves a small layer's gradient by O(1/sqrt(#elements))
        tol = 5e-3 if over.get('act') == 'relu' else 1e-4
        if path == 'tc':
            # 3xTF32 products carry ~1e-6 relative error (A/B-tested per op at <= 5e-6 against the fp32
            # kernels); through the LeakyReLU kinks a pre-activation within that distance of 0 flips a
            # derivative bit against the fp64 oracle, which moves a whole-layer gradient by O(1e-3).
            tol = max(tol, 3e-3)
        assert rel_fro(grads[name], p.grad) <= tol, name


def test_golden_fixture_h64(path):
    """tests/golden/model_h64.npz was produced by tests/golden/make_golden.py."""
    from tests.golden import make_golden as G
    gtol = 1e-4 if path == 'fp32' else 3e-3
    gold = np.load(os.path.join(GOLD, 'model_h64.npz'))
    over = {k: G.CFG[k] for k in ('uvh', 'uvw', 'imh', 'imw')}
    m, params, got, _ = run_pair(over, B=G.B, seed=G.SEED)
    pred, gt, per, vis = got
    assert np.abs(pred.cpu().numpy() - gold['pred_camspc']).max() <= 2e-5
    assert np.abs(vis['pred'].cpu().numpy() - gold['pred_uv']).max() <= 2e-5
    np.testing.assert_allclose(per.cpu().numpy(), gold['per_example_loss'], rtol=1e-4)
    grads = m.export_grads()
    names = sorted(grads)
    np.testing.assert_allclose([float(grads[n].double().norm()) for n in names], gold['grad_l2norm'], rtol=20 * gtol)
    for k in gold.files:
        if k.startswith('grad:'):
            g = grads[k[5:]].cpu().numpy()
            assert np.linalg.norm(g - gold[k]) <= gtol * np.linalg.norm(gold[k]), k


def test_cfg4_wide_query_stack(path):
    m, params, got, want = run_pair(dict(uvh=64, uvw=64, imh=64, imw=64), c_extra=59)
    assert float((got[0].double().cpu() - want[0].detach()).abs().max()) <= 2e-5
    grads = m.export_grads()
    for name in ('query.0.0.kernel', 'query.6.1.kernel', 'obs.3.0.kernel'):
        assert rel_fro(grads[name], params[name].grad) <= (1e-4 if path == 'fp32' else 3e-3), name


def test_sss_depth1024_forward():
    """dragon_sss family (depth 1024, 18 layers) at the smallest legal UV size."""
    from util import synth
    m, cfg = make_model(uvh=256, uvw=256, imh=256, imw=256, depth=1024)
    oc = ocfg(cfg)
    bt = synth.make_batch(1, 256, 256, seed=5)
    params = O.init_params(oc, seed=3, dtype=torch.float32)
    m.build(5, 3)
    m.load_params(params)
    assert m.flat_params.numel() >= 53841543
    pred, _, _, _ = m(bt, mode='test')
    with torch.no_grad():
        want, _, _, _ = O.model_call({k: v.double() for k, v in params.items()}, oc,
                                     tuple(t.double() if torch.is_tensor(t) else t for t in bt), 'test')
    assert float((pred.double().cpu() - want).abs().max()) <= 5e-5


@pytest.mark.parametrize('K', [1, 6])
def test_multi_observation_call(K):
    """_call with K observations (cfg3 uses K=6) and obs_weights."""
    from util import synth
    m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64)
    oc = ocfg(cfg)
    params = O.init_params(oc, seed=9, dtype=torch.float64)
    m.build(5, 3)
    m.load_params(params)
    torch.manual_seed(K)
    qx = torch.rand(2, 64, 64, 5)
    obs = [torch.rand(2, 64, 64, 3) - 0.5 for _ in range(K)]
    got = m._call(qx, obs)
    with torch.no_grad():
        want = O.net_call(params, oc, qx.double(), [o.double() for o in obs])
    assert float((got.double().cpu() - want).abs().max()) <= 2e-5
    if K > 1:
        w = torch.rand(2, K)
        got = m._call(qx, obs, obs_weights=w)
        with torch.no_grad():
            want = O.net_call(params, oc, qx.double(), [o.double() for o in obs], obs_weights=w.double())
        assert float((got.double().cpu() - want).abs().max()) <= 2e-5


def test_obs_override_equals_live_path_and_extract_feat():
    """SURVEY 8c(6): the nlt_test override path fed with the live features of
    the same single observation reproduces the live path; extract_feat/infer
    follow nlt_test.py:78-127."""
    import nlt_test
    from util import synth
    m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64)
    oc = ocfg(cfg)
    params = O.init_params(oc, seed=11, dtype=torch.float64)
    m.build(5, 3)
    m.load_params(params)
    train_batches = [synth.make_batch(2, 64, 64, seed=s) for s in (21, 22)]
    feat = nlt_test.extract_feat(m, train_batches, n_obs_batches=-1)
    want = O.extract_feat(params, oc, [(b[1].double(), b[5].double()) for b in train_batches])
    assert len(feat) == 7
    for f, w in zip(feat, want):
        assert f.shape[0] == 1 and float((f.double().cpu() - w.detach()).abs().max()) <= 2e-5
    test_batch = synth.make_batch(3, 64, 64, seed=23)
    outs = nlt_test.infer(m, [test_batch], feat)
    with torch.no_grad():
        ov = [w.expand(3, -1, -1, -1) for w in want]
        p64, _, _, _ = O.model_call(params, oc, tuple(t.double() if torch.is_tensor(t) else t for t in test_batch),
                                    'test', obs_override=ov)
    assert float((outs[0].double().cpu() - p64).abs().max()) <= 2e-5
    # live path == override path when the override IS the live features (B=1, K=1)
    b1 = synth.make_batch(1, 64, 64, seed=24)
    live, _, _, _ = m(b1, mode='test')
    x = (b1[9] - b1[8]).cuda()
    feats = []
    for layer in m.net['obs'].layers:
        x = layer(x)
        feats.append(x)
    over, _, _, _ = m.call(b1, 'test', obs_override=feats)
    assert torch.equal(live, over)


def test_train_steps_match_oracle_amsgrad():
    """Three full train steps (fwd, bwd, AMSGrad) track the fp64 oracle (strict fp32 kernels: AMSGrad's
    m/sqrt(v) turns a derivative-bit flip into an O(lr) parameter difference)."""
    import trainvali
    import nlt_native as nat
    with nat.options(tc=0):
        from util import synth
        m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64, depth=64)
        oc = ocfg(cfg)
        params = O.init_params(oc, seed=13, dtype=torch.float64)
        m.build(5, 3)
        m.load_params(params)
        strategy = trainvali.Strategy()
        opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
        st = {k: [torch.zeros_like(v) for _ in range(3)] for k, v in params.items()}
        for step in range(1, 4):
            bt = synth.make_batch(2, 64, 64, seed=100 + step)
            loss, _ = trainvali.distributed_train_step(strategy, m, bt, opt, 2)
            ps = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
            l64 = O.train_loss(ps, oc, tuple(t.double() if torch.is_tensor(t) else t for t in bt), 2)
            l64.backward()
            assert abs(float(loss) - float(l64)) <= 1e-4 * abs(float(l64))
            for k in params:
                p, mm, v, vh = O.amsgrad_step(params[k], ps[k].grad, *st[k], step, 1e-3)
                params[k], st[k] = p, [mm, v, vh]
    got = m.export_params()
    for k in params:
        assert float((got[k].double().cpu() - params[k]).abs().max()) <= 5e-5, k


def test_model_api_surface():
    m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64)
    assert [hasattr(m, 'net_query_layer%d' % i) for i in range(14)] == [True] * 14
    assert [hasattr(m, 'net_obs_layer%d' % i) for i in range(7)] == [True] * 7
    assert len(m.net['obs'].layers) == 7 and len(m.net['query'].layers) == 14
    with pytest.raises(ValueError):
        m.call(None, 'bogus')
    assert m.trainable_variables == []       # lazily built, like Keras
    m.build()
    assert sum(v.numel() for v in m.trainable_variables) == 3368071


def test_cfg5_relight_sweep_psnr_vs_oracle(path):
    """cfg5 in miniature (SURVEY 8d): a relight/view sweep is forward-only inference with the cached
    observation features (nlt_test.py semantics), samples sharded round-robin over ranks; quality is
    reported as PSNR(new output, restated-reference output) with xiuminglib's luma PSNR: >= 80 dB."""
    import nlt_test
    from util import synth
    m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64)
    oc = ocfg(cfg)
    params = O.init_params(oc, seed=17, dtype=torch.float64)
    m.build(5, 3)
    m.load_params(params)
    feat = nlt_test.extract_feat(m, [synth.make_batch(2, 64, 64, seed=31)])
    want_feat = O.extract_feat(params, oc, [(b[1].double(), b[5].double()) for b in [synth.make_batch(2, 64, 64, seed=31)]])
    world = 2                                   # two virtual ranks, round-robin sample ownership
    samples = [synth.make_batch(1, 64, 64, seed=200 + i) for i in range(6)]
    worst = 1e9
    for rank in range(world):
        mine = samples[rank::world]
        outs = nlt_test.infer(m, mine, feat)
        for bt, got in zip(mine, outs):
            with torch.no_grad():
                ref, _, _, _ = O.model_call(params, oc, tuple(t.double() if torch.is_tensor(t) else t for t in bt),
                                            'test', obs_override=want_feat)
            worst = min(worst, O.psnr_luma(got[0].cpu().numpy(), ref[0].numpy()))
    assert worst >= 80.0, worst


def test_uint8_inputs_are_bit_identical_to_float32_inputs():
    """A batch whose image tensors arrive as uint8 (datasets with `uint8_inputs`, a quarter of the PCIe bytes) gives
    exactly the outputs of the float32 batch: v / 255 on the device is the host's float32(v / 255.0)."""
    from util import synth
    m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64)
    m.build(5, 3)
    bt = synth.make_batch(2, 64, 64, seed=3)
    u8 = synth.as_uint8(bt)
    assert u8[1].dtype == torch.uint8 and u8[4].dtype == torch.float32
    a = m(bt, mode='vali')
    b = m(u8, mode='vali')
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(a[3]['pred'], b[3]['pred'])


def test_pack_ahead_and_extra_wgrad_streams_do_not_change_results():
    """Scheduling switches only: weight planes packed on the pack stream (engine.PACK_AHEAD) and weight gradients on
    1 / 2 / 3 side streams must give bit-identical predictions and gradients (same kernels, same order per buffer)."""
    import engine
    from util import synth
    saved = (engine.PACK_AHEAD, engine.N_SIDE_STREAMS)
    outs = []
    try:
        for pack, nside in ((False, 1), (True, 1), (True, 2), (True, 3)):
            engine.PACK_AHEAD, engine.N_SIDE_STREAMS = pack, nside
            m, cfg = make_model(uvh=128, uvw=128, imh=64, imw=64)
            m.build(5, 3)
            bt = synth.make_batch(2, 128, 64, seed=11)
            pred, gt, kw, _ = m(bt, mode='train')
            m.set_loss_grad_scale(0.5)
            m.compute_loss(pred, gt, **kw)
            m.backward()
            torch.cuda.synchronize()
            outs.append((pred.clone(), m.bucket.grad.clone()))
    finally:
        engine.PACK_AHEAD, engine.N_SIDE_STREAMS = saved
    for pred, grad in outs[1:]:
        assert torch.equal(pred, outs[0][0])
        assert torch.equal(grad, outs[0][1])
