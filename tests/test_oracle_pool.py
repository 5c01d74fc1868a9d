"""The pooling U-Net's oracle (oracle/pool_oracle.py) against direct-loop restatements, known answers and adjoint
identities.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import nlt_oracle as O
from oracle import pool_oracle as P


def _t(a):
    return torch.as_tensor(np.asarray(a, dtype=np.float64))


@pytest.mark.parametrize('shape', [(2, 6, 8, 3), (1, 5, 7, 4), (2, 1, 1, 2), (1, 3, 1, 5), (3, 9, 4, 1)])
def test_pools_agree_with_direct_loops(shape):
    rng = np.random.default_rng(sum(shape))
    x = rng.standard_normal(shape)
    x[..., 0] = np.round(x[..., 0])                       # many ties in one channel
    y_loop, arg_loop = P.np_max_pool_same(x)
    assert np.array_equal(P.max_pool_same(_t(x)).numpy(), y_loop)
    assert np.array_equal(P.first_argmax(_t(x)).numpy(), arg_loop)
    np.testing.assert_allclose(P.avg_pool_same(_t(x)).numpy(), P.np_avg_pool_same(x), rtol=1e-15, atol=1e-15)


def test_pool_known_answers_odd_sizes_ties_and_flat_windows():
    # 3 x 3: windows {(0,0),(0,1),(1,0),(1,1)}, {(0,2),(1,2)}, {(2,0),(2,1)}, {(2,2)}
    x = _t([[1, 2, 3], [4, 5, 6], [7, 8, 9]]).reshape(1, 3, 3, 1)
    assert P.max_pool_same(x).flatten().tolist() == [5, 6, 8, 9]
    assert P.avg_pool_same(x).flatten().tolist() == [3.0, 4.5, 7.5, 9.0]       # divisor = valid taps (4, 2, 2, 1)
    # forced ties: the gradient goes to the FIRST maximum in row-major tap order
    x = _t([[2, 7, 1, 1], [7, 7, 1, 1]]).reshape(1, 2, 4, 1).requires_grad_(True)
    P.max_pool_same(x).sum().backward()
    assert x.grad.flatten().tolist() == [0, 1, 1, 0, 0, 0, 0, 0]
    assert P.first_argmax(x).flatten().tolist() == [1, 0]
    # all-equal window: the first tap; -inf padding never wins
    x = _t(np.full((1, 3, 3, 1), -5.0)).requires_grad_(True)
    y = P.max_pool_same(x)
    assert y.flatten().tolist() == [-5.0] * 4
    y.sum().backward()
    assert x.grad.flatten().tolist() == [1, 0, 1, 0, 0, 0, 1, 0, 1]
    # avg adjoint at a clipped edge: d_y / valid taps
    x = _t(np.zeros((1, 3, 3, 1))).requires_grad_(True)
    P.avg_pool_same(x).sum().backward()
    assert x.grad.flatten().tolist() == [.25, .25, .5, .25, .25, .5, .5, .5, 1.0]


def test_upsample_matches_hand_stencils_and_direct_loops():
    # 1-D along W (H = 1): out[2i] = .25 x[i-1] + .75 x[i], out[2i+1] = .75 x[i] + .25 x[i+1], clamped
    x = _t([1.0, 5.0, 3.0]).reshape(1, 1, 3, 1)
    y = P.upsample2x_bilinear(x)
    assert y.shape == (1, 2, 6, 1)
    want = [1.0, 0.75 * 1 + 0.25 * 5, 0.25 * 1 + 0.75 * 5, 0.75 * 5 + 0.25 * 3, 0.25 * 5 + 0.75 * 3, 3.0]
    assert y[0, 0, :, 0].tolist() == want and y[0, 1, :, 0].tolist() == want
    # a single pixel replicates
    assert P.upsample2x_bilinear(_t([[[[2.5]]]])).flatten().tolist() == [2.5] * 4
    rng = np.random.default_rng(3)
    for shape in ((2, 3, 4, 3), (1, 1, 5, 2), (1, 4, 1, 1), (2, 7, 6, 4)):
        x = rng.standard_normal(shape)
        np.testing.assert_allclose(P.upsample2x_bilinear(_t(x)).numpy(), P.np_upsample2x(x), rtol=0, atol=1e-14)


@pytest.mark.parametrize('shape', [(2, 5, 7, 3), (1, 1, 1, 2), (1, 8, 6, 4), (1, 1, 9, 1)])
def test_adjoint_identities(shape):
    """<U x, g> = <x, U^T g> for the upsample and <A x, g> = <x, A^T g> for the average pool, with U^T / A^T the
    autograd adjoints the oracle's gradients use."""
    g0 = torch.Generator().manual_seed(sum(shape))
    for op, oshape in ((P.upsample2x_bilinear, (shape[0], 2 * shape[1], 2 * shape[2], shape[3])),
                       (P.avg_pool_same, (shape[0], -(-shape[1] // 2), -(-shape[2] // 2), shape[3]))):
        x = torch.randn(shape, generator=g0, dtype=torch.float64).requires_grad_(True)
        g = torch.randn(oshape, generator=g0, dtype=torch.float64)
        y = op(x)
        assert y.shape == oshape
        (xt,) = torch.autograd.grad(y, x, g)
        lhs, rhs = float((y * g).sum().detach()), float((x * xt).sum().detach())
        assert abs(lhs - rhs) <= 1e-12 * max(1.0, abs(lhs)), (op.__name__, lhs, rhs)


def test_pool_model_channels_and_parameters():
    cfg = dict(depth0=16, depth=256, kernel=2, stride=1, norm='None', act='leakyrelu', pool='max', use_obs=True)
    ch = P.model_channels(cfg, 5, 3)
    assert ch['query'][7] == [('conv', 1024, 128, 2, 1), ('deconv', 128, 128, 2, 1), ('deconv', 128, 128, 2, 1)]
    assert ch['query'][12] == [('conv', 40, 4, 2, 1), ('deconv', 4, 4, 2, 1), ('deconv', 4, 4, 2, 1)]
    assert ch['query'][1] == [('conv', 32, 16, 2, 1), ('conv', 16, 16, 2, 1)]
    assert ch['obs'] == O.model_channels(dict(cfg, pool='None'), 5, 3)['obs']
    params = P.init_params(cfg, seed=1)
    assert params['query.7.0.kernel'].shape == (2, 2, 1024, 128) and params['query.7.2.kernel'].shape == (2, 2, 128, 128)
    assert 'query.7.3.kernel' not in params and 'query.6.2.kernel' not in params
    # no pool: the plain oracle, unchanged
    assert P.model_channels(dict(cfg, pool='None'), 5, 3) == O.model_channels(dict(cfg, pool='None'), 5, 3)


def test_pool_network_forward_shapes_and_obs_override():
    cfg = dict(depth0=16, depth=32, kernel=2, stride=1, norm="pixel", act="leakyrelu", pool="avg", use_obs=True,
               skip_connect_base=True, uvh=16, uvw=16, imh=16, imw=16)
    params = P.init_params(cfg, seed=2, dtype=torch.float64)
    g = torch.Generator().manual_seed(0)
    q = torch.randn(2, 16, 16, 5, generator=g, dtype=torch.float64)
    o = torch.randn(2, 16, 16, 3, generator=g, dtype=torch.float64)
    y = P.net_call(params, cfg, q, [o])
    assert y.shape == (2, 16, 16, 3)
    # a batch-1 override equals the same override tiled to the batch
    feats = []
    x = o[:1]
    _, contracting = O.network_plan(cfg['depth0'], cfg['depth'])
    for li in range(sum(contracting)):
        x = P.apply_layer(params, cfg, 'obs', li, x)
        feats.append(x)
    a = P.net_call(params, cfg, q, [o], obs_override=feats)
    b = P.net_call(params, cfg, q, [o], obs_override=[f.expand(2, -1, -1, -1).clone() for f in feats])
    assert torch.equal(a, b)
