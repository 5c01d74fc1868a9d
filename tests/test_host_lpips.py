"""LPIPS on the host: the frozen-graph reader (util/tf_graphdef.py), the two float64 oracles of oracle/lpips_oracle.py
against each other and against finite differences, and how the config enables or refuses the term.  The graph is the
reference's own file, which build() copies into oracle/_ref/; without it these tests skip."""
import os

import numpy as np
import pytest
import torch

from oracle import lpips_oracle as LP


@pytest.fixture(scope='module')
def graph():
    path = LP.graph_path()
    if path is None:
        pytest.skip('the LPIPS graph is not in oracle/_ref/ (build() copies it from a reference checkout)')
    return path


@pytest.fixture(scope='module')
def weights(graph):
    from util import tf_graphdef
    return tf_graphdef.load_lpips_alex(graph)


def test_reader_accepts_the_reference_graph(weights):
    from util import tf_graphdef
    assert sorted(weights) == sorted(['scale', 'shift'] + ['%s%d' % (k, i) for k in 'wb' for i in range(1, 6)]
                                     + ['lin%d' % i for i in range(1, 6)])
    for i, (co, ci, k, _, _) in enumerate(tf_graphdef.ALEX, 1):
        assert weights['w%d' % i].shape == (co, ci, k, k) and weights['b%d' % i].shape == (co,)
        assert weights['lin%d' % i].shape == (co,) and (weights['lin%d' % i] >= 0).all()
    assert all(v.dtype == np.float32 for v in weights.values())
    # LPIPS's scaling layer: (x - shift) / scale with shift (-.030, -.088, -.188) and scale (.458, .448, .450)
    np.testing.assert_allclose(weights['scale'], 1 / np.array([.458, .448, .450]), rtol=1e-6)
    np.testing.assert_allclose(weights['shift'], np.array([.030, .088, .188]) / np.array([.458, .448, .450]),
                               rtol=1e-6)


def _doctored(graph, tmp_path, old, new, count=1):
    buf = open(graph, 'rb').read()
    assert buf.count(old) >= count, old
    out = tmp_path / 'doctored.pb'
    out.write_bytes(buf.replace(old, new, count))
    return str(out)


def _node_bytes(graph, name):
    """The serialized NodeDef of `name` (the reader's own decoder finds it; the test then edits bytes inside it)."""
    from util.tf_ckpt import _parse_fields
    for num, _, v in _parse_fields(open(graph, 'rb').read()):
        if num == 1 and any(n == 1 and x == name.encode() for n, _, x in _parse_fields(v)):
            return v
    raise KeyError(name)


def test_reader_rejects_doctored_graphs(graph, tmp_path):
    from util import tf_graphdef
    # conv1's stride 4 -> 2 (strides list [1, 4, 4, 1] of node convolution_6)
    node = _node_bytes(graph, 'convolution_6')
    assert b'\x1a\x04\x01\x04\x04\x01' in node
    bad = node.replace(b'\x1a\x04\x01\x04\x04\x01', b'\x1a\x04\x01\x02\x02\x01')
    with pytest.raises(ValueError, match='stride'):
        tf_graphdef.load_lpips_alex(_doctored(graph, tmp_path, node, bad))
    # conv3's pad 1 -> 2 (the int32 [4, 2] constant of Pad_4, stored as tensor_content)
    pad = tf_graphdef.load_graph(graph)['Pad_4'].inputs[1]
    node = _node_bytes(graph, pad)
    ones = np.array([[0, 0], [0, 0], [1, 1], [1, 1]], np.int32).tobytes()
    assert ones in node
    bad = node.replace(ones, np.array([[0, 0], [0, 0], [2, 2], [2, 2]], np.int32).tobytes())
    with pytest.raises(ValueError, match='pad'):
        tf_graphdef.load_lpips_alex(_doctored(graph, tmp_path, node, bad))
    # truncated file
    out = tmp_path / 'truncated.pb'
    out.write_bytes(open(graph, 'rb').read()[:5000000])
    with pytest.raises(ValueError):
        tf_graphdef.load_lpips_alex(str(out))
    with pytest.raises(FileNotFoundError):
        tf_graphdef.load_lpips_alex(str(tmp_path / 'missing.pb'))


@pytest.mark.parametrize('shape', [(2, 64, 64), (1, 96, 128)])
def test_graph_interpreter_and_restatement_agree(graph, weights, shape):
    from util import tf_graphdef
    nodes = tf_graphdef.load_graph(graph)
    rng = np.random.default_rng(sum(shape))
    gt = rng.random(shape + (3,))
    pred = np.clip(gt + 0.1 * rng.standard_normal(gt.shape), 0, 1)
    a = LP.graph_lpips(nodes, pred, gt)
    b = LP.lpips_torch(weights, torch.from_numpy(pred), torch.from_numpy(gt)).numpy()
    assert a.shape == (shape[0],) and (a > 0).all()
    np.testing.assert_allclose(b, a, rtol=1e-12, atol=0)


def test_restatement_gradient_matches_finite_differences(weights):
    rng = np.random.default_rng(1)
    gt = torch.from_numpy(rng.random((1, 35, 39, 3)))
    pred = (gt + 0.1 * torch.from_numpy(rng.standard_normal(gt.shape))).clamp(0.05, 0.95).requires_grad_(True)
    LP.lpips_torch(weights, pred, gt).sum().backward()
    g = pred.grad
    h = 1e-6
    for idx in [(0, 0, 0, 0), (0, 17, 20, 1), (0, 34, 38, 2), (0, 10, 3, 0), (0, 30, 11, 2)]:
        p1, p0 = pred.detach().clone(), pred.detach().clone()
        p1[idx] += h
        p0[idx] -= h
        fd = float(LP.lpips_torch(weights, p1, gt) - LP.lpips_torch(weights, p0, gt)) / (2 * h)
        assert abs(fd - float(g[idx])) <= 1e-6 * max(abs(fd), 1e-3), (idx, fd, float(g[idx]))


def test_config_enables_or_refuses_the_term(graph, tmp_path):
    import losses
    import models
    from util import io as ioutil
    Model = models.get_model_class('nlt')
    with pytest.raises(NotImplementedError, match='lpips_weights'):
        Model(ioutil.make_config(loss='barron,1e+0lpips'))
    with pytest.raises(FileNotFoundError):
        Model(ioutil.make_config(loss='barron,1e+0lpips', lpips_weights=str(tmp_path / 'missing.pb')))
    wrong = tmp_path / 'wrong.pb'
    wrong.write_bytes(open(graph, 'rb').read()[:100000])
    with pytest.raises(ValueError):
        Model(ioutil.make_config(loss='barron,1e+0lpips', lpips_weights=str(wrong)))
    m = Model(ioutil.make_config(loss='barron,1e+0lpips', lpips_weights=graph))
    assert [(w, type(f).__name__) for w, f in m.wloss] == [(1.0, 'Barron'), (1.0, 'LPIPS')]
    with pytest.raises(NotImplementedError, match='per_ch'):
        losses.LPIPS(per_ch=True, weights_path=graph)
    with pytest.raises(NotImplementedError, match='sample weights'):
        m.wloss[1][1](torch.zeros(1, 32, 32, 3), torch.zeros(1, 32, 32, 3), weights=torch.ones(1, 32, 32, 1))


def test_fetch_keeps_a_verified_copy(graph, monkeypatch, tmp_path):
    monkeypatch.setattr(LP, 'REFERENCE', str(tmp_path / 'no_reference_here'))
    assert LP.fetch_graph() == graph and os.path.isfile(graph)
