"""Host side of the pooling U-Net (`pool = max | avg`, stride 1): network wiring, geometry checks and checkpoint keys.
CPU only (no kernel is launched)."""
import numpy as np
import pytest
import torch

from oracle import pool_oracle as P


def _cpu_model(uv=64, **over):
    import models
    from util import io as ioutil
    cfg = ioutil.make_config(uvh=uv, uvw=uv, imh=uv, imw=uv, **over)
    model = models.get_model_class('nlt')(cfg)
    model.register_trainable()
    model.device = torch.device('cpu')
    model.build(5, 3)
    return model


@pytest.mark.parametrize('kind', ['max', 'avg'])
def test_pool_network_structure(kind):
    from networks import convnet
    net = convnet.Network(16, 256, 2, 1, norm_type='None', act_type='leakyrelu', pool_type=kind)
    assert len(net.layers) == 14
    assert net.is_contracting == [True] * 7 + [False] * 7
    assert net.spatsize_changes == [1] + [0.5] * 6 + [2] * 6 + [1]
    kinds = [[(c.kind, c.k, c.s, c.cout, c.act) for c in blk.convs] for blk in net.layers]
    assert kinds[0] == [('conv', 1, 1, 16, None)] and net.layers[0].pool is None
    assert kinds[1] == [('conv', 2, 1, 16, 'leakyrelu'), ('conv', 2, 1, 16, 'leakyrelu')]
    assert kinds[7] == [('conv', 2, 1, 128, None), ('deconv', 2, 1, 128, 'leakyrelu'), ('deconv', 2, 1, 128, 'leakyrelu')]
    for li in range(1, 7):
        assert net.layers[li].pool.kind == kind and not net.layers[li].upconv
    for li in range(7, 13):
        assert net.layers[li].pool is None and net.layers[li].upconv
        assert kinds[li][0][:3] == ('conv', 2, 1) and kinds[li][0][4] is None      # upconv: linear 2x2 conv
    assert kinds[13] == [('conv', 1, 1, 3, None)]
    # distinct pool objects per block, and norm layers after the two deconvs only
    assert len({id(net.layers[li].pool) for li in range(1, 7)}) == 6
    px = convnet.Network(16, 256, 2, 1, norm_type='pixel', act_type='leakyrelu', pool_type=kind)
    assert px.layers[8].norms[0] is None and [n.kind for n in px.layers[8].norms[1:]] == ['pixel', 'pixel']
    assert [c.act for c in px.layers[8].convs] == [None, None, None]


def test_pool_with_stride_2_raises_with_reason():
    from networks import convnet
    for kind in ('max', 'avg'):
        with pytest.raises(NotImplementedError, match='stride=1'):
            convnet.Network(16, 256, 2, 2, norm_type='None', act_type='relu', pool_type=kind)
    with pytest.raises(NotImplementedError):
        convnet.Network(16, 256, 2, 1, norm_type='None', act_type='relu', pool_type='min')


@pytest.mark.parametrize('kind,kernel', [('max', 2), ('avg', 3)])
def test_pool_model_parameters_follow_the_oracle(kind, kernel):
    model = _cpu_model(stride=1, pool=kind, kernel=kernel)
    cfg = dict(depth0=16, depth=256, kernel=kernel, stride=1, norm='None', act='leakyrelu', pool=kind, use_obs=True)
    params = P.init_params(cfg, seed=0)
    mine = {n: c for n, c in model.named_convs()}
    assert set(k.rsplit('.', 1)[0] for k in params) == set(mine)
    for name, c in mine.items():
        assert tuple(c.kernel.shape) == tuple(params[name + '.kernel'].shape), name
    n = sum(v.numel() for v in params.values())
    assert sum(v.numel() for v in model.trainable_variables) == n
    if kernel == 2:
        assert n == 3455683          # pinned: 2x2 kernels, 5 / 3 input channels
    # the flat bucket covers every layer, including the three-conv up blocks
    assert model.bucket.n >= n and len(model.bucket.layers) == len(mine)


def test_uv_size_not_divisible_raises_before_any_launch():
    from util import synth
    model = _cpu_model(uv=96, stride=1, pool='max')
    bt = synth.make_batch(1, 96, 96, seed=0)
    with pytest.raises(ValueError, match='multiple of 2\\*\\*6'):
        model(bt, mode='train')
    with pytest.raises(ValueError):
        model._call(torch.zeros(1, 64, 80, 5), [torch.zeros(1, 64, 80, 3)])
    # stride 2 without a pool keeps accepting any size (unchanged)
    _cpu_model(uv=96)._check_uv_size(96, 40)


def test_tf_checkpoint_round_trip_of_a_pool_model(tmp_path):
    """The up block's conv0 sits in the nested upconv Sequential: layer_with_weights-0/layer_with_weights-0; the
    deconvs are layer_with_weights-1 / -2.  Keys and Adam slots round-trip."""
    import trainvali
    from util import ckpt, tf_ckpt
    model = _cpu_model(stride=1, pool='max')
    opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
    g = torch.Generator().manual_seed(4)
    model.flat_params.copy_(torch.randn(model.flat_params.numel(), generator=g))
    opt.m, opt.v, opt.vhat = (torch.rand(model.flat_params.numel(), generator=g) for _ in range(3))
    opt.iterations = 7
    prefix = str(tmp_path / 'ckpt-7')
    tf_ckpt.save_nlt_state(prefix, ckpt.state_dict(model, opt, step=7))
    raw = tf_ckpt.load_bundle(prefix)
    sfx = '/.ATTRIBUTES/VARIABLE_VALUE'
    assert raw['net/net_query_layer7/layer_with_weights-0/layer_with_weights-0/kernel' + sfx].shape == (2, 2, 1024, 128)
    assert raw['net/net_query_layer7/layer_with_weights-1/kernel' + sfx].shape == (2, 2, 128, 128)
    assert raw['net/net_query_layer12/layer_with_weights-2/bias' + sfx].shape == (4,)
    assert 'net/net_query_layer7/layer_with_weights-0/kernel' + sfx not in raw
    assert 'net/net_query_layer3/layer_with_weights-0/kernel' + sfx in raw                      # down blocks: flat
    assert ('net/net_query_layer9/layer_with_weights-0/layer_with_weights-0/bias/.OPTIMIZER_SLOT/optimizer/vhat'
            + sfx) in raw
    state = tf_ckpt.load_nlt_state(prefix)
    assert 'net/net_query_layer7/conv0/kernel' in state and 'optimizer/m/net_query_layer12/conv2/bias' in state
    other = _cpu_model(stride=1, pool='max')
    other_opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
    assert ckpt.restore(prefix, other, other_opt) == 7
    for (n1, c1), (n2, c2) in zip(model.named_convs(), other.named_convs()):
        assert n1 == n2 and torch.equal(c1.kernel, c2.kernel) and torch.equal(c1.bias, c2.bias)
    for slot in ('m', 'v', 'vhat'):
        a, b = ckpt._slot_views(model, getattr(opt, slot)), ckpt._slot_views(other, getattr(other_opt, slot))
        assert all(torch.equal(a[k], b[k]) for k in a)
    assert np.int64(state['step']) == 7
