"""norm = pixel / instance (nlt/networks/elements.py:97-121): the CUDA ops against the oracle restatement, and whole-model
forward + backward with either norm.  'instance' has no upstream oracle (tf.contrib is gone in TF2, SURVEY D2): it is
checked against this repo's own restatement only."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nlt_oracle as O   # noqa: E402
from tests.test_gpu_model import make_model, ocfg, rel_fro   # noqa: E402


@pytest.mark.parametrize('kind', ['pixel', 'instance'])
@pytest.mark.parametrize('N,H,W,C', [(2, 8, 8, 16), (3, 33, 17, 4), (1, 64, 64, 64), (2, 40, 40, 256), (2, 5, 7, 1024)])
@pytest.mark.parametrize('act', ['leakyrelu', None])
def test_norm_layer_forward_backward(kind, N, H, W, C, act):
    import engine
    dev = torch.device('cuda')
    torch.manual_seed(N * 100 + C)
    x = torch.randn(N, H, W, C) * 2 + 0.3
    L = engine.NormLayer(kind, act)
    L.build(C, dev)
    g = b = None
    if kind == 'instance':
        L.kernel.copy_(1 + 0.3 * torch.randn(C))
        L.bias.copy_(0.3 * torch.randn(C))
        g, b = L.kernel.double().cpu().requires_grad_(True), L.bias.double().cpu().requires_grad_(True)
    x64 = x.double().requires_grad_(True)
    y64 = O.norm(x64, kind, g, b)
    if act:
        y64 = O.act(y64, act)
    tape = engine.Tape()
    xa = engine.Act(x.to(dev).contiguous(), act=None, needs_grad=True)
    y = L.forward(xa, tape)
    assert float((y.t.double().cpu() - y64.detach()).abs().max()) <= 2e-5 * max(1.0, float(y64.abs().max()))
    gy = torch.randn_like(y64)
    y64.backward(gy)
    dz = gy * (torch.where(y64 > 0, 1.0, 0.3) if act == 'leakyrelu' else 1.0)     # the consumer applies act' from y
    y.grad = dz.float().to(dev).contiguous()
    tape.backward()
    assert rel_fro(xa.grad, x64.grad) <= 2e-5
    if kind == 'instance':
        assert rel_fro(L.gkernel, g.grad) <= 2e-5 and rel_fro(L.gbias, b.grad) <= 2e-5


@pytest.mark.parametrize('kind', ['pixel', 'instance'])
def test_model_with_norm_forward_backward(kind):
    """Whole model with conv -> norm -> act blocks (fp32 kernels; the masked-oracle argument of test_gpu_parity.py
    applies unchanged, so the strict bars are used on the activation-branch-agnostic quantities)."""
    import nlt_native as nat
    from util import synth
    with nat.options(tc=0):
        m, cfg = make_model(uvh=64, uvw=64, imh=64, imw=64, norm=kind)
        oc = ocfg(cfg)
        B = 2
        bt = synth.make_batch(B, 64, 64, seed=11)
        params = O.init_params(oc, seed=7, dtype=torch.float64)
        m.build(5, 3)
        m.load_params(params)
        for v in params.values():
            v.requires_grad_(True)
        p64, g64, _, _ = O.model_call(params, oc, tuple(t.double() if torch.is_tensor(t) else t for t in bt), 'train')
        (O.l2_loss(g64, p64, keep_batch=True).sum() / B).backward()
        pred, gt, kw, _ = m(bt, mode='train')
        kw['keep_batch'] = True
        m.set_loss_grad_scale(1.0 / B)
        m.compute_loss(pred, gt, **kw)
        m.backward()
    assert float((pred.double().cpu() - p64.detach()).abs().max()) <= 5e-5
    grads = m.export_grads()
    assert set(grads) == set(params)
    # a conv bias in front of an instance norm has an identically zero gradient (the norm removes the mean):
    # compare those on an absolute scale, everything else relatively
    scale = max(float(params[k].grad.norm()) for k in params)
    worst = max((rel_fro(grads[k], params[k].grad) if float(params[k].grad.norm()) > 1e-9 * scale
                 else float(grads[k].double().norm().cpu()) / scale, k) for k in params)
    assert worst[0] <= 3e-3, worst          # plain oracle: includes LeakyReLU derivative-bit flips
    # checkpoint keys carry the norm parameters
    if kind == 'instance':
        from util import ckpt
        st = ckpt.state_dict(m)
        assert 'net/net_query_layer3/norm0/kernel' in st and st['net/net_obs_layer2/norm1/bias'].shape == (32,)
