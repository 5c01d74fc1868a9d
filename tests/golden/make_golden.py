"""Generates the committed fixtures of tests/golden/.

  python tests/golden/make_golden.py REFERENCE_CHECKOUT   # rewrites the .npz files

* gen_feat_n_reference.npz -- outputs of the REFERENCE's own
  nlt/util/net.py:gen_feat_n (the only module on the path importable without
  TensorFlow), imported from a checkout of google/neural-light-transport.
* model_h64.npz -- fp64 run of oracle/nlt_oracle.py (the restated reference) on
  a seeded 64x64 dragon_specular-shaped problem: forward, loss, gradients.
  NOTE: this pins the oracle against regressions; the reference itself has no
  golden for this path (parity unpinned, SURVEY.md 8c).
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, 'neural-light-transport_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import nlt_oracle as O   # noqa: E402
from util import synth               # noqa: E402

CFG = dict(depth0=16, depth=256, kernel=2, stride=2, norm='None', act='leakyrelu', pool='None',
           use_obs=True, skip_connect_base=True, imh=64, imw=64, uvh=64, uvw=64)
B, SEED = 2, 1234


def batch(dtype):
    b = synth.make_batch(B, CFG['uvh'], CFG['imh'], seed=SEED)
    return tuple(t.to(dtype) if torch.is_tensor(t) else t for t in b)


def compute(dtype=torch.float64):
    params = O.init_params(CFG, seed=7, dtype=dtype)
    for v in params.values():
        v.requires_grad_(True)
    bt = batch(dtype)
    pred, gt, _, to_vis = O.model_call(params, CFG, bt, 'train')
    per_ex = O.l2_loss(gt, pred, keep_batch=True)
    loss = per_ex.sum() / B
    loss.backward()
    out = {'pred_camspc': pred.detach().numpy(), 'gt_camspc': gt.detach().numpy(),
           'pred_uv': to_vis['pred'].detach().numpy(), 'per_example_loss': per_ex.detach().numpy()}
    names = sorted(params)
    out['grad_l2norm'] = np.array([float(params[n].grad.norm()) for n in names])
    out['grad_sum'] = np.array([float(params[n].grad.sum()) for n in names])
    for n in ('query.0.0.kernel', 'query.13.0.kernel', 'obs.0.0.kernel', 'query.1.0.bias', 'query.12.1.kernel'):
        out['grad:' + n] = params[n].grad.numpy()
    return out


def main():
    spec = importlib.util.spec_from_file_location('refnet', os.path.join(sys.argv[1], 'nlt', 'util', 'net.py'))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    gf = {}
    for a, b in [(16, 256), (16, 1024), (16, 64), (8, 64), (4, 4), (16, 16), (5, 100), (2, 8), (32, 512)]:
        for f in (3, 1, 4):
            if b >= f:
                gf['%d_%d_%d' % (a, b, f)] = np.array(ref.gen_feat_n(a, b, f))
    np.savez(os.path.join(HERE, 'gen_feat_n_reference.npz'), **gf)
    np.savez_compressed(os.path.join(HERE, 'model_h64.npz'), **compute())
    print('wrote goldens')


if __name__ == '__main__':
    main()
