"""CPU oracle of the U-Net built with `pool = max | avg`.  TEST INFRASTRUCTURE ONLY.

Restates, in fp64 PyTorch-CPU ops, what the reference computes when a network is built with a pool
(nlt/networks/convnet.py:50-80, nlt/networks/elements.py:42-48, 81-94):

  down block  conv -> norm -> act -> conv -> norm -> act -> pool       (pool: 2x2 / stride 2, padding 'same')
  up block    UpSampling2D(2, 'bilinear') -> Conv2D(n, 2, 'same') (linear, bias) -> deconv -> norm -> act -> ...

on top of oracle/nlt_oracle.py, whose conv, norm, activation, resampler and resize restatements are reused unchanged.
The external ops are restated from their published behaviour; TensorFlow cannot be installed offline, so two facts
stay unpinned (DESIGN.md section 8):
  * which maximum TF 2.2's MaxPoolGrad routes a tie to on the GPU (cuDNN does not document it; TF's own CPU/GPU kernels
    and torch's CPU kernel take the first maximum in row-major order, which is what this oracle does);
  * whether Keras 2.2's UpSampling2D calls the v2 (half-pixel) or the v1 (corner-aligned) resize.  v2 is restated.
The direct-loop functions at the end (np_*) restate the pools and the upsample from their definitions, independently
of the tensor formulation, and pin it in tests/test_oracle_pool.py.
"""
import math

import numpy as np
import torch

from oracle import nlt_oracle as O


# ----------------------------------------------------------------------------
# external ops
# ----------------------------------------------------------------------------
def _taps(x, fill):
    """[B,H,W,C] -> [4,B,ceil(H/2),ceil(W/2),C] window taps in row-major order, and the per-tap validity [4,1,Ho,Wo,1];
    odd sizes pad the right / bottom edge with `fill` (the SAME window is clipped there)."""
    B, H, W, C = x.shape
    Ho, Wo = -(-H // 2), -(-W // 2)
    xp = torch.nn.functional.pad(x, (0, 0, 0, 2 * Wo - W, 0, 2 * Ho - H), value=fill)
    valid = torch.zeros(1, 2 * Ho, 2 * Wo, 1, dtype=torch.bool, device=x.device)
    valid[:, :H, :W] = True
    taps = [xp[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)]
    vals = [valid[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)]
    return torch.stack(taps), torch.stack(vals)


def first_argmax(x):
    """Index (0..3, row-major tap order) of the FIRST maximum of every 2x2 window of x: [B,Ho,Wo,C] int64."""
    taps, valid = _taps(x.detach(), -math.inf)
    best = taps[0].clone()
    arg = torch.zeros(best.shape, dtype=torch.int64, device=x.device)
    for t in range(1, 4):
        take = valid[t] & (taps[t] > best)
        best = torch.where(take, taps[t], best)
        arg = torch.where(take, torch.full_like(arg, t), arg)
    return arg


def max_pool_same(x, argmax=None):
    """tf.keras.layers.MaxPooling2D(2, 2, 'same') (elements.py:81-94).  The gradient goes to the window's first maximum
    in row-major order, or to the taps `argmax` names (the masked-oracle tests pass the product's)."""
    taps, _ = _taps(x, -math.inf)
    if argmax is None:
        argmax = first_argmax(x)
    return torch.gather(taps, 0, argmax.unsqueeze(0)).squeeze(0)


def avg_pool_same(x):
    """tf.keras.layers.AveragePooling2D(2, 2, 'same'): the mean over the VALID taps of each window."""
    taps, valid = _taps(x, 0.0)
    s = ((taps[0] + taps[1]) + taps[2]) + taps[3]
    return s / valid.sum(dim=0).to(x.dtype)


def upsample2x_bilinear(x):
    """tf.keras.layers.UpSampling2D(2, interpolation='bilinear') = tf.image.resize(x, (2H, 2W)), half-pixel centres."""
    return O.resize_bilinear(x, 2 * x.shape[1], 2 * x.shape[2])


# ----------------------------------------------------------------------------
# network
# ----------------------------------------------------------------------------
def has_pool(cfg):
    return str(cfg.get('pool', 'None')).lower() != 'none'


def model_channels(cfg, c_query, c_obs):
    """nlt_oracle.model_channels for a pooling network: per net, per layer, per conv (kind, Cin, Cout, k, s).  Up blocks
    list the upconv's conv first: ('conv', Cin, n, 2, 1), ('deconv', n, n, k, s), ('deconv', n, n, k, 1)."""
    chans = O.model_channels(cfg, c_query, c_obs)
    if not has_pool(cfg):
        return chans
    plan, _ = O.network_plan(cfg['depth0'], cfg['depth'])
    q = []
    for (kind, n), convs in zip(plan, chans['query']):
        if kind == 'up':
            cin = convs[0][1]
            convs = [('conv', cin, n, 2, 1), ('deconv', n, n, convs[0][3], convs[0][4]), convs[1]]
        q.append(convs)
    return {'query': q, 'obs': chans['obs']}


def init_params(cfg, c_query=5, c_obs=3, seed=0, dtype=torch.float32, bias_range=0.1):
    """nlt_oracle.init_params over model_channels above (norm parameters ride on the convs followed by a norm)."""
    g = torch.Generator().manual_seed(seed)
    chans = model_channels(cfg, c_query, c_obs)
    params = {}
    for net in ('query', 'obs'):
        for li, convs in enumerate(chans[net]):
            for ci, (kind, cin, cout, k, _s) in enumerate(convs):
                limit = math.sqrt(6.0 / (k * k * (cin + cout)))
                shape = (k, k, cin, cout) if kind == 'conv' else (k, k, cout, cin)
                w = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * limit
                b = (torch.rand((cout,), generator=g, dtype=torch.float64) * 2 - 1) * bias_range
                params['%s.%d.%d.kernel' % (net, li, ci)] = w.to(dtype)
                params['%s.%d.%d.bias' % (net, li, ci)] = b.to(dtype)
                normed = len(convs) >= 2 and ci >= len(convs) - 2
                if str(cfg.get('norm', 'None')) == 'instance' and normed:
                    params['%s.%d.%d.norm.kernel' % (net, li, ci)] = \
                        (1.0 + 0.2 * (torch.rand((cout,), generator=g, dtype=torch.float64) - 0.5)).to(dtype)
                    params['%s.%d.%d.norm.bias' % (net, li, ci)] = \
                        (0.2 * (torch.rand((cout,), generator=g, dtype=torch.float64) - 0.5)).to(dtype)
    return params


def _act(x, type_, key):
    """Activation of the conv / norm named `key` ('query.3.1'); tests substitute the product's branch masks."""
    return O.act(x, type_)


def _pool(x, kind, key):
    """Pool of the block named `key` ('query.3.pool'); tests substitute the product's argmax."""
    return max_pool_same(x) if kind == 'max' else avg_pool_same(x)


def apply_layer(params, cfg, net, li, x):
    """One entry of Network.layers of a pooling network (nlt_oracle.apply_layer otherwise)."""
    if not has_pool(cfg):
        return O.apply_layer(params, cfg, net, li, x)
    assert cfg['stride'] == 1, 'pooling networks take stride 1'
    plan, _ = O.network_plan(cfg['depth0'], cfg['depth'])
    kind = plan[li][0]
    a, nm = cfg['act'], cfg.get('norm', 'None')
    w = lambda ci: params['%s.%d.%d.kernel' % (net, li, ci)]
    b = lambda ci: params['%s.%d.%d.bias' % (net, li, ci)]
    g = lambda ci: params.get('%s.%d.%d.norm.kernel' % (net, li, ci))
    bt = lambda ci: params.get('%s.%d.%d.norm.bias' % (net, li, ci))
    key = lambda ci: '%s.%d.%d' % (net, li, ci)
    if kind == 'conv1x1':
        return O.conv2d_same(x, w(0), b(0), 1)
    if kind == 'down':
        x = _act(O.norm(O.conv2d_same(x, w(0), b(0), 1), nm, g(0), bt(0)), a, key(0))
        x = _act(O.norm(O.conv2d_same(x, w(1), b(1), 1), nm, g(1), bt(1)), a, key(1))
        return _pool(x, cfg['pool'], '%s.%d.pool' % (net, li))
    x = O.conv2d_same(upsample2x_bilinear(x), w(0), b(0), 1)                 # upconv: linear
    x = _act(O.norm(O.conv2d_transpose_same(x, w(1), b(1), 1), nm, g(1), bt(1)), a, key(1))
    return _act(O.norm(O.conv2d_transpose_same(x, w(2), b(2), 1), nm, g(2), bt(2)), a, key(2))


def net_call(params, cfg, query_x, obs_xs, obs_override=None):
    """Model._call (nlt/models/nlt.py:141-199), the walk of nlt_oracle.net_call over apply_layer above."""
    _, contracting = O.network_plan(cfg['depth0'], cfg['depth'])
    use_obs = cfg.get('use_obs', True)
    featmaps, query_y = [], None
    for li, contr in enumerate(contracting):
        if contr:
            obs_ys = [apply_layer(params, cfg, 'obs', li, x) for x in obs_xs]
            obs_agg = torch.stack(obs_ys, dim=-1).mean(dim=-1)
            obs_xs = obs_ys
            query_y = apply_layer(params, cfg, 'query', li, query_x)
            if use_obs:
                if obs_override is not None:
                    obs_agg = obs_override[li]
                    if obs_agg.shape[0] != query_y.shape[0]:                  # batch-1 override (nlt_test.py:84)
                        obs_agg = obs_agg.expand(query_y.shape[0], -1, -1, -1)
                query_x = torch.cat((query_y, obs_agg), dim=-1)
            else:
                query_x = query_y
            featmaps.append(query_x)
        else:
            if featmaps:
                query_x = torch.cat((query_x, featmaps.pop()), dim=-1)
            query_y = apply_layer(params, cfg, 'query', li, query_x)
            query_x = query_y
    return query_y


def model_call(params, cfg, batch, mode, obs_override=None):
    """Model.call (nlt/models/nlt.py:89-139) of nlt_oracle.model_call over net_call above."""
    id_, base, cvis, lvis, warp, rgb, rgb_camspc, nn_id, nn_base, nn_rgb, nn_rgb_camspc = batch
    x = torch.cat((base, cvis, lvis), dim=3)
    y_obs = [nn_rgb[k] - nn_base[k] for k in range(nn_rgb.shape[0])] if nn_rgb.dim() == 5 else [nn_rgb - nn_base]
    pred = net_call(params, cfg, x, y_obs, obs_override=obs_override)
    if cfg.get('skip_connect_base', True):
        pred = pred + base
    warp = torch.stack((warp[..., 0] * cfg['uvw'], warp[..., 1] * cfg['uvh']), dim=3)
    fg = O.set_left_top_corner(torch.ones_like(pred), 0)
    base = O.set_left_top_corner(base, 0)
    pred = O.set_left_top_corner(pred, 0)
    fg_c = O.resize_bilinear(O.resampler(fg, warp), cfg['imh'], cfg['imw'])
    pred_c = O.resize_bilinear(O.resampler(pred, warp), cfg['imh'], cfg['imw'])
    if mode in ('train', 'vali'):
        return pred_c, O.alpha_blend(rgb_camspc, fg_c)
    return pred_c, None


# ----------------------------------------------------------------------------
# direct-loop restatements (numpy, small sizes)
# ----------------------------------------------------------------------------
def np_max_pool_same(x):
    """y[o] = max over the valid taps of window o; also returns the first-maximum tap (row-major) per output."""
    B, H, W, C = x.shape
    Ho, Wo = -(-H // 2), -(-W // 2)
    y = np.zeros((B, Ho, Wo, C))
    arg = np.zeros((B, Ho, Wo, C), dtype=np.int64)
    for b in range(B):
        for oy in range(Ho):
            for ox in range(Wo):
                for c in range(C):
                    best, bt = None, 0
                    for t, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
                        iy, ix = 2 * oy + dy, 2 * ox + dx
                        if iy < H and ix < W and (best is None or x[b, iy, ix, c] > best):
                            best, bt = x[b, iy, ix, c], t
                    y[b, oy, ox, c], arg[b, oy, ox, c] = best, bt
    return y, arg


def np_avg_pool_same(x):
    B, H, W, C = x.shape
    Ho, Wo = -(-H // 2), -(-W // 2)
    y = np.zeros((B, Ho, Wo, C))
    for oy in range(Ho):
        for ox in range(Wo):
            n, s = 0, 0.0
            for dy in (0, 1):
                for dx in (0, 1):
                    if 2 * oy + dy < H and 2 * ox + dx < W:
                        s = s + x[:, 2 * oy + dy, 2 * ox + dx]
                        n += 1
            y[:, oy, ox] = s / n
    return y


def np_upsample2x(x):
    """The 1-D stencil out[2i] = .25 x[i-1] + .75 x[i], out[2i+1] = .75 x[i] + .25 x[i+1] (index clamped), applied
    along H and then along W."""
    def along(a, axis):
        n = a.shape[axis]
        out = []
        for i in range(n):
            lo, hi = max(i - 1, 0), min(i + 1, n - 1)
            t = lambda j: np.take(a, j, axis=axis)
            out += [0.25 * t(lo) + 0.75 * t(i), 0.75 * t(i) + 0.25 * t(hi)]
        return np.stack(out, axis=axis)
    return along(along(np.asarray(x, dtype=np.float64), 1), 2)
