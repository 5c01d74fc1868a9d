"""CPU oracle for the NLT UV-space hot path.  TEST INFRASTRUCTURE ONLY.

This file is a restatement, in plain PyTorch-CPU ops, of the arithmetic that
google/neural-light-transport runs on its per-texel forward/backward path.  It
exists so that the CUDA product path (neural-light-transport_b200/) can be
checked; it is NOT part of the product.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs may import it.

PARITY UNPINNED: the reference has no test, golden tensor or checkpoint for
this path (SURVEY.md section 4 / 8c) and TensorFlow cannot be imported here, so
this restatement is pinned only by (i) hand-computed known-answer vectors,
(ii) an independent direct-loop numpy restatement (oracle/np_ref.py), and
(iii) the one docstring example the reference carries (util/net.py:23).

Every function cites the reference file:line it follows (paths relative to a
checkout of google/neural-light-transport).  External-op semantics (TF 2.2 Conv2D/Conv2DTranspose 'same',
tfa.image.resampler 0.10, tf.image.resize, Keras Adam(amsgrad)) are restated
from their published behaviour; see SURVEY.md section 8c.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------
# channel schedule -- nlt/util/net.py:18-56
# ----------------------------------------------------------------------------
def gen_feat_n(min_n, max_n, final_n=3):
    """nlt/util/net.py:18-56 (numbers of channels per block, excluding the
    first full-resolution 1x1 layer)."""
    assert max_n >= min_n and max_n >= final_n
    lo, hi = int(np.log2(min_n)), int(np.log2(max_n))
    seq = [2 ** i for i in range(lo + 1, hi + 1)]
    if not seq or seq[0] != min_n:
        seq = [min_n] + seq
    if seq[-1] != max_n:
        seq.append(max_n)
    seq = seq + seq[::-1]
    seq += [2 ** i for i in range(int(np.log2(seq[-1])) - 1,
                                  int(np.log2(final_n)), -1)]
    while seq and seq[-1] < final_n:
        seq.pop()
    seq.append(final_n)
    return seq


# ----------------------------------------------------------------------------
# layer plan -- nlt/networks/convnet.py:31-90
# ----------------------------------------------------------------------------
def network_plan(depth0, depth):
    """Returns [(kind, n_out)], is_contracting, following convnet.py:41-87.
    kind in {'conv1x1', 'down', 'up'}."""
    n_feat = gen_feat_n(depth0, depth)
    plan, contracting = [('conv1x1', n_feat[0])], [True]
    prev = 0
    for n in n_feat[:-1]:
        if n >= prev:            # convnet.py:49 -- 256 -> 256 is "contracting"
            plan.append(('down', n))
            contracting.append(True)
        else:
            plan.append(('up', n))
            contracting.append(False)
        prev = n
    plan.append(('conv1x1', n_feat[-1]))
    contracting.append(False)
    return plan, contracting


# ----------------------------------------------------------------------------
# external-op restatements
# ----------------------------------------------------------------------------
def same_pad(n, k, s):
    """TF 'SAME': out=ceil(n/s); total=max((out-1)s+k-n,0); before=total//2."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def conv2d_same(x, w, b, s):
    """tf.keras.layers.Conv2D(padding='same') -- elements.py:26-31.
    x NHWC, w (kh,kw,Ci,Co) Keras layout, b (Co,) or None."""
    kh, kw = w.shape[0], w.shape[1]
    pt, pb = same_pad(x.shape[1], kh, s)
    pl, pr = same_pad(x.shape[2], kw, s)
    xn = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
    y = F.conv2d(xn, w.permute(3, 2, 0, 1), b, stride=s)
    return y.permute(0, 2, 3, 1)


def conv2d_transpose_same(x, w, b, s):
    """tf.keras.layers.Conv2DTranspose(padding='same') -- elements.py:34-39.
    Output n*s; equals the input-gradient of the SAME forward conv from size
    n*s.  x NHWC, w (kh,kw,Co,Ci) Keras layout (no flip)."""
    kh, kw = w.shape[0], w.shape[1]
    n_h, n_w = x.shape[1] * s, x.shape[2] * s
    pt, _ = same_pad(n_h, kh, s)
    pl, _ = same_pad(n_w, kw, s)
    full = F.conv_transpose2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1),
                              None, stride=s)
    need_h, need_w = pt + n_h, pl + n_w
    if full.shape[2] < need_h or full.shape[3] < need_w:
        full = F.pad(full, (0, max(need_w - full.shape[3], 0),
                            0, max(need_h - full.shape[2], 0)))
    y = full[:, :, pt:pt + n_h, pl:pl + n_w]
    if b is not None:
        y = y + b.view(1, -1, 1, 1)
    return y.permute(0, 2, 3, 1)


def act(x, type_):
    """elements.py:69-78."""
    if type_ == 'relu':
        return F.relu(x)
    if type_ == 'leakyrelu':
        return F.leaky_relu(x, 0.3)
    if type_ == 'elu':
        return F.elu(x, 1.0)
    raise NotImplementedError(type_)


def norm(x, type_, gamma=None, beta=None):
    """elements.py:51-66: None, 'pixel' (:103-121) and 'instance' (:97-100).  The instance branch restates
    tf.contrib.layers.instance_norm(center=True, scale=True, epsilon=1e-6) -- per sample and channel over H x W, biased
    variance; upstream that call does not exist in TF 2.2 (SURVEY D2), so this branch pins only this repo's own
    kernels.  'batch' / 'layer' are unshipped and outside the oracle."""
    if type_ is None or str(type_).lower() == 'none':
        return x
    if type_ == 'pixel':         # elements.py:103-121
        return x * torch.rsqrt((x * x).mean(dim=3, keepdim=True) + 1.0e-8)
    if type_ == 'instance':
        mean = x.mean(dim=(1, 2), keepdim=True)
        var = ((x - mean) ** 2).mean(dim=(1, 2), keepdim=True)
        y = (x - mean) * torch.rsqrt(var + 1.0e-6)
        if gamma is not None:
            y = y * gamma + beta
        return y
    raise NotImplementedError(type_)


def resampler(data, warp):
    """tfa.image.resampler (0.10.0) -- call sites nlt/models/nlt.py:112-114.
    data [B,H,W,C]; warp [B,h,w,2] in pixels, (...,0)=x, (...,1)=y, pixel
    centres at integers.  Out-of-range taps contribute zero; a sample point
    outside (-1,W)x(-1,H) gives zero."""
    B, H, W, C = data.shape
    x, y = warp[..., 0], warp[..., 1]
    inside = (x > -1) & (y > -1) & (x < W) & (y < H)
    fx, fy = torch.floor(x), torch.floor(y)
    cx, cy = fx + 1, fy + 1
    dx, dy = cx - x, cy - y
    flat = data.reshape(B, H * W, C)

    def tap(ix, iy):
        ok = inside & (ix >= 0) & (iy >= 0) & (ix <= W - 1) & (iy <= H - 1)
        idx = (iy.clamp(0, H - 1) * W + ix.clamp(0, W - 1)).long()
        g = torch.gather(flat, 1, idx.reshape(B, -1, 1).expand(-1, -1, C))
        return g.reshape(*warp.shape[:3], C) * ok.unsqueeze(-1).to(data.dtype)

    out = (dx * dy).unsqueeze(-1) * tap(fx, fy) \
        + ((1 - dx) * (1 - dy)).unsqueeze(-1) * tap(cx, cy) \
        + (dx * (1 - dy)).unsqueeze(-1) * tap(fx, cy) \
        + ((1 - dx) * dy).unsqueeze(-1) * tap(cx, fy)
    return out


def resize_bilinear(x, new_h, new_w):
    """tf.image.resize default (bilinear, half-pixel centres, no antialias)
    -- nlt/util/img.py:113-116.  Exact identity when sizes match."""
    B, H, W, C = x.shape
    if (H, W) == (new_h, new_w):
        return x

    def weights(n_in, n_out):
        scale = n_in / n_out
        src = (torch.arange(n_out, dtype=x.dtype) + 0.5) * scale - 0.5
        f = torch.floor(src)
        lo = f.clamp(min=0).long()
        hi = torch.ceil(src).clamp(max=n_in - 1).long()
        return lo, hi, src - f

    ylo, yhi, yl = weights(H, new_h)
    xlo, xhi, xl = weights(W, new_w)
    top = x[:, ylo][:, :, xlo] * (1 - xl).view(1, 1, -1, 1) \
        + x[:, ylo][:, :, xhi] * xl.view(1, 1, -1, 1)
    bot = x[:, yhi][:, :, xlo] * (1 - xl).view(1, 1, -1, 1) \
        + x[:, yhi][:, :, xhi] * xl.view(1, 1, -1, 1)
    return top * (1 - yl).view(1, -1, 1, 1) + bot * yl.view(1, -1, 1, 1)


def set_left_top_corner(x, val):
    """nlt/util/img.py:179-185 (mask multiply: texel (0,0) *= val)."""
    mask = torch.ones_like(x)
    mask[:, 0, 0, :] = val
    return mask * x


def alpha_blend(t1, alpha):
    """nlt/util/img.py:74-89 with tensor2=None."""
    return t1 * alpha + torch.zeros_like(t1) * (1 - alpha)


# ----------------------------------------------------------------------------
# parameters
# ----------------------------------------------------------------------------
def model_channels(cfg, c_query, c_obs):
    """Replays the lazy Keras build driven by Model._call (models/nlt.py:
    141-199) and returns, per net, the list (per layer) of per-conv
    (kind, Cin, Cout, k, s).  kind: 'conv' | 'deconv'."""
    plan, contracting = network_plan(cfg['depth0'], cfg['depth'])
    k, s = cfg['kernel'], cfg['stride']
    use_obs = cfg.get('use_obs', True)
    q_layers, o_layers = [], []
    q_in, o_in = c_query, c_obs
    skips = []
    for (kind, n), contr in zip(plan, contracting):
        if contr:
            if kind == 'conv1x1':
                o_layers.append([('conv', o_in, n, 1, 1)])
                q_layers.append([('conv', q_in, n, 1, 1)])
            else:
                o_layers.append([('conv', o_in, n, k, s), ('conv', n, n, k, 1)])
                q_layers.append([('conv', q_in, n, k, s), ('conv', n, n, k, 1)])
            o_in = n
            q_in = n + n if use_obs else n
            skips.append(q_in)
        else:
            if skips:
                q_in = q_in + skips.pop()
            if kind == 'conv1x1':
                q_layers.append([('conv', q_in, n, 1, 1)])
            else:
                q_layers.append([('deconv', q_in, n, k, s),
                                 ('deconv', n, n, k, 1)])
            q_in = n
    return {'query': q_layers, 'obs': o_layers}


def init_params(cfg, c_query=5, c_obs=3, seed=0, dtype=torch.float32,
                bias_range=0.1):
    """Keras-default Glorot-uniform kernels; biases U[-r, r) (non-zero on
    purpose so that bias paths are exercised; Keras default is zeros)."""
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
                if str(cfg.get('norm', 'None')) == 'instance' and len(convs) == 2:
                    # scale ~ 1, centre ~ 0 (tf.contrib defaults are exactly 1 / 0; perturbed so both are exercised)
                    params['%s.%d.%d.norm.kernel' % (net, li, ci)] = \
                        (1.0 + 0.2 * (torch.rand((cout,), generator=g, dtype=torch.float64) - 0.5)).to(dtype)
                    params['%s.%d.%d.norm.bias' % (net, li, ci)] = \
                        (0.2 * (torch.rand((cout,), generator=g, dtype=torch.float64) - 0.5)).to(dtype)
    return params


# ----------------------------------------------------------------------------
# the model -- nlt/models/nlt.py
# ----------------------------------------------------------------------------
def apply_layer(params, cfg, net, li, x):
    """One entry of Network.layers (convnet.py:44, 50-59, 67-76, 85)."""
    plan, _ = network_plan(cfg['depth0'], cfg['depth'])
    kind = plan[li][0]
    s, a, nm = cfg['stride'], cfg['act'], cfg.get('norm', 'None')
    if str(cfg.get('pool', 'None')).lower() != 'none':
        raise NotImplementedError('pool=%s' % cfg['pool'])
    w = lambda ci: params['%s.%d.%d.kernel' % (net, li, ci)]
    b = lambda ci: params['%s.%d.%d.bias' % (net, li, ci)]
    if kind == 'conv1x1':
        return conv2d_same(x, w(0), b(0), 1)
    g = lambda ci: params.get('%s.%d.%d.norm.kernel' % (net, li, ci))     # instance norm: scale / centre
    bt = lambda ci: params.get('%s.%d.%d.norm.bias' % (net, li, ci))
    if kind == 'down':
        x = act(norm(conv2d_same(x, w(0), b(0), s), nm, g(0), bt(0)), a)
        return act(norm(conv2d_same(x, w(1), b(1), 1), nm, g(1), bt(1)), a)
    x = act(norm(conv2d_transpose_same(x, w(0), b(0), s), nm, g(0), bt(0)), a)
    return act(norm(conv2d_transpose_same(x, w(1), b(1), 1), nm, g(1), bt(1)), a)


def net_call(params, cfg, query_x, obs_xs, obs_weights=None, obs_override=None):
    """Model._call -- nlt/models/nlt.py:141-199."""
    _, contracting = network_plan(cfg['depth0'], cfg['depth'])
    use_obs = cfg.get('use_obs', True)
    if obs_weights is not None:
        obs_weights = obs_weights.reshape(obs_weights.shape[0], 1, 1, 1, -1)
    featmaps = []
    query_y = None
    for li, contr in enumerate(contracting):
        if contr:
            obs_ys = [apply_layer(params, cfg, 'obs', li, x) for x in obs_xs]
            obs_agg = torch.stack(obs_ys, dim=-1)                 # :161
            if obs_weights is not None:
                obs_agg = obs_weights * obs_agg                   # :162-163
            obs_agg = obs_agg.mean(dim=-1)                        # :164
            obs_xs = obs_ys                                       # :166
            query_y = apply_layer(params, cfg, 'query', li, query_x)
            if use_obs:
                if obs_override is not None:
                    obs_agg = obs_override[li]                    # :172-173
                query_x = torch.cat((query_y, obs_agg), dim=-1)   # :174
            else:
                query_x = query_y
            featmaps.append(query_x)                              # :180
        else:
            if featmaps:
                query_x = torch.cat((query_x, featmaps.pop()), dim=-1)  # :184-190
            query_y = apply_layer(params, cfg, 'query', li, query_x)
            query_x = query_y
    return query_y


def model_call(params, cfg, batch, mode, obs_override=None):
    """Model.call -- nlt/models/nlt.py:89-139.  batch is the 11-tuple."""
    if mode not in ('train', 'vali', 'test'):
        raise ValueError(mode)
    id_, base, cvis, lvis, warp, rgb, rgb_camspc, nn_id, nn_base, nn_rgb, \
        nn_rgb_camspc = batch
    x = torch.cat((base, cvis, lvis), dim=3)                      # :95
    if nn_rgb.dim() == 5:       # K observations, k-major [K,B,H,W,3] (SURVEY 8d cfg3; `_call` takes a list, :153-164)
        y_obs = [nn_rgb[k] - nn_base[k] for k in range(nn_rgb.shape[0])]
    else:
        y_obs = [nn_rgb - nn_base]                                # :96
    pred = net_call(params, cfg, x, y_obs, obs_override=obs_override)
    if cfg.get('skip_connect_base', True):
        pred = pred + base                                        # :101-102
    warp = torch.stack((warp[..., 0] * cfg['uvw'],
                        warp[..., 1] * cfg['uvh']), dim=3)        # :104-106
    fg = set_left_top_corner(torch.ones_like(pred), 0)
    base = set_left_top_corner(base, 0)
    pred = set_left_top_corner(pred, 0)
    fg_c = resize_bilinear(resampler(fg, warp), cfg['imh'], cfg['imw'])
    base_c = resize_bilinear(resampler(base, warp), cfg['imh'], cfg['imw'])
    pred_c = resize_bilinear(resampler(pred, warp), cfg['imh'], cfg['imw'])
    to_vis = {'id': id_, 'nn_id': nn_id, 'base_camspc': base_c, 'pred': pred,
              'pred_camspc': pred_c, 'nn_camspc': nn_rgb_camspc}
    if mode in ('train', 'vali'):
        gt_c = alpha_blend(rgb_camspc, fg_c)                      # :132-133
        to_vis['gt'] = rgb
        to_vis['gt_camspc'] = gt_c
        return pred_c, gt_c, {}, to_vis
    return pred_c, None, None, to_vis


def model_call_multi_obs(params, cfg, query_x, obs_list, base, warp):
    """K-observation variant used for cfg3-style synthetic tests: same as
    model_call's tensor path but with an explicit observation list (the
    reference's _call accepts any K; call() passes K=1)."""
    pred = net_call(params, cfg, query_x, obs_list)
    if cfg.get('skip_connect_base', True):
        pred = pred + base
    warp = torch.stack((warp[..., 0] * cfg['uvw'], warp[..., 1] * cfg['uvh']), 3)
    pred = set_left_top_corner(pred, 0)
    return resize_bilinear(resampler(pred, warp), cfg['imh'], cfg['imw'])


def l2_loss(gt, pred, keep_batch=False):
    """losses.L2 -- nlt/losses.py:39-53."""
    se = ((gt - pred) ** 2).mean(dim=-1)
    return se.mean(dim=(1, 2)) if keep_batch else se.mean()


def extract_feat(params, cfg, samples):
    """nlt/nlt_test.py:97-127.  samples: list of (base, rgb) batches."""
    _, contracting = network_plan(cfg['depth0'], cfg['depth'])
    n_obs_layers = sum(contracting)
    feats = None
    for base, rgb in samples:
        x = rgb - base
        feat = []
        for li in range(n_obs_layers):
            x = apply_layer(params, cfg, 'obs', li, x)
            feat.append(x)
        feats = feat if feats is None else \
            [torch.cat((a, b_), 0) for a, b_ in zip(feats, feat)]
    return [f.mean(dim=0, keepdim=True) for f in feats]


# ----------------------------------------------------------------------------
# train step -- nlt/trainvali.py:122-127, 272-281
# ----------------------------------------------------------------------------
def train_loss(params, cfg, batch, global_bs):
    """per-example loss -> sum / global_bs  (trainvali.py:274-278)."""
    pred, gt, kw, _ = model_call(params, cfg, batch, 'train')
    per_ex = l2_loss(gt, pred, keep_batch=True)
    return per_ex.sum() / global_bs


def amsgrad_step(p, g, m, v, vhat, t, lr, beta1=0.9, beta2=0.999, eps=1e-7):
    """tf.keras.optimizers.Adam(amsgrad=True) dense update (TF 2.2):
    lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m,v EMA; vhat=max(vhat,v);
    p -= lr_t*m/(sqrt(vhat)+eps).  t is the 1-based step count."""
    lr_t = lr * math.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
    m = m + (g - m) * (1 - beta1)
    v = v + (g * g - v) * (1 - beta2)
    vhat = torch.maximum(vhat, v)
    p = p - lr_t * m / (torch.sqrt(vhat) + eps)
    return p, m, v, vhat


def psnr_luma(im1, im2):
    """xiuminglib.metric.PSNR (third_party/xiuminglib/xiuminglib/metric.py:
    105-151): clip to [0,1], luma 0.2126/0.7152/0.0722, drange 1."""
    a = np.clip(np.asarray(im1, dtype=np.float64), 0, 1)
    b = np.clip(np.asarray(im2, dtype=np.float64), 0, 1)
    wts = np.array([0.2126, 0.7152, 0.0722])
    mse = np.mean((a @ wts - b @ wts) ** 2)
    return float(10 * np.log10(1.0 / mse)) if mse > 0 else float('inf')
