#!/usr/bin/env python
"""Times the U-Net of `pool = max | avg`: the dragon_specular network (depth0 16, depth 256, leakyrelu) with stride 1,
for kernel 2 and 3, at UV 1024 x 1024, batch 8, with the shipped 5 / 3 input channels.

Per arm it reports:
  * the graph-replayed training step (trainvali.GraphedTrainStep: forward, L2, backward, AMSGrad), timed with CUDA
    events over --steps replays on two rotating device-resident batches, as bench.py times its step;
  * the peak device memory of the arm;
  * from one eager step with per-call CUDA events (engine.PROF, a separate pass), the share of the profiled step time
    spent in the upsamples and in the upconv convs (forward, input gradient, weight gradient);
and, once, the time of each of the four new kernels at the shapes the step runs (CUDA events over --reps launches),
their algorithmic bytes over that time, and the device copy rate measured in the same process (tools/hbm_copy.py's
method).  Writes one JSON file (--out) with the card's name and power limit.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'neural-light-transport_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.hbm_copy import power_limit   # noqa: E402
from tools.loss_bench import copy_rate   # noqa: E402


def make_config(pool, kernel, uv):
    from util import io as ioutil
    return ioutil.make_config(uvh=uv, uvw=uv, imh=uv, imw=uv, loss='l2', depth0=16, depth=256, kernel=kernel, stride=1,
                              pool=pool)


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_table(B, uv, reps, gbps):
    """The four kernels at the step's largest shapes: pools at level 1 (16 channels, uv^2 -> (uv/2)^2), upsample of
    level 12's 40-channel concat ((uv/2)^2 -> uv^2).  Bytes: every tensor read or written once."""
    import nlt_native as nat
    lib, st = nat.lib(), nat.stream
    dev = torch.device('cuda')
    out = {}
    x = torch.randn(B, uv, uv, 16, device=dev)
    y = torch.empty(B, uv // 2, uv // 2, 16, device=dev)
    dx = torch.empty_like(x)
    for kind, code in (('max', 0), ('avg', 1)):
        ms = event_ms(lambda: nat.check(lib.nlt_pool2x2_fwd(nat.ptr(x), B, uv, uv, 16, code, nat.ptr(y), st())), reps)
        nb = 4 * (x.numel() + y.numel())
        out['pool2x2_fwd_%s' % kind] = {'shape': [B, uv, uv, 16], 'ms': ms, 'bytes': nb}
        # beta = 0, with the LeakyReLU mask (the mask is x itself, as in the step): x, d_y read, d_x written
        ms = event_ms(lambda: nat.check(lib.nlt_pool2x2_bwd(nat.ptr(x), nat.ptr(y), B, uv, uv, 16, code, 0.0,
                                                            nat.ptr(x), 2, nat.ptr(dx), st())), reps)
        nb = 4 * (2 * x.numel() + y.numel())
        out['pool2x2_bwd_%s' % kind] = {'shape': [B, uv, uv, 16], 'ms': ms, 'bytes': nb}
    del x, y, dx
    h = uv // 2
    x = torch.randn(B, h, h, 40, device=dev)
    y = torch.empty(B, uv, uv, 40, device=dev)
    dx = torch.empty_like(x)
    ms = event_ms(lambda: nat.check(lib.nlt_upsample2x_bilinear_fwd(nat.ptr(x), B, h, h, 40, nat.ptr(y), st())), reps)
    out['upsample2x_fwd'] = {'shape': [B, h, h, 40], 'ms': ms, 'bytes': 4 * (x.numel() + y.numel())}
    ms = event_ms(lambda: nat.check(lib.nlt_upsample2x_bilinear_bwd(nat.ptr(y), B, h, h, 40, 0.0, None, 0, nat.ptr(dx),
                                                                    st())), reps)
    out['upsample2x_bwd'] = {'shape': [B, h, h, 40], 'ms': ms, 'bytes': 4 * (x.numel() + y.numel())}
    for v in out.values():
        v['GBps'] = v['bytes'] / (v['ms'] * 1e-3) / 1e9
        v['of_copy_rate'] = v['GBps'] / gbps
    return out


def upsample_share(model, bt, B):
    """One eager step with per-call events: ms of the upsamples and the upconv convs, and of everything profiled."""
    import engine
    engine.PROF.enabled = True
    try:
        pred, gt, kw, _ = model(bt, mode='train')
        kw['keep_batch'] = True
        model.set_loss_grad_scale(1.0 / B)
        model.compute_loss(pred, gt, **kw)
        model.backward()
        prof = engine.PROF.summary()
    finally:
        engine.PROF.enabled = False
    upconv = {'query.%d.0' % li for li, blk in enumerate(model.net['query'].layers) if blk.upconv}
    total = sum(v['ms'] for v in prof.values())
    up = sum(v['ms'] for k, v in prof.items() if 'upsample2x' in k)
    conv = sum(v['ms'] for k, v in prof.items() if k.split(' ')[1] in upconv)
    pool = sum(v['ms'] for k, v in prof.items() if '.pool ' in k)
    return {'profiled_ms': total, 'upsample_ms': up, 'upconv_conv_ms': conv, 'pool_ms': pool,
            'upsample_share': up / total, 'upsample_plus_upconv_share': (up + conv) / total,
            'pool_share': pool / total}


def run_arm(pool, kernel, B, uv, steps, warmup):
    import models
    import trainvali
    from util import synth
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model = models.get_model_class('nlt')(make_config(pool, kernel, uv))
    model.register_trainable()
    model.build(5, 3)
    opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
    dev = model.device
    bts = [tuple(t.to(dev) if torch.is_tensor(t) else t for t in synth.make_batch(B, uv, uv, seed=1235 + i))
           for i in range(2)]
    share = upsample_share(model, bts[0], B)
    step = trainvali.GraphedTrainStep(trainvali.Strategy(), model, opt, B)
    for i in range(max(warmup, 3)):
        step(bts[i % 2])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        loss, _ = step(bts[i % 2])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    rec = {'pool': pool, 'kernel': kernel, 'batch': B, 'uv': uv, 'step_ms': ms, 'steps': steps,
           'full_step_in_graph': bool(step.full_step_in_graph), 'loss': float(loss),
           'peak_mem_GB': torch.cuda.max_memory_allocated() / 1e9, 'n_params': int(model.flat_params.numel()),
           'eager_profile': share}
    del step, model, opt, bts
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--uv', type=int, default=1024)
    ap.add_argument('--arms', default='max:2,avg:2,max:3,avg:3')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'pool_bench.py measures a GPU'
    gbps = copy_rate()
    res = {'device': torch.cuda.get_device_name(), 'power_limit_and_max_sm_clock': power_limit(),
           'copy_rate_GBps': gbps, 'kernels': kernel_table(args.batch, args.uv, args.reps, gbps), 'arms': []}
    for arm in args.arms.split(','):
        pool, k = arm.split(':')
        res['arms'].append(run_arm(pool, int(k), args.batch, args.uv, args.steps, args.warmup))
        print(json.dumps(res['arms'][-1]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != 'arms'}))


if __name__ == '__main__':
    main()
