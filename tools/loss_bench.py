#!/usr/bin/env python
"""Times the four training-loss entry points (nlt_l2_loss, nlt_l1_loss, nlt_ssim_loss, nlt_barron_loss), each with its
gradient and captured in a CUDA graph, at the cfg4 loss shape (batch 8, 1024 x 1024 x 3) and at batch 32, with CUDA
events.  Each is reported as algorithmic bytes (pred and gt read, d_pred written: 12 B per element) over kernel time,
next to a device copy rate measured in the same run (the method of tools/hbm_copy.py).  For SSIM it also counts the
FP32 operations of the separable formulation and says which lower bound, bytes at the copy rate or FMAs at the data
sheet's FP32 rate, is larger.  With --step it also times the graphed cfg4 training step (trainvali.GraphedTrainStep,
batch 8) for `loss = l2`, `ssim`, `l1` and `barron,1e+0ssim`.  Writes one JSON file (--out) with the card's name and
power limit.
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

FP32_PEAK_TFLOPS = 67.0     # H100 SXM data sheet, dense FP32 (at up to 700 W)


def ssim_flops(B, H, W, grad=True):
    """FP32 operations of SSIM per the formula, separable window, no halo recompute: per input element and channel 4
    products (x*y, x*x + y*y) and per output pixel 4 maps x 2 passes x 11 FMAs, ~30 operations for L, CS and the
    coefficients; the gradient adds 3 maps x 2 passes x 11 FMAs and 4 operations per input element."""
    n_in, n_out = B * H * W * 3, B * (H - 10) * (W - 10) * 3
    f = 4 * n_in + n_out * (4 * 2 * 11 * 2 + 30)
    if grad:
        f += n_in * (3 * 2 * 11 * 2 + 4)
    return f


def copy_rate(gb=2.0, reps=10):
    n = int(gb * 1e9) // 4
    src = torch.ones(n, dtype=torch.float32, device='cuda')
    dst = torch.empty_like(src)
    dst.copy_(src)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float('inf')
    for _ in range(reps):
        e0.record()
        dst.copy_(src)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    del src, dst
    return 2 * n * 4 / (best * 1e-3) / 1e9


def graph_ms(fn, reps):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def loss_calls(B, H, W):
    import nlt_native as nat
    lib = nat.lib()
    g = torch.Generator(device='cuda').manual_seed(B)
    gt = torch.rand(B, H, W, 3, generator=g, device='cuda')
    pred = (gt + 0.05 * torch.randn(B, H, W, 3, generator=g, device='cuda')).contiguous()
    per = H * W * 3
    loss = torch.empty(B, device='cuda')
    d = torch.empty_like(pred)
    P = nat.ptr
    scale = 1.0 / B

    def ws(nbytes):
        assert nbytes > 0
        return torch.empty((nbytes + 3) // 4, device='cuda')
    w_l2, w_l1 = ws(lib.nlt_l2_loss_workspace_bytes(B, per)), ws(lib.nlt_l1_loss_workspace_bytes(B, per))
    w_ssim, w_bar = ws(lib.nlt_ssim_loss_workspace_bytes(B, H, W)), ws(lib.nlt_barron_loss_workspace_bytes(B, H, W, 5))
    calls = {
        'nlt_l2_loss': lambda: nat.check(lib.nlt_l2_loss(P(pred), P(gt), B, per, scale, P(loss), P(d), P(w_l2),
                                                         nat.stream())),
        'nlt_l1_loss': lambda: nat.check(lib.nlt_l1_loss(P(pred), P(gt), B, per, scale, P(loss), P(d), P(w_l1),
                                                         nat.stream())),
        'nlt_ssim_loss': lambda: nat.check(lib.nlt_ssim_loss(P(pred), P(gt), B, H, W, 1.0, scale, P(loss), P(d),
                                                             P(w_ssim), nat.stream())),
        'nlt_barron_loss': lambda: nat.check(lib.nlt_barron_loss(P(pred), P(gt), None, B, H, W, 5, 0.01,
                                                                 1.185495232349193, scale, P(loss), P(d), P(w_bar),
                                                                 nat.stream())),
    }
    return calls, (gt, pred, loss, d, w_l2, w_l1, w_ssim, w_bar)


def step_ms(loss, steps, warmup):
    import bench
    import trainvali
    from util import io as ioutil
    wl = bench.WORKLOADS['cfg4']
    cfg = ioutil.make_config(uvh=wl['uv'], uvw=wl['uv'], imh=wl['uv'], imw=wl['uv'], loss=loss, depth0=16,
                             depth=wl['depth'], kernel=wl['kernel'], stride=2)
    real = bench.make_config
    bench.make_config = lambda w: cfg
    try:
        run = bench.TrainRun(trainvali.Strategy(), wl, wl['batch'], wl['batch'])
    finally:
        bench.make_config = real
    ms = [run.measure_resident(steps, warmup)[0] for _ in range(3)]
    del run
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--step', action='store_true', help='also time the graphed cfg4 step per objective')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', required=True, help='JSON file to write (e.g. profiles/h100_losses.json)')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'loss_bench.py measures a GPU'
    rec = {'device': torch.cuda.get_device_name(), 'power_limit_and_max_sm_clock': power_limit(),
           'copy_GBps': copy_rate(), 'fp32_datasheet_TFLOPS': FP32_PEAK_TFLOPS, 'losses': []}
    for B in (8, 32):
        H = W = 1024
        calls, keep = loss_calls(B, H, W)
        nbytes = 12 * B * H * W * 3
        for name, fn in calls.items():
            ms = graph_ms(fn, args.reps)
            row = {'entry': name, 'shape': [B, H, W, 3], 'ms': ms, 'algorithmic_bytes': nbytes,
                   'GBps': nbytes / (ms * 1e-3) / 1e9}
            row['of_copy_rate'] = row['GBps'] / rec['copy_GBps']
            if name == 'nlt_ssim_loss':
                fl = ssim_flops(B, H, W)
                t_bytes = nbytes / (rec['copy_GBps'] * 1e9) * 1e3
                t_fma = fl / (FP32_PEAK_TFLOPS * 1e12) * 1e3
                row.update({'flops': fl, 'TFLOPS': fl / (ms * 1e-3) / 1e12, 'bytes_bound_ms': t_bytes,
                            'fp32_bound_ms': t_fma, 'larger_bound': 'bytes' if t_bytes >= t_fma else 'fp32 FMA'})
            rec['losses'].append(row)
            print(json.dumps(row))
        del calls, keep
        torch.cuda.empty_cache()
    if args.step:
        rec['cfg4_step_ms'] = {}
        for loss in ('l2', 'ssim', 'l1', 'barron,1e+0ssim'):
            rec['cfg4_step_ms'][loss] = step_ms(loss, args.steps, args.warmup)
            print(json.dumps({'loss': loss, 'cfg4_step_ms': rec['cfg4_step_ms'][loss]}))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(rec, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
