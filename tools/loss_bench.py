#!/usr/bin/env python
"""Times the four training-loss entry points (nlt_l2_loss, nlt_l1_loss, nlt_ssim_loss, nlt_barron_loss), each with its
gradient and captured in a CUDA graph, at the cfg4 loss shape (batch 8, 1024 x 1024 x 3) and at batch 32, with CUDA
events.  Each is reported as algorithmic bytes (pred and gt read, d_pred written: 12 B per element) over kernel time,
next to a device copy rate measured in the same run (the method of tools/hbm_copy.py).  For SSIM it also counts the
FP32 operations of the separable formulation and says which lower bound, bytes at the copy rate or FMAs at the data
sheet's FP32 rate, is larger.  With --step it also times the graphed cfg4 training step (trainvali.GraphedTrainStep,
batch 8) for `loss = l2`, `ssim`, `l1`, `barron,1e+0ssim`, `barron` and `barron,1e+0lpips`.

nlt_lpips_loss (when build() has put the reference's LPIPS graph in oracle/_ref/) is timed at 4 x 512^2 and 8 x 1024^2
with its gradient, on the default conv route and with option tc = 0, and reported as conv TFLOP/s (shape-derived:
the forward of both images plus the input gradients of pred) next to a TF32 GEMM rate measured in the same run, with
the share of conv1 (forward and input gradient, timed alone on the same kernels).  Writes one JSON file (--out) with
the card's name and power limit.
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


# AlexNet of LPIPS: (Cout, Cin, k, stride, pad); maxpool 3x3 / s2 after conv1 and conv2
ALEX = ((64, 3, 11, 4, 2), (192, 64, 5, 1, 2), (384, 192, 3, 1, 1), (256, 384, 3, 1, 1), (256, 256, 3, 1, 1))


def alex_lattices(H, W):
    out, h, w = [], H, W
    for i, (co, ci, k, s, p) in enumerate(ALEX):
        if i in (1, 2):
            h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        out.append((h, w))
    return out


def lpips_conv_flops(B, H, W):
    """(all, conv1) conv FLOPs of one nlt_lpips_loss call with its gradient: forwards of 2B images, input gradients
    of B images (2 FLOPs per multiply-add)."""
    per = [2 * h * w * co * ci * k * k for (co, ci, k, _, _), (h, w) in zip(ALEX, alex_lattices(H, W))]
    return 3 * B * sum(per), 3 * B * per[0]


def tf32_gemm_tflops(n=8192, reps=20):
    a = torch.randn(n, n, device='cuda')
    b = torch.randn(n, n, device='cuda')
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        ms = graph_ms(lambda: torch.mm(a, b), reps)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return 2 * n ** 3 / (ms * 1e-3) / 1e12


def lpips_rows(reps, tf32):
    import ctypes as C
    import nlt_native as nat
    from oracle import lpips_oracle
    from util import tf_graphdef
    path = lpips_oracle.graph_path()
    if path is None:
        return None
    lib = nat.lib()
    host = tf_graphdef.load_lpips_alex(path)
    t = {k: torch.from_numpy(v).cuda() for k, v in host.items()}
    wts = nat.LpipsWeights()
    wts.scale, wts.shift = nat.ptr(t['scale']), nat.ptr(t['shift'])
    for i in range(5):
        wts.w[i], wts.b[i], wts.lin[i] = (nat.ptr(t['%s%d' % (k, i + 1)]) for k in ('w', 'b', 'lin'))
    rows = []
    for B, H, W in ((4, 512, 512), (8, 1024, 1024)):
        g = torch.Generator(device='cuda').manual_seed(B)
        gt = torch.rand(B, H, W, 3, generator=g, device='cuda')
        pred = (gt + 0.05 * torch.randn(B, H, W, 3, generator=g, device='cuda')).clamp(0, 1).contiguous()
        loss, d = torch.empty(B, device='cuda'), torch.empty_like(pred)
        need = lib.nlt_lpips_loss_workspace_bytes(B, H, W)
        ws = torch.empty((need + 3) // 4, device='cuda')
        fn = lambda: nat.check(lib.nlt_lpips_loss(nat.ptr(pred), nat.ptr(gt), wts, B, H, W, 1.0 / B, nat.ptr(loss),
                                                  nat.ptr(d), nat.ptr(ws), need, nat.stream()))
        # conv1 alone: its forward on 2B images and its input gradient on B images, on the kernels the call uses
        (h1, w1) = alex_lattices(H, W)[0]
        x = torch.empty(2 * B, H, W, 3, device='cuda')
        y = torch.empty(2 * B, h1, w1, 64, device='cuda')

        def desc(dgrad):
            dd = nat.GConvDesc()
            dd.kh = dd.kw = 11
            dd.stride, dd.pad_t, dd.pad_l, dd.nseg, dd.Cout = 4, 2, 2, 1, 3 if dgrad else 64
            dd.w = nat.ptr(t['w1'])
            dd.w_tap_stride = 1
            if dgrad:
                dd.N, dd.Hin, dd.Win, dd.Hout, dd.Wout, dd.transposed = B, h1, w1, H, W, 1
                dd.seg_ptr[0], dd.seg_C[0] = nat.ptr(y), 64
                dd.w_c_stride, dd.w_n_stride = 3 * 121, 121
            else:
                dd.N, dd.Hin, dd.Win, dd.Hout, dd.Wout = 2 * B, H, W, h1, w1
                dd.seg_ptr[0], dd.seg_C[0] = nat.ptr(x), 3
                dd.w_c_stride, dd.w_n_stride = 121, 3 * 121
            return dd
        df, db = desc(False), desc(True)
        conv1 = lambda: (nat.check(lib.nlt_gconv_fwd(C.byref(df), nat.ptr(t['b1']), 1, 0.0, None, 0, nat.ptr(y),
                                                     nat.stream())),
                         nat.check(lib.nlt_gconv_fwd(C.byref(db), None, 0, 0.0, None, 0, nat.ptr(x), nat.stream())))
        fl, fl1 = lpips_conv_flops(B, H, W)
        row = {'entry': 'nlt_lpips_loss', 'shape': [B, H, W, 3], 'conv_flops': fl, 'conv1_flops': fl1}
        for tc in (1, 0):
            with nat.options(tc=tc):
                ms = graph_ms(fn, reps)
                ms1 = graph_ms(conv1, reps)
            key = 'tc%d' % tc
            row[key] = {'ms': ms, 'conv_TFLOPS': fl / (ms * 1e-3) / 1e12, 'of_tf32_gemm': fl / (ms * 1e-3) / 1e12 / tf32,
                        'conv1_ms': ms1, 'conv1_share': ms1 / ms}
        rows.append(row)
        print(json.dumps(row))
        del pred, gt, loss, d, ws, x, y
        torch.cuda.empty_cache()
    return rows


def step_ms(loss, steps, warmup):
    import bench
    import trainvali
    from oracle import lpips_oracle
    from util import io as ioutil
    wl = bench.WORKLOADS['cfg4']
    extra = {'lpips_weights': lpips_oracle.graph_path()} if 'lpips' in loss else {}
    cfg = ioutil.make_config(uvh=wl['uv'], uvw=wl['uv'], imh=wl['uv'], imw=wl['uv'], loss=loss, depth0=16,
                             depth=wl['depth'], kernel=wl['kernel'], stride=2, **extra)
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
    rec['tf32_gemm_TFLOPS'] = tf32_gemm_tflops()
    rec['lpips'] = lpips_rows(args.reps, rec['tf32_gemm_TFLOPS'])
    if args.step:
        rec['cfg4_step_ms'] = {}
        for loss in ('l2', 'ssim', 'l1', 'barron,1e+0ssim', 'barron', 'barron,1e+0lpips'):
            rec['cfg4_step_ms'][loss] = step_ms(loss, args.steps, args.warmup)
            print(json.dumps({'loss': loss, 'cfg4_step_ms': rec['cfg4_step_ms'][loss]}))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(rec, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
