#!/usr/bin/env python
"""Achievable device-memory bandwidth: a device-to-device copy of --gb GB (default 2), timed with CUDA events,
best of --reps runs.  Counts the bytes read plus the bytes written, so the result is directly comparable with the
per-op GB/s of `bench.py --profile-out` (algorithmic bytes over kernel time).  Prints one JSON line with the card
name and, when nvidia-smi is available, its power limit, because the number belongs to both.
"""
import argparse
import json
import subprocess

import torch


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gb', type=float, default=2.0, help='size of the copied buffer in GB')
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'hbm_copy.py measures a GPU'
    n = int(args.gb * 1e9) // 4
    src = torch.ones(n, dtype=torch.float32, device='cuda')
    dst = torch.empty_like(src)
    dst.copy_(src)                          # warm-up
    torch.cuda.synchronize()
    best = float('inf')
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.reps):
        e0.record()
        dst.copy_(src)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    moved = 2 * n * 4
    print(json.dumps({'device': torch.cuda.get_device_name(), 'power_limit_and_max_sm_clock': power_limit(),
                      'copy_bytes': n * 4, 'bytes_moved': moved, 'best_ms': best,
                      'GBps': moved / (best * 1e-3) / 1e9, 'reps': args.reps}))


if __name__ == '__main__':
    main()
