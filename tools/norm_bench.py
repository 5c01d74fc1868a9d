#!/usr/bin/env python
"""Times nlt_instnorm_fwd / nlt_instnorm_bwd (and the pixel-norm pair) at the shapes a norm layer sees at cfg4's batch:
the level-0 map 8 x 1024^2 x 16 and 8 x 64^2 x 256, with CUDA events over --reps launches.

--other LIB.so times a second build of the library (say, the parent commit's) in the same process, the two builds
alternating over --rounds rounds, so that a difference between them is not a difference between moments on a shared
host.  Reports per build and shape the median over the rounds, the algorithmic bytes (every tensor read or written
once: forward x + y, backward x + dz + dx) over that time, the device copy rate measured in the same process
(tools/hbm_copy.py's method), and the card's name and power limit.  Writes one JSON file (--out).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'neural-light-transport_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.hbm_copy import power_limit   # noqa: E402
from tools.loss_bench import copy_rate   # noqa: E402
from tools.pool_bench import event_ms    # noqa: E402

SHAPES = [(8, 1024 * 1024, 16), (8, 64 * 64, 256)]
NAMES = ('nlt_pixelnorm_fwd', 'nlt_pixelnorm_bwd', 'nlt_instnorm_workspace_bytes', 'nlt_instnorm_fwd', 'nlt_instnorm_bwd')


def load(path):
    """The norm entry points of one build of the library, with the signatures nlt_native declares."""
    import nlt_native as nat
    if path is None:
        return nat.lib()
    handle = C.CDLL(os.path.abspath(path))
    for name in NAMES:
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = nat._SIGS[name]
    return handle


def ops(lib, x, dz, gamma, beta):
    import nlt_native as nat
    N, HW, Cn = x.shape
    y = torch.empty_like(x)
    mean, rstd = torch.empty(N * Cn, device=x.device), torch.empty(N * Cn, device=x.device)
    dg, db = torch.empty(Cn, device=x.device), torch.empty(Cn, device=x.device)
    ws = torch.empty(lib.nlt_instnorm_workspace_bytes(N, HW, Cn) // 4, device=x.device)
    p, st = nat.ptr, nat.stream
    fwd = lambda: nat.check(lib.nlt_instnorm_fwd(p(x), p(gamma), p(beta), N, HW, Cn, 2, 1e-6, p(y), p(mean), p(rstd),
                                                 p(ws), st()))
    bwd = lambda: nat.check(lib.nlt_instnorm_bwd(p(x), p(dz), p(gamma), p(mean), p(rstd), N, HW, Cn, p(y), p(dg), p(db),
                                                 0, p(ws), st()))
    pfwd = lambda: nat.check(lib.nlt_pixelnorm_fwd(p(x), N * HW, Cn, 2, p(y), st()))
    pbwd = lambda: nat.check(lib.nlt_pixelnorm_bwd(p(x), p(dz), N * HW, Cn, p(y), st()))
    nb = 4 * x.numel()
    return {'instnorm_fwd': (fwd, 2 * nb), 'instnorm_bwd': (bwd, 3 * nb), 'pixelnorm_fwd': (pfwd, 2 * nb),
            'pixelnorm_bwd': (pbwd, 3 * nb)}, (mean, rstd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--other', default=None, help='a second build of libnlt_b200.so to alternate with')
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'norm_bench.py measures a GPU'
    dev = torch.device('cuda')
    builds = {'tree': load(None)}
    if args.other:
        builds['other'] = load(args.other)
    gbps = copy_rate()
    res = {'device': torch.cuda.get_device_name(), 'power_limit_and_max_sm_clock': power_limit(),
           'copy_rate_GBps': gbps, 'reps': args.reps, 'rounds': args.rounds, 'shapes': {}}
    for N, HW, Cn in SHAPES:
        gen = torch.Generator(dev).manual_seed(Cn)
        x = torch.randn(N, HW, Cn, device=dev, generator=gen) * 0.5 + 3.0
        dz = torch.randn(N, HW, Cn, device=dev, generator=gen)
        gamma, beta = torch.ones(Cn, device=dev), torch.zeros(Cn, device=dev)
        table = {b: ops(lib, x, dz, gamma, beta) for b, lib in builds.items()}
        ms = {b: {k: [] for k in table[b][0]} for b in builds}
        for _ in range(args.rounds):
            for b in builds:                      # the builds alternate inside every round
                for k, (fn, _) in table[b][0].items():
                    ms[b][k].append(event_ms(fn, args.reps))
        rec = {}
        for b in builds:
            rec[b] = {}
            for k, (_, nb) in table[b][0].items():
                med = statistics.median(ms[b][k])
                rec[b][k] = {'ms_median': med, 'ms_min': min(ms[b][k]), 'ms_max': max(ms[b][k]), 'bytes': nb,
                             'GBps': nb / (med * 1e-3) / 1e9, 'of_copy_rate': nb / (med * 1e-3) / 1e9 / gbps}
        if args.other:                            # what the two builds' statistics say about the same input
            (m0, r0), (m1, r1) = table['tree'][1], table['other'][1]
            rec['rstd_rel_diff_tree_vs_other'] = float(((r0 - r1).abs() / r0).max())
            rec['mean_rel_diff_tree_vs_other'] = float(((m0 - m1).abs() / m0.abs()).max())
        res['shapes']['%dx%dx%d' % (N, HW, Cn)] = rec
        print(json.dumps({'%dx%dx%d' % (N, HW, Cn): rec}), flush=True)
        del x, dz, table
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
