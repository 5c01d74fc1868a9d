#!/usr/bin/env python
"""Multi-GPU correctness check of the data-parallel step (run under torchrun on N GPUs):

  * N ranks, each with its shard of a global batch, run GraphedTrainStep (whole step incl. the overlapped NCCL
    all-reduce and the AMSGrad update captured in ONE CUDA graph) for a few steps;
  * rank 0 then replays the same global batches on a single-replica model (same initial weights) and compares the
    parameters and the losses: the only differences are fp32 summation order across the batch shards.

Prints one JSON line on rank 0; exit code 1 on mismatch.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'neural-light-transport_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    import models
    import trainvali
    from util import io as ioutil, synth
    strategy = trainvali.Strategy()
    world, rank = strategy.world, strategy.rank
    uv, per_rank, steps = 256, 2, 4
    gbs = per_rank * world
    cfg = ioutil.make_config(uvh=uv, uvw=uv, imh=uv, imw=uv, loss='l2')

    def make_model():
        m = models.get_model_class('nlt')(cfg)
        m.register_trainable()
        m.seed = 11
        m.build(5, 3)
        return m

    batches = [synth.make_batch(gbs, uv, uv, seed=500 + s) for s in range(steps)]
    shard = lambda b: tuple((t[rank * per_rank:(rank + 1) * per_rank].cuda() if torch.is_tensor(t)
                             else t[rank * per_rank:(rank + 1) * per_rank]) for t in b)
    model = make_model()
    opt = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
    step = trainvali.GraphedTrainStep(strategy, model, opt, gbs)
    losses = []
    for b in batches:
        loss, _ = step(shard(b))
        losses.append(float(loss))
    torch.cuda.synchronize()
    in_graph = bool(step.full_step_in_graph)
    # eager multi-rank path as well (overlapped all-reduce outside a graph)
    model_e = make_model()
    opt_e = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
    losses_e = []
    for b in batches:
        loss, _ = trainvali.distributed_train_step(strategy, model_e, shard(b), opt_e, gbs)
        losses_e.append(float(loss))
    torch.cuda.synchronize()
    strategy.barrier()
    ok = True
    out = None
    if rank == 0:
        single = trainvali.Strategy.__new__(trainvali.Strategy)
        single.world, single.rank, single.local_rank = 1, 0, 0
        ref = make_model()
        opt_r = trainvali.Adam(learning_rate=1e-3, amsgrad=True)
        losses_r = []
        for b in batches:
            loss, _ = trainvali.distributed_train_step(single, ref, tuple(t.cuda() if torch.is_tensor(t) else t for t in b),
                                                       opt_r, gbs)
            losses_r.append(float(loss))
        torch.cuda.synchronize()
        def cmp(a, b):
            d = (a.flat_params - b.flat_params).abs()
            disp = (b.flat_params - make_model().flat_params).norm()
            return float(d.max()), float(d.norm() / disp)
        g_max, g_rel = cmp(model, ref)
        e_max, e_rel = cmp(model_e, ref)
        l_err = max(abs(a - b) / abs(b) for a, b in zip(losses, losses_r))
        le_err = max(abs(a - b) / abs(b) for a, b in zip(losses_e, losses_r))
        ok = g_rel <= 2e-2 and e_rel <= 2e-2 and l_err <= 1e-5 and le_err <= 1e-5
        out = {'world': world, 'steps': steps, 'collectives_in_graph': in_graph, 'graph_vs_single_max': g_max,
               'graph_vs_single_rel_displacement': g_rel, 'eager_vs_single_max': e_max,
               'eager_vs_single_rel_displacement': e_rel, 'loss_rel_graph': l_err, 'loss_rel_eager': le_err, 'ok': ok}
        print(json.dumps(out))
    # leave without tearing the communicator down: on 2 GPUs the result above was printed and the processes then sat
    # in destroy_process_group() until the job timed out -- rank 1 reaches it minutes before rank 0
    # (which still computes the single-replica reference) while CUDA graphs holding NCCL kernels are alive
    if world > 1:
        torch.distributed.barrier()
        torch.cuda.synchronize()
    sys.stdout.flush()
    sys.stderr.flush()
    os._exit(0 if ok else 1)


if __name__ == '__main__':
    main()
