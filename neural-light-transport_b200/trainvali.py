"""Data-parallel training step -- host mirror of nlt/trainvali.py:254-325.

The reference replicates in-graph with tf.distribute.MirroredStrategy; here it
is one process per GPU (torchrun), the batch sharded along the view x light
axis, and ONE all-reduce(SUM) over the flat fp32 gradient bucket per step
(NCCL over NVLink/NVSwitch), followed by one fused AMSGrad launch.
"""
import os

import torch
import torch.distributed as dist

import nlt_native as nat


class Strategy:
    """Stand-in for tf.distribute.{OneDevice,Mirrored}Strategy
    (trainvali.py:254-264): rank / world size of the torchrun job."""

    def __init__(self, backend=None):
        self.world = int(os.environ.get('WORLD_SIZE', '1'))
        self.rank = int(os.environ.get('RANK', '0'))
        self.local_rank = int(os.environ.get('LOCAL_RANK', '0'))
        if self.world > 1 and not dist.is_initialized():
            if backend is None:
                backend = 'nccl' if torch.cuda.is_available() else 'gloo'
            if backend == 'nccl':
                torch.cuda.set_device(self.local_rank)
            dist.init_process_group(backend)
        if torch.cuda.is_available():
            torch.cuda.set_device(self.local_rank if self.world > 1 else torch.cuda.current_device())

    @property
    def num_replicas_in_sync(self):
        return self.world

    def all_reduce_sum_(self, t):
        if self.world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return t

    def all_reduce_sum_async(self, t):
        """Starts the SUM all-reduce of `t` ordered after the work already queued on the current stream; returns
        the work handle (`.wait()` makes the then-current stream wait for it).  None with one replica."""
        if self.world > 1:
            return dist.all_reduce(t, op=dist.ReduceOp.SUM, async_op=True)
        return None

    def barrier(self):
        if self.world > 1:
            dist.barrier()


def get_strategy(device='gpu'):
    if device == 'gpu':
        return Strategy()
    if device == 'cpu':
        # the reference offers OneDeviceStrategy('/cpu:0'); this hot path has
        # no CPU implementation by design
        raise NotImplementedError('device=cpu: the CUDA hot path has no CPU fallback')
    raise NotImplementedError(device)


class Adam:
    """tf.keras.optimizers.Adam(learning_rate, amsgrad=True) over the model's
    flat parameter bucket (trainvali.py:122-127); Keras defaults b1 .9,
    b2 .999, eps 1e-7.

    `device_step=True` keeps the step counter on the device (nlt_amsgrad_step_dev), which makes the update
    capturable in a CUDA graph; `iterations` stays the host mirror of the same count."""

    def __init__(self, learning_rate=1e-3, beta_1=0.9, beta_2=0.999, epsilon=1e-7, amsgrad=False, clipnorm=None):
        if not amsgrad:
            raise NotImplementedError('only amsgrad=True is on the accelerated path')
        if clipnorm is not None:
            raise NotImplementedError('clipnorm (mgm > 0) is out of parity scope (SURVEY.md 8c)')
        self.lr, self.b1, self.b2, self.eps = learning_rate, beta_1, beta_2, epsilon
        self.iterations = 0
        self.m = self.v = self.vhat = None
        self.step_dev = None

    def _state(self, flat_p):
        if self.m is None:
            self.m, self.v, self.vhat = (torch.zeros_like(flat_p) for _ in range(3))
        if self.step_dev is None:
            self.step_dev = torch.full((1,), self.iterations, dtype=torch.int32, device=flat_p.device)

    @staticmethod
    def _flat(gv):
        g0, v0 = gv[0]
        base_g, flat_p = g0._base, v0._base
        if base_g is None or flat_p is None or any(g._base is not base_g or v._base is not flat_p for g, v in gv):
            raise ValueError('apply_gradients expects views of the model\'s flat parameter/gradient buckets')
        return base_g[:flat_p.numel()], flat_p

    def apply_gradients(self, grads_and_vars, grad_scale=1.0, device_step=False):
        flat_g, flat_p = self._flat(list(grads_and_vars))
        self._state(flat_p)
        self.iterations += 1
        from engine import PROF
        if PROF.enabled:       # 4 state reads + 1 gradient read + 4 writes per parameter
            return PROF.run('opt amsgrad', 4 * 9 * flat_p.numel(), lambda: self._launch(flat_p, flat_g, grad_scale,
                                                                                      device_step))
        self._launch(flat_p, flat_g, grad_scale, device_step)

    def _launch(self, flat_p, flat_g, grad_scale, device_step):
        if device_step:
            nat.check(nat.lib().nlt_amsgrad_step_dev(
                nat.ptr(flat_p), nat.ptr(flat_g), nat.ptr(self.m), nat.ptr(self.v), nat.ptr(self.vhat),
                flat_p.numel(), self.step_dev.data_ptr(), self.lr, self.b1, self.b2, self.eps, grad_scale,
                nat.stream()))
        else:
            nat.check(nat.lib().nlt_amsgrad_step(
                nat.ptr(flat_p), nat.ptr(flat_g), nat.ptr(self.m), nat.ptr(self.v), nat.ptr(self.vhat),
                flat_p.numel(), self.iterations, self.lr, self.b1, self.b2, self.eps, grad_scale, nat.stream()))
            self.step_dev.fill_(self.iterations)

    # ---- checkpoint state (util/ckpt.py) ----
    def state_dict(self):
        return {'iterations': self.iterations, 'm': self.m, 'v': self.v, 'vhat': self.vhat}

    def load_state(self, iterations, m, v, vhat):
        self.iterations = int(iterations)
        self.m, self.v, self.vhat = m, v, vhat
        self.step_dev = torch.full((1,), self.iterations, dtype=torch.int32, device=m.device)


class GradReducer:
    """The gradient all-reduce of the data-parallel step (the reference's implicit cross-replica SUM inside
    `optimizer.apply_gradients` under `strategy.run`, nlt/trainvali.py:279-284, plus the `strategy.reduce(SUM)`
    of the loss at :317) as at most TWO collectives over the flat bucket, the first overlapped with backward:

      * the bucket is laid out in the order backward() produces the weight gradients (models/nlt.py:build), so its
        head -- decoder + deep encoder levels, ~90 % of the parameters -- is complete long before the
        full-resolution levels have finished; its all-reduce is launched asynchronously from the stream that
        issued the last weight gradient of the head (engine.WGRAD_HOOK) and runs under the rest of backward;
      * the tail (shallow levels, a few hundred KB) and the per-replica loss (one extra slot behind the
        gradients) go out in ONE final collective.

    With one replica nothing is launched.  Works eagerly and under CUDA-graph capture (the NCCL stream forks from
    and joins back into the capturing stream)."""

    def __init__(self, strategy, model, overlap=True):
        self.strategy, self.model = strategy, model
        self.overlap = overlap
        self.work = None
        self.split_layer, self.split = None, 0

    def begin(self):
        import engine
        self.work = None
        if self.strategy.world > 1 and self.overlap and self.model.bucket is not None:
            self.split_layer, self.split = self.model.bucket.split_point()
            engine.WGRAD_HOOK = self._hook if self.split_layer is not None else None

    def _hook(self, layer):
        import engine
        if layer is not self.split_layer or self.work is not None:
            return
        head = self.model.bucket.grad[:self.split]
        if engine.USE_SIDE_STREAM:
            engine.join_side_streams()
            with torch.cuda.stream(engine.side_stream()):      # ordered after the wgrad launches issued so far
                self.work = self.strategy.all_reduce_sum_async(head)
            head.record_stream(engine.side_stream())
        else:
            self.work = self.strategy.all_reduce_sum_async(head)

    def finish(self, weighted_loss):
        """Completes the reduction; returns the global loss (a device scalar)."""
        import engine
        engine.WGRAD_HOOK = None
        bucket = self.model.bucket
        if self.strategy.world == 1:
            return weighted_loss.clone()
        bucket.loss_slot.copy_(weighted_loss.reshape(1))
        start = 0
        if self.work is not None:
            self.work.wait()                                   # current stream waits for the head's collective
            self.work = None
            start = self.split
        self.strategy.all_reduce_sum_(bucket.grad_with_loss()[start:])
        return bucket.loss_slot[0].clone()


def distributed_train_step(strategy, model, batch, optimizer, global_bs):
    """trainvali.py:267-290: per-replica train_step, gradient all-reduce,
    loss SUM.  `batch` is this rank's shard of the global batch."""
    assert model.trainable_registered, \
        "Register the trainable layers before using `trainable_variables`"
    reducer = GradReducer(strategy, model)

    def train_step(batch):
        pred, gt, loss_kwargs, partial_to_vis = model(batch, mode='train')
        loss_kwargs['keep_batch'] = True  # keep the batch dimension
        model.set_loss_grad_scale(1.0 / global_bs)
        per_example_loss = model.compute_loss(pred, gt, **loss_kwargs)
        weighted_loss = per_example_loss.sum() / global_bs   # tf.nn.compute_average_loss
        reducer.begin()
        model.backward()
        loss = reducer.finish(weighted_loss)                 # gradient (+ loss) all-reduce, overlapped with backward
        optimizer.apply_gradients(zip(model.gradients, model.trainable_variables))
        return loss, partial_to_vis

    return train_step(batch)


class GraphedTrainStep:
    """distributed_train_step with the WHOLE step of one replica -- forward, loss, backward, the gradient
    all-reduce (overlapped with backward, see GradReducer) and the fused AMSGrad update with its step counter on
    the device -- captured ONCE in a CUDA graph (shapes are static).  Every activation and gradient buffer lives in
    the graph's private pool and the scratch buffers whose addresses the kernels bake in (packed weight planes, TMA
    descriptors, wgrad partials) belong to this object (engine.use_workspaces), so nothing an eager call does later
    can move memory under a replay.  Per step: copy the batch into the static input buffers, replay.
    Same semantics as nlt/trainvali.py:267-290.

    `graph_collectives=False` keeps the collectives and the optimiser outside the graph (replay -> all-reduce ->
    AMSGrad), which is also the automatic fallback when capturing NCCL fails."""

    def __init__(self, strategy, model, optimizer, global_bs, graph_collectives=True):
        import engine
        self.strategy, self.model, self.optimizer, self.global_bs = strategy, model, optimizer, global_bs
        self.graph = None
        self.static_batch = None
        self.loss = None
        self.to_vis = None
        self.graph_collectives = graph_collectives
        self.full_step_in_graph = False
        self._ws = (engine.Workspace(), engine.Workspace())
        self.reducer = GradReducer(strategy, model)

    def _body(self, batch, with_update):
        model = self.model
        pred, gt, loss_kwargs, to_vis = model(batch, mode='train')
        loss_kwargs['keep_batch'] = True
        model.set_loss_grad_scale(1.0 / self.global_bs)
        per_example_loss = model.compute_loss(pred, gt, **loss_kwargs)
        weighted_loss = per_example_loss.sum() / self.global_bs
        if with_update:
            self.reducer.begin()
        model.backward()
        if with_update:
            loss = self.reducer.finish(weighted_loss)
            self.optimizer.apply_gradients(zip(model.gradients, model.trainable_variables), device_step=True)
            return loss, to_vis
        return weighted_loss, to_vis

    def _capture(self, batch):
        import engine
        from models.nlt import _dev_tensor
        dev = self.model.device
        # uint8 image tensors become v / 255 here, as in the eager step (models/nlt.py:_dev_tensor)
        self.static_batch = tuple(_dev_tensor(t, dev, out=torch.empty(t.shape, dtype=torch.float32, device=dev))
                                  if torch.is_tensor(t) else t for t in batch)
        with engine.use_workspaces(*self._ws):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):  # warm-up: lazy build, one-time CUDA attribute calls, scratch sizing
                for _ in range(2):
                    self._body(self.static_batch, with_update=False)
            torch.cuda.current_stream().wait_stream(side)
            if self.strategy.world > 1:
                # NCCL creates its communicator at the first collective, which cannot happen inside a capture
                self.strategy.all_reduce_sum_(torch.zeros(1, device=dev))
            torch.cuda.synchronize()
            # the warm-up ran on a side stream: its freed activation blocks stay cached for that stream, where the
            # graph's private pool cannot reuse them.  Returning them first keeps the step's peak at one set of
            # activations (cfg4 at batch 32 does not fit in 80 GB otherwise)
            torch.cuda.empty_cache()
            it0 = self.optimizer.iterations
            self.optimizer._state(self.model.flat_params)
            for full in ([True, False] if self.graph_collectives else [False]):
                try:
                    graph = torch.cuda.CUDAGraph()
                    l0, t0 = nat.launch_count(), nat.tc_launch_count()
                    with torch.cuda.graph(graph):
                        self.loss, self.to_vis = self._body(self.static_batch, with_update=full)
                    self.graph, self.full_step_in_graph = graph, full
                    break
                except RuntimeError:
                    if not full:
                        raise
                    engine.WGRAD_HOOK = None
                    torch.cuda.synchronize()
            # kernels of this library inside ONE replay (the counters only see the capture)
            self.captured_launches = nat.launch_count() - l0
            self.captured_tc_launches = nat.tc_launch_count() - t0
            self.optimizer.iterations = it0      # the capture itself applied no update

    def __call__(self, batch):
        assert self.model.trainable_registered, \
            "Register the trainable layers before using `trainable_variables`"
        if self.graph is None:
            self._capture(batch)
        if batch is not self.static_batch:
            from models.nlt import _dev_tensor
            for dst, src in zip(self.static_batch, batch):
                if torch.is_tensor(dst):
                    _dev_tensor(src, dst.device, out=dst)     # uint8 -> v / 255, like the eager step
        self.graph.replay()
        if self.full_step_in_graph:
            self.optimizer.iterations += 1       # host mirror of the device step counter
            return self.loss, self.to_vis
        self.reducer.work = None
        loss = self.reducer.finish(self.loss)
        self.optimizer.apply_gradients(zip(self.model.gradients, self.model.trainable_variables))
        return loss, self.to_vis


def distributed_vali_step(strategy, model, batch, global_bs):
    """trainvali.py:296-312."""
    pred, gt, loss_kwargs, to_vis = model(batch, mode='vali')
    loss_kwargs['keep_batch'] = True
    per_example_loss = model.compute_loss(pred, gt, **loss_kwargs)
    weighted_loss = per_example_loss.sum() / global_bs
    loss = strategy.all_reduce_sum_(weighted_loss.clone())
    return loss, to_vis


def batch_source(config, strategy, steps, device='cuda', mode='train', seed=None):
    """This rank's shards of `steps` global batches (trainvali.py:72-90).

    Real data when `<data_root>.json` exists: `datasets.get_dataset_class(config dataset)` -> pipeline ->
    `.shard(world, rank)` (the reference's `experimental_distribute_dataset`), cycling over epochs; the tensors
    arrive pinned and are copied to `device` asynchronously.  Otherwise (no NLT data on this machine) synthetic
    batches of the configured shape (util/synth.py)."""
    import os
    from util import synth
    bs = config.getint('DEFAULT', 'bs')
    data_root = config.get('DEFAULT', 'data_root', fallback='')
    if data_root and os.path.exists(data_root.rstrip('/') + '.json'):
        import datasets
        geti = lambda k, d: config.getint('DEFAULT', k, fallback=d)
        pre, par = geti('prefetch_buffer_size', -1), geti('n_map_parallel_calls', -1)
        ds = datasets.get_dataset_class(config.get('DEFAULT', 'dataset', fallback='nlt'))(
            config, mode, shuffle_buffer_size=geti('shuffle_buffer_size', 64),
            prefetch_buffer_size=None if pre < 0 else pre, n_map_parallel_calls=None if par < 0 else par)
        pipe = ds.build_pipeline(seed=seed, no_batch=config.getboolean('DEFAULT', 'no_batch', fallback=False))
        pipe = pipe.shard(strategy.world, strategy.rank)
        done = 0
        while done < steps:
            n_before = done
            for batch in pipe:
                yield tuple(t.to(device, non_blocking=True) if torch.is_tensor(t) else t for t in batch)
                done += 1
                if done >= steps:
                    return
            if done == n_before:
                raise RuntimeError('dataset pipeline produced no batch')
        return
    local_bs = max(bs // strategy.world, 1)
    for step in range(steps):
        yield synth.make_batch(local_bs, config.getint('DEFAULT', 'uvh'), config.getint('DEFAULT', 'imh'),
                               seed=1234 + step * strategy.world + strategy.rank, device=device)


def make_optimizer(config):
    """nlt/trainvali.py:120-127: Adam(lr, amsgrad=True[, clipnorm=mgm if mgm > 0])."""
    lr = config.getfloat('DEFAULT', 'lr')
    mgm = config.getfloat('DEFAULT', 'mgm', fallback=-1.0)
    if mgm > 0:
        # the reference clips each gradient tensor to norm mgm; that path is TF-version dependent and not part of
        # the accelerated step -- refuse instead of silently training without clipping
        raise NotImplementedError('mgm = %g > 0 (per-tensor clipnorm) is not on the accelerated path' % mgm)
    return Adam(learning_rate=lr, amsgrad=True)


def main(argv=None):
    """Same CLI flags as the reference (--config --debug --device).  Trains from the on-disk dataset named by
    the config when it exists (datasets/nlt.py), else on synthetic batches of the configured shape; resumes from
    and writes checkpoints under `<outroot>/<xname>/checkpoints` like nlt/trainvali.py:129-141, 221-226."""
    import argparse
    import models
    from util import io as ioutil, ckpt as ckptutil
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='dragon_specular.ini')
    ap.add_argument('--debug', action='store_true')
    ap.add_argument('--device', default='gpu')
    ap.add_argument('--steps', type=int, default=4, help='train steps per epoch on synthetic data')
    args = ap.parse_args(argv)
    strategy = get_strategy(args.device)
    config = ioutil.read_config(args.config)
    Model = models.get_model_class(config.get('DEFAULT', 'model'))
    model = Model(config)
    model.register_trainable()
    optimizer = make_optimizer(config)
    global_bs = config.getint('DEFAULT', 'bs')
    outroot = config.get('DEFAULT', 'outroot', fallback='')
    manager = None
    if outroot:
        xname = config.get('DEFAULT', 'xname', fallback='run').format(**dict(config['DEFAULT']))
        keep = config.getint('DEFAULT', 'keep_recent_epochs', fallback=-1)
        manager = ckptutil.CheckpointManager(os.path.join(outroot, xname, 'checkpoints'), keep if keep > 0 else None)
    epochs = 1 if args.debug else config.getint('DEFAULT', 'epochs', fallback=1)
    ckpt_period = config.getint('DEFAULT', 'ckpt_period', fallback=1)
    steps = 1 if args.debug else args.steps
    step = 0
    resumed = False
    for epoch in range(epochs):
        for batch in batch_source(config, strategy, steps, device='cuda', seed=epoch):
            if manager is not None and not resumed:
                # parameters exist once the first batch has fixed the channel counts (Keras builds lazily too)
                model.build(batch[1].shape[-1] + batch[2].shape[-1] + batch[3].shape[-1], batch[9].shape[-1])
                restored = manager.restore_latest(model, optimizer)
                if restored is not None:
                    step = restored
                    if strategy.rank == 0:
                        print('Resumed from step:\n\t%s' % manager.latest_checkpoint)
                elif strategy.rank == 0:
                    print('Started from scratch')
                resumed = True
            loss, _ = distributed_train_step(strategy, model, batch, optimizer, global_bs)
            step += 1
            if strategy.rank == 0:
                print('epoch %d step %d loss %.6f' % (epoch, step, float(loss)))
        if manager is not None and strategy.rank == 0 and (epoch + 1) % ckpt_period == 0:
            print('Checkpoint saved:\n\t%s' % manager.save(model, optimizer, step))


if __name__ == '__main__':
    main()
