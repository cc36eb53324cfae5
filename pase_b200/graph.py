"""CUDA-graph capture of one whole training step (H2D of the waveform batch, encoder
forward + backward through the C-ABI kernels, optimizer update, D2H of the loss) so that a
step is ONE launch: the hot loop is launch-bound on the host once the kernels take only a
few ms.  Buffers of the encoder plan are static by construction (EncoderPlan), TMA
descriptors are kernel parameters, so the captured graph is replayable as is.

GraphedEncoderStep captures the encoder with a given loss; GraphedTrainStep captures the PASE /
PASE+ training step with its workers, fed by a DeviceBatcher plan uploaded before each replay.
"""
import random

import numpy as np
import torch


def _refresh_hyperparams(opt, stream):
    """FlatAdam keeps its hyper-parameter table at one address; write the current lr / betas /
    eps / weight decay into it on the replay stream, so that a scheduler's change between two
    replays reaches the captured update."""
    segments = getattr(opt, "_segments", None)
    if segments is not None:
        with torch.cuda.stream(stream):
            segments()


class GraphedEncoderStep(object):
    """step(x_host) -> loss (python float).  `x_host` must be a pinned CPU tensor of the shape
    given at construction; `loss_fn(y) -> scalar tensor`; the optimizer must be capturable."""

    def __init__(self, model, optimizer, loss_fn, shape, device, pre_step=None, post_backward=None,
                 warmup=3, stream=None, resident=False, x_init=None,
                 capture_error_mode="global", between=None, prefetch=False):
        self.model, self.opt, self.loss_fn = model, optimizer, loss_fn
        self.x_static = torch.zeros(shape, dtype=torch.float32, device=device)
        self.x_host = torch.zeros(shape, dtype=torch.float32).pin_memory()
        self.loss_host = torch.zeros((), dtype=torch.float32).pin_memory()
        if x_init is not None:               # batch used by the warm-up steps
            self.x_host.copy_(x_init)
            self.x_static.copy_(x_init)
        self.pre_step, self.post_backward = pre_step, post_backward
        # `between`: a callable that runs EAGERLY between two captured halves of the step
        # ([H2D, forward, backward, post_backward] and [optimizer, D2H]).  Data parallelism
        # puts its NCCL all-reduce there: the collective is never captured, only ordered on
        # the same stream between two graph replays.
        self.between = between
        self.resident = resident        # True: input stays in HBM, no H2D / D2H in the graph
        # prefetch: the H2D copy of the NEXT step's batch (pinned host -> one of two device
        # staging buffers, on a copy stream) overlaps the current step's compute; the step
        # itself starts with a device-to-device copy out of the staging buffer.  Same bytes
        # per step, every copy still inside the caller's timed region -- the usual
        # double-buffered input pipeline of a training loop.
        self.prefetch = bool(prefetch) and not resident
        if self.prefetch:
            self.stage = [torch.zeros(shape, dtype=torch.float32, device=device) for _ in (0, 1)]
            self.h2d_done = [torch.cuda.Event(), torch.cuda.Event()]
            self.copy_stream = torch.cuda.Stream(device=device)
            self._k = 0
            self._primed = False
        # capture on the stream the model's autograd nodes already live on: an AccumulateGrad
        # node created on another stream invalidates the capture
        self.stream = stream if stream is not None else torch.cuda.Stream(device=device)
        self.graph = self.graph_b = None
        # "thread_local" when other threads of the process issue CUDA calls during the
        # capture (e.g. an NCCL process group's watchdog)
        self.capture_error_mode = capture_error_mode
        self._loss = None
        self._capture(warmup)

    def _part_a(self):
        if not self.resident and not self.prefetch:
            self.x_static.copy_(self.x_host, non_blocking=True)
        if self.pre_step is not None:
            self.pre_step()
        y = self.model(self.x_static)
        self._loss = self.loss_fn(y)
        self._loss.backward()
        if self.post_backward is not None:
            self.post_backward()

    def _part_b(self):
        self.opt.step()
        if not self.resident:
            self.loss_host.copy_(self._loss.detach(), non_blocking=True)

    def _one(self):
        self._part_a()
        if self.between is not None:
            self.between()
        self._part_b()

    def _capture(self, warmup):
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            for _ in range(warmup):
                self.opt.zero_grad(set_to_none=True)
                self._one()
        self.stream.synchronize()
        torch.cuda.current_stream().wait_stream(self.stream)
        self.opt.zero_grad(set_to_none=True)
        mode = self.capture_error_mode
        g = torch.cuda.CUDAGraph()
        if self.between is None:
            with torch.cuda.graph(g, stream=self.stream, capture_error_mode=mode):
                self._one()
        else:
            with torch.cuda.graph(g, stream=self.stream, capture_error_mode=mode):
                self._part_a()
            with torch.cuda.stream(self.stream):
                self.between()
            gb = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gb, stream=self.stream, pool=g.pool(), capture_error_mode=mode):
                self._part_b()
            self.graph_b = gb
        self.graph = g

    def step(self, x_host=None):
        """Replays the captured step.  The batch is read from the pinned staging buffer
        ``self.x_host`` (a data loader writes batches straight into it); passing ``x_host``
        copies it there first."""
        if x_host is not None:
            self.x_host.copy_(x_host)
        if self.prefetch:
            k = self._k
            with torch.cuda.stream(self.stream):
                if not self._primed:             # first call: nothing was prefetched yet
                    self.stage[k].copy_(self.x_host, non_blocking=True)
                    self._primed = True
                else:
                    self.stream.wait_event(self.h2d_done[k])
                self.x_static.copy_(self.stage[k], non_blocking=True)      # D2D, ~2 us
            # next batch -> the other staging buffer, concurrently with this step's compute
            # (its previous reader, the step before this one, has completed: step() syncs)
            with torch.cuda.stream(self.copy_stream):
                self.stage[1 - k].copy_(self.x_host, non_blocking=True)
                self.h2d_done[1 - k].record(self.copy_stream)
            self._k = 1 - k
        _refresh_hyperparams(self.opt, self.stream)
        self.graph.replay()
        if self.graph_b is not None:
            with torch.cuda.stream(self.stream):
                self.between()
            self.graph_b.replay()
        if self.resident:
            return None
        self.stream.synchronize()
        return float(self.loss_host)


def spc_minions(model):
    """The SPCMinion heads of a ``pase`` model in the order its forward calls them (regression
    workers, then classification workers), i.e. the order of their draws."""
    from .minions import SPCMinion
    workers = list(model.regression_workers) + list(model.classification_workers)
    return [m for w in workers for m in w.modules() if isinstance(m, SPCMinion)]


class TrainPlanner(object):
    """Host side of one PASE/PASE+ training step: the batch plan of ``DeviceBatcher.plan`` and
    the frames of every SPC head, drawn in the order the eager loop draws them (the batch, then
    the step's SPC frames; the next batch's draws come after).  ``rng``: None (the global
    random, np.random and torch generators) or a (random.Random, np.random.RandomState,
    torch.Generator) triple, as for ``plan()``; the SPC frames come from its first member."""

    def __init__(self, model, batcher):
        self.batcher = batcher
        self.spc = spc_minions(model)
        self.Tq = model.frontend.frame_counts(batcher.T)[-1]
        for m in self.spc:
            if not m.frames_ok(self.Tq):
                M = m.seq_pad + m.ctxt_frames
                raise ValueError("TrainPlanner: chunk_size %d gives T'=%d frames, which leave the "
                                 "SPC head %s no current frame (range(%d, %d) is empty); use a "
                                 "longer chunk" % (batcher.T, self.Tq, m.name, M + 1, self.Tq - M))

    def __call__(self, indices, rng=None):
        """-> (BatchPlan, int64 numpy table: the plan's table then t, future_t, past_t of each
        SPC head)."""
        plan = self.batcher.plan(indices, rng)
        py = random if rng is None else rng[0]
        frames = [f for m in self.spc for f in m.draw_frames(self.Tq, py)]
        return plan, np.concatenate([plan.table, np.asarray(frames, dtype=np.int64)])


def _world(group):
    """Ranks of `group` (None: no data parallelism, 1)."""
    if group is None:
        return 1
    import torch.distributed as dist
    return dist.get_world_size(group)


def _all_gather(t, group, device):
    """Every rank's CPU tensor `t` (one shape on all ranks), in rank order, as CPU tensors.  It
    travels on `device` unless the group's backend is gloo alone."""
    import torch.distributed as dist
    if dist.get_backend(group) != "gloo":
        t = t.to(device)
    parts = [torch.empty_like(t) for _ in range(dist.get_world_size(group))]
    dist.all_gather(parts, t.contiguous(), group=group)
    return [p.cpu() for p in parts]


class GraphedTrainStep(object):
    """One PASE/PASE+ training step from a resident corpus as one CUDA-graph replay: batch
    assembly (``DeviceBatcher``), the encoder, every worker head and its loss, the summed
    ('base' scheduler) loss, backward and the single ``FlatAdam`` update.

        step = GraphedTrainStep(model, engine, batcher, B)
        for indices in BatchSampler(RandomSampler(range(len(wavs))), B, drop_last=True):
            step(indices)                 # plan on the host, upload, replay; does not wait
            if bidx % log_freq == 0:
                losses = step.losses()    # {'total': float, name: float, ...}

    ``model``: a ``pase_b200.pase.pase`` on CUDA in train mode; ``engine``: a ``FlatAdam`` over
    its parameters with ``bind_encoder(model.frontend)`` applied (not ``peer_dp``);
    ``batcher``: a ``DeviceBatcher``.  Each call is exactly one step on its own batch: the first
    `warmup` calls run eagerly through the code that is captured, the next one captures and
    replays, every later one replays.  The host draws and stages the next step's plan while the
    device runs the current one; lr changes (``param_groups``, ``views()``) between two calls
    take effect at the next step.  The step runs on its own stream; each call orders the caller's
    current stream after it (and the step after the caller's earlier work), so eager work the
    caller queues between calls, such as a validation pass or a checkpoint, sees the finished
    step without a host synchronise.

    Data parallelism (``group``: a ``torch.distributed`` process group of W > 1 ranks, one
    process per GPU of one node): each rank builds its own step over its own replica, engine,
    batcher and batches of B, and a step on rank r is the step above on rank r's batch with the
    update on the mean over ranks of the flat gradient.  With ``FlatAdam(peer_dp=True)`` over
    the same group the step stays one replay: ``pase_adam_flat_dp`` averages the gradients and
    stores the same new parameters into every rank's buffer inside it.  With a plain
    ``FlatAdam`` the step is two replays, [batch, forward, losses, backward] and [update, loss
    copy], with ``engine.reduce_grads(group)`` run eagerly on the step stream between them; no
    collective is captured.  Every rank must be built with the same ``warmup`` and called in
    lockstep, the same number of times: a rank that skips a step leaves its peers waiting in
    the update.  ``losses()`` is then collective too."""

    def __init__(self, model, engine, batcher, batch_size, warmup=3, stream=None, group=None):
        from .optim import FlatAdam
        if int(warmup) < 1:
            raise ValueError("GraphedTrainStep: warmup=%d; at least one eager step builds the "
                             "constants and buffers the capture reads" % warmup)
        if not model.training:
            raise ValueError("GraphedTrainStep: the model is in eval mode; call model.train()")
        if not isinstance(engine, FlatAdam):
            raise TypeError("GraphedTrainStep: the engine must be a FlatAdam, got %s"
                            % type(engine).__name__)
        if engine.peer_dp:
            if group is None:
                raise NotImplementedError("GraphedTrainStep: a FlatAdam(peer_dp=True) engine "
                                          "needs group=, the process group it was built over")
            import torch.distributed as dist

            def resolved(g):
                return dist.group.WORLD if g is None else g
            if resolved(engine._group) is not resolved(group):
                raise ValueError("GraphedTrainStep: the FlatAdam(peer_dp=True) engine was built "
                                 "over another process group than `group`")
        sunk = {id(p) for _, p in model.frontend.named_parameters() if p.requires_grad}
        if getattr(model.frontend, "grad_sink", None) is None or engine._sunk != sunk:
            raise ValueError("GraphedTrainStep: call engine.bind_encoder(model.frontend) first")
        if int(batch_size) < 1:
            raise ValueError("GraphedTrainStep: batch_size=%d" % batch_size)
        self.planner = TrainPlanner(model, batcher)
        params = list(model.parameters())
        if not params or not all(p.is_cuda for p in params):
            raise ValueError("GraphedTrainStep: the model must live on a CUDA device")
        self.model, self.engine, self.batcher = model, engine, batcher
        self.B, self.warmup = int(batch_size), int(warmup)
        self.device = params[0].device
        self.group, self.world = group, _world(group)
        # a plain engine averages the gradients with a collective between two graphs
        self.split = self.world > 1 and engine._peer is None
        # total_loss's order: classification workers, then regression workers
        self.names = ["total"] + [w.name for w in list(model.classification_workers) +
                                  list(model.regression_workers)]
        self.stream = stream if stream is not None else torch.cuda.Stream(device=self.device)
        self.loss_host = torch.zeros(len(self.names), dtype=torch.float32).pin_memory()
        self.done = torch.cuda.Event()
        self.table = None                 # the graph's static plan table, sized by the first plan
        self.graph = self.graph_b = None
        self._vec = None
        self._plans = []
        self.calls = 0
        self._k = 0

    def _alloc(self, n):
        self.table = torch.zeros(n, dtype=torch.int64, device=self.device)
        # two page-locked staging tables: the host fills one while the other's copy is queued
        self._stage = [torch.zeros(n, dtype=torch.int64).pin_memory() for _ in (0, 1)]
        self._staged = [torch.cuda.Event(), torch.cuda.Event()]

    def _forward_backward(self):
        """The step's first part as it is captured: everything reads the static table."""
        from .pase import total_loss
        eng, model = self.engine, self.model
        nb = self.table.numel() - 3 * len(self.planner.spc)
        eng.zero_grad(set_to_none=True)
        batch = self.batcher.run(self.table[:nb])
        for i, m in enumerate(self.planner.spc):
            m.frame_table = self.table[nb + 3 * i:nb + 3 * i + 3]
        try:
            _, _, preds, labels = model(batch)
        finally:
            for m in self.planner.spc:
                m.frame_table = None
        tot, losses = total_loss(model, preds, labels)
        self._vec = torch.stack([tot.detach()] + [losses[n].detach() for n in self.names[1:]])
        tot.backward()
        if self.split:
            # the heads' gradients into the flat buffer inside the graph, so the eager
            # all-reduce after it reads this replay's gradients
            eng.pack_grads()

    def _update(self):
        self.engine.step()
        self.loss_host.copy_(self._vec, non_blocking=True)

    def _run(self):
        self._forward_backward()
        if self.split:
            self.engine.reduce_grads(self.group)
        self._update()

    def _capture(self):
        # "thread_local": a process group's watchdog thread may query CUDA during the capture
        mode = "thread_local" if self.world > 1 else "global"
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=self.stream, capture_error_mode=mode):
            if self.split:
                self._forward_backward()
            else:
                self._run()
        if self.split:
            gb = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gb, stream=self.stream, pool=g.pool(), capture_error_mode=mode):
                self._update()
            self.graph_b = gb
        self.graph = g
        # the graph holds raw addresses of the encoder's and decoders' plan buffers; keep those
        # plans alive when their caches evict them (other shapes run eagerly between replays,
        # e.g. validation batches)
        self._plans = [p for m in self.model.modules()
                       for p in getattr(m, "_plans", {}).values()]

    def __call__(self, indices, rng=None):
        indices = [int(i) for i in indices]
        if len(indices) != self.B:
            raise ValueError("GraphedTrainStep: a batch of %d indices, the step was built for %d"
                             % (len(indices), self.B))
        _, table = self.planner(indices, rng)
        if self.table is None:
            self._alloc(table.size)
        elif table.size != self.table.numel():
            raise RuntimeError("GraphedTrainStep: the plan has %d entries, the captured step %d"
                               % (table.size, self.table.numel()))
        k = self._k
        self._staged[k].synchronize()          # the copy that last read this buffer has run
        self._stage[k].numpy()[:] = table
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            self.table.copy_(self._stage[k], non_blocking=True)
            self._staged[k].record(self.stream)
            self.engine._segments()              # lr changes, into the table at its address
            if self.calls < self.warmup:
                self._run()
            else:
                if self.graph is None:
                    self._capture()
                self.graph.replay()
                if self.split:
                    self.engine.reduce_grads(self.group)
                    self.graph_b.replay()
            self.done.record(self.stream)
        # work the caller queues next (an eager validation pass, reading or saving parameters)
        # runs after this step on the device; the host does not wait
        torch.cuda.current_stream(self.device).wait_stream(self.stream)
        self._k = 1 - k
        self.calls += 1

    def losses(self):
        """{'total': ..., worker name: ...} (python floats, each worker's loss times its
        loss_weight) of the last step issued; waits for that step only.  With a process group,
        each entry is the mean over ranks (summed in rank order), i.e. the loss of the global
        batch; collective: every rank calls it after the same steps."""
        if self.calls == 0:
            raise RuntimeError("GraphedTrainStep.losses: no step has run yet")
        self.done.synchronize()
        vals = self.loss_host.tolist()
        if self.world > 1:
            rows = [r.tolist() for r in _all_gather(self.loss_host, self.group, self.device)]
            vals = [sum(r[j] for r in rows) / self.world for j in range(len(vals))]
        return dict(zip(self.names, vals))


class GraphedEvalStep(object):
    """The validation pass of the reference trainer (``_eval``, trainer.py:282-337) from a
    resident corpus, one CUDA-graph replay per batch: batch assembly (``DeviceBatcher``), the
    encoder in eval mode (BatchNorm on its running statistics) and every worker under
    ``no_grad``, and each worker's unweighted loss with their fp32 sum (``pase.eval_losses``).

        ev = GraphedEvalStep(model, va_batcher, B)      # model on CUDA
        model.eval()
        for indices in BatchSampler(RandomSampler(range(len(va_pool))), B, drop_last=True):
            ev(indices)                   # plan on the host, upload, replay; does not wait
        running_loss = ev.losses()        # {worker: [per batch], ..., 'total': [...]}, one D2H
        ev.reset()                        # before the next pass
        model.train()

    Batch k of a pass writes row k of a device table of ``max_batches`` rows (default: the
    drop_last batches of the batcher's pool); the row index travels in the uploaded plan, so a
    call neither waits nor reads anything back.  ``losses()`` copies the pass's rows to the host
    once and returns the reference's ``running_loss`` layout (classification workers, regression
    workers, then 'total'), which its ``eval_logger`` takes as it is.  The host draws are the
    eager pass's, in its order: the batch, then the three frames of each SPC head
    (``TrainPlanner``).  Fused regression heads (``model.fuse_regression_loss``) run their
    loss-only epilogue, as they do eagerly under ``no_grad``.

    The replay reads the parameters and BatchNorm running statistics by address, so a pass sees
    what the training steps before it wrote, and it writes none of them.  Like
    ``GraphedTrainStep`` it runs on its own stream, after the caller's earlier work and with the
    caller's stream ordered after it; it holds every encoder and decoder plan that existed at
    capture.  A ``GraphedTrainStep`` at the same batch size shares the (3B, T) encoder plan
    with it: both graphs write its buffers, which is safe because each call is ordered after
    the caller's earlier work and the caller after it, so the two never run at once.  The first
    `warmup` calls run eagerly through the code that is captured.

    Data parallelism (``group``: a process group of W > 1 ranks, as for ``GraphedTrainStep``):
    each rank replays its own shard of the validation batches.  The first call of a pass (after
    construction or ``reset()``) first broadcasts rank 0's buffers, the BatchNorm running
    statistics, in place into every rank's, so every rank evaluates the model rank 0 would
    save.  ``losses()`` is collective and returns every rank's rows, rank-major."""

    def __init__(self, model, batcher, batch_size, max_batches=None, warmup=3, stream=None,
                 group=None):
        if int(warmup) < 1:
            raise ValueError("GraphedEvalStep: warmup=%d; at least one eager batch builds the "
                             "constants and buffers the capture reads" % warmup)
        if int(batch_size) < 1:
            raise ValueError("GraphedEvalStep: batch_size=%d" % batch_size)
        self.planner = TrainPlanner(model, batcher)
        params = list(model.parameters())
        if not params or not all(p.is_cuda for p in params):
            raise ValueError("GraphedEvalStep: the model must live on a CUDA device")
        self.B, self.warmup = int(batch_size), int(warmup)
        if max_batches is None:
            max_batches = len(batcher.wavs) // self.B
        if int(max_batches) < 1:
            raise ValueError("GraphedEvalStep: max_batches=%d" % max_batches)
        self.model, self.batcher = model, batcher
        self.max_batches = int(max_batches)
        self.device = params[0].device
        self.group, self.world = group, _world(group)
        # running_loss's order (trainer.py:306-326)
        self.names = [w.name for w in list(model.classification_workers) +
                      list(model.regression_workers)] + ["total"]
        self.stream = stream if stream is not None else torch.cuda.Stream(device=self.device)
        self.out = torch.zeros(self.max_batches, len(self.names), dtype=torch.float32,
                               device=self.device)
        self.out_host = torch.zeros(self.max_batches, len(self.names),
                                    dtype=torch.float32).pin_memory()
        self.done = torch.cuda.Event()
        self.table = None                 # the graph's static plan table, sized by the first plan
        self.graph = None
        self._plans = []
        self.calls = 0
        self.k = 0                        # batches of the current pass
        self._k = 0

    def _alloc(self, n):
        self.table = torch.zeros(n, dtype=torch.int64, device=self.device)
        self._stage = [torch.zeros(n, dtype=torch.int64).pin_memory() for _ in (0, 1)]
        self._staged = [torch.cuda.Event(), torch.cuda.Event()]

    def _run(self):
        """One batch as it is captured: everything reads the static table [plan | SPC frames |
        row]."""
        from .pase import eval_losses
        model = self.model
        nb = self.table.numel() - 1 - 3 * len(self.planner.spc)
        with torch.no_grad():
            batch = self.batcher.run(self.table[:nb])
            for i, m in enumerate(self.planner.spc):
                m.frame_table = self.table[nb + 3 * i:nb + 3 * i + 3]
            try:
                _, _, preds, labels = model(batch)
            finally:
                for m in self.planner.spc:
                    m.frame_table = None
            tot, losses = eval_losses(model, preds, labels)
            vec = torch.stack([losses[n].reshape(()) for n in self.names[:-1]] +
                              [tot.reshape(())])
            self.out.index_copy_(0, self.table[-1:], vec[None])

    def __call__(self, indices, rng=None):
        if self.model.training:
            raise ValueError("GraphedEvalStep: the model is in train mode; call model.eval() "
                             "before the pass (BatchNorm must use its running statistics)")
        indices = [int(i) for i in indices]
        if len(indices) != self.B:
            raise ValueError("GraphedEvalStep: a batch of %d indices, the pass was built for %d"
                             % (len(indices), self.B))
        if self.k >= self.max_batches:
            raise RuntimeError("GraphedEvalStep: the loss table holds %d batches and this pass "
                               "has filled it; call reset() to start the next pass"
                               % self.max_batches)
        _, table = self.planner(indices, rng)
        table = np.append(table, np.int64(self.k))
        if self.table is None:
            self._alloc(table.size)
        elif table.size != self.table.numel():
            raise RuntimeError("GraphedEvalStep: the plan has %d entries, the captured pass %d"
                               % (table.size, self.table.numel()))
        if self.world > 1 and self.k == 0:
            # on the caller's stream, which the replay below waits for
            from .dp import broadcast_buffers
            import torch.distributed as dist
            broadcast_buffers(self.model, src=dist.get_global_rank(self.group, 0),
                              group=self.group)
        k = self._k
        self._staged[k].synchronize()          # the copy that last read this buffer has run
        self._stage[k].numpy()[:] = table
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            self.table.copy_(self._stage[k], non_blocking=True)
            self._staged[k].record(self.stream)
            if self.calls < self.warmup:
                self._run()
            else:
                if self.graph is None:
                    g = torch.cuda.CUDAGraph()
                    mode = "thread_local" if self.world > 1 else "global"
                    with torch.cuda.graph(g, stream=self.stream, capture_error_mode=mode):
                        self._run()
                    self.graph = g
                    self._plans = [p for m in self.model.modules()
                                   for p in getattr(m, "_plans", {}).values()]
                self.graph.replay()
            self.done.record(self.stream)
        torch.cuda.current_stream(self.device).wait_stream(self.stream)
        self._k = 1 - k
        self.k += 1
        self.calls += 1

    def losses(self):
        """{worker name: [loss of batch 0, 1, ...], ..., 'total': [...]} (python floats) of the
        batches of the current pass; one device-to-host copy, waits for the pass only.  With a
        process group: rank 0's batches, then rank 1's, ...; collective, and it raises on every
        rank when the ranks ran different numbers of batches in the pass."""
        n = self.k
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            self.out_host[:n].copy_(self.out[:n], non_blocking=True)
            self.done.record(self.stream)
        self.done.synchronize()
        rows = self.out_host[:n].tolist()
        if self.world > 1:
            counts = [int(c) for c in _all_gather(torch.tensor([n], dtype=torch.int64),
                                                  self.group, self.device)]
            if len(set(counts)) > 1:
                raise RuntimeError("GraphedEvalStep.losses: the ranks ran %s batches in this "
                                   "pass; every rank must run the same number" % counts)
            if n:
                rows = [r for part in _all_gather(self.out_host[:n].clone(), self.group,
                                                  self.device) for r in part.tolist()]
        return {name: [r[j] for r in rows] for j, name in enumerate(self.names)}

    def reset(self):
        """Start the next pass at row 0 (the draws continue from the generators' state)."""
        self.k = 0


class PipelinedDPStep(object):
    """Data-parallel training step of the encoder with the gradient all-reduce HIDDEN behind
    the tail of backward (SURVEY.md 8e: pure DP, one flat gradient buffer).

    The flat gradient buffer of ``FlatAdam`` is ordered [blocks 0..split-1 | everything else].
    One step =
        graph A1   H2D, forward, loss, backward of the output layer / QRNN / blocks >= split;
                   those gradients are final in the flat buffer when A1 ends
        eager      NCCL all-reduce (average) of the UPPER bucket (~98 % of the bytes) on a
                   side stream ...
        graph A2   ... while the backward of blocks split-1 .. 0 -- the two largest
                   activations, ~40 % of the backward time -- runs on the main stream
        eager      NCCL all-reduce of the LOWER bucket (blocks 0..split-1: ~1 MB)
        graph B    one pase_adam_flat launch, D2H of the loss
    Collectives are never captured; they are ordered against the graph replays with events.
    ``optimizer`` must be a FlatAdam whose FIRST parameters are exactly the encoder's blocks
    < split (see ``order_params``)."""

    @staticmethod
    def order_params(model, split):
        """Parameter list for FlatAdam: blocks 0..split-1 first (the lower bucket)."""
        lower, upper = [], []
        for name, p in model.named_parameters():
            if not p.requires_grad:
                continue
            head = name.split(".")
            is_lower = head[0] == "blocks" and int(head[1]) < split
            (lower if is_lower else upper).append(p)
        return lower + upper, len(lower)

    def __init__(self, model, optimizer, loss_fn, shape, device, split=3, n_lower=None,
                 group=None, stream=None, resident=False, warmup=3, x_init=None):
        import torch.distributed as dist
        from . import encoder as enc
        self.dist, self.enc = dist, enc
        self.model, self.opt, self.loss_fn, self.split, self.group = model, optimizer, loss_fn, \
            split, group
        if getattr(model, "grad_sink", None) is None:
            optimizer.bind_encoder(model)
        self.sink = model.grad_sink
        if n_lower is None:
            n_lower = sum(1 for n, p in model.named_parameters() if p.requires_grad and
                          n.startswith("blocks.") and int(n.split(".")[1]) < split)
        first_upper = optimizer._offsets[n_lower] if n_lower < len(optimizer._offsets) else optimizer.n
        lo_ids = {id(p) for p in optimizer._plist[:n_lower]}
        want = {id(p) for n, p in model.named_parameters() if p.requires_grad and
                n.startswith("blocks.") and int(n.split(".")[1]) < split}
        if lo_ids != want:
            raise ValueError("PipelinedDPStep: the optimizer's first %d parameters must be the "
                             "encoder's blocks < %d (use PipelinedDPStep.order_params)"
                             % (n_lower, split))
        self.lower = optimizer.flat_grad[:first_upper]
        self.upper = optimizer.flat_grad[first_upper:]
        self.x_static = torch.zeros(shape, dtype=torch.float32, device=device)
        self.x_host = torch.zeros(shape, dtype=torch.float32).pin_memory()
        self.loss_host = torch.zeros((), dtype=torch.float32).pin_memory()
        if x_init is not None:
            self.x_host.copy_(x_init)
            self.x_static.copy_(x_init)
        self.resident = resident
        self.stream = stream if stream is not None else torch.cuda.Stream(device=device)
        self.comm = torch.cuda.Stream(device=device)
        self.ev_upper = torch.cuda.Event()
        self._loss = self._gen = None
        self.gA1 = self.gA2 = self.gB = None
        self._capture(warmup)

    # -- the pieces ----------------------------------------------------------------------
    def _a1(self):
        enc = self.enc
        if not self.resident:
            self.x_static.copy_(self.x_host, non_blocking=True)
        m = self.model
        m._sinc_consts(self.x_static.device)
        plan = m._plan(self.x_static.shape[0], self.x_static.shape[2], self.x_static.device)
        params = dict(m.named_parameters())
        with torch.no_grad():
            y, _ = enc.encoder_forward(plan, m, self.x_static, params, True, True)
        yl = y.detach().requires_grad_(True)
        self._loss = self.loss_fn(yl)
        self._loss.backward()
        self._gen = enc.encoder_backward_steps(plan, m, params, yl.grad.contiguous(), None, True,
                                               self.sink, self.split)
        next(self._gen)                                  # ... up to the split

    def _a2(self):
        try:
            next(self._gen)
            raise RuntimeError("encoder_backward_steps yielded twice")
        except StopIteration:
            pass
        self._gen = None

    def _b(self):
        self.opt.step()
        if not self.resident:
            self.loss_host.copy_(self._loss.detach(), non_blocking=True)

    def _reduce(self, t):
        dist = self.dist
        if dist.get_backend(self.group) == "nccl":
            dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group)
        else:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
            t.mul_(1.0 / dist.get_world_size(self.group))

    def _reduce_upper_async(self):
        """on the side stream, after everything enqueued on the main stream so far"""
        self.ev_upper.record(self.stream)
        self.comm.wait_event(self.ev_upper)
        with torch.cuda.stream(self.comm):
            self._reduce(self.upper)

    def _reduce_lower_and_join(self):
        with torch.cuda.stream(self.stream):
            self._reduce(self.lower)
            self.stream.wait_stream(self.comm)

    def _eager(self):
        self._a1()
        self._reduce_upper_async()
        self._a2()
        self._reduce_lower_and_join()
        self._b()

    def _capture(self, warmup):
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            for _ in range(warmup):
                self._eager()
        self.stream.synchronize()
        self.comm.synchronize()
        torch.cuda.current_stream().wait_stream(self.stream)
        g1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1, stream=self.stream):
            self._a1()
        self._reduce_upper_async()
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g2, stream=self.stream, pool=g1.pool()):
            self._a2()
        self._reduce_lower_and_join()
        g3 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g3, stream=self.stream, pool=g1.pool()):
            self._b()
        self.gA1, self.gA2, self.gB = g1, g2, g3

    def step(self, x_host=None):
        if x_host is not None:
            self.x_host.copy_(x_host)
        _refresh_hyperparams(self.opt, self.stream)
        with torch.cuda.stream(self.stream):
            self.gA1.replay()
            self._reduce_upper_async()
            self.gA2.replay()
            self._reduce_lower_and_join()
            self.gB.replay()
        if self.resident:
            return None
        self.stream.synchronize()
        return float(self.loss_host)
