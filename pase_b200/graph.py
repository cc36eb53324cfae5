"""CUDA-graph capture of one whole training step (H2D of the waveform batch, encoder
forward + backward through the C-ABI kernels, optimizer update, D2H of the loss) so that a
step is ONE launch: the hot loop is launch-bound on the host once the kernels take only a
few ms.  Buffers of the encoder plan are static by construction (EncoderPlan), TMA
descriptors are kernel parameters, so the captured graph is replayable as is.
"""
import torch


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
        self.graph.replay()
        if self.graph_b is not None:
            with torch.cuda.stream(self.stream):
                self.between()
            self.graph_b.replay()
        if self.resident:
            return None
        self.stream.synchronize()
        return float(self.loss_host)


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
