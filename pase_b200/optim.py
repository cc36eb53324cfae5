"""Flat-buffer Adam / RAdam (SURVEY.md 8f N4).

The reference trains with one optimizer per worker plus one for the frontend
(pase/models/WorkerScheduler/trainer.py:86-143) and steps them one after the other
(worker_scheduler.py:66-73): 13 x (zero_grad + multi-tensor step).  The optimizers are
``torch.optim.Adam``, or the reference's own ``RAdam`` for ``--fe_opt radam`` /
``--min_opt radam``.  ``FlatAdam`` keeps every parameter, gradient and moment of ALL those
groups in four flat fp32 buffers and updates them with ONE kernel launch (``pase_adam_flat``),
with per-group learning rates / betas / eps / weight decay and algorithm (``"adam"`` or
``"radam"``, mixed freely).  The gradient buffer is the same flat buffer the data-parallel
all-reduce works on (``pase_b200.dp.FlatGradAllReducer``), so a step is: backward -> one NCCL
all-reduce -> one optimizer launch.

Drop-in surface: ``param_groups`` (LR schedulers mutate ``group['lr']``), ``step()``,
``zero_grad()``, ``state_dict()`` / ``load_state_dict()`` in torch.optim.Adam's own format,
or the reference RAdam's for RAdam groups (so ``Saver`` checkpoints interchange with the
reference's), and ``views()``: one per-group facade with ``step()`` / ``zero_grad()`` /
``state_dict()`` / ``load_state_dict()`` for callers that hold a
dict of optimizers like the reference's ``backprop_scheduler`` -- the facades' steps are
deferred and the single launch happens when the last group has stepped.
"""
import torch

from . import ops


def _ru4(n):
    return (n + 3) // 4 * 4


# the segment table's algorithm code of each supported update
ALGORITHMS = {"adam": 0, "radam": 1}


def _algorithm(name):
    if name not in ALGORITHMS:
        raise ValueError("FlatAdam: algorithm=%r; supported: %s"
                         % (name, ", ".join(repr(a) for a in ALGORITHMS)))
    return name


class FlatAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
                 grad_buffer=None, grad_scale=1.0, peer_dp=False, group=None, algorithm="adam"):
        """algorithm (default of every group; a group may set its own ``"algorithm"`` key):
        ``"adam"`` is torch.optim.Adam (L2 weight decay added to the gradient); ``"radam"`` is
        the reference's RAdam (pase/models/WorkerScheduler/radam.py: rectified steps from the
        step where rho >= 5, momentum-SGD steps before it, decoupled weight decay).  Each RAdam
        group computes its own step size; the reference's RAdam caches one per step for all
        groups of an instance, which differs only for an instance with several groups of
        different lr, a layout the reference trainer never builds.

        peer_dp=True (torch.distributed initialised, one process per GPU of ONE node): the
        flat parameter / gradient buffers are CUDA-IPC peer-mapped across the ranks and
        ``step()`` becomes ``pase_adam_flat_dp`` -- gradient averaging (reduce-scatter),
        the Adam update of this rank's 1/world shard and the parameter all-gather in ONE
        kernel over NVLink, no collective call (``reduce_grads()`` turns into a no-op).  The
        Adam moments are then sharded: ``consolidate_state()`` (collective) before
        ``state_dict()``."""
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                        algorithm=_algorithm(algorithm))
        super().__init__(params, defaults)
        for g in self.param_groups:
            _algorithm(g["algorithm"])
        plist = [p for g in self.param_groups for p in g["params"]]
        if not plist:
            raise ValueError("FlatAdam: no parameters")
        dev = plist[0].device
        if any(p.dtype != torch.float32 or p.device != dev for p in plist):
            raise ValueError("FlatAdam: parameters must be fp32 on one device")
        # segment = one param group; every parameter starts at a multiple of 4 elements
        self._offsets, self._ranges, off = [], [], 0
        for g in self.param_groups:
            start = off
            for p in g["params"]:
                self._offsets.append(off)
                off = _ru4(off + p.numel())
            self._ranges.append((start, off))
        self.n = off
        f32 = dict(dtype=torch.float32, device=dev)
        self.peer_dp = bool(peer_dp)
        self._peer = None
        self._group = group
        if peer_dp:
            import torch.distributed as dist
            if not (dist.is_available() and dist.is_initialized()):
                raise RuntimeError("FlatAdam(peer_dp=True) needs an initialised process group")
            if grad_buffer is not None:
                raise ValueError("FlatAdam: peer_dp allocates its own gradient buffer")
            world = dist.get_world_size(group)
            if world > 1:
                from .peer import PeerAlloc, PeerGroup
                allocs = {"param": PeerAlloc(self.n, torch.float32, dev),
                          "grad": PeerAlloc(self.n, torch.float32, dev),
                          "flag": PeerAlloc(2 * world, torch.int32, dev)}
                self._peer = PeerGroup(allocs, group)
                self._peer_sync = torch.zeros(2, dtype=torch.int32, device=dev)   # epoch, done
        if self._peer is not None:
            self.flat_param = self._peer.allocs["param"].tensor
            self.flat_grad = self._peer.allocs["grad"].tensor
        else:
            self.flat_param = torch.zeros(self.n, **f32)
            if grad_buffer is not None and grad_buffer.numel() != self.n:
                raise ValueError("FlatAdam: grad_buffer has %d elements, layout needs %d"
                                 % (grad_buffer.numel(), self.n))
            self.flat_grad = grad_buffer if grad_buffer is not None else torch.zeros(self.n, **f32)
        self.exp_avg = torch.zeros(self.n, **f32)
        self.exp_avg_sq = torch.zeros(self.n, **f32)
        self.grad_scale = float(grad_scale)
        self._plist = plist
        self._pviews, self._gviews = [], []
        for p, o in zip(plist, self._offsets):
            pv = self.flat_param[o:o + p.numel()].view_as(p)
            pv.copy_(p.data)
            p.data = pv                                   # parameters become views
            self._pviews.append(pv)
            self._gviews.append(self.flat_grad[o:o + p.numel()].view_as(p))
        self.steps = torch.zeros(len(self.param_groups), **f32)       # device step counts
        self._table = None
        self._table_key = None
        self._pending = set()
        self._sunk = set()

    # ---- gradient buffer protocol (shared with dp.FlatGradAllReducer) -----------------
    def attach_grads(self):
        for p, v in zip(self._plist, self._gviews):
            p.grad = v

    def pack_grads(self):
        """Gradients autograd allocated outside the flat buffer are copied in (one
        multi-tensor copy); parameters without a gradient contribute zeros."""
        srcs, dsts = [], []
        sunk = self._sunk
        for p, v in zip(self._plist, self._gviews):
            if id(p) in sunk:                 # written in place by the encoder's kernels
                continue
            if p.grad is None:
                v.zero_()
            elif p.grad.data_ptr() != v.data_ptr():
                srcs.append(p.grad)
                dsts.append(v)
        if srcs:
            torch._foreach_copy_(dsts, srcs)
        self.attach_grads()

    def zero_grad(self, set_to_none=False):
        """One memset of the flat gradient buffer; ``.grad`` stays a view of it.  Parameters
        bound through ``bind_encoder`` keep their views even with set_to_none (their
        gradients are overwritten, not accumulated)."""
        if set_to_none:
            for p in self._plist:
                if id(p) not in self._sunk:
                    p.grad = None
        else:
            self.flat_grad.zero_()
            self.attach_grads()

    def bind_encoder(self, encoder):
        """Make the encoder's backward kernels write their gradients straight into this
        optimizer's flat gradient buffer (``WaveFe.grad_sink``): no autograd accumulation, no
        per-parameter copies.  The encoder's gradients are then OVERWRITTEN by each backward
        (one encoder call per step); other modules' gradients keep autograd's semantics."""
        byid = {id(p): v for p, v in zip(self._plist, self._gviews)}
        sink = {}
        for name, p in encoder.named_parameters():
            if p.requires_grad:
                if id(p) not in byid:
                    raise ValueError("FlatAdam.bind_encoder: %s is not optimised here" % name)
                sink[name] = byid[id(p)]
        encoder.grad_sink = sink
        self._sunk = {id(p) for _, p in encoder.named_parameters() if p.requires_grad}
        self.attach_grads()
        return self

    def reduce_grads(self, group=None):
        """Data parallelism: ONE all-reduce (average) of the flat gradient buffer."""
        import torch.distributed as dist
        if self._peer is not None:
            return self.flat_grad            # averaged inside step() (pase_adam_flat_dp)
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            self.pack_grads()
            if dist.get_backend(group) == "nccl":
                dist.all_reduce(self.flat_grad, op=dist.ReduceOp.AVG, group=group)
            else:
                dist.all_reduce(self.flat_grad, op=dist.ReduceOp.SUM, group=group)
                self.flat_grad.mul_(1.0 / dist.get_world_size(group))
        return self.flat_grad

    # ---- the update ------------------------------------------------------------------
    def _segments(self):
        """The device table of per-group hyper-parameters and algorithm.  It is allocated once and keeps its
        address: a captured ``pase_adam_flat`` launch reads whatever the table holds at replay
        time, so a changed lr / betas / eps / weight decay is written into the same tensor, by
        a copy ordered on the current stream after every earlier update that read it."""
        key = tuple((g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"],
                     ALGORITHMS[_algorithm(g["algorithm"])]) for g in self.param_groups)
        if key != self._table_key:
            import struct
            raw = b"".join(
                struct.pack("<qqffffffq", a, b, float(k[0]), float(k[1]), float(k[2]), float(k[3]),
                            float(k[4]), float(k[5]), i)
                for i, ((a, b), k) in enumerate(zip(self._ranges, key)))
            src = torch.frombuffer(bytearray(raw), dtype=torch.int64)
            dev = self.flat_param.device
            if self._table is None:
                self._table = torch.empty(src.numel(), dtype=torch.int64, device=dev)
            if dev.type == "cuda":
                # page-locked: the copy is asynchronous, and the caching host allocator keeps
                # the source alive until it has executed
                src = src.pin_memory()
            self._table.copy_(src, non_blocking=True)
            self._table_key = key
        return self._table

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.pack_grads()
        self.steps += 1.0
        if self._peer is not None:
            pg = self._peer
            ops.call("pase_adam_flat_dp", pg.table("param"), pg.table("grad"), pg.table("flag"),
                     self.exp_avg, self.exp_avg_sq, self.n, self._segments(),
                     len(self.param_groups), self.steps, pg.world, pg.rank,
                     self._peer_sync[0:1], self._peer_sync[1:2])
            return loss
        ops.call("pase_adam_flat", self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq,
                 self.n, self._segments(), len(self.param_groups), self.steps, self.grad_scale)
        return loss

    def shard_range(self):
        """[lo, hi) of the flat index space whose Adam moments this rank maintains."""
        if self._peer is None:
            return 0, self.n
        per = ((self.n + 3) // 4 + self._peer.world - 1) // self._peer.world
        return min(per * self._peer.rank * 4, self.n), min(per * (self._peer.rank + 1) * 4, self.n)

    def consolidate_state(self):
        """peer_dp: gather every rank's shard of (exp_avg, exp_avg_sq) so that ``state_dict()``
        is complete on every rank.  Collective -- call it on all ranks before checkpointing."""
        if self._peer is None:
            return
        import torch.distributed as dist
        per = ((self.n + 3) // 4 + self._peer.world - 1) // self._peer.world * 4
        for buf in (self.exp_avg, self.exp_avg_sq):
            pad = torch.zeros(per * self._peer.world, dtype=buf.dtype, device=buf.device)
            pad[:self.n] = buf
            lo = per * self._peer.rank
            dist.all_gather_into_tensor(pad, pad[lo:lo + per].clone(), group=self._group)
            buf.copy_(pad[:self.n])

    # ---- torch.optim.Adam / reference RAdam-compatible persistence ----------------------
    def state_dict(self):
        """torch.optim.Adam's format for Adam groups; for RAdam groups the reference RAdam's:
        an int ``step`` and only lr / betas / eps / weight_decay in the group."""
        state, groups, idx = {}, [], 0
        steps = self.steps.detach().cpu()
        for gi, g in enumerate(self.param_groups):
            radam = g["algorithm"] == "radam"
            ids = []
            for p in g["params"]:
                o = self._offsets[idx]
                state[idx] = {"step": int(steps[gi]) if radam else steps[gi].clone(),
                              "exp_avg": self.exp_avg[o:o + p.numel()].view_as(p).clone(),
                              "exp_avg_sq": self.exp_avg_sq[o:o + p.numel()].view_as(p).clone()}
                ids.append(idx)
                idx += 1
            if radam:
                gd = {k: g[k] for k in ("lr", "betas", "eps", "weight_decay")}
                gd.update(params=ids)
            else:
                gd = {k: v for k, v in g.items() if k not in ("params", "algorithm")}
                gd.update(params=ids, amsgrad=False, maximize=False, foreach=None,
                          capturable=False, differentiable=False, fused=None)
            groups.append(gd)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        """Either format; the groups keep their algorithm, which neither format records."""
        first = 0
        for gi, sg in enumerate(sd["param_groups"][:len(self.param_groups)]):
            self._load_group(gi, sg, sd["state"], first)
            first += len(self.param_groups[gi]["params"])

    def _load_group(self, gi, sg, state, first):
        """Group gi from a saved group ``sg`` whose parameters are ``state[first + j]``."""
        g = self.param_groups[gi]
        for k in ("lr", "betas", "eps", "weight_decay"):
            if k in sg:
                g[k] = tuple(sg[k]) if k == "betas" else sg[k]
        base = sum(len(h["params"]) for h in self.param_groups[:gi])
        step = None
        for j, p in enumerate(g["params"]):
            st = state.get(first + j, state.get(str(first + j)))
            if st is not None:
                o = self._offsets[base + j]
                self.exp_avg[o:o + p.numel()].view_as(p).copy_(st["exp_avg"])
                self.exp_avg_sq[o:o + p.numel()].view_as(p).copy_(st["exp_avg_sq"])
                step = float(st["step"])
        if step is not None:
            self.steps[gi] = step
        self._table_key = None

    # ---- per-group facades for callers that hold a dict of optimizers -------------------
    def views(self):
        """One facade per param group, in order (e.g. frontend, then each worker)."""
        return [_GroupView(self, i) for i in range(len(self.param_groups))]

    def _view_step(self, gi):
        self._pending.add(gi)
        if len(self._pending) == len(self.param_groups):
            self._pending.clear()
            self.step()


class _GroupView(object):
    """What ``backprop_scheduler`` needs from an optimizer (worker_scheduler.py:43-75):
    ``zero_grad()`` and ``step()``; plus ``param_groups`` for the LR schedulers and
    ``state_dict`` / ``load_state_dict`` for the per-worker ``Saver``.  ``step()`` is deferred: the one kernel launch
    happens when the last group of the engine has stepped."""

    def __init__(self, engine, gi):
        self.engine, self.gi = engine, gi

    @property
    def param_groups(self):
        return [self.engine.param_groups[self.gi]]

    def zero_grad(self, set_to_none=False):
        a, b = self.engine._ranges[self.gi]
        self.engine.flat_grad[a:b].zero_()
        self.engine.attach_grads()

    def step(self, closure=None):
        self.engine._view_step(self.gi)

    def state_dict(self):
        full = self.engine.state_dict()
        ids = full["param_groups"][self.gi]["params"]
        remap = {old: new for new, old in enumerate(ids)}
        g = dict(full["param_groups"][self.gi])
        g["params"] = list(range(len(ids)))
        return {"state": {remap[i]: full["state"][i] for i in ids}, "param_groups": [g]}

    def load_state_dict(self, sd):
        self.engine._load_group(self.gi, sd["param_groups"][0], sd["state"], 0)
