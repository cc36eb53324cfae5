"""Pure data parallelism over waveform chunks (SURVEY.md 8e): one process per GPU,
model replicated, per-rank BatchNorm statistics (exactly N independent reference runs),
and ONE NCCL all-reduce per step over a single flat fp32 gradient buffer (31 MB for the
PASE+ encoder, 119 MB with every workers+ head).  No per-parameter collectives.

Usage after ``tot_loss.backward()`` (worker_scheduler.py:64)::

    reducer.all_reduce()        # packs whatever autograd produced, then one collective

``all_reduce()`` is safe under every ``zero_grad`` convention: gradients that are already
views of the flat buffer (``zero_grad(set_to_none=False)``, or ``attach()`` + ``zero()``)
are reduced in place; gradients that autograd allocated freshly (``set_to_none=True``, the
torch >= 2.0 default that the reference's ``optim.zero_grad()`` calls hit) are packed with one
multi-tensor copy first and ``.grad`` is re-pointed at the reduced views; parameters without
a gradient contribute zeros.  With CUDA graphs the pack is captured with the backward
(``post_backward=reducer.pack``) and only the collective (``reduce()``) runs between the two
graph replays.
"""
import torch
import torch.distributed as dist


def broadcast_parameters_and_buffers(module, src=0, group=None):
    """One-off replica alignment (what DDP does at construction): parameters and buffers
    (BatchNorm running statistics, step counters) of rank `src` overwrite the others'.
    Afterwards BatchNorm buffers evolve per rank (exactly N independent reference runs, the
    reference has no SyncBN); checkpoint rank 0's."""
    _broadcast_in_place([p.data for p in module.parameters()] +
                        [b.data for b in module.buffers()], src, group)


def broadcast_buffers(module, src=0, group=None):
    """Rank `src`'s buffers (BatchNorm running statistics, step counters) into every rank's, in
    place: CUDA graphs that read them by address see the new values (what DDP's
    ``broadcast_buffers`` gives before a forward)."""
    _broadcast_in_place([b.data for b in module.buffers()], src, group)


def _broadcast_in_place(tensors, src, group):
    """One broadcast per (dtype, device) of the concatenated tensors, copied back into them."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return
    by_dtype = {}
    for t in tensors:
        by_dtype.setdefault((t.dtype, t.device), []).append(t)
    for (_, _), ts in by_dtype.items():
        flat = torch.cat([t.reshape(-1) for t in ts])
        dist.broadcast(flat, src=src, group=group)
        off = 0
        for t in ts:
            t.copy_(flat[off:off + t.numel()].view_as(t))
            off += t.numel()


class FlatGradAllReducer(object):
    def __init__(self, params, process_group=None, attach=True):
        self.params = [p for p in params if p.requires_grad]
        self.group = process_group
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        self.views, off = [], 0
        for p in self.params:
            self.views.append(self.flat[off:off + p.numel()].view_as(p))
            off += p.numel()
        if attach:
            self.attach()
        self.nbytes = n * 4

    def attach(self):
        for p, v in zip(self.params, self.views):
            p.grad = v

    def detach(self):
        for p in self.params:
            p.grad = None

    def zero(self):
        self.flat.zero_()

    def world(self):
        if dist.is_available() and dist.is_initialized():
            return dist.get_world_size(self.group)
        return 1

    def reduce(self):
        """The collective alone: average the flat buffer over ranks (NCCL: ReduceOp.AVG, one
        kernel; other backends: SUM then scale)."""
        w = self.world()
        if w > 1:
            if dist.get_backend(self.group) == "nccl":
                dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=self.group)
            else:
                dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
                self.flat.mul_(1.0 / w)
        return self.flat

    def pack(self):
        """Bring every gradient into the flat buffer (one multi-tensor copy for the ones that
        are not views of it yet, zeros for parameters without a gradient) and re-point
        ``.grad`` at the views.  No collective."""
        srcs, dsts = [], []
        for p, v in zip(self.params, self.views):
            if p.grad is None:
                v.zero_()
            elif p.grad.data_ptr() != v.data_ptr():
                srcs.append(p.grad)
                dsts.append(v)
        if srcs:
            torch._foreach_copy_(dsts, srcs)
        self.attach()
        return self.flat

    def all_reduce(self):
        """pack() + reduce(): correct whatever ``zero_grad`` flavour ran before backward."""
        self.pack()
        return self.reduce()

    pack_and_reduce = all_reduce
