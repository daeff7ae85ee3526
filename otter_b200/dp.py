"""Data parallelism of the hot path: one flat fp32 gradient buffer, ONE all-reduce per step.

Replaces `accelerator.prepare(model)` + `accelerator.backward(loss)` (DDP bucketed all-reduce,
pipeline/train/instruction_following.py:200,219-222,491-494; SURVEY.md §2.3 / §8e): the batch dimension
shards across ranks with no other collective.  Every trainable parameter's `.grad` is a view into one
contiguous buffer; the wgrad GEMM epilogues write straight into it (`_otb_grad` sink, otter_b200.params),
so the step ends with a single mean all-reduce over NVLink/NVSwitch (NCCL via torch.distributed: `AVG` on the fp32
buffer, `SUM` with 1/world_size folded into the up-cast on the bf16 wire format; on CPU tests the same code runs over gloo).
"""
import torch
import torch.distributed as dist


class _CommHandle:
    """Completion handle of a reduced-precision all-reduce: wait() also copies the averaged gradients back into
    the fp32 buffer the `.grad` views alias."""
    averaged = True

    def __init__(self, owner, work, divide_by):
        self.owner, self.work, self.divide_by = owner, work, divide_by

    def wait(self):
        if self.work is not None:
            self.work.wait()
        o = self.owner
        if self.divide_by and o.comm.is_cuda and o.comm.dtype == torch.bfloat16 and o.flat.dtype == torch.float32:
            from . import functional as F                      # one pass: up-cast with the 1/world_size folded in
            F.cast_f32_scaled(o.comm, o.flat, 1.0 / self.divide_by)
            return True
        if self.divide_by:
            o.comm.div_(self.divide_by)
        o.flat.copy_(o.comm)
        return True


class FlatGradBuffer:
    def __init__(self, params, device=None, dtype=torch.float32, comm_dtype=None, nccl_registered=False,
                 direct_params=None, reduce_op="sum"):
        """direct_params (only with a reduced-precision comm_dtype): parameters whose gradient is produced by ONE wgrad
        GEMM per step (the nn.Linear weights of the perceiver / gated blocks).  Their kernel sink is the bf16 WIRE
        buffer itself — the epilogue rounds once to the wire format, which is also what autocast's backward hands the
        reference (a bf16 weight gradient cast up to fp32) — so the 7 GB cast pass in front of the collective
        disappears; `.grad` (fp32) is filled by the one up-cast after the collective.  Gradient accumulation over
        several backward passes per step is not available for these parameters (the sink refuses a second write)."""
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("no trainable parameters")
        if reduce_op not in ("sum", "avg"):
            raise ValueError("reduce_op must be 'sum' or 'avg'")
        # Wire-format collectives reduce with SUM and fold 1/world_size into the up-cast that follows: NCCL implements AVG
        # on floating types as pre-multiplied sum, which its in-switch (NVLS) algorithms do not take, so AVG pins the
        # collective to RING.  'avg' keeps ncclAvg.
        self.reduce_op = reduce_op
        direct_ids = {id(p) for p in (direct_params or [])}
        if direct_ids and (comm_dtype is None or comm_dtype == dtype):
            raise ValueError("direct_params needs a reduced-precision comm_dtype")
        # direct-sink parameters first, so that everything still produced in fp32 is ONE contiguous tail to cast
        self.params = [p for p in self.params if id(p) in direct_ids] + [p for p in self.params if id(p) not in direct_ids]
        self.n_direct_params = sum(1 for p in self.params if id(p) in direct_ids)
        device = device or self.params[0].device
        # 16-byte aligned segments so vectorised epilogue stores stay legal
        self.offsets, off = [], 0
        for p in self.params:
            self.offsets.append(off)
            off += (p.numel() + 3) // 4 * 4
        self.numel = off
        self.direct_numel = self.offsets[self.n_direct_params] if self.n_direct_params < len(self.params) else off
        if self.n_direct_params == 0:
            self.direct_numel = 0
        self._pools = []
        self._registered = bool(nccl_registered)
        self.flat = self._alloc(off, dtype, device)
        # optional wire format of the collective (SURVEY.md §8e budgets the bf16 payload: 2.36 GB instead of 4.72 GB);
        # gradients are still produced, accumulated and handed to the optimizer in `dtype`
        self.comm = None
        if comm_dtype is not None and comm_dtype != dtype:
            self.comm = self._alloc(off, comm_dtype, device)
        self.views = []
        for p, o in zip(self.params, self.offsets):
            view = self.flat[o:o + p.numel()].view(p.shape)
            if p.dtype != dtype:
                raise TypeError(f"FlatGradBuffer({dtype}) needs {dtype} parameters (fp32 master weights); got {p.dtype}")
            self.views.append(view)
            p.grad = view
            if dtype == torch.float32:
                p._otb_grad = view          # sink used by otter_b200 backward kernels
                p._otb_grad_live = False
        for p, o in zip(self.params[:self.n_direct_params], self.offsets):
            p._otb_grad = self.comm[o:o + p.numel()].view(p.shape)      # the wgrad epilogue writes the wire format

    def _alloc(self, n, dtype, device):
        """Plain zero-filled allocation, or (nccl_registered=True) one drawn from NCCL's own allocator and registered
        with the communicator, so the collective can run zero-copy / in-switch (NVLS) on the user buffer instead of
        staging through NCCL's internal buffers.  Needs an initialised NCCL process group; fails loudly otherwise."""
        if not self._registered:
            return torch.zeros(n, device=device, dtype=dtype)
        if not (dist.is_available() and dist.is_initialized()) or dist.get_backend() != "nccl":
            raise RuntimeError("nccl_registered=True needs an initialised NCCL process group")
        backend = dist.distributed_c10d._get_default_group()._get_backend(torch.device(device))
        pool = torch.cuda.MemPool(backend.mem_allocator)
        with torch.cuda.use_mem_pool(pool):
            t = torch.zeros(n, device=device, dtype=dtype)
        backend.register_mem_pool(pool)
        self._pools.append(pool)              # keep the pool (and the registration) alive with the buffer
        return t

    def begin_step(self):
        """Start a step.  Parameters whose gradients are written by otter_b200 kernels (`_otb_sink_user`, learned
        on first use) are only marked empty — the first kernel write overwrites, later ones accumulate, so the
        multi-GB buffer needs no zero-fill pass.  Parameters that receive gradients through plain autograd
        accumulation (e.g. LM embeddings) are zeroed here, like optimizer.zero_grad().

        `optimizer.zero_grad()` (set_to_none=True is the default, and what the reference's loop calls:
        pipeline/train/instruction_following.py:213) detaches `.grad` from the flat buffer; every view is re-attached
        here, so begin_step() is the only reset a train loop needs and the kernels' sinks, `.grad` and the buffer the
        all-reduce sends stay one and the same memory."""
        for p, view in zip(self.params, self.views):
            if p.grad is None or p.grad.data_ptr() != view.data_ptr():
                p.grad = view
            if getattr(p, "_otb_sink_user", False):
                p._otb_grad_live = False
            else:
                view.zero_()

    def finish_step(self):
        """Kernel-written sinks nobody touched this step (unused parameters) must read as zero before the reduce.
        Also repairs the aliasing if `optimizer.zero_grad()` ran AFTER begin_step(): a gradient autograd then
        accumulated outside the buffer is copied in, and every `.grad` is a view of the buffer again."""
        for p, view in zip(self.params, self.views):
            sink = getattr(p, "_otb_sink_user", False)
            if sink and not p._otb_grad_live:
                p._otb_grad.zero_()
            g = p.grad
            if g is None or g.data_ptr() != view.data_ptr():
                if g is not None and not sink:
                    view.copy_(g)
                p.grad = view

    def all_reduce(self, group=None, async_op=False):
        """The one collective of the step: mean over ranks (DDP semantics)."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            if self.direct_numel:       # single rank: the wire-format sinks still have to reach the fp32 `.grad` views
                self.flat[:self.direct_numel].copy_(self.comm[:self.direct_numel])
            return None
        if self.comm is not None:
            # cast on the current stream, ahead of the collective: everything, or only the fp32-produced tail when the
            # big gradients were written in the wire format by the kernels
            d = self.direct_numel
            if d < self.numel:
                self.comm[d:].copy_(self.flat[d:])
            if dist.get_backend(group) == "gloo":
                w = dist.all_reduce(self.comm, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
                h = _CommHandle(self, w if async_op else None, dist.get_world_size(group))
            elif self.reduce_op == "sum":
                w = dist.all_reduce(self.comm, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
                h = _CommHandle(self, w if async_op else None, dist.get_world_size(group))
            else:
                w = dist.all_reduce(self.comm, op=dist.ReduceOp.AVG, group=group, async_op=async_op)
                h = _CommHandle(self, w if async_op else None, 0)
            if not async_op:
                h.wait()
                return None
            return h
        if dist.get_backend(group) == "gloo":          # gloo has no AVG
            w = dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
            if not async_op:
                self.flat.div_(dist.get_world_size(group))
            return w
        return dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=group, async_op=async_op)

    def grad_norm(self):
        return self.flat.norm()

    def nbytes(self):
        return self.flat.numel() * self.flat.element_size()

    def comm_nbytes(self):
        """Bytes each rank contributes to the step's all-reduce."""
        buf = self.comm if self.comm is not None else self.flat
        return buf.numel() * buf.element_size()


def shard_batch(global_batch, rank, world_size):
    """Contiguous, near-equal split of the batch dimension: rank r owns [start, stop)."""
    base, rem = divmod(global_batch, world_size)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)
