"""CPU, world_size 2 over gloo: the N>1 path of otter_b200.dp — batch sharding and the single flat-buffer
gradient all-reduce (mean over ranks = DDP semantics, SURVEY.md §8e)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from otter_b200.dp import FlatGradBuffer, shard_batch


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q, comm_dtype=None, async_op=False):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(0)                                   # identical weights on all ranks
    lin = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 3))
    lin[0].bias.requires_grad_(False)                      # a frozen parameter must be skipped
    flat = FlatGradBuffer(lin.parameters(), device="cpu", comm_dtype=comm_dtype)
    assert flat.numel % 4 == 0 and all(o % 4 == 0 for o in flat.offsets)
    g = torch.Generator().manual_seed(7)
    X = torch.randn(8, 6, generator=g)                     # the GLOBAL batch, same on both ranks
    lo, hi = shard_batch(8, rank, world)
    flat.begin_step()
    loss = lin(X[lo:hi]).pow(2).mean()
    loss.backward()                                        # autograd accumulates into the flat views
    flat.finish_step()
    work = flat.all_reduce(async_op=async_op)
    if work is not None:
        work.wait()
        if not getattr(work, "averaged", False):
            flat.flat.div_(world)
    # reference: full-batch gradient on one process (equal shards => mean of shard grads == full-batch grad)
    ref = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 3))
    ref.load_state_dict(lin.state_dict())
    ref(X).pow(2).mean().backward()
    rtol, atol = (1e-5, 1e-6) if comm_dtype is None else (2e-2, 2e-3)       # bf16 wire format: 8 mantissa bits
    ok = all(torch.allclose(p.grad, r.grad, rtol=rtol, atol=atol)
             for p, r in zip(lin.parameters(), ref.parameters()) if p.requires_grad)
    views_ok = all(p.grad.data_ptr() >= flat.flat.data_ptr() for p in flat.params)
    q.put((rank, ok, views_ok, flat.numel))
    dist.destroy_process_group()


def _run_world2(*extra):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q) + extra) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(timeout=60) for p in procs]
    assert all(ok and views for _, ok, views, _ in res), res
    assert res[0][3] == res[1][3]


def test_flat_allreduce_world2():
    _run_world2()


def test_flat_allreduce_world2_async():
    _run_world2(None, True)


def test_flat_allreduce_world2_bf16_wire():
    """Reduced-precision wire format (SURVEY.md §8e's 2.36 GB payload): gradients stay fp32 on both sides."""
    _run_world2(torch.bfloat16, False)
    _run_world2(torch.bfloat16, True)


def test_shard_batch_partitions_exactly():
    for n in (1, 7, 8, 256):
        for w in (1, 2, 3, 8):
            spans = [shard_batch(n, r, w) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [b - a for a, b in spans]
            assert max(sizes) - min(sizes) <= 1


def test_zero_grad_set_to_none_keeps_the_flat_buffer_live():
    """The reference's loop calls optimizer.zero_grad() (set_to_none=True by default) every step
    (pipeline/train/instruction_following.py:213): `.grad` must be a view of the flat buffer again after
    begin_step(), in either call order, and a kernel-sink parameter whose `.grad` was dropped must still be seen
    by the optimizer."""
    torch.manual_seed(0)
    lin = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 3))
    flat = FlatGradBuffer(lin.parameters(), device="cpu")
    opt = torch.optim.SGD(lin.parameters(), lr=0.1)
    sink = lin[1].weight                                   # pretend an otter_b200 wgrad epilogue writes this one
    X = torch.randn(4, 6)
    for order in ("zero_then_begin", "begin_then_zero", "zero_then_begin"):
        if order == "zero_then_begin":
            opt.zero_grad()
            flat.begin_step()
        else:
            flat.begin_step()
            opt.zero_grad()
        assert order == "begin_then_zero" or all(p.grad is not None for p in flat.params)
        before = [p.detach().clone() for p in lin.parameters()]
        # the "kernel" path: gradient written straight into the sink view, autograd gets None for it
        sink.requires_grad_(False)
        lin(X).pow(2).mean().backward()
        sink.requires_grad_(True)
        sink._otb_grad.fill_(0.25)
        sink._otb_grad_live = True
        sink._otb_sink_user = True
        flat.finish_step()
        for p, v in zip(flat.params, flat.views):
            assert p.grad is not None and p.grad.data_ptr() == v.data_ptr()
        assert flat.flat.abs().sum() > 0
        opt.step()
        for p, b in zip(lin.parameters(), before):
            assert not torch.equal(p.detach(), b), "optimizer skipped a parameter"
        assert torch.allclose(sink.detach(), before[2] - 0.1 * 0.25)


def _worker_direct(rank, world, port, q):
    """bf16 wire format with DIRECT sinks: the (emulated) wgrad kernel writes bf16 straight into the comm buffer."""
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(0)
    lin = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 3))
    direct = [lin[0].weight, lin[1].weight]
    flat = FlatGradBuffer(lin.parameters(), device="cpu", comm_dtype=torch.bfloat16, direct_params=direct)
    assert flat.params[:2] == direct and flat.direct_numel == 32 + 16          # 30 -> 32, 15 -> 16 (16-byte segments)
    assert all(p._otb_grad.dtype == torch.bfloat16 for p in direct) and lin[0].bias._otb_grad.dtype == torch.float32
    g = torch.Generator().manual_seed(7)
    X = torch.randn(8, 6, generator=g)
    lo, hi = shard_batch(8, rank, world)
    ref = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 3))
    ref.load_state_dict(lin.state_dict())
    ref(X).pow(2).mean().backward()
    flat.begin_step()
    shard = torch.nn.Sequential(torch.nn.Linear(6, 5), torch.nn.Linear(5, 3))
    shard.load_state_dict(lin.state_dict())
    shard(X[lo:hi]).pow(2).mean().backward()
    from otter_b200.params import GradSink
    sink = GradSink()
    for p, sp in zip(lin.parameters(), shard.parameters()):                    # the "kernels" write through the sinks
        buf, acc = sink.target(p)
        assert not acc
        buf.copy_(sp.grad)
    flat.finish_step()
    w = flat.all_reduce(async_op=True)
    w.wait()
    ok = all(torch.allclose(p.grad, r.grad, rtol=2e-2, atol=2e-3) for p, r in zip(lin.parameters(), ref.parameters()))
    second_write_refused = False
    try:
        GradSink().target(direct[0])
    except RuntimeError:
        second_write_refused = True
    q.put((rank, ok and second_write_refused, all(p.grad.dtype == torch.float32 for p in lin.parameters()), flat.numel))
    dist.destroy_process_group()


def test_flat_allreduce_world2_bf16_direct_sinks():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_direct, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(timeout=60) for p in procs]
    assert all(ok and views for _, ok, views, _ in res), res


def test_reduce_op_argument():
    """The wire-format collective reduces with SUM (1/world_size folded into the up-cast) by default; 'avg' keeps ncclAvg;
    anything else is rejected.  (On gloo both arms are SUM + divide.)"""
    import pytest
    from otter_b200.dp import FlatGradBuffer
    lin = torch.nn.Linear(8, 8)
    assert FlatGradBuffer(lin.parameters(), device="cpu", comm_dtype=torch.bfloat16).reduce_op == "sum"
    assert FlatGradBuffer(lin.parameters(), device="cpu", comm_dtype=torch.bfloat16, reduce_op="avg").reduce_op == "avg"
    with pytest.raises(ValueError, match="reduce_op"):
        FlatGradBuffer(lin.parameters(), device="cpu", reduce_op="max")
