"""Parameter plumbing: bf16 compute shadows of fp32 master weights, and gradient sinks.

The reference trains fp32 weights under `autocast(bf16)` (pipeline/train/instruction_following.py:311-314):
autocast re-casts each weight to bf16 for the matmul.  Here the cast is an explicit kernel
(otb_cast_f32_bf16) whose result is cached until the parameter changes (`_version` bump by the
optimizer / load_state_dict), so a step pays for it exactly once per weight.

Gradient sinks: by default backward returns fresh fp32 gradients to autograd.  When a parameter
carries `_otb_grad` (an fp32 view into the flat data-parallel gradient buffer, see otter_b200.dp),
the wgrad GEMM epilogue writes/accumulates straight into it and autograd receives None — no gather
copy before the single NCCL all-reduce.
"""
import weakref

import torch

from . import functional as F

# id(param) -> (version, data_ptr, converted tensor, weakref(param)).  The weakref guards against CPython
# re-using an id (and the allocator re-using the address) for a different parameter after the old one died.
_shadow = {}
_f32 = {}


def _ref(cache, p):
    """weakref whose callback drops the cache entry (and its device buffer) when the parameter dies."""
    key = id(p)

    def _drop(r, cache=cache, key=key):
        hit = cache.get(key)
        if hit is not None and hit[3] is r:
            del cache[key]

    return weakref.ref(p, _drop)


def _lookup(cache, p, ver, ptr):
    hit = cache.get(id(p))
    if hit is not None and hit[3]() is not p:
        del cache[id(p)]
        return None, None
    if hit is not None and hit[0] == ver and hit[1] == ptr:
        return hit, hit[2]
    return hit, None


def bf16_of(p):
    """bf16 compute copy of a weight (identity for bf16 parameters)."""
    t = p.detach() if isinstance(p, torch.nn.Parameter) or p.requires_grad else p
    if t.dtype == torch.bfloat16:
        return t if t.is_contiguous() else t.contiguous()
    ver, ptr = p._version, t.data_ptr()
    hit, val = _lookup(_shadow, p, ver, ptr)
    if val is not None:
        return val
    out = hit[2] if (hit is not None and hit[2].shape == t.shape and hit[2].device == t.device) else None
    out = F.cast_bf16(t.float() if t.dtype != torch.float32 else t, out)
    _shadow[id(p)] = (ver, ptr, out, _ref(_shadow, p))
    return out


def f32_of(p):
    """fp32 view/copy of a small parameter (LayerNorm affine, bias, gate)."""
    t = p.detach()
    if t.dtype == torch.float32:
        return t if t.is_contiguous() else t.contiguous()
    ver, ptr = p._version, t.data_ptr()
    _, val = _lookup(_f32, p, ver, ptr)
    if val is not None:
        return val
    out = t.float().contiguous()
    _f32[id(p)] = (ver, ptr, out, _ref(_f32, p))
    return out


def invalidate(params):
    """Force the bf16 shadows of `params` to be re-derived on next use (what an optimizer step implies);
    the shadow buffers themselves are kept and overwritten in place."""
    for p in params:
        hit = _shadow.get(id(p))
        if hit is not None:
            _shadow[id(p)] = (-1, hit[1], hit[2], hit[3])


# (id, data_ptr, shadow ptr) of every member -> (device table, total blocks): the table of one refresh() call
_tables = {}


def refresh(params):
    """Re-derive the bf16 shadows of all fp32 `params` in ONE multi-tensor launch (what `invalidate` + lazy
    `bf16_of` do in one launch per weight).  The pointer table is built on first use — outside any CUDA-graph
    capture — and reused while the parameters and their shadow buffers stay where they are."""
    todo = []
    for p in params:
        t = p.detach()
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or t.data_ptr() % 16:
            continue                                    # bf16_of() handles these one by one
        hit = _shadow.get(id(p))
        if hit is not None and hit[3]() is not p:
            hit = None
        out = hit[2] if (hit is not None and hit[2].shape == t.shape and hit[2].device == t.device) else \
            torch.empty(t.shape, device=t.device, dtype=torch.bfloat16)
        todo.append((p, t, out))
    if not todo:
        return
    key = tuple((id(p), t.data_ptr(), out.data_ptr()) for p, t, out in todo)
    ent = _tables.get(key)
    if ent is None:
        rows, blk = [], 0
        for p, t, out in todo:
            rows.append([t.data_ptr(), out.data_ptr(), t.numel(), blk])
            blk += (t.numel() + F.CAST_MULTI_BLOCK - 1) // F.CAST_MULTI_BLOCK
        if len(_tables) > 8:
            _tables.clear()
        ent = (torch.tensor(rows, dtype=torch.int64, device=todo[0][1].device), blk)
        _tables[key] = ent
    F.cast_bf16_multi(ent[0], len(todo), ent[1])
    for p, t, out in todo:
        hit = _shadow.get(id(p))
        ref = hit[3] if (hit is not None and hit[3]() is p) else _ref(_shadow, p)
        _shadow[id(p)] = (p._version, t.data_ptr(), out, ref)


def install_optimizer_hook(optimizer, params=None):
    """Re-derive the bf16 compute copies after every `optimizer.step()`.

    The caches above are keyed on `(data_ptr, _version)`.  In-place updates through the public API bump `_version`
    (torch optimizers, `load_state_dict`), but updates made through `.data` do not — `p.data.copy_()`, DeepSpeed's fp32
    flat-partition updates (ZeRO 1/2, which the reference's accelerate configs use), EMA swaps — and the kernels would
    keep computing with stale bf16 weights.  This registers a step post-hook that invalidates the shadows of `params`
    (default: every parameter of the optimizer's groups); returns the hook handle."""
    if params is None:
        params = [p for g in optimizer.param_groups for p in g["params"]]
    params = list(params)

    def _hook(opt, args, kwargs):
        invalidate(params)
        _f32.clear()

    return optimizer.register_step_post_hook(_hook)


def clear_caches():
    _shadow.clear()
    _f32.clear()
    _tables.clear()


class GradSink:
    """Resolves where a parameter's gradient is written during backward."""

    def __init__(self):
        self.returned = {}

    def target(self, p):
        """-> (fp32 tensor to write, accumulate flag)."""
        buf = getattr(p, "_otb_grad", None)
        if buf is not None:
            acc = bool(getattr(p, "_otb_grad_live", False)) and bool(getattr(p, "_otb_sink_user", False))
            if acc and buf.dtype != torch.float32:
                raise RuntimeError("a wire-format (bf16) gradient sink takes one write per step: gradient accumulation "
                                   "over several backward passes needs FlatGradBuffer without direct_params")
            p._otb_grad_live = True
            p._otb_sink_user = True
            return buf, acc
        if id(p) in self.returned:          # second contribution within the same backward
            return self.returned[id(p)], True
        t = torch.empty(p.shape, device=p.device, dtype=torch.float32)
        self.returned[id(p)] = t
        return t, False

    def target_f32(self, p):
        """target() for a gradient a row-wise kernel writes (norm weights, biases): those need an fp32 sink."""
        g, acc = self.target(p)
        if g.dtype != torch.float32:
            raise RuntimeError("only weights produced by one wgrad GEMM can take a bf16 gradient sink (FlatGradBuffer "
                               "direct_params); norm weights and biases need an fp32 one")
        return g, acc

    def result(self, p):
        """What backward() returns to autograd for this parameter."""
        t = self.returned.get(id(p))
        if t is None:
            return None
        return t if p.dtype == torch.float32 else t.to(p.dtype)


def trainable_params(module):
    """The module's parameters, as extra inputs of its autograd Function, when grad mode is on and any of them requires
    grad (autograd then asks the Function for their gradients); () otherwise, which keeps the frozen path's inputs."""
    ps = tuple(module.parameters())
    return ps if torch.is_grad_enabled() and any(p.requires_grad for p in ps) else ()


def linear_param_grads(sink, lin, dout, inp):
    """Gradients of an nn.Linear's weight (wgrad GEMM) and bias (column sum), for those that require grad."""
    if lin.weight.requires_grad:
        g, acc = sink.target(lin.weight)
        F.linear_wgrad(dout, inp, out=g, accumulate=acc)
    if lin.bias is not None and lin.bias.requires_grad:
        g, acc = sink.target_f32(lin.bias)
        F.grouped_colsum(dout, 1, 1, out=g.view(1, -1), accumulate=acc)
