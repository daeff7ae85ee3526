"""fp32-grade path ("parity mode"): reproduces the reference's fp32 forward within the north star's 1e-3 rel / 1e-5 abs
on the CUDA path itself, and — for the trainable perceiver / gated cross-attention blocks — its fp32 autograd gradients
within 1e-3 as well.  Selected with `with otter_b200.precision("fp32"):`.

Dense contractions run on the wgmma GEMM (three-term bf16 split, six cross products over a 6x longer reduction —
functional.linear_f32; dgrad and wgrad go through the same routine on transposed operands); LayerNorm, softmax/attention,
activation derivative, gate and row-bias gradients are fp32 CUDA-core kernels (csrc/otb_fp32.cu, csrc/otb_fp32_bwd.cu).
Pure data movement (drop CLS, concat CLS token, im2col, transposes, broadcast of the latents) is torch indexing; autograd's
own fan-in accumulation (a tensor consumed by two branches) is a torch add.  The CLIP tower is frozen: forward only.
Production numerics (bf16 operands, otter_b200.blocks) are untouched; this mode is never timed.
"""
import contextlib
import weakref

import torch

from . import functional as F
from .params import f32_of

_state = {"fp32": False}


@contextlib.contextmanager
def precision(mode):
    assert mode in ("bf16", "fp32")
    old = _state["fp32"]
    _state["fp32"] = (mode == "fp32")
    try:
        yield
    finally:
        _state["fp32"] = old


def is_fp32():
    return _state["fp32"]


def require_no_grad(*tensors):
    """The CLIP tower has no backward in either mode (frozen on the hot path, modeling_otter.py:851-858)."""
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise RuntimeError("otter_b200 precision('fp32'): the CLIP tower is forward-only (frozen); "
                           "call it under torch.no_grad() or freeze its parameters")


def _needs_grad(*tensors):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


_w6 = {}


def w6_of(p, pad_to=None, transpose=False):
    """Cached split3_concat(W, pattern B) of a weight [N, K] (optionally zero-padded along K); transpose=True splits
    W^T [K, N] instead — the B operand of dgrad."""
    key = (id(p), pad_to, transpose)
    hit = _w6.get(key)
    if hit is not None and hit[0]() is p and hit[1] == p._version and hit[2] == p.data_ptr():
        return hit[3]
    w = f32_of(p).reshape(p.shape[0], -1)
    if transpose:
        w = w.t()
    if pad_to is not None and w.shape[1] < pad_to:
        w = torch.nn.functional.pad(w, (0, pad_to - w.shape[1]))
    out = F.split3_concat(w.contiguous(), 1)

    def _drop(r, key=key):
        hit = _w6.get(key)
        if hit is not None and hit[0] is r:
            del _w6[key]

    _w6[key] = (weakref.ref(p, _drop), p._version, p.data_ptr(), out)
    return out


def _wgrad(dy, x):
    """dW [N, K] = dy^T x, tokens as the reduction dimension (zero-padded to a multiple of 8; transposes = data movement)."""
    M, N = dy.shape
    K = x.shape[1]
    Mp = (M + 7) // 8 * 8
    dyT = dy.new_zeros((N, Mp))
    dyT[:, :M] = dy.t()
    xT = x.new_zeros((K, Mp))
    xT[:, :M] = x.t()
    return F.linear_f32(dyT, F.split3_concat(xT, 1), K)


class _LinFn(torch.autograd.Function):
    """y = act(x W^T + bias) * tanh(gate) + residual, every option optional (reference: nn.Linear + GELU + gate + skip)."""

    @staticmethod
    def forward(ctx, x, weight, bias, gate, residual, act):
        N = weight.shape[0]
        g32 = f32_of(gate) if gate is not None else None
        pre = F.linear_f32(x, w6_of(weight), N, bias=bias)
        f = F.epilogue_f32(pre, act=act) if act else pre
        out = F.epilogue_f32(f, scale_ptr=g32, scale_tanh=True, residual=residual) if (gate is not None or residual is not None) else f
        ctx.act, ctx.weight, ctx.gate, ctx.has_bias = act, weight, gate, bias is not None
        ctx.save_for_backward(x, pre if act else None, f if gate is not None else None)
        return out

    @staticmethod
    def backward(ctx, dy):
        x, pre, f = ctx.saved_tensors
        weight, gate = ctx.weight, ctx.gate
        need = ctx.needs_input_grad
        if ctx.has_bias and need[2]:
            raise NotImplementedError("fp32-grade backward: bias gradients are not implemented (only the frozen CLIP has biases)")
        dy = dy.contiguous()
        d_res = dy if need[4] else None
        d_gate = None
        df = dy
        if gate is not None:
            g32 = f32_of(gate)
            if need[3]:
                d_gate = F.gate_grad_f32(dy, f, g32).view(gate.shape).to(gate.dtype)
            df = F.epilogue_f32(dy, scale_ptr=g32, scale_tanh=True)
        dpre = F.act_bwd_f32(df, pre, ctx.act) if ctx.act else df
        dx = F.linear_f32(dpre, w6_of(weight, transpose=True), weight.shape[1]) if need[0] else None
        dw = _wgrad(dpre, x).to(weight.dtype) if need[1] else None
        return dx, dw, None, d_gate, d_res, None


def lin(x, weight, *, bias=None, act=0, gate=None, residual=None):
    if _needs_grad(x, weight, bias, gate, residual):
        return _LinFn.apply(x, weight, bias, gate, residual, act)
    return F.linear_f32(x, w6_of(weight), weight.shape[0], bias=bias, act=act,
                        scale_ptr=f32_of(gate) if gate is not None else None, scale_tanh=gate is not None, residual=residual)


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        ctx.eps, ctx.gamma = eps, gamma
        ctx.save_for_backward(x)
        return F.layernorm_fwd_f32(x, f32_of(gamma), f32_of(beta), eps)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx, dg, db = F.layernorm_bwd_f32(dy.contiguous(), x, f32_of(ctx.gamma), ctx.eps, need_dx=need[0],
                                         need_params=need[1] or need[2])
        dt = ctx.gamma.dtype
        return dx, (dg.to(dt) if need[1] else None), (db.to(dt) if need[2] else None), None


def layer_norm(x, ln_weight, ln_bias, eps=1e-5):
    if _needs_grad(x, ln_weight, ln_bias):
        return _LayerNormFn.apply(x, ln_weight, ln_bias, eps)
    return F.layernorm_fwd_f32(x, f32_of(ln_weight), f32_of(ln_bias), eps)


def _attn_spec(q, kv1, kv2, tt, P, H, Sq, Sk1, Sk2, n_per_media, T_img, mask_ge):
    inner = H * 64
    return F.AttnSpec(q, 0, kv1, 0, inner, P, H, Sq, Sk1, 0.125, kv2=kv2, k2_col0=0, v2_col0=inner, Sk2=Sk2, text_time=tt,
                      n_per_media=n_per_media, T_img=T_img, dtype=torch.float32, mask_ge=mask_ge)


class _AttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, kv1, kv2, tt, dims):
        out = F.attn_fwd_f32(_attn_spec(q, kv1, kv2, tt, *dims))
        ctx.dims, ctx.tt = dims, tt
        ctx.save_for_backward(q, kv1, kv2, out)
        return out

    @staticmethod
    def backward(ctx, dout):
        q, kv1, kv2, out = ctx.saved_tensors
        dq, dkv1, dkv2 = F.attn_bwd_f32(_attn_spec(q, kv1, kv2, ctx.tt, *ctx.dims), out, dout.contiguous())
        return dq, dkv1, dkv2, None, None


def attention(q, kv1, kv2, tt, *dims):
    """dims = (P, H, Sq, Sk1, Sk2, n_per_media, T_img, mask_ge); K at column 0, V at column H*64 of each key source."""
    if _needs_grad(q, kv1, kv2):
        return _AttnFn.apply(q, kv1, kv2, tt, dims)
    return F.attn_fwd_f32(_attn_spec(q, kv1, kv2, tt, *dims))


class _RowBiasFn(torch.autograd.Function):
    """x[r] + table[(r // div) % mod]  (frame / media-time embeddings, modeling_otter.py:224-229)."""

    @staticmethod
    def forward(ctx, x, table, div, mod):
        ctx.div, ctx.mod, ctx.table = div, mod, table
        return F.add_rowbias_f32(x, f32_of(table).reshape(-1, x.shape[1])[:mod].contiguous(), div, mod)

    @staticmethod
    def backward(ctx, dy):
        t = ctx.table
        dt = None
        if ctx.needs_input_grad[1]:
            dt = F.rowbias_grad_f32(dy.contiguous(), ctx.div, ctx.mod, t.numel() // dy.shape[1]).view(t.shape).to(t.dtype)
        return dy, dt, None, None


def add_rowbias(x, table, div, mod):
    if _needs_grad(x, table):
        return _RowBiasFn.apply(x, table, div, mod)
    return F.add_rowbias_f32(x, f32_of(table).reshape(-1, x.shape[1])[:mod].contiguous(), div, mod)


class _BroadcastLatentsFn(torch.autograd.Function):
    """latents [n, D] -> [BT * n, D] (modeling_otter.py:232); the gradient sums over the BT copies."""

    @staticmethod
    def forward(ctx, latents, BT):
        n, D = latents.shape
        ctx.n, ctx.dtype = n, latents.dtype
        return f32_of(latents).unsqueeze(0).expand(BT, n, D).reshape(BT * n, D).contiguous()

    @staticmethod
    def backward(ctx, dy):
        return F.rowbias_grad_f32(dy.contiguous(), 1, ctx.n, ctx.n).to(ctx.dtype), None


def _f32_2d(t, cols):
    t = t.reshape(-1, cols)
    return t.float().contiguous() if (t.dtype != torch.float32 or not t.is_contiguous()) else t


def perceiver_block(blk, x2d, lat2d, BT):
    n1, n2 = x2d.shape[0] // BT, lat2d.shape[0] // BT
    ff = blk.feed_forward
    xn = layer_norm(x2d, blk.norm_media.weight, blk.norm_media.bias)
    ln = layer_norm(lat2d, blk.norm_latents.weight, blk.norm_latents.bias)
    q = lin(ln, blk.to_q.weight)
    kv_x, kv_l = lin(xn, blk.to_kv.weight), lin(ln, blk.to_kv.weight)
    o = attention(q, kv_x, kv_l, None, BT, blk.heads, n2, n1, n2, 0, 0, False)
    lat1 = lin(o, blk.to_out.weight, residual=lat2d)
    h = layer_norm(lat1, ff[0].weight, ff[0].bias)
    h = lin(h, ff[1].weight, act=1)
    return lin(h, ff[3].weight, residual=lat1)


def resample_media(rs, media2d, BT):
    lat = _BroadcastLatentsFn.apply(rs.latents, BT)
    for blk in rs.layers:
        lat = perceiver_block(blk, media2d, lat, BT)
    return layer_norm(lat, rs.norm.weight, rs.norm.bias, rs.norm.eps)


def resampler_forward(rs, x):
    b, T, Fr, v, D = x.shape
    media = _f32_2d(x, D)
    if rs.frame_embs is not None:
        media = add_rowbias(media, rs.frame_embs, v, Fr)
    if rs.media_time_embs is not None:
        media = add_rowbias(media, rs.media_time_embs, Fr * v, T)
    return resample_media(rs, media, b * T).view(b, T, rs.latents.shape[0], D)


def masked_cross_attention(att, x2d, media2d, tt, B, L, T_img, n, gate=None, residual=None):
    xn = layer_norm(x2d, att.norm.weight, att.norm.bias)
    q = lin(xn, att.to_q.weight)
    kv = lin(media2d, att.to_kv.weight)
    o = attention(q, kv, None, tt, B, att.heads, L, T_img * n, 0, n, T_img, not att.only_attend_immediate_media)
    return lin(o, att.to_out.weight, gate=gate, residual=residual)


def gated_block(gb, x2d, media2d, tt, B, L, T_img, n):
    ff = gb.feed_forward
    x1 = masked_cross_attention(gb.attn, x2d, media2d, tt, B, L, T_img, n, gate=gb.attn_gate, residual=x2d)
    h = layer_norm(x1, ff[0].weight, ff[0].bias)
    h = lin(h, ff[1].weight, act=1)
    return lin(h, ff[3].weight, gate=gb.ff_gate, residual=x1)


def clip_last_hidden(clip, pixel_values):
    cfg, vm = clip.config, clip.vision_model
    D, P, heads, eps = cfg.hidden_size, cfg.patch_size, cfg.num_attention_heads, cfg.layer_norm_eps
    N = pixel_values.shape[0]
    cols = torch.nn.functional.unfold(pixel_values.float(), P, stride=P).transpose(1, 2)      # data movement only
    np_ = cols.shape[1]
    K = cols.shape[2]
    Kp = (K + 7) // 8 * 8
    cols = torch.nn.functional.pad(cols.reshape(N * np_, K), (0, Kp - K)).contiguous()
    pe = F.linear_f32(cols, w6_of(vm.embeddings.patch_embedding.weight, pad_to=Kp), D)
    cls = f32_of(vm.embeddings.class_embedding).reshape(1, 1, D).expand(N, 1, D)
    h = torch.cat([cls, pe.view(N, np_, D)], dim=1).reshape(N * (np_ + 1), D).contiguous()   # data movement only
    S = np_ + 1
    h = F.add_rowbias_f32(h, f32_of(vm.embeddings.position_embedding.weight), 1, S)
    h = F.layernorm_fwd_f32(h, f32_of(vm.pre_layrnorm.weight), f32_of(vm.pre_layrnorm.bias), eps)
    for l in vm.encoder.layers:
        a = l.self_attn
        x = F.layernorm_fwd_f32(h, f32_of(l.layer_norm1.weight), f32_of(l.layer_norm1.bias), eps)
        q = lin(x, a.q_proj.weight, bias=f32_of(a.q_proj.bias))
        k = lin(x, a.k_proj.weight, bias=f32_of(a.k_proj.bias))
        v = lin(x, a.v_proj.weight, bias=f32_of(a.v_proj.bias))
        kv = torch.cat([k, v], dim=1)                                                         # data movement only
        o = F.attn_fwd_f32(F.AttnSpec(q, 0, kv, 0, D, N, heads, S, S, 0.125, dtype=torch.float32))
        h = lin(o, a.out_proj.weight, bias=f32_of(a.out_proj.bias), residual=h)
        x = F.layernorm_fwd_f32(h, f32_of(l.layer_norm2.weight), f32_of(l.layer_norm2.bias), eps)
        x = lin(x, l.mlp.fc1.weight, bias=f32_of(l.mlp.fc1.bias), act=2)
        h = lin(x, l.mlp.fc2.weight, bias=f32_of(l.mlp.fc2.bias), residual=h)
    return h.view(N, S, D)
