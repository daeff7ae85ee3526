"""LLaMA decoder layer on the otter_b200 kernels — SURVEY.md §8f rank 1 (the LM of OTTER-Video-LLaMA7B, config c3).

Mirrors `LlamaDecoderLayer` (/root/reference/xformers_model/llama.py:262-320; the reference falls back to HF's identical
`transformers.models.llama` classes when xformers is absent, modeling_otter.py:52-54): same sub-module and parameter names
(`input_layernorm`, `self_attn.{q,k,v,o}_proj`, `post_attention_layernorm`, `mlp.{gate,up,down}_proj`), no biases.
Otter freezes the LM by default (modeling_otter.py:897-905), and so do the constructor and swap_llama_layers: backward
then produces the input gradient only.  Parameters set to `requires_grad` afterwards (`train_lang_encoder`,
`train_full_model`, partial unfreezing) also receive their gradients: the seven wgrad GEMMs and the RMSNorm weight
gradients (otb_rmsnorm_bwd_params), written through `params.GradSink`.

  RMSNorm -> q / k / v GEMMs into one [rows, (H + 2 kv) * 128] buffer -> rotary embedding in place (rotate_half,
     head dim 128) -> causal attention (otb_lm_attn_*, no key bias) -> o_proj GEMM (+residual)
     -> RMSNorm -> gate / up GEMMs -> silu(g) * u -> down GEMM (+residual)
head_dim must be 128 (LLaMA-7B: 4096 = 32 x 128); training path (no KV cache); default position ids.
Grouped-query attention (kv < H K/V heads: Llama-2-70B, Llama-3) and the linear / llama3 / yarn RoPE scalings are
covered too: the RoPE table (inverse frequencies and yarn's cos / sin factor) comes from HF's own LlamaRotaryEmbedding,
so none of the scaling formulas is restated here.  `dynamic` and `longrope` depend on the sequence length at run time
and are not covered.
`swap_llama_layers(model)` replaces the decoder layers of an HF `LlamaForCausalLM` by this class, sharing the Parameter
objects.  Attention masks: the kernel applies the causal mask only, which equals HF's causal + padding mask at every
non-pad position when padding is on the RIGHT (the training collate, SURVEY.md §8f-2); a forward pre-hook on the LlamaModel
checks the 2-D mask once per forward and raises on left padding.  Incremental decoding with a KV cache (generation — out of
the hot path, SURVEY.md §8 "out of scope") is handed to the original HF layer, which is what the reference itself runs.
"""
import math

import torch
from torch import nn

from . import functional as F
from . import lora as L
from . import params as P

BF16 = torch.bfloat16


class _FrozenLlamaLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, layer, B, S, *params):   # params: layer.parameters() when any of them trains, else empty
        a, m = layer.self_attn, layer.mlp
        D, H = layer.hidden_size, layer.num_heads
        Dkv = layer.num_key_value_heads * 128
        x2 = x.reshape(B * S, D)
        w_in, w_post = P.f32_of(layer.input_layernorm.weight), P.f32_of(layer.post_attention_layernorm.weight)
        h1, r1 = F.rmsnorm_fwd(x2, w_in, layer.eps)                                        # llama.py:296
        qkv = torch.empty((B * S, D + 2 * Dkv), device=x.device, dtype=BF16)
        lq, lv = L.adapter(a.q_proj), L.adapter(a.v_proj)          # LoRA on q / v (otter_b200.lora), else None
        seed = L.layer_seed(x.device, lq, lv)
        xas = []                                                   # xa = dropout(h1) A^T of each adapter
        if lq is None:
            F.linear_fwd(h1, P.bf16_of(a.q_proj.weight), out=qkv[:, :D])                   # :222-224
        else:
            xas.append(L.kernel_fwd(h1, P.bf16_of(a.q_proj.weight), lq, qkv[:, :D], seed, 0))
        F.linear_fwd(h1, P.bf16_of(a.k_proj.weight), out=qkv[:, D:D + Dkv])
        if lv is None:
            F.linear_fwd(h1, P.bf16_of(a.v_proj.weight), out=qkv[:, D + Dkv:])
        else:
            xas.append(L.kernel_fwd(h1, P.bf16_of(a.v_proj.weight), lv, qkv[:, D + Dkv:], seed, 1))
        _rope(layer, qkv, S, False)                                                        # :229-230
        o, lse = F.lm_attn_fwd(qkv, B, S, H, slopes=None, causal=True, scale=1.0 / math.sqrt(128),
                               **_kv_kw(layer))                                             # :241-246
        x1 = F.linear_fwd(o, P.bf16_of(a.o_proj.weight), residual=x2)                      # :254,304
        h2, r2 = F.rmsnorm_fwd(x1, w_post, layer.eps)                                      # :308
        g = F.linear_fwd(h2, P.bf16_of(m.gate_proj.weight))
        u = F.linear_fwd(h2, P.bf16_of(m.up_proj.weight))
        hh = F.swiglu_fwd(g, u)                                                            # :184
        y = F.linear_fwd(hh, P.bf16_of(m.down_proj.weight), residual=x1)                   # :309-310
        ctx.layer, ctx.B, ctx.S, ctx.params = layer, B, S, params
        ctx.lora = (lq, lv, seed)
        # the weight GEMMs' other operands (the RMSNorm outputs and the SwiGLU output, the bits the forward GEMMs read)
        # are kept only for the weights that train: a layer that trains only its LoRA adapters keeps h1 alone
        keep = (h1 if L.needs_input(a.q_proj, a.k_proj, a.v_proj) else None,
                h2 if L.needs_input(m.gate_proj, m.up_proj) else None, hh if L.needs_input(m.down_proj) else None)
        ctx.save_for_backward(x2, r1, qkv, o, lse, x1, r2, g, u, *(keep if params else ()), *xas)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        layer, B, S = ctx.layer, ctx.B, ctx.S
        x2, r1, qkv, o, lse, x1, r2, g, u = ctx.saved_tensors[:9]
        a, m = layer.self_attn, layer.mlp
        D, H = layer.hidden_size, layer.num_heads
        dy2 = dy.reshape(B * S, D)
        if dy2.dtype != BF16 or not dy2.is_contiguous():
            dy2 = dy2.to(BF16).contiguous()
        train = bool(ctx.params)
        h1, h2, hh = ctx.saved_tensors[9:12] if train else (None, None, None)
        xas = list(ctx.saved_tensors[12 if train else 9:])
        sink = P.GradSink() if train else None

        def wgrad(lin, dout, inp):
            if train:
                P.linear_param_grads(sink, lin, dout, inp)

        def rms_kw(norm):
            """No extra arguments for a frozen norm weight: the frozen path's call, unchanged."""
            if not (train and norm.weight.requires_grad):
                return {}
            gw, acc = sink.target_f32(norm.weight)
            return {"dweight": gw, "accumulate": acc}

        dh = F.linear_dgrad(dy2, P.bf16_of(m.down_proj.weight))
        wgrad(m.down_proj, dy2, hh)
        dg, du = F.swiglu_bwd(dh, g, u)
        dh2 = F.linear_dgrad(dg, P.bf16_of(m.gate_proj.weight))
        dh2 = F.linear_dgrad(du, P.bf16_of(m.up_proj.weight), residual=dh2)
        wgrad(m.gate_proj, dg, h2)
        wgrad(m.up_proj, du, h2)
        dx1 = F.rmsnorm_bwd(dh2, x1, r2, P.f32_of(layer.post_attention_layernorm.weight), add=dy2,
                            **rms_kw(layer.post_attention_layernorm))
        do = F.linear_dgrad(dx1, P.bf16_of(a.o_proj.weight))
        wgrad(a.o_proj, dx1, o)
        dqkv = F.lm_attn_bwd(do, qkv, o, lse, B, S, H, slopes=None, causal=True, scale=1.0 / math.sqrt(128),
                             **_kv_kw(layer))
        _rope(layer, dqkv, S, True)
        Dkv = layer.num_key_value_heads * 128
        dh1 = F.linear_dgrad(dqkv[:, :D], P.bf16_of(a.q_proj.weight))
        dh1 = F.linear_dgrad(dqkv[:, D:D + Dkv], P.bf16_of(a.k_proj.weight), residual=dh1)
        dh1 = F.linear_dgrad(dqkv[:, D + Dkv:], P.bf16_of(a.v_proj.weight), residual=dh1)
        lq, lv, seed = ctx.lora
        if lq is not None:                                        # LoRA: the adapters' share of dh1, A / B gradients
            dh1 = L.kernel_bwd(sink, dqkv[:, :D], h1, xas.pop(0), lq, seed, 0, dh1)
        if lv is not None:
            dh1 = L.kernel_bwd(sink, dqkv[:, D + Dkv:], h1, xas.pop(0), lv, seed, 1, dh1)
        wgrad(a.q_proj, dqkv[:, :D], h1)                          # gradients after the inverse RoPE, as the dgrad
        wgrad(a.k_proj, dqkv[:, D:D + Dkv], h1)
        wgrad(a.v_proj, dqkv[:, D + Dkv:], h1)
        dx = F.rmsnorm_bwd(dh1, x2, r1, P.f32_of(layer.input_layernorm.weight), add=dx1, **rms_kw(layer.input_layernorm))
        if train:
            return (dx.view(dy.shape), None, None, None) + tuple(sink.result(p) for p in ctx.params)
        return dx.view(dy.shape), None, None, None


def _kv_kw(layer):
    """Extra attention arguments: none for multi-head attention, so that path makes exactly the calls it always made."""
    kv = layer.num_key_value_heads
    return {} if kv == layer.num_heads else {"kv_heads": kv}


def _rope(layer, buf, S, backward):
    """Rotary embedding in place on the q and k blocks of the fused projection buffer (or of its gradient)."""
    H, kv = layer.num_heads, layer.num_key_value_heads
    if not layer.table_rope:                                   # multi-head attention, default RoPE: theta in the kernel
        if backward:
            F.rope128_(buf, H, S, 2, layer.rope_theta, backward=True)
        else:
            F.rope128_(buf, H, S, 2, layer.rope_theta)
        return
    inv, sc = layer.rope_inv_freq(buf.device), layer.rope_attention_scaling
    if kv == H:
        F.rope128_freqs_(buf, H, S, 2, inv, sc, backward=backward)
    else:                                                      # q block (H heads), then k block (kv heads)
        F.rope128_freqs_(buf[:, :H * 128], H, S, 1, inv, sc, backward=backward)
        F.rope128_freqs_(buf[:, H * 128:(H + kv) * 128], kv, S, 1, inv, sc, backward=backward)


def rope_table(hidden_size, num_attention_heads, rope_parameters, max_position_embeddings=None):
    """(inv_freq fp32 [64] on the CPU, attention_scaling) of HF's LlamaRotaryEmbedding for these RoPE parameters."""
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
    kw = {} if max_position_embeddings is None else {"max_position_embeddings": max_position_embeddings}
    cfg = LlamaConfig(hidden_size=hidden_size, num_attention_heads=num_attention_heads, rope_parameters=dict(rope_parameters),
                      **kw)
    rot = LlamaRotaryEmbedding(cfg, device="cpu")
    return rot.inv_freq.detach().float().clone(), float(rot.attention_scaling)


class _RMSNormParams(nn.Module):
    def __init__(self, d, eps):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d))
        self.variance_epsilon = eps


class _Attn(nn.Module):
    def __init__(self, d, d_kv):
        super().__init__()
        self.q_proj, self.k_proj = nn.Linear(d, d, bias=False), nn.Linear(d, d_kv, bias=False)
        self.v_proj, self.o_proj = nn.Linear(d, d_kv, bias=False), nn.Linear(d, d, bias=False)


class _MLP(nn.Module):
    def __init__(self, d, i):
        super().__init__()
        self.gate_proj, self.up_proj = nn.Linear(d, i, bias=False), nn.Linear(d, i, bias=False)
        self.down_proj = nn.Linear(i, d, bias=False)


class FrozenLlamaDecoderLayer(nn.Module):
    """Drop-in for HF's `LlamaDecoderLayer`, constructed frozen; parameters set to `requires_grad` afterwards receive their
    gradients too.  (The name is kept: checkpoints and isinstance checks use it.)
    num_key_value_heads: K/V heads (grouped-query attention; default: num_attention_heads).  rope_parameters: HF's
    `config.rope_parameters` dict (rope_type default / linear / llama3 / yarn; default: {"rope_type": "default",
    "rope_theta": rope_theta}); max_position_embeddings is passed to HF's RoPE initialisation (yarn may read it)."""

    def __init__(self, hidden_size, num_attention_heads, intermediate_size, rms_norm_eps=1e-6, rope_theta=10000.0, *,
                 num_key_value_heads=None, rope_parameters=None, max_position_embeddings=None):
        super().__init__()
        if hidden_size != num_attention_heads * 128:
            raise ValueError("FrozenLlamaDecoderLayer: head_dim must be 128 (LLaMA-7B: 4096 = 32 x 128)")
        kv = num_attention_heads if num_key_value_heads is None else int(num_key_value_heads)
        if kv <= 0 or num_attention_heads % kv != 0:
            raise ValueError(f"FrozenLlamaDecoderLayer: num_key_value_heads = {kv} must divide {num_attention_heads} heads")
        rp = dict(rope_parameters) if rope_parameters else {"rope_type": "default", "rope_theta": rope_theta}
        rope_type = rp.get("rope_type", "default")
        if rope_type not in _TABLE_ROPE_TYPES:
            raise ValueError(f"FrozenLlamaDecoderLayer: rope_type {rope_type!r} is not covered (one of {_TABLE_ROPE_TYPES})")
        rope_theta = rp.get("rope_theta", rope_theta)
        self.hidden_size, self.num_heads, self.eps, self.rope_theta = hidden_size, num_attention_heads, rms_norm_eps, rope_theta
        self.num_key_value_heads, self.rope_type = kv, rope_type
        # multi-head attention with default RoPE keeps the theta-driven kernel; everything else uses HF's table
        self.table_rope = not (kv == num_attention_heads and rope_type == "default")
        self.rope_attention_scaling = 1.0
        self._rope_freqs = {}                       # device -> fp32 [64] (plain attribute: module dtype casts leave it fp32)
        if self.table_rope:
            inv, self.rope_attention_scaling = rope_table(hidden_size, num_attention_heads, rp, max_position_embeddings)
            self._rope_freqs[torch.device("cpu")] = inv
        self.self_attn = _Attn(hidden_size, kv * 128)
        self.mlp = _MLP(hidden_size, intermediate_size)
        self.input_layernorm = _RMSNormParams(hidden_size, rms_norm_eps)
        self.post_attention_layernorm = _RMSNormParams(hidden_size, rms_norm_eps)
        self.requires_grad_(False)

    def rope_inv_freq(self, device):
        """The fp32 [64] inverse-frequency table on `device` (copied there once)."""
        t = self._rope_freqs.get(device)
        if t is None:
            t = self._rope_freqs[device] = self._rope_freqs[torch.device("cpu")].to(device)
        return t

    def forward(self, hidden_states, attention_mask=None, position_ids=None, past_key_value=None, past_key_values=None,
                output_attentions=False, use_cache=False, **kwargs):
        if past_key_value is not None or past_key_values is not None:
            hf = self.__dict__.get("_hf_layer")
            if hf is None:
                raise NotImplementedError("FrozenLlamaDecoderLayer: training path only (no KV cache)")
            kw = dict(kwargs, attention_mask=attention_mask, position_ids=position_ids, use_cache=use_cache)
            kw["past_key_values" if past_key_values is not None else "past_key_value"] = \
                past_key_values if past_key_values is not None else past_key_value
            return hf(hidden_states, **kw)
        if output_attentions:
            raise NotImplementedError("output_attentions is not available from the fused attention kernel")
        B, S, _ = hidden_states.shape
        if position_ids is not None:
            want = torch.arange(S, device=position_ids.device)
            if position_ids.shape[-1] != S or not bool((position_ids.reshape(-1, S) == want).all()):
                raise NotImplementedError("only the default position_ids (arange) are supported")
        xb = hidden_states if hidden_states.dtype == BF16 else hidden_states.to(BF16)
        y = _FrozenLlamaLayerFn.apply(xb.contiguous(), self, B, S, *P.trainable_params(self))
        return y.to(hidden_states.dtype)          # HF 5.x decoder layers return the tensor (SURVEY.md §8a-7)


def _share_parameters(new, old):
    for name, _ in list(new.named_parameters()):
        mod_path, _, leaf = name.rpartition(".")
        src, dst = old.get_submodule(mod_path), new.get_submodule(mod_path)
        p = getattr(src, leaf)
        if tuple(p.shape) != tuple(getattr(dst, leaf).shape):
            raise ValueError(f"{name}: shape {tuple(p.shape)} does not fit FrozenLlamaDecoderLayer")
        dst._parameters[leaf] = p          # the SAME Parameter object: .to() / optimizer / checkpoint see one tensor


def _right_padding_check(module, args, kwargs):
    mask = kwargs.get("attention_mask")
    if mask is not None and mask.dim() == 2 and mask.shape[1] > 1:
        m = mask.to(torch.bool)
        if bool((m[:, 1:] & ~m[:, :-1]).any()):
            raise NotImplementedError("FrozenLlamaDecoderLayer applies the causal mask only: attention_mask must be "
                                      "right-padded (ones then zeros per row)")
    elif mask is not None and not isinstance(mask, dict) and mask.dim() != 2:
        raise NotImplementedError("FrozenLlamaDecoderLayer: pass the 2-D padding mask, not a prepared 4-D mask")
    return None


_TABLE_ROPE_TYPES = ("default", "linear", "llama3", "yarn")


def swappable(cfg):
    """True when the HF LlamaConfig describes layers this module covers: head_dim 128, multi-head or grouped-query
    attention (num_key_value_heads divides num_attention_heads), default / linear / llama3 / yarn RoPE, no biases."""
    rp = getattr(cfg, "rope_parameters", None) or {}
    rope_type = rp.get("rope_type", "default") if isinstance(rp, dict) else "default"
    hd = getattr(cfg, "head_dim", None) or cfg.hidden_size // cfg.num_attention_heads
    kv = getattr(cfg, "num_key_value_heads", None) or cfg.num_attention_heads
    return (hd == 128 and cfg.hidden_size == cfg.num_attention_heads * 128
            and cfg.num_attention_heads % kv == 0
            and rope_type in _TABLE_ROPE_TYPES and not getattr(cfg, "attention_bias", False) and not getattr(cfg, "mlp_bias", False)
            and getattr(cfg, "hidden_act", "silu") == "silu" and cfg.hidden_size % 64 == 0 and cfg.intermediate_size % 64 == 0)


def swap_llama_layers(llama_model, keep_hf_for_cache=True):
    """Replace the decoder layers of an HF LlamaForCausalLM / LlamaModel by FrozenLlamaDecoderLayer (Parameters shared)."""
    model = llama_model.model if hasattr(llama_model, "model") else llama_model
    cfg = model.config
    if not swappable(cfg):
        raise ValueError("swap_llama_layers: this LlamaConfig is outside FrozenLlamaDecoderLayer's coverage (see swappable())")
    rp = getattr(cfg, "rope_parameters", None) or {}
    theta = rp.get("rope_theta", getattr(cfg, "rope_theta", 10000.0))
    kv = getattr(cfg, "num_key_value_heads", None) or cfg.num_attention_heads
    rope_kw = {}
    if kv != cfg.num_attention_heads or rp.get("rope_type", "default") != "default":
        rope_kw = dict(num_key_value_heads=kv, rope_parameters=rp,
                       max_position_embeddings=getattr(cfg, "max_position_embeddings", None))
    for i, old in enumerate(model.layers):
        new = FrozenLlamaDecoderLayer(cfg.hidden_size, cfg.num_attention_heads, cfg.intermediate_size, cfg.rms_norm_eps, theta,
                                      **rope_kw)
        _share_parameters(new, old)
        new.requires_grad_(False)
        if keep_hf_for_cache:
            new.__dict__["_hf_layer"] = old            # not a registered sub-module: no duplicate state-dict keys
        model.layers[i] = new
    if not getattr(model, "_otb_mask_hook", False):
        model.register_forward_pre_hook(_right_padding_check, with_kwargs=True)
        model._otb_mask_hook = True
    return llama_model
