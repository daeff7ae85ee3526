"""Frozen MPT decoder layer on the otter_b200 kernels (SURVEY.md §8f rank 1).

Mirrors `MPTBlock` (/root/reference/src/otter_ai/models/mpt/blocks.py:23-88) — same sub-module and parameter names
(`norm_1`, `attn.Wqkv`, `attn.out_proj`, `norm_2`, `ffn.up_proj`, `ffn.down_proj`), same `forward()` signature and
return tuple — for the configuration OTTER-Image-MPT7B ships: multi-head attention, `attn_impl: torch` semantics
(mpt/attention.py:22-84), ALiBi key bias, causal mask, erf-GELU MLP, dropouts 0.  The layer is FROZEN in Otter
(modeling_otter.py:905 freezes the LM): backward produces the input gradient only — five dgrad GEMMs, the causal
attention backward and two LayerNorm backwards; no wgrad, and the bf16 weight copies are cast once.

head_dim must be 128 (MPT-7B / LLaMA-7B); there is no CPU path.
"""
import math

import torch
from torch import nn

from . import functional as F
from . import params as P


def alibi_slopes(n_heads, alibi_bias_max=8, device=None):
    """mpt/attention.py:447-454 gen_slopes -> fp32 [H]."""
    n2 = 2 ** math.ceil(math.log2(n_heads))
    m = torch.arange(1, n2 + 1, dtype=torch.float32, device=device) * (alibi_bias_max / n2)
    slopes = 1.0 / torch.pow(2, m)
    if n2 != n_heads:
        slopes = torch.cat([slopes[1::2], slopes[::2]])[:n_heads]
    return slopes.contiguous()


class _FrozenMPTBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, blk, B, S):
        D, H = blk.d_model, blk.n_heads
        x2 = x.reshape(B * S, D)
        g1, b1 = P.f32_of(blk.norm_1.weight), blk._beta(blk.norm_1)
        g2, b2 = P.f32_of(blk.norm_2.weight), blk._beta(blk.norm_2)
        w_qkv, w_out = P.bf16_of(blk.attn.Wqkv.weight), P.bf16_of(blk.attn.out_proj.weight)
        w_up, w_down = P.bf16_of(blk.ffn.up_proj.weight), P.bf16_of(blk.ffn.down_proj.weight)

        a, mean1, rstd1 = F.layernorm_fwd(x2, g1, b1)
        qkv = F.linear_fwd(a, w_qkv, bias=blk._bias(blk.attn.Wqkv))
        o, lse = F.lm_attn_fwd(qkv, B, S, H, slopes=blk.slopes, causal=True, scale=blk.softmax_scale)
        x1 = F.linear_fwd(o, w_out, bias=blk._bias(blk.attn.out_proj), residual=x2)
        m, mean2, rstd2 = F.layernorm_fwd(x1, g2, b2)
        z = torch.empty((B * S, w_up.shape[0]), device=x.device, dtype=torch.bfloat16)
        h = F.linear_fwd(m, w_up, bias=blk._bias(blk.ffn.up_proj), act=1, aux_out=z)
        y = F.linear_fwd(h, w_down, bias=blk._bias(blk.ffn.down_proj), residual=x1)
        ctx.blk, ctx.B, ctx.S = blk, B, S
        ctx.save_for_backward(x2, mean1, rstd1, qkv, o, lse, x1, mean2, rstd2, z)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        blk, B, S = ctx.blk, ctx.B, ctx.S
        x2, mean1, rstd1, qkv, o, lse, x1, mean2, rstd2, z = ctx.saved_tensors
        D, H = blk.d_model, blk.n_heads
        dy2 = dy.reshape(B * S, D)
        if dy2.dtype != torch.bfloat16 or dy2.stride(-1) != 1:
            dy2 = dy2.to(torch.bfloat16).contiguous()
        g1, g2 = P.f32_of(blk.norm_1.weight), P.f32_of(blk.norm_2.weight)
        w_qkv, w_out = P.bf16_of(blk.attn.Wqkv.weight), P.bf16_of(blk.attn.out_proj.weight)
        w_up, w_down = P.bf16_of(blk.ffn.up_proj.weight), P.bf16_of(blk.ffn.down_proj.weight)

        dz = F.linear_dgrad(dy2, w_down, aux_in=z)                       # (dy W_down) * gelu'(z)
        dm = F.linear_dgrad(dz, w_up)
        dx1, _, _ = F.layernorm_bwd(dm, x1, mean2, rstd2, g2, add=dy2, want_param_grads=False)   # + residual branch
        do = F.linear_dgrad(dx1, w_out)
        dqkv = F.lm_attn_bwd(do, qkv, o, lse, B, S, H, slopes=blk.slopes, causal=True, scale=blk.softmax_scale)
        da = F.linear_dgrad(dqkv, w_qkv)
        dx, _, _ = F.layernorm_bwd(da, x2, mean1, rstd1, g1, add=dx1, want_param_grads=False)
        return dx.view(dy.shape), None, None, None


class _Attn(nn.Module):
    def __init__(self, d_model, bias):
        super().__init__()
        self.Wqkv = nn.Linear(d_model, 3 * d_model, bias=bias)
        self.out_proj = nn.Linear(d_model, d_model, bias=bias)


class _MLP(nn.Module):
    def __init__(self, d_model, expansion_ratio, bias):
        super().__init__()
        self.up_proj = nn.Linear(d_model, expansion_ratio * d_model, bias=bias)
        self.down_proj = nn.Linear(expansion_ratio * d_model, d_model, bias=bias)


class FrozenMPTBlock(nn.Module):
    """Drop-in for a frozen `MPTBlock` (state-dict keys identical); trains nothing, propagates input gradients."""

    def __init__(self, d_model, n_heads, expansion_ratio=4, no_bias=True, alibi=True, alibi_bias_max=8,
                 softmax_scale=None):
        super().__init__()
        if d_model != n_heads * 128:
            raise ValueError("FrozenMPTBlock: head_dim must be 128 (MPT-7B: 4096 = 32 x 128)")
        self.d_model, self.n_heads = d_model, n_heads
        self.norm_1 = nn.LayerNorm(d_model, eps=1e-5, bias=not no_bias)
        self.attn = _Attn(d_model, bias=not no_bias)
        self.norm_2 = nn.LayerNorm(d_model, eps=1e-5, bias=not no_bias)
        self.ffn = _MLP(d_model, expansion_ratio, bias=not no_bias)
        self.alibi, self.alibi_bias_max = alibi, alibi_bias_max
        self.softmax_scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(128)
        self.slopes = None
        self._zeros = None
        self.requires_grad_(False)

    def _beta(self, ln):
        if ln.bias is not None:
            return P.f32_of(ln.bias)
        if self._zeros is None or self._zeros.device != ln.weight.device:
            self._zeros = torch.zeros(self.d_model, device=ln.weight.device, dtype=torch.float32)
        return self._zeros

    @staticmethod
    def _bias(lin):
        return P.f32_of(lin.bias) if lin.bias is not None else None

    def forward(self, x, past_key_value=None, attn_bias=None, attention_mask=None, is_causal=True):
        if past_key_value is not None or not is_causal:
            raise NotImplementedError("FrozenMPTBlock: training path only (causal, no KV cache)")
        if attention_mask is not None:
            # Right padding needs no key mask under a causal mask (a real token never sees a later pad key, and the
            # ALiBi key bias is a per-row constant shift away from the relative form); anything else is refused.
            am = attention_mask.to(torch.bool)
            if not bool((am[:, 1:] <= am[:, :-1]).all()):
                raise NotImplementedError("FrozenMPTBlock: only right-padded batches (no interior / left padding)")
        if self.alibi and (self.slopes is None or self.slopes.device != x.device):
            self.slopes = alibi_slopes(self.n_heads, self.alibi_bias_max, device=x.device)
        B, S, _ = x.shape
        xb = x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)
        y = _FrozenMPTBlockFn.apply(xb.contiguous(), self, B, S)
        return (y, None, past_key_value)


# =================================================================================================
# MPTModel / MPTForCausalLM on the otter_b200 kernels (SURVEY.md §8f rank 1; harness mode M2)
#   reference: src/otter_ai/models/mpt/modeling_mpt.py:40-293 (MPTModel), :280-436 (MPTForCausalLM),
#              configuration_mpt.py:29-140 (MPTConfig)
# The class is NAMED MPTForCausalLM: OtterLMMixin dispatches on the class name (modeling_otter.py:500-509) and
# `_infer_decoder_layers_attr_name` maps it to `transformer.blocks`; state-dict keys equal the reference's
# (`transformer.wte.weight`, `transformer.blocks.{i}.{norm_1,attn.Wqkv,attn.out_proj,norm_2,ffn.up_proj,
# ffn.down_proj}.weight`, `transformer.norm_f.weight`), so reference checkpoints load unchanged.
# Scope: the configuration OTTER-Image-MPT7B ships (ALiBi, multi-head attention, no biases, tied embeddings,
# dropouts 0).  The decoder layers are frozen in Otter (modeling_otter.py:897-905): input gradients only.  The tied
# embedding IS trained there (:905): it receives the gather gradient (torch index op) and the un-embedding wgrad.
# No KV cache: generate() re-runs the whole prefix each step (correct, O(n^2) — the decode path is not the hot path).
# =================================================================================================
from transformers import PretrainedConfig, PreTrainedModel  # noqa: E402
from transformers.generation import GenerationMixin  # noqa: E402
from transformers.modeling_outputs import BaseModelOutputWithPast, CausalLMOutputWithPast  # noqa: E402

_ATTN_DEFAULTS = {"attn_type": "multihead_attention", "attn_pdrop": 0.0, "attn_impl": "triton", "qk_ln": False,
                  "clip_qkv": None, "softmax_scale": None, "prefix_lm": False, "attn_uses_sequence_id": False,
                  "alibi": False, "alibi_bias_max": 8}


class MPTConfig(PretrainedConfig):
    """configuration_mpt.py:29-140 (same field names and defaults; `init_config` is accepted and ignored)."""
    model_type = "mpt"

    def __init__(self, d_model=2048, n_heads=16, n_layers=24, expansion_ratio=4, max_seq_len=2048, vocab_size=50368,
                 resid_pdrop=0.0, emb_pdrop=0.0, learned_pos_emb=True, attn_config=None, init_device="cpu",
                 logit_scale=None, no_bias=False, verbose=0, embedding_fraction=1.0,
                 norm_type="low_precision_layernorm", use_cache=False, init_config=None, **kwargs):
        self.d_model, self.n_heads, self.n_layers = d_model, n_heads, n_layers
        self.expansion_ratio, self.max_seq_len, self.vocab_size = expansion_ratio, max_seq_len, vocab_size
        self.resid_pdrop, self.emb_pdrop, self.learned_pos_emb = resid_pdrop, emb_pdrop, learned_pos_emb
        self.attn_config = dict(_ATTN_DEFAULTS, **(attn_config or {}))
        self.init_device, self.logit_scale, self.no_bias, self.verbose = init_device, logit_scale, no_bias, verbose
        self.embedding_fraction, self.norm_type, self.use_cache = embedding_fraction, norm_type, use_cache
        self.init_config = init_config or {}
        kwargs.pop("name", None)
        kwargs.pop("loss_fn", None)
        kwargs.setdefault("tie_word_embeddings", True)
        super().__init__(**kwargs)
        self.hidden_size = d_model                     # read by OtterLMMixin.init_otter (modeling_otter.py:473)
        self.num_hidden_layers = n_layers
        self.num_attention_heads = n_heads


def _as_bf16(t):
    return t if t.dtype == torch.bfloat16 else t.to(torch.bfloat16)


class _FrozenLayerNormFn(torch.autograd.Function):
    """LayerNorm with frozen affine parameters: input gradient only (norm_f, modeling_mpt.py:292)."""

    @staticmethod
    def forward(ctx, x2, w, beta):
        y, mean, rstd = F.layernorm_fwd(x2, P.f32_of(w), beta)
        ctx.save_for_backward(x2, mean, rstd)
        ctx.w = w
        return y

    @staticmethod
    def backward(ctx, dy):
        x2, mean, rstd = ctx.saved_tensors
        dx, _, _ = F.layernorm_bwd(_as_bf16(dy).contiguous(), x2, mean, rstd, P.f32_of(ctx.w), want_param_grads=False)
        return dx, None, None


class _UnembedFn(torch.autograd.Function):
    """logits = h wte^T with the TIED embedding (modeling_mpt.py:418-421): dgrad to h, wgrad to wte when trainable."""

    @staticmethod
    def forward(ctx, h2, wte):
        ctx.save_for_backward(h2)
        ctx.wte = wte
        return F.linear_fwd(h2, P.bf16_of(wte))

    @staticmethod
    def backward(ctx, dlogits):
        (h2,) = ctx.saved_tensors
        wte = ctx.wte
        dl = _as_bf16(dlogits).contiguous()
        dh = F.linear_dgrad(dl, P.bf16_of(wte)) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1]:
            sink = P.GradSink()
            g, acc = sink.target(wte)
            F.linear_wgrad(dl, h2, out=g, accumulate=acc)
            dw = sink.result(wte)
        return dh, dw


class MPTModel(nn.Module):
    """modeling_mpt.py:40-293 — wte -> n_layers x MPTBlock -> norm_f."""

    def __init__(self, config):
        super().__init__()
        ac = config.attn_config
        if not ac["alibi"] or ac["attn_type"] != "multihead_attention" or ac["prefix_lm"] or ac["qk_ln"] \
                or ac["clip_qkv"] or ac["attn_uses_sequence_id"]:
            raise NotImplementedError("otter_b200 MPT: the OTTER-Image-MPT7B configuration only (ALiBi multi-head "
                                      "attention, no prefix-LM / qk_ln / clip_qkv / sequence ids)")
        if config.emb_pdrop or config.resid_pdrop or ac["attn_pdrop"]:
            raise NotImplementedError("otter_b200 MPT: dropout probabilities must be 0 (as shipped)")
        self.config = config
        self.embedding_fraction = config.embedding_fraction
        self.wte = nn.Embedding(config.vocab_size, config.d_model)
        self.blocks = nn.ModuleList([
            FrozenMPTBlock(config.d_model, config.n_heads, config.expansion_ratio, no_bias=config.no_bias, alibi=True,
                           alibi_bias_max=ac["alibi_bias_max"], softmax_scale=ac["softmax_scale"])
            for _ in range(config.n_layers)])
        self.norm_f = nn.LayerNorm(config.d_model, eps=1e-5, bias=not config.no_bias)
        self.is_causal = True
        self._zeros = None

    def get_input_embeddings(self):
        return self.wte

    def set_input_embeddings(self, value):
        self.wte = value

    def forward(self, input_ids, past_key_values=None, attention_mask=None, prefix_mask=None, sequence_id=None,
                return_dict=None, output_attentions=None, output_hidden_states=None, use_cache=None,
                inputs_embeds=None):
        if inputs_embeds is not None:
            raise NotImplementedError("inputs_embeds is not implemented for MPT.")          # modeling_mpt.py:209-210
        if output_attentions:
            raise NotImplementedError("output_attentions is not implemented for the fused attention kernel")
        if attention_mask is not None:
            # ONE host read per forward for both checks (the reference syncs here too, modeling_mpt.py:203): left
            # padding in training is the reference's error; interior padding is what the fused causal kernel cannot
            # express.  A right-padded mask needs no key mask under causality, so the layers get attention_mask=None.
            am = attention_mask.bool()
            left_pad = am[:, 0].sum() != am.shape[0]
            ragged = ~(am[:, 1:] <= am[:, :-1]).all()
            left_pad, ragged = (bool(v) for v in torch.stack([left_pad, ragged]).tolist())
            if left_pad and self.training:                                                 # modeling_mpt.py:203-204
                raise NotImplementedError("MPT does not support training with left padding.")
            if left_pad or ragged:
                raise NotImplementedError("otter_b200 MPT: only right-padded batches (no interior / left padding)")
            attention_mask = None
        S = input_ids.size(1)
        assert S <= self.config.max_seq_len, \
            f"Cannot forward input with seq_len={S}, this model only supports seq_len<={self.config.max_seq_len}"
        x = self.wte(input_ids)                                                            # :226 (ALiBi: no wpe)
        if self.embedding_fraction != 1:                                                   # :255-259
            x = x * self.embedding_fraction + x.detach() * (1 - self.embedding_fraction)
        x = _as_bf16(x)
        hs = () if output_hidden_states else None
        for block in self.blocks:                                                          # :270-283
            if output_hidden_states:
                hs = hs + (x,)
            x, _, _ = block(x, past_key_value=None, attn_bias=None, attention_mask=attention_mask,
                            is_causal=self.is_causal)
        B = x.shape[0]
        if self.norm_f.bias is not None:
            beta = P.f32_of(self.norm_f.bias)
        else:
            if self._zeros is None or self._zeros.device != x.device:
                self._zeros = torch.zeros(self.config.d_model, device=x.device, dtype=torch.float32)
            beta = self._zeros
        x = _FrozenLayerNormFn.apply(x.reshape(B * S, -1).contiguous(), self.norm_f.weight, beta).view(B, S, -1)   # :292
        if output_hidden_states:
            hs = hs + (x,)
        return BaseModelOutputWithPast(last_hidden_state=x, past_key_values=None, hidden_states=hs, attentions=None)


class MPTPreTrainedModel(PreTrainedModel):
    config_class = MPTConfig
    base_model_prefix = "model"
    _no_split_modules = ["FrozenMPTBlock"]

    def _init_weights(self, module):
        return None


class MPTForCausalLM(MPTPreTrainedModel, GenerationMixin):
    """modeling_mpt.py:280-436: same constructor check, accessors, forward() signature and shifted loss."""
    _tied_weights_keys = []

    def __init__(self, config):
        super().__init__(config)
        if not config.tie_word_embeddings:
            raise ValueError("MPTForCausalLM only supports tied word embeddings")
        self.transformer = MPTModel(config)
        self.logit_scale = None
        if config.logit_scale is not None:
            ls = config.logit_scale
            if isinstance(ls, str):
                if ls == "inv_sqrt_d_model":
                    ls = 1 / math.sqrt(config.d_model)
                else:
                    raise ValueError(f"logit_scale={ls!r} is not recognized as an option; use numeric value or "
                                     "'inv_sqrt_d_model'.")
            self.logit_scale = ls

    def get_input_embeddings(self):
        return self.transformer.wte

    def set_input_embeddings(self, value):
        self.transformer.wte = value

    def get_output_embeddings(self):
        return self.transformer.wte

    def set_output_embeddings(self, new_embeddings):
        self.transformer.wte = new_embeddings

    def set_decoder(self, decoder):
        self.transformer = decoder

    def get_decoder(self):
        return self.transformer

    def forward(self, input_ids, past_key_values=None, attention_mask=None, prefix_mask=None, sequence_id=None,
                labels=None, return_dict=None, output_attentions=None, output_hidden_states=None, use_cache=None,
                inputs_embeds=None, **unused):
        if inputs_embeds is not None:
            raise NotImplementedError("inputs_embeds has to be None (for hf/peft support).")   # modeling_mpt.py:398-399
        out = self.transformer(input_ids=input_ids, past_key_values=None, attention_mask=attention_mask,
                               prefix_mask=prefix_mask, sequence_id=sequence_id, return_dict=return_dict,
                               output_attentions=output_attentions, output_hidden_states=output_hidden_states,
                               use_cache=False)
        h = out.last_hidden_state
        B, S, D = h.shape
        wte = self.transformer.wte.weight
        V = wte.shape[0]
        if V % 8:
            raise ValueError(f"vocab_size {V} must be a multiple of 8 for the tensor-core un-embedding "
                             "(resize_token_embeddings pads to a multiple of 8 for MPT's 50432-style vocabularies)")
        logits = _UnembedFn.apply(h.reshape(B * S, D), wte).view(B, S, V)                     # :418-421
        if self.logit_scale is not None:
            logits = logits * self.logit_scale                                                  # :423-426
        loss = None
        if labels is not None:                                                                  # :428-436
            from .losses import shifted_cross_entropy
            loss = shifted_cross_entropy(logits, labels.to(logits.device))
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=None, hidden_states=out.hidden_states,
                                      attentions=None)

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, inputs_embeds=None, attention_mask=None,
                                      **kwargs):
        """No KV cache: every decode step re-runs the whole prefix (modeling_mpt.py:456-483 minus the cache slice)."""
        if inputs_embeds is not None:
            raise NotImplementedError("inputs_embeds is not implemented for MPT yet")
        return {"input_ids": input_ids, "attention_mask": attention_mask, "past_key_values": None, "use_cache": False}
