"""Otter / OpenFlamingo module classes on the otter_b200 kernels.

Drop-in boundary (SURVEY.md §8b): same class names, constructor kwargs, forward() signatures, error
behaviour and state-dict keys as /root/reference/src/otter_ai/models/otter/modeling_otter.py, so
checkpoints load both ways and pipeline/train / pipeline/demos call sites work unchanged — but every
forward/backward below runs on the sm_90a kernels of libotter_b200.so (via otter_b200.blocks).
There is no eager/PyTorch fallback: CPU tensors are rejected.

Numerics: bf16 operands, fp32 accumulation / softmax / LayerNorm statistics — the reference's
`autocast(bf16)` training recipe (pipeline/train/instruction_following.py:311-314).
"""
import random
from typing import List, Optional

import torch
import torch.nn as nn

from . import fp32_path
from . import functional as F
from .blocks import (BroadcastRowsFn, GatedCrossAttentionBlockFn, LayerNormFn, MaskedCrossAttentionFn,
                     MediaFromClipFn, PerceiverBlockFn, _as_bf16_2d)
from .modeling_clip import CLIPVisionModel

BF16 = torch.bfloat16


def exists(val):
    return val is not None


def _check_heads(dim_head):
    if dim_head != 64:
        raise ValueError("otter_b200 attention kernels are built for dim_head == 64 (the Otter / Flamingo value)")


class _AddRowBiasFn(torch.autograd.Function):
    """x [rows,D] + bias[(row // div) % mod]   (frame_embs broadcast, modeling_otter.py:224-226)."""

    @staticmethod
    def forward(ctx, x, bias, div, mod):
        from .params import f32_of
        if mod > bias.shape[0]:       # the kernel indexes bias[(row // div) % mod] unchecked
            raise ValueError(f"{mod} frames / media per sample but the embedding table holds {bias.shape[0]} rows "
                             "(max_num_frames / max_num_media, modeling_otter.py:224-229)")
        ctx.bias, ctx.cfg = bias, (div, mod)
        return F.add_rowbias(x, f32_of(bias)[:mod].contiguous(), div, mod)

    @staticmethod
    def backward(ctx, dy):
        from .params import GradSink
        bias = ctx.bias
        div, mod = ctx.cfg
        sink = GradSink()
        g, acc = sink.target(bias)
        if not acc:
            g.zero_()
        F.grouped_colsum(_as_bf16_2d(dy, bias.shape[-1]), div, mod, out=g[:mod], accumulate=acc)
        return (dy if ctx.needs_input_grad[0] else None), sink.result(bias), None, None


# =================================================================================================
# Perceiver
# =================================================================================================
class OtterPerceiverBlock(nn.Module):
    """reference :129-184 — cross-attention of latents over (media ++ latents) + feed-forward."""

    def __init__(self, *, dim: int, dim_head: int = 64, heads: int = 8, mult: int = 4):
        super().__init__()
        _check_heads(dim_head)
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner_dim = dim_head * heads
        self.norm_media = nn.LayerNorm(dim)
        self.norm_latents = nn.LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, inner_dim * 2, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)
        self.feed_forward = nn.ModuleList(
            [nn.LayerNorm(dim), nn.Linear(dim, dim * mult, bias=False), nn.GELU(), nn.Linear(dim * mult, dim, bias=False)])

    def _apply2d(self, x2d, lat2d, BT, need_dx):
        ff = self.feed_forward
        return PerceiverBlockFn.apply(x2d, lat2d, BT, need_dx, self.heads, self.norm_media.weight, self.norm_media.bias,
                                      self.norm_latents.weight, self.norm_latents.bias, self.to_q.weight,
                                      self.to_kv.weight, self.to_out.weight, ff[0].weight, ff[0].bias, ff[1].weight,
                                      ff[3].weight)

    def forward(self, x: torch.Tensor, latents: torch.Tensor) -> torch.Tensor:
        """x (b, T, n1, D) media features, latents (b, T, n2, D) -> (b, T, n2, D)."""
        b, T, n2, D = latents.shape
        if fp32_path.is_fp32():
            out = fp32_path.perceiver_block(self, fp32_path._f32_2d(x, D), fp32_path._f32_2d(latents, D), b * T)
            return out.view(b, T, n2, D).to(latents.dtype)
        out = self._apply2d(_as_bf16_2d(x, D), _as_bf16_2d(latents, D), b * T, x.requires_grad)
        return out.view(b, T, n2, D).to(latents.dtype)


class OtterPerceiverResampler(nn.Module):
    """reference :187-235."""
    _block_cls = None          # Flamingo twin: FlamingoPerceiverBlock

    def __init__(self, *, dim: int, depth: int = 6, dim_head: int = 64, heads: int = 8, num_latents: int = 64,
                 max_num_media: Optional[int] = None, max_num_frames: Optional[int] = None, ff_mult: int = 4):
        super().__init__()
        self.latents = nn.Parameter(torch.randn(num_latents, dim))
        self.frame_embs = nn.Parameter(torch.randn(max_num_frames, dim)) if exists(max_num_frames) else None
        self.media_time_embs = nn.Parameter(torch.randn(max_num_media, 1, dim)) if exists(max_num_media) else None
        self.layers = nn.ModuleList(
            [(self._block_cls or OtterPerceiverBlock)(dim=dim, dim_head=dim_head, heads=heads, mult=ff_mult)
             for _ in range(depth)])
        self.norm = nn.LayerNorm(dim)

    def resample_media(self, media2d, BT):
        """media2d bf16 [BT*n1, D] (frame/time embeddings already added) -> bf16 [BT*n, D]."""
        n, D = self.latents.shape
        lat = BroadcastRowsFn.apply(self.latents, BT * n, 1, n)                       # :232
        need_dx = media2d.requires_grad
        for block in self.layers:                                                      # :233-234
            lat = block._apply2d(media2d, lat, BT, need_dx)
        return LayerNormFn.apply(lat, self.norm.weight, self.norm.bias, self.norm.eps)  # :235

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x (b, T, F, v, D) -> (b, T, n, D)."""
        b, T, Fr, v, D = x.shape
        if fp32_path.is_fp32():
            return fp32_path.resampler_forward(self, x).to(x.dtype)
        media = _as_bf16_2d(x, D)
        if exists(self.frame_embs):                                                    # :224-226
            media = _AddRowBiasFn.apply(media, self.frame_embs, v, Fr)
        if exists(self.media_time_embs):                                               # :228-229 (never set by Otter)
            media = _AddRowBiasFn.apply(media, self.media_time_embs.view(-1, D), Fr * v, T)
        out = self.resample_media(media, b * T)
        return out.view(b, T, self.latents.shape[0], D).to(x.dtype if x.dtype != torch.float64 else torch.float32)


# =================================================================================================
# Gated cross-attention
# =================================================================================================
def _text_time_for(media_locations, attend_previous):
    if media_locations is None:
        return None
    return F.text_time(media_locations, attend_previous)


class OtterMaskedCrossAttention(nn.Module):
    """reference :238-340."""

    def __init__(self, *, dim: int, dim_visual: int, dim_head: int = 64, heads: int = 8,
                 only_attend_immediate_media: bool = True):
        super().__init__()
        _check_heads(dim_head)
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner_dim = dim_head * heads
        self.norm = nn.LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim_visual, inner_dim * 2, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)
        self.only_attend_immediate_media = only_attend_immediate_media

    def forward(self, x: torch.Tensor, media: torch.Tensor, media_locations: Optional[torch.BoolTensor] = None,
                attend_previous: bool = True) -> torch.Tensor:
        """x (B, T_txt, D), media (B, T_img, n, D_img), media_locations bool (B, T_txt) -> (B, T_txt, D)."""
        B, L, D = x.shape
        _, T_img, n = media.shape[:3]
        tt = _text_time_for(media_locations, attend_previous)
        if fp32_path.is_fp32():
            out = fp32_path.masked_cross_attention(self, fp32_path._f32_2d(x, D),
                                                   fp32_path._f32_2d(media, media.shape[-1]), tt, B, L, T_img, n)
            return out.view(B, L, D).to(x.dtype)
        out = MaskedCrossAttentionFn.apply(_as_bf16_2d(x, D), _as_bf16_2d(media, media.shape[-1]), tt, B, L, T_img, n,
                                           self.heads, self.norm.weight, self.norm.bias, self.to_q.weight,
                                           self.to_kv.weight, self.to_out.weight, not self.only_attend_immediate_media)
        return out.view(B, L, D).to(x.dtype)


class OtterGatedCrossAttentionBlock(nn.Module):
    """reference :343-395 — tanh-gated masked cross-attention + tanh-gated feed-forward."""
    _attn_cls = None           # Flamingo twin: FlamingoMaskedCrossAttention

    def __init__(self, *, dim: int, dim_visual: int, dim_head: int = 64, heads: int = 8, ff_mult: int = 4,
                 only_attend_immediate_media: bool = True):
        super().__init__()
        self.attn = (self._attn_cls or OtterMaskedCrossAttention)(
            dim=dim, dim_visual=dim_visual, dim_head=dim_head, heads=heads,
            only_attend_immediate_media=only_attend_immediate_media)
        self.attn_gate = nn.Parameter(torch.tensor([0.0]))
        self.feed_forward = nn.ModuleList(
            [nn.LayerNorm(dim), nn.Linear(dim, dim * ff_mult, bias=False), nn.GELU(),
             nn.Linear(dim * ff_mult, dim, bias=False)])
        self.ff_gate = nn.Parameter(torch.tensor([0.0]))

    def forward_2d(self, x2d, media2d, tt, B, L, T_img, n):
        a, ff = self.attn, self.feed_forward
        return GatedCrossAttentionBlockFn.apply(x2d, media2d, tt, B, L, T_img, n, a.heads, a.norm.weight, a.norm.bias,
                                                a.to_q.weight, a.to_kv.weight, a.to_out.weight, self.attn_gate,
                                                ff[0].weight, ff[0].bias, ff[1].weight, ff[3].weight, self.ff_gate,
                                                not a.only_attend_immediate_media)

    def forward(self, x: torch.Tensor, media: torch.Tensor, media_locations: Optional[torch.BoolTensor] = None,
                attend_previous: bool = True) -> torch.Tensor:
        B, L, D = x.shape
        _, T_img, n = media.shape[:3]
        tt = _text_time_for(media_locations, attend_previous)
        if fp32_path.is_fp32():
            out = fp32_path.gated_block(self, fp32_path._f32_2d(x, D), fp32_path._f32_2d(media, media.shape[-1]), tt,
                                        B, L, T_img, n)
            return out.view(B, L, D).to(x.dtype)
        out = self.forward_2d(_as_bf16_2d(x, D), _as_bf16_2d(media, media.shape[-1]), tt, B, L, T_img, n)
        return out.view(B, L, D).to(x.dtype)


# =================================================================================================
# LM wiring (state holders, no arithmetic)
# =================================================================================================
class OtterLayer(nn.Module):
    """reference :398-442 — gated block (optional) in front of a frozen decoder layer; vision features and
    media locations arrive through side-channel state."""

    def __init__(self, gated_cross_attn_layer: nn.Module, decoder_layer: nn.Module):
        super().__init__()
        self.gated_cross_attn_layer = gated_cross_attn_layer
        self.decoder_layer = decoder_layer
        self.vis_x = None
        self.media_locations = None

    def is_conditioned(self) -> bool:
        return self.vis_x is not None

    def condition_vis_x(self, vis_x) -> None:
        self.vis_x = vis_x

    def condition_media_locations(self, media_locations) -> None:
        self.media_locations = media_locations

    def condition_attend_previous(self, attend_previous) -> None:
        self.attend_previous = attend_previous

    def forward(self, lang_x: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, **decoder_layer_kwargs):
        if self.gated_cross_attn_layer is not None:
            if self.vis_x is None:
                raise ValueError("vis_x must be conditioned before forward pass")
            if self.media_locations is None:
                raise ValueError("media_locations must be conditioned before forward pass")
            lang_x = self.gated_cross_attn_layer(lang_x, self.vis_x, media_locations=self.media_locations,
                                                 attend_previous=self.attend_previous)
        return self.decoder_layer(lang_x, attention_mask=attention_mask, **decoder_layer_kwargs)


_DECODER_LAYERS_ATTR = {
    "opt": "model.decoder.layers", "gptneo": "transformer.h", "gptj": "transformer.h", "gpt-j": "transformer.h",
    "pythia": "gpt_neox.layers", "llama": "model.layers", "RWForCausalLM": "transformer.h",
    "MPTForCausalLM": "transformer.blocks", "MosaicGPT": "transformer.blocks",
}


def _infer_decoder_layers_attr_name(model: nn.Module):
    name = model.__class__.__name__.lower()
    for k, v in _DECODER_LAYERS_ATTR.items():
        if k.lower() in name:
            return v
    raise ValueError("We require the attribute name for the nn.ModuleList in the decoder storing the transformer "
                     "block layers. Please supply this string manually.")


def extend_instance(obj, mixin):
    """Re-class an instance as (mixin, original class) — the mixin's forward must come first in the MRO."""
    base = obj.__class__
    obj.__class__ = type(base.__name__, (mixin, base), {})


def getattr_recursive(obj, att):
    for part in (att.split(".") if att else []):
        obj = getattr(obj, part)
    return obj


def setattr_recursive(obj, att, val):
    head, _, leaf = att.rpartition(".")
    setattr(getattr_recursive(obj, head), leaf, val)


class OtterLMMixin(nn.Module):
    """reference :445-520 — mixed INTO the language model instance."""
    _layer_cls = None          # OtterLayer / OtterGatedCrossAttentionBlock (Flamingo twin: its own class names, which
    _gated_cls = None          # `_no_split_modules` and checkpoints' module reprs refer to)

    def set_decoder_layers_attr_name(self, decoder_layers_attr_name):
        self.decoder_layers_attr_name = decoder_layers_attr_name

    def _get_decoder_layers(self):
        return getattr_recursive(self, self.decoder_layers_attr_name)

    def _set_decoder_layers(self, value):
        setattr_recursive(self, self.decoder_layers_attr_name, value)

    def init_otter(self, media_token_id: int, vis_hidden_size: int, cross_attn_every_n_layers: int,
                   use_media_placement_augmentation: bool):
        layers = self._get_decoder_layers()
        wrapped = []
        for idx, dec in enumerate(layers):
            gated = None
            if (idx + 1) % cross_attn_every_n_layers == 0:
                gated = (self._gated_cls or OtterGatedCrossAttentionBlock)(dim=self.config.hidden_size,
                                                                           dim_visual=vis_hidden_size)
            wrapped.append((self._layer_cls or OtterLayer)(gated, dec))
        self._set_decoder_layers(nn.ModuleList(wrapped))
        self.media_token_id = media_token_id
        self.use_media_placement_augmentation = use_media_placement_augmentation
        self.initialized_otter = True

    def forward(self, *input, **kwargs):
        if not getattr(self, "initialized_otter", False):
            raise ValueError("Otter layers are not initialized. Please call `init_otter` first.")
        input_ids = kwargs["input_ids"] if "input_ids" in kwargs else input[0]
        media_locations = input_ids == self.media_token_id            # bool [B, L] — bit-exact index tensor
        attend_previous = (random.random() < 0.5) if self.use_media_placement_augmentation else True
        for layer in self._get_decoder_layers():
            layer.condition_media_locations(media_locations)
            layer.condition_attend_previous(attend_previous)
        return super().forward(*input, **kwargs)

    def is_conditioned(self) -> bool:
        return all(l.is_conditioned() for l in self._get_decoder_layers())

    def clear_conditioned_layers(self) -> None:
        for layer in self._get_decoder_layers():
            layer.condition_vis_x(None)
            layer.condition_media_locations(None)
            layer.condition_attend_previous(None)


# =================================================================================================
# a-1  vision encoding shared by OtterModel / OtterForConditionalGeneration  (:975-997)
# =================================================================================================
def encode_vision_x(vision_encoder, perceiver, vision_x):
    assert vision_x.ndim == 6, "vision_x should be of shape (b, T_img, F, C, H, W)"
    b, T, Fr = vision_x.shape[:3]
    pixels = vision_x.reshape(b * T * Fr, *vision_x.shape[3:])
    if fp32_path.is_fp32() and isinstance(vision_encoder, CLIPVisionModel):
        with torch.no_grad():                                                  # frozen tower, as on the bf16 path
            feats = fp32_path.clip_last_hidden(vision_encoder, pixels)[:, 1:, :]
        return perceiver(feats.reshape(b, T, Fr, feats.shape[1], feats.shape[2]))
    if isinstance(vision_encoder, CLIPVisionModel):
        hidden = vision_encoder.last_hidden_bf16(pixels)                       # bf16 [bTF, 1+v, D]
        media = MediaFromClipFn.apply(hidden, perceiver.frame_embs, Fr)        # drop CLS (+frame_embs) fused
        if exists(perceiver.media_time_embs):
            media = _AddRowBiasFn.apply(media, perceiver.media_time_embs.view(-1, media.shape[-1]),
                                        Fr * (hidden.shape[1] - 1), T)
        out = perceiver.resample_media(media, b * T)
        n, D = perceiver.latents.shape
        return out.view(b, T, n, D)
    feats = vision_encoder(pixels)[0][:, 1:, :]                                # foreign vision tower
    return perceiver(feats.reshape(b, T, Fr, feats.shape[1], feats.shape[2]))


def __getattr__(name):
    """Lazy re-export of the HF-level classes (they import `transformers`, which is slow to load)."""
    if name in ("OtterConfig", "OtterPreTrainedModel", "OtterModel", "OtterForConditionalGeneration", "AutoTokenizer"):
        from . import otter_hf
        return getattr(otter_hf, name)
    raise AttributeError(name)
