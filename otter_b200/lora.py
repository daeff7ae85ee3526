"""LoRA adapters with peft's module layout, on the otter_b200 decoder layers.

The reference puts peft's LoRA on the language model when the Otter config carries `lora_config = {r, lora_alpha,
lora_dropout}` (modeling_otter.py:808-829): adapters on `q_proj` / `v_proj` (LLaMA) or `Wqkv` (MPT), and `init_weights`
unfreezes every parameter whose name contains "lora" (:889-894).  peft wraps each targeted Linear in a LoraLayer and
forwards `.weight` to the base weight; the otter_b200 decoder layers read `.weight` directly, so under peft the adapters
would never reach the kernels.  This module builds the same layout without peft, and the decoder layers
(lm_llama.py, lm_mpt.py) run the adapters on their kernel path:

  * `LoraLinear`: peft's attribute names (`base_layer`, `lora_A` / `lora_B` / `lora_dropout` ModuleDicts keyed
    "default", `scaling`), peft's default initialisation (kaiming_uniform_(a=sqrt(5)) for A, zeros for B) and peft's
    formula as its own torch forward: base(x) + lora_B(lora_A(dropout(x))) * scaling.  That forward serves the layers
    that stay stock HF code (configs the kernel layers do not cover, OTB_LLAMA_LAYERS=0, and the HF layer generate()
    uses for KV-cache steps).
  * `wrap_lora`: replaces the targeted Linears and returns a shell laid out like peft's PeftModelForCausalLM, so state-dict
    keys read `base_model.model.<path>.base_layer.weight`, `<path>.lora_A.default.weight` [r, in] and
    `<path>.lora_B.default.weight` [out, r] (peft >= 0.7) and reference LoRA checkpoints load.
"""
import math

import torch
from torch import nn

from . import functional as F
from . import params as P

ADAPTER = "default"


class LoraLinear(nn.Module):
    """An nn.Linear with one LoRA adapter, peft's layout and default initialisation."""

    def __init__(self, base_layer, r, lora_alpha, lora_dropout=0.0):
        super().__init__()
        if not isinstance(base_layer, nn.Linear):
            raise TypeError(f"LoraLinear wraps an nn.Linear, got {type(base_layer).__name__}")
        if r <= 0:
            raise ValueError(f"LoRA rank r = {r} must be positive")
        self.base_layer = base_layer
        self.in_features, self.out_features = base_layer.in_features, base_layer.out_features
        self.r, self.lora_alpha = {ADAPTER: int(r)}, {ADAPTER: lora_alpha}
        self.scaling = {ADAPTER: lora_alpha / r}
        w = base_layer.weight
        self.lora_A = nn.ModuleDict({ADAPTER: nn.Linear(self.in_features, r, bias=False, device=w.device, dtype=w.dtype)})
        self.lora_B = nn.ModuleDict({ADAPTER: nn.Linear(r, self.out_features, bias=False, device=w.device, dtype=w.dtype)})
        self.lora_dropout = nn.ModuleDict({ADAPTER: nn.Dropout(p=float(lora_dropout))})
        nn.init.kaiming_uniform_(self.lora_A[ADAPTER].weight, a=math.sqrt(5))
        nn.init.zeros_(self.lora_B[ADAPTER].weight)

    # peft's LoraLayer forwards these to the base layer too
    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return self.base_layer.bias

    def forward(self, x):
        result = self.base_layer(x)
        a, b = self.lora_A[ADAPTER], self.lora_B[ADAPTER]
        xa = x.to(a.weight.dtype)
        return result + (b(a(self.lora_dropout[ADAPTER](xa))) * self.scaling[ADAPTER]).to(result.dtype)


def adapter(lin):
    """(A [r, in], B [out, r], scaling, dropout p or 0 when the dropout module is in eval mode) of a LoraLinear, or None
    for a plain Linear."""
    if not isinstance(lin, LoraLinear):
        return None
    drop = lin.lora_dropout[ADAPTER]
    return (lin.lora_A[ADAPTER].weight, lin.lora_B[ADAPTER].weight, lin.scaling[ADAPTER],
            drop.p if drop.training else 0.0)


def needs_input(*lins):
    """True when the backward needs the input of one of these Linears (or LoraLinears): a weight that requires grad (its
    wgrad GEMM), or an adapter A that does (dA = dxa^T dropout(input))."""
    for lin in lins:
        ad = adapter(lin)
        if lin.weight.requires_grad or (ad is not None and ad[0].requires_grad):
            return True
    return False


def draw_seed(device):
    """64-bit key of one layer call's adapter dropout masks, drawn from torch's generator of `device`: the CUDA
    generator's (seed, offset) pair, whose offset is then advanced, so no host-device synchronisation is needed and
    torch.manual_seed reproduces the sequence of masks."""
    if device.type == "cuda":
        idx = device.index if device.index is not None else torch.cuda.current_device()
        gen = torch.cuda.default_generators[idx]
        seed, off = gen.initial_seed(), gen.get_offset()
        gen.set_offset(off + 4)
    else:
        seed, off = int(torch.randint(0, 2 ** 62, (1,)).item()), 0
    return _splitmix64(_splitmix64(seed) ^ off)


def layer_seed(device, *adapters):
    """The dropout key of one decoder-layer call: drawn only when an adapter drops something (None otherwise)."""
    return draw_seed(device) if any(ad is not None and ad[3] > 0 for ad in adapters) else None


# ---- an adapted projection on the kernels (h: the norm output feeding it, A [r, in], B [out, r], s = scaling) ----
def kernel_fwd(h, w, ad, out, seed, stream_id, bias=None):
    """out = h W^T (+ bias) + s (dropout(h) A^T) B^T.  The base projection goes to a temporary that the adapter GEMM
    reads as its epilogue residual (alpha = s), so out = bf16(s xa B^T + bf16(base)): with B = 0 that is the unadapted
    projection bit for bit.  Returns xa = dropout(h) A^T (bf16 [rows, r]), which the B gradient needs."""
    A, B, s, p = ad
    base = F.linear_fwd(h, w, bias=bias)
    hd = F.lora_dropout(h, p, seed, stream_id) if p > 0 else h
    xa = F.linear_fwd(hd, P.bf16_of(A))
    F.linear_fwd(xa, P.bf16_of(B), alpha=s, residual=base, out=out)
    return xa


def kernel_bwd(sink, dout, h, xa, ad, seed, stream_id, dh):
    """Adapter part of the backward of kernel_fwd.  dout: gradient of the projection output; dh: the bf16 gradient of h
    accumulated so far (updated in place, or replaced: the returned tensor is the result).
      dxa = s dout B;  dB = s dout^T xa;  dA = dxa^T dropout(h);  dh += dropout_bwd(dxa A)
    dropout(h) is regenerated from the key rather than kept from the forward.  A, B gradients go through `sink` (None:
    nothing trains) for those that require grad."""
    A, B, s, p = ad
    dxa = F.linear_dgrad(dout, P.bf16_of(B), alpha=s)
    if sink is not None and B.requires_grad:
        g, acc = sink.target(B)
        F.linear_wgrad(dout, xa, out=g, accumulate=acc, alpha=s)
    if sink is not None and A.requires_grad:
        hd = F.lora_dropout(h, p, seed, stream_id) if p > 0 else h
        g, acc = sink.target(A)
        F.linear_wgrad(dxa, hd, out=g, accumulate=acc)
    if p > 0:
        return F.lora_dropout_bwd_add_(F.linear_dgrad(dxa, P.bf16_of(A)), dh, p, seed, stream_id)
    return F.linear_dgrad(dxa, P.bf16_of(A), residual=dh)


def _splitmix64(z):
    z = (z + 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & 0xFFFFFFFFFFFFFFFF
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & 0xFFFFFFFFFFFFFFFF
    return z ^ (z >> 31)


# ---- peft's PeftModelForCausalLM / LoraModel layout ----
class _Forwarding(nn.Module):
    """Attribute lookups that nn.Module does not resolve go to the wrapped module (peft's __getattr__ chain)."""
    _inner = None

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            if name == self._inner or name.startswith("__"):
                raise
            return getattr(super().__getattr__(self._inner), name)


class LoraModel(_Forwarding):
    """peft's tuners.lora.LoraModel: `.model` is the language model with its targeted Linears replaced."""
    _inner = "model"

    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, *args, **kwargs):
        return self.model(*args, **kwargs)


class LoraModelForCausalLM(_Forwarding):
    """peft's PeftModelForCausalLM layout: `.base_model` (a LoraModel) holds the language model at `.base_model.model`."""
    _inner = "base_model"

    def __init__(self, model, r, lora_alpha, lora_dropout, target_modules):
        super().__init__()
        self.base_model = LoraModel(model)
        self.peft_config = {ADAPTER: {"r": r, "lora_alpha": lora_alpha, "lora_dropout": lora_dropout,
                                      "target_modules": list(target_modules), "task_type": "CAUSAL_LM"}}

    def forward(self, *args, **kwargs):
        return self.base_model.model(*args, **kwargs)

    def generate(self, *args, **kwargs):
        return self.base_model.model.generate(*args, **kwargs)


def _kernel_layer_types():
    from .lm_llama import FrozenLlamaDecoderLayer
    from .lm_mpt import FrozenMPTBlock
    return (FrozenLlamaDecoderLayer, FrozenMPTBlock)


def _matches(name, targets):
    """peft's suffix rule: the module name equals a target or ends with "." + target."""
    return any(name == t or name.endswith("." + t) for t in targets)


def wrap_lora(lang_encoder, r, lora_alpha, lora_dropout, target_modules):
    """Put a LoRA adapter on every nn.Linear of `lang_encoder` whose name matches `target_modules` (peft's suffix rule)
    and return the peft-layout shell around it, of a class named f"{type(lang_encoder).__name__}LoRA".  As peft does,
    every parameter of the language model except the adapters is frozen (Otter's init_weights then applies its policy).

    r must be a multiple of 8 for adapters inside the otter_b200 decoder layers: the adapter GEMMs have r as an output
    width or as the extent of an MN-major operand, both of which the GEMM needs in 16-byte rows.  Adapters on stock HF
    layers take any r.  A swapped LLaMA layer's KV-cache HF layer (`_hf_layer`) receives the same LoraLinear objects, so
    cached generation decodes with the adapters."""
    targets = [target_modules] if isinstance(target_modules, str) else list(target_modules)
    kernel_types = _kernel_layer_types()
    owners = {}                                    # module name -> the kernel decoder layer it lies in
    hf_hosts = {}                                  # module name -> module whose __dict__ holds an `_hf_layer`
    for name, mod in lang_encoder.named_modules():
        if isinstance(mod, kernel_types):
            owners[name] = mod
        if "_hf_layer" in mod.__dict__:
            hf_hosts[name] = mod
    todo = [(n, m) for n, m in lang_encoder.named_modules() if n and isinstance(m, nn.Linear) and _matches(n, targets)]
    if not todo:
        raise ValueError(f"wrap_lora: no nn.Linear of {type(lang_encoder).__name__} matches {targets}")

    def enclosing(name, table):
        for prefix, mod in table.items():
            if prefix == "" or name.startswith(prefix + "."):
                return prefix, mod
        return None, None

    for name, lin in todo:
        if enclosing(name, owners)[1] is not None and r % 8:
            raise ValueError(f"wrap_lora: r = {r} must be a multiple of 8 for the adapter on {name}: it runs inside an "
                             "otter_b200 decoder layer, whose GEMMs need 16-byte rows (r % 8 == 0)")
    for name, lin in todo:
        new = LoraLinear(lin, r, lora_alpha, lora_dropout)
        parent, _, leaf = name.rpartition(".")
        setattr(lang_encoder.get_submodule(parent) if parent else lang_encoder, leaf, new)
        host_name, host = enclosing(name, hf_hosts)
        if host is not None:                                             # the KV-cache HF layer shares the adapter
            rel_parent, _, rel_leaf = (name[len(host_name) + 1:] if host_name else name).rpartition(".")
            hf = host.__dict__["_hf_layer"]
            setattr(hf.get_submodule(rel_parent) if rel_parent else hf, rel_leaf, new)
    for n, p in lang_encoder.named_parameters():
        p.requires_grad_("lora_" in n)
    cls = type(f"{type(lang_encoder).__name__}LoRA", (LoraModelForCausalLM,), {})
    return cls(lang_encoder, r, lora_alpha, lora_dropout, targets)
