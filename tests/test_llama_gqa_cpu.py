"""CPU: grouped-query attention (GQA) and scaled RoPE in the frozen LLaMA decoder layer (otter_b200/lm_llama.py).

- `llama_layer_gqa`, the LLaMA-layer oracle extended with K/V head groups and a scaled RoPE table (built from the helpers
  of oracle/restatement_llama.py; tests/test_llama_gqa_gpu.py uses it too), against HF's LlamaDecoderLayer,
  fp32, forward and input gradient, for 2 and 4 query heads per K/V head and one K/V head (MQA), with each covered
  rope_type.
- The autograd wiring of _FrozenLlamaLayerFn for GQA / scaled RoPE with the kernels replaced by torch formulas.
- swappable() / swap_llama_layers on GQA and scaled-RoPE configs.
- The C ABI: struct sizes unchanged, the new entry point exported, kv_heads that do not divide H rejected before any
  launch.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import restatement_llama as RL


def llama_layer_gqa(x, p, num_heads, eps=1e-6, rope_theta=10000.0, num_kv_heads=None, inv_freq=None, attn_scale=1.0):
    """One LLaMA decoder layer, as RL.llama_layer, with grouped-query attention (K/V head h // (num_heads //
    num_kv_heads) serves query head h: HF's repeat_kv) and a RoPE table: inv_freq [hd/2] with cos and sin multiplied by
    attn_scale (HF's linear / llama3 / yarn scaling).  By default the frequencies come from rope_theta."""
    B, S, D = x.shape
    hd = D // num_heads
    kvh = num_heads if num_kv_heads is None else num_kv_heads
    h = RL.rms_norm(x, p["input_layernorm.weight"], eps)
    sp = lambda t, n: t.view(B, S, n, hd).transpose(1, 2)
    q = sp(h @ p["self_attn.q_proj.weight"].t(), num_heads)
    k, v = (sp(h @ p[f"self_attn.{n}_proj.weight"].t(), kvh) for n in ("k", "v"))
    if inv_freq is None:
        inv_freq = 1.0 / (rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
    fr = torch.arange(S, dtype=torch.float32)[:, None] * inv_freq[None].to(torch.float32)
    emb = torch.cat((fr, fr), -1)
    cos, sin = emb.cos()[None, None], emb.sin()[None, None]
    if attn_scale != 1.0:
        cos, sin = cos * attn_scale, sin * attn_scale
    q, k = q * cos + RL.rotate_half(q) * sin, k * cos + RL.rotate_half(k) * sin
    if kvh != num_heads:                                                            # repeat_kv
        k, v = k.repeat_interleave(num_heads // kvh, dim=1), v.repeat_interleave(num_heads // kvh, dim=1)
    sim = (q @ k.transpose(-1, -2)) / math.sqrt(hd)
    sim = sim.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
    o = (sim.softmax(-1) @ v).transpose(1, 2).reshape(B, S, D)
    x1 = x + o @ p["self_attn.o_proj.weight"].t()
    h2 = RL.rms_norm(x1, p["post_attention_layernorm.weight"], eps)
    g, u = h2 @ p["mlp.gate_proj.weight"].t(), h2 @ p["mlp.up_proj.weight"].t()
    return x1 + (torch.nn.functional.silu(g) * u) @ p["mlp.down_proj.weight"].t()


ROPES = {
    "default": {"rope_type": "default", "rope_theta": 10000.0},
    "linear": {"rope_type": "linear", "rope_theta": 10000.0, "factor": 4.0},
    "llama3": {"rope_type": "llama3", "rope_theta": 500000.0, "factor": 8.0, "low_freq_factor": 1.0,
               "high_freq_factor": 4.0, "original_max_position_embeddings": 64},
    "yarn": {"rope_type": "yarn", "rope_theta": 10000.0, "factor": 4.0, "original_max_position_embeddings": 64},
}


def _cfg(D, H, kv, rope, **kw):
    from transformers import LlamaConfig
    cfg = LlamaConfig(hidden_size=D, num_attention_heads=H, num_key_value_heads=kv, intermediate_size=3 * D,
                      num_hidden_layers=1, vocab_size=32, max_position_embeddings=256, rms_norm_eps=1e-6,
                      rope_parameters=dict(ROPES[rope]), **kw)
    cfg._attn_implementation = "eager"
    return cfg


def _hf_layer_and_grad(cfg, B, S, seed=0):
    from transformers.models.llama import modeling_llama as M
    torch.manual_seed(seed)
    layer = M.LlamaDecoderLayer(cfg, layer_idx=0)
    with torch.no_grad():
        for _, p_ in layer.named_parameters():
            if p_.dim() == 1:
                p_.add_(0.1 * torch.randn_like(p_))
    rope = M.LlamaRotaryEmbedding(cfg)
    x = torch.randn(B, S, cfg.hidden_size, requires_grad=True)
    pos = torch.arange(S)[None].expand(B, S)
    mask = torch.full((S, S), float("-inf")).triu(1)[None, None].expand(B, 1, S, S)
    out = layer(x, attention_mask=mask, position_ids=pos, position_embeddings=rope(x, pos))
    out = out[0] if isinstance(out, tuple) else out
    w = torch.randn_like(out)
    (out * w).sum().backward()
    return layer, rope, x, out, w


# ------------------------------------------------------------------------------------------------------------------
# oracle vs HF
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rope", list(ROPES))
@pytest.mark.parametrize("H,kv", [(4, 2), (4, 1), (8, 2)])
def test_oracle_matches_hf_gqa_layer(H, kv, rope):
    B, S, D = 2, 37, H * 64
    cfg = _cfg(D, H, kv, rope)
    layer, rot, x, out, w = _hf_layer_and_grad(cfg, B, S)
    p = {k: v.detach().clone() for k, v in layer.state_dict().items()}
    xr = x.detach().clone().requires_grad_(True)
    ref = llama_layer_gqa(xr, p, H, eps=cfg.rms_norm_eps, num_kv_heads=kv, inv_freq=rot.inv_freq,
                         attn_scale=rot.attention_scaling)
    (ref * w).sum().backward()
    assert torch.allclose(ref, out, rtol=1e-4, atol=1e-5)
    assert torch.allclose(xr.grad, x.grad, rtol=1e-3, atol=1e-5)


def test_extended_oracle_reduces_to_the_mha_oracle():
    """Defaults, and explicit num_kv_heads = H with the default table and attn_scale 1, give RL.llama_layer's result
    bit for bit."""
    torch.manual_seed(3)
    B, S, D, H = 1, 19, 256, 2
    p = {"input_layernorm.weight": torch.randn(D), "post_attention_layernorm.weight": torch.randn(D)}
    for n in ("q", "k", "v", "o"):
        p[f"self_attn.{n}_proj.weight"] = torch.randn(D, D) / 16
    p.update({"mlp.gate_proj.weight": torch.randn(64, D) / 16, "mlp.up_proj.weight": torch.randn(64, D) / 16,
              "mlp.down_proj.weight": torch.randn(D, 64) / 8})
    x = torch.randn(B, S, D)
    a = RL.llama_layer(x, p, H)
    inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))
    assert torch.equal(a, llama_layer_gqa(x, p, H))
    assert torch.equal(a, llama_layer_gqa(x, p, H, num_kv_heads=H, inv_freq=inv, attn_scale=1.0))


# ------------------------------------------------------------------------------------------------------------------
# wiring of _FrozenLlamaLayerFn, kernels replaced by torch formulas
# ------------------------------------------------------------------------------------------------------------------
def _rot(x):
    return torch.cat((-x[..., 64:], x[..., :64]), -1)


@pytest.fixture
def torch_kernels(monkeypatch):
    from otter_b200 import functional as F
    from otter_b200 import params as P
    calls = []

    def rmsnorm_fwd(x, w, eps, want_rstd=True):
        rstd = torch.rsqrt(x.float().pow(2).mean(-1) + eps)
        return x.float() * rstd[:, None] * w, rstd

    def rmsnorm_bwd(dy, x, rstd, w, add=None):
        xh = x.float() * rstd[:, None]
        g = dy.float() * w
        dx = rstd[:, None] * (g - xh * (g * xh).mean(-1, keepdim=True))
        return dx if add is None else dx + add

    def linear_fwd(x, w, *, out=None, residual=None, **kw):
        assert not kw
        y = x @ w.t()
        if residual is not None:
            y = y + residual
        if out is not None:
            out.copy_(y)
            return out
        return y

    def linear_dgrad(dy, w, *, residual=None, **kw):
        assert not kw
        dx = dy @ w
        return dx if residual is None else dx + residual

    def _apply_rope(buf, H, S, nblk, inv, scale, backward):
        rows = buf.shape[0]
        ang = (torch.arange(rows) % S).float()[:, None] * inv[None]
        cos = torch.cat((ang, ang), -1).cos()[:, None, None] * scale
        sin = torch.cat((ang, ang), -1).sin()[:, None, None] * scale
        if backward:
            sin = -sin
        v = buf[:, :nblk * H * 128].reshape(rows, nblk, H, 128)
        buf[:, :nblk * H * 128] = (v * cos + _rot(v) * sin).reshape(rows, -1)
        return buf

    def rope128_(buf, H, S, nblk, theta, backward=False):
        calls.append(("rope128_", H, nblk))
        inv = 1.0 / (theta ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))
        return _apply_rope(buf, H, S, nblk, inv, 1.0, backward)

    def rope128_freqs_(buf, H, S, nblk, inv_freq, attn_scale=1.0, backward=False):
        calls.append(("rope128_freqs_", H, nblk))
        assert inv_freq.dtype == torch.float32 and inv_freq.shape == (64,)
        return _apply_rope(buf, H, S, nblk, inv_freq, attn_scale, backward)

    def _attn(qkv, B, S, H, kv):
        D, Dkv = H * 128, kv * 128
        sp = lambda t, n: t.reshape(B, S, n, 128).transpose(1, 2)
        q, k, v = sp(qkv[:, :D], H), sp(qkv[:, D:D + Dkv], kv), sp(qkv[:, D + Dkv:], kv)
        k, v = k.repeat_interleave(H // kv, 1), v.repeat_interleave(H // kv, 1)
        s = (q @ k.transpose(-1, -2)) / math.sqrt(128)
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
        return (s.softmax(-1) @ v).transpose(1, 2).reshape(B * S, D)

    def lm_attn_fwd(qkv, B, S, H, *, slopes=None, causal=True, scale=None, kv_heads=None):
        assert slopes is None and causal
        calls.append(("lm_attn_fwd", kv_heads))
        return _attn(qkv, B, S, H, kv_heads or H), torch.zeros(B, H, S)

    def lm_attn_bwd(dout, qkv, out, lse, B, S, H, *, slopes=None, causal=True, scale=None, kv_heads=None):
        calls.append(("lm_attn_bwd", kv_heads))
        q = qkv.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            return torch.autograd.grad(_attn(q, B, S, H, kv_heads or H), q, dout)[0]

    def swiglu_bwd(dh, g, u):
        gr, ur = g.detach().requires_grad_(True), u.detach().requires_grad_(True)
        with torch.enable_grad():
            return torch.autograd.grad(torch.nn.functional.silu(gr) * ur, (gr, ur), dh)

    for name, fn in dict(rmsnorm_fwd=rmsnorm_fwd, rmsnorm_bwd=rmsnorm_bwd, linear_fwd=linear_fwd, linear_dgrad=linear_dgrad,
                         rope128_=rope128_, rope128_freqs_=rope128_freqs_, lm_attn_fwd=lm_attn_fwd, lm_attn_bwd=lm_attn_bwd,
                         swiglu_fwd=lambda g, u: torch.nn.functional.silu(g) * u, swiglu_bwd=swiglu_bwd).items():
        monkeypatch.setattr(F, name, fn)
    monkeypatch.setattr(P, "bf16_of", lambda p: p.detach().float())
    monkeypatch.setattr(P, "f32_of", lambda p: p.detach().float())
    from otter_b200 import lm_llama
    monkeypatch.setattr(lm_llama, "BF16", torch.float32)          # keep the stand-in arithmetic in fp32
    return calls


@pytest.mark.parametrize("H,kv,rope", [(2, 1, "llama3"), (4, 2, "yarn"), (4, 4, "linear"), (4, 2, "default")])
def test_frozen_llama_gqa_wiring_matches_hf(torch_kernels, H, kv, rope):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    B, S, D = 2, 21, H * 128
    cfg = _cfg(D, H, kv, rope)
    hf, _, x, out, w = _hf_layer_and_grad(cfg, B, S)
    mine = FrozenLlamaDecoderLayer(D, H, 3 * D, num_key_value_heads=kv, rope_parameters=cfg.rope_parameters,
                                   max_position_embeddings=cfg.max_position_embeddings)
    mine.load_state_dict(hf.state_dict(), strict=True)
    x2 = x.detach().clone().requires_grad_(True)
    y = mine(x2, position_ids=torch.arange(S)[None])
    (y * w).sum().backward()
    assert torch.allclose(y, out, rtol=1e-4, atol=1e-5)
    assert torch.allclose(x2.grad, x.grad, rtol=1e-3, atol=1e-5)
    assert all(p.grad is None for p in mine.parameters())
    rope_calls = [c for c in torch_kernels if c[0].startswith("rope")]
    if kv == H:                                   # q and k blocks in one call
        assert rope_calls == [("rope128_freqs_", H, 2)] * 2
    else:                                         # q block, then the narrower k block
        assert rope_calls == [("rope128_freqs_", H, 1), ("rope128_freqs_", kv, 1)] * 2
    want_kv = None if kv == H else kv
    assert [c for c in torch_kernels if c[0].startswith("lm_attn")] == [("lm_attn_fwd", want_kv), ("lm_attn_bwd", want_kv)]


def test_mha_default_layer_keeps_the_theta_kernel(torch_kernels):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    layer = FrozenLlamaDecoderLayer(256, 2, 512, rope_theta=5e5)
    assert not layer.table_rope and layer.num_key_value_heads == 2
    layer(torch.randn(1, 5, 256))
    assert torch_kernels == [("rope128_", 2, 2), ("lm_attn_fwd", None)]


# ------------------------------------------------------------------------------------------------------------------
# swappable() / swap_llama_layers
# ------------------------------------------------------------------------------------------------------------------
def _big_cfg(**kw):
    from transformers import LlamaConfig
    base = dict(hidden_size=4096, intermediate_size=14336, num_attention_heads=32, num_key_value_heads=8,
                num_hidden_layers=1, vocab_size=128, max_position_embeddings=131072)
    base.update(kw)
    return LlamaConfig(**base)


def test_swappable_accepts_gqa_and_scaled_rope():
    from otter_b200.lm_llama import swappable
    llama31_8b = _big_cfg(rope_parameters={"rope_type": "llama3", "rope_theta": 500000.0, "factor": 8.0,
                                           "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                           "original_max_position_embeddings": 8192})
    llama2_70b = _big_cfg(hidden_size=8192, intermediate_size=28672, num_attention_heads=64, num_key_value_heads=8,
                          max_position_embeddings=4096)
    yarn = _big_cfg(num_key_value_heads=32, rope_parameters={"rope_type": "yarn", "rope_theta": 10000.0, "factor": 4.0,
                                                             "original_max_position_embeddings": 32768})
    linear = _big_cfg(num_key_value_heads=1, rope_parameters={"rope_type": "linear", "rope_theta": 10000.0, "factor": 2.0})
    for cfg in (llama31_8b, llama2_70b, yarn, linear):
        assert swappable(cfg), cfg


def test_swappable_rejects_what_is_not_covered():
    from otter_b200.lm_llama import swappable
    dyn = _big_cfg(rope_parameters={"rope_type": "dynamic", "rope_theta": 10000.0, "factor": 2.0})
    longrope = _big_cfg()
    longrope.rope_parameters = {"rope_type": "longrope", "rope_theta": 10000.0, "short_factor": [1.0] * 64,
                                "long_factor": [1.0] * 64, "original_max_position_embeddings": 4096}
    not_dividing = _big_cfg()
    not_dividing.num_key_value_heads = 6
    hd64 = _big_cfg(num_attention_heads=64, num_key_value_heads=8)
    attn_bias = _big_cfg(attention_bias=True)
    mlp_bias = _big_cfg(mlp_bias=True)
    for cfg in (dyn, longrope, not_dividing, hd64, attn_bias, mlp_bias):
        assert not swappable(cfg), cfg


def test_layer_rejects_uncovered_arguments():
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    with pytest.raises(ValueError, match="divide"):
        FrozenLlamaDecoderLayer(512, 4, 1024, num_key_value_heads=3)
    with pytest.raises(ValueError, match="rope_type"):
        FrozenLlamaDecoderLayer(512, 4, 1024, rope_parameters={"rope_type": "dynamic", "rope_theta": 1e4, "factor": 2.0})


def test_swap_keeps_state_dict_keys_and_shapes_of_a_gqa_model():
    from transformers import LlamaForCausalLM
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer, swap_llama_layers
    cfg = _cfg(512, 4, 2, "llama3", )
    cfg.num_hidden_layers = 2
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg)
    before = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    swap_llama_layers(model)
    after = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    assert after == before
    assert after["model.layers.0.self_attn.k_proj.weight"] == (256, 512)
    for layer in model.model.layers:
        assert isinstance(layer, FrozenLlamaDecoderLayer)
        assert layer.num_key_value_heads == 2 and layer.rope_type == "llama3" and layer.table_rope
        assert torch.equal(layer.rope_inv_freq(torch.device("cpu")), model.model.rotary_emb.inv_freq.float())
        assert layer.rope_attention_scaling == model.model.rotary_emb.attention_scaling


# ------------------------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_lm_attn_struct_sizes_unchanged():
    from otter_b200 import _lib
    lib = _lib.load()
    assert lib.otb_abi_sizeof(3) == 96 == C.sizeof(_lib.LmAttnDesc)
    assert lib.otb_abi_sizeof(4) == 64 == C.sizeof(_lib.LmAttnGrads)
    assert _lib.LmAttnDesc.kv_heads.offset == 92 and _lib.LmAttnDesc._fields_[-1][0] == "kv_heads"


def test_rope_freqs_symbol_exported():
    from otter_b200 import _lib
    lib = _lib.load()
    assert hasattr(lib, "otb_rope128_freqs") and "otb_rope128_freqs" in _lib.SIGNATURES
    launches = lib.otb_launch_count()
    rc = lib.otb_rope128_freqs(C.c_void_p(0x10000), 256, 4, 1, 4, 2, None, 1.0, 0, None)     # no table
    assert rc == 1 and b"otb_rope128_freqs" in lib.otb_last_error()
    rc = lib.otb_rope128_freqs(C.c_void_p(0x10000), 256, 4, 1, 4, 2, C.c_void_p(0x20000), 0.0, 0, None)   # scale 0
    assert rc == 1
    assert lib.otb_launch_count() == launches


def test_kv_heads_not_dividing_h_is_rejected_without_a_launch():
    from otter_b200 import _lib
    lib = _lib.load()
    launches = lib.otb_launch_count()
    d = _lib.LmAttnDesc()
    d.qkv, d.out, d.lse = C.c_void_p(0x10000), C.c_void_p(0x20000), C.c_void_p(0x30000)
    d.ld_qkv, d.ld_out = 8 * 128, 4 * 128
    d.qkv_cols, d.q_col0, d.k_col0, d.v_col0, d.out_col0 = 8 * 128, 0, 4 * 128, 6 * 128, 0
    d.B, d.H, d.S, d.head_dim, d.causal, d.scale = 1, 4, 16, 128, 1, 128 ** -0.5
    for kv in (3, -1, 8):
        d.kv_heads = kv
        assert lib.otb_lm_attn_fwd(C.byref(d), None) == 1
        assert b"kv_heads" in lib.otb_last_error()
        g = _lib.LmAttnGrads()
        g.dout, g.dqkv, g.dq_ws = C.c_void_p(0x40000), C.c_void_p(0x50000), C.c_void_p(0x60000)
        g.ld_dout, g.ld_dqkv = 4 * 128, 8 * 128
        assert lib.otb_lm_attn_bwd(C.byref(d), C.byref(g), None) == 1
    d.kv_heads = 2                                 # grouped backward without a workspace: rejected too
    g.dq_ws = None
    assert lib.otb_lm_attn_bwd(C.byref(d), C.byref(g), None) == 1
    assert b"workspace" in lib.otb_last_error()
    assert lib.otb_launch_count() == launches
