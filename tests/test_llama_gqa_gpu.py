"""GPU: grouped-query attention (GQA) and table-driven (scaled) RoPE on the sm_90a kernels, and the LLaMA layers, HF model
and Otter model that use them.

- otb_lm_attn_fwd / _bwd with kv_heads < H against float64, with the metric of tests/test_attention_edges_gpu.py: O, LSE,
  dQ and the group-summed dK / dV, at the 64 / 128 tile edges and at S = 2048 with 32 heads / 8 K/V heads; a NaN canary
  through the C ABI with offset column blocks; bit-identical repeated backward runs.
- otb_rope128_freqs against float64 for each covered rope_type, q and k blocks of different head counts, forward and
  backward; with HF's default table it agrees with otb_rope128.
- FrozenLlamaDecoderLayer with GQA + llama3 / yarn against the oracle; a Llama-3-style LlamaForCausalLM swapped and
  unswapped; an OtterForConditionalGeneration over that LM.  The layer's oracle is llama_layer_gqa of
  tests/test_llama_gqa_cpu.py.
"""
import ctypes as C

import pytest
import torch

from oracle.ref_shims import FakeTokenizer
from test_llama_gqa_cpu import llama_layer_gqa
from test_attention_edges_gpu import _Canvas, _check, _heads, _mask64, _rnd, _stack, ref_attention

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
def _gqa_inputs(B, S, H, kv, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = _rnd(g, B * S, (H + 2 * kv) * 128, scale=0.8).to(DEV)
    dout = _rnd(g, B * S, H * 128, scale=0.5).to(DEV)
    return qkv, dout


def _gqa_refs(qkv, q0, k0, v0, dout, o, B, S, H, kv):
    """Per query head h: float64 attention over K/V head h // (H / kv); dK / dV summed over the group."""
    grp = H // kv
    allowed, _ = _mask64(B, S, S, DEV, causal=True)
    hq, hk, hv = _heads(qkv, B, S, q0, H, 128), _heads(qkv, B, S, k0, kv, 128), _heads(qkv, B, S, v0, kv, 128)
    hdo, ho = _heads(dout, B, S, 0, H, 128), _heads(o, B, S, 0, H, 128)
    refs = [ref_attention(hq[:, h], hk[:, h // grp], hv[:, h // grp], 128 ** -0.5, allowed, dout=hdo[:, h], o_given=ho[:, h])
            for h in range(H)]
    dk = torch.stack([sum(refs[j * grp + r]["dk"] for r in range(grp)) for j in range(kv)], 1)
    dv = torch.stack([sum(refs[j * grp + r]["dv"] for r in range(grp)) for j in range(kv)], 1)
    return refs, dk, dv


def _run_gqa(tag, B, S, H, kv):
    from otter_b200 import functional as F
    qkv, dout = _gqa_inputs(B, S, H, kv, S * 10 + H + kv + B)
    out, lse = F.lm_attn_fwd(qkv, B, S, H, kv_heads=kv)
    dqkv = F.lm_attn_bwd(dout, qkv, out, lse, B, S, H, kv_heads=kv)
    torch.cuda.synchronize()
    D, Dkv = H * 128, kv * 128
    refs, dk, dv = _gqa_refs(qkv, 0, D, D + Dkv, dout, out, B, S, H, kv)
    _check(f"{tag} O", _heads(out, B, S, 0, H, 128), _stack(refs, "o"))
    _check(f"{tag} lse", lse, _stack(refs, "lse"), lse=True)
    _check(f"{tag} dq", _heads(dqkv, B, S, 0, H, 128), _stack(refs, "dq"))
    _check(f"{tag} dk", _heads(dqkv, B, S, D, kv, 128), dk)
    _check(f"{tag} dv", _heads(dqkv, B, S, D + Dkv, kv, 128), dv)
    return qkv, dout, out, lse, dqkv


@pytest.mark.parametrize("B,S,H,kv", [
    # group sizes 2, 4, 8 and one K/V head (MQA); S at the 64-key backward and 128-key forward tile edges
    (2, 1, 4, 2), (1, 63, 8, 2), (2, 64, 8, 1), (1, 65, 2, 1), (2, 127, 4, 2), (1, 128, 8, 1), (2, 129, 16, 2),
    (1, 193, 4, 1), (2, 320, 8, 4),
])
def test_gqa_attention_fwd_bwd(B, S, H, kv):
    _run_gqa(f"gqa[{B}-{S}-{H}-{kv}]", B, S, H, kv)


def test_gqa_attention_llama3_8b_shape():
    """S = 2048, 32 query heads, 8 K/V heads (Llama-3-8B / Llama-3.1-8B attention)."""
    _run_gqa("gqa-llama3-8b", 1, 2048, 32, 8)


def test_gqa_backward_is_bit_deterministic():
    from otter_b200 import functional as F
    B, S, H, kv = 2, 320, 8, 2
    qkv, dout = _gqa_inputs(B, S, H, kv, 7)
    out, lse = F.lm_attn_fwd(qkv, B, S, H, kv_heads=kv)
    a = F.lm_attn_bwd(dout, qkv, out, lse, B, S, H, kv_heads=kv)
    b = F.lm_attn_bwd(dout, qkv, out, lse, B, S, H, kv_heads=kv)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("B,S,H,kv", [(2, 130, 4, 2), (1, 64, 4, 1)])
def test_canary_gqa_lm_attn_fwd_bwd(B, S, H, kv):
    """Column blocks at offsets other than functional's: K first, then V, then Q; a NaN-filled workspace."""
    from otter_b200 import _lib
    lib = _lib.load()
    D, Dkv = H * 128, kv * 128
    qkv, dout = _gqa_inputs(B, S, H, kv, 5 + S)
    k0, v0, q0 = 8, Dkv + 24, 2 * Dkv + 40
    width = D + 2 * Dkv
    cqkv = _Canvas(B * S + 3, width + 64).put(qkv[:, D:D + Dkv], k0).put(qkv[:, D + Dkv:], v0).put(qkv[:, :D], q0)
    co, clse = _Canvas(B * S + 2, D + 64), _Canvas(1, B * H * S + 5, torch.float32)
    o_view, lse_view = co.own(B * S, 24, 24 + D), clse.own(1, 0, B * H * S)
    d = _lib.LmAttnDesc()
    d.qkv, d.out, d.lse, d.alibi_slopes = cqkv.ptr(), co.ptr(), clse.ptr(), None
    d.ld_qkv, d.ld_out = cqkv.t.stride(0), co.t.stride(0)
    d.qkv_cols, d.q_col0, d.k_col0, d.v_col0, d.out_col0 = width + 48, q0, k0, v0, 24
    d.B, d.H, d.S, d.head_dim, d.causal, d.scale, d.kv_heads = B, H, S, 128, 1, 128 ** -0.5, kv
    _lib.check(lib.otb_lm_attn_fwd(C.byref(d), _stream()), "otb_lm_attn_fwd")
    torch.cuda.synchronize()
    co.check("gqa otb_lm_attn_fwd out")
    clse.check("gqa otb_lm_attn_fwd lse")

    cdo = _Canvas(B * S + 2, D + 32).put(dout, 16)
    cdqkv = _Canvas(B * S + 3, width + 64)
    dk_view, dv_view = cdqkv.own(B * S, 8, 8 + Dkv), cdqkv.own(B * S, Dkv + 16, 2 * Dkv + 16)
    dq_view = cdqkv.own(B * S, 2 * Dkv + 24, 2 * Dkv + 24 + D)
    ws = torch.full((3, B * S, H * 128), float("nan"), dtype=torch.float32, device=DEV)
    gr = _lib.LmAttnGrads()
    gr.dout, gr.dqkv, gr.dq_ws = cdo.ptr(), cdqkv.ptr(), C.c_void_p(ws.data_ptr())
    gr.ld_dout, gr.ld_dqkv = cdo.t.stride(0), cdqkv.t.stride(0)
    gr.dout_cols, gr.dout_col0, gr.dq_col0, gr.dk_col0, gr.dv_col0 = D + 24, 16, 2 * Dkv + 24, 8, Dkv + 16
    _lib.check(lib.otb_lm_attn_bwd(C.byref(d), C.byref(gr), _stream()), "otb_lm_attn_bwd")
    torch.cuda.synchronize()
    cdqkv.check("gqa otb_lm_attn_bwd dqkv")

    refs, dk, dv = _gqa_refs(qkv, 0, D, D + Dkv, dout, o_view, B, S, H, kv)
    _check("canary gqa O", _heads(o_view, B, S, 0, H, 128), _stack(refs, "o"))
    _check("canary gqa lse", lse_view.reshape(B, H, S), _stack(refs, "lse"), lse=True)
    _check("canary gqa dq", _heads(dq_view, B, S, 0, H, 128), _stack(refs, "dq"))
    _check("canary gqa dk", _heads(dk_view, B, S, 0, kv, 128), dk)
    _check("canary gqa dv", _heads(dv_view, B, S, 0, kv, 128), dv)


# ------------------------------------------------------------------------------------------------------------------
# table-driven RoPE
# ------------------------------------------------------------------------------------------------------------------
ROPES = {
    "default": {"rope_type": "default", "rope_theta": 500000.0},
    "linear": {"rope_type": "linear", "rope_theta": 10000.0, "factor": 4.0},
    "llama3": {"rope_type": "llama3", "rope_theta": 500000.0, "factor": 8.0, "low_freq_factor": 1.0,
               "high_freq_factor": 4.0, "original_max_position_embeddings": 8192},
    "yarn": {"rope_type": "yarn", "rope_theta": 10000.0, "factor": 4.0, "original_max_position_embeddings": 4096},
}
A_ROPE = B_ROPE = 2.0 ** -7        # tests/test_rowwise_edges_gpu.py: bf16 output rounding + bf16 inputs to the rotation


def _rope_ratio(got, ref):
    """Per head (last dim 128): |got - ref| <= 2^-7 |ref| + 2^-7 rms(ref head)."""
    got, ref = got.double(), ref.double()
    rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    return ((got - ref).abs() / (A_ROPE * ref.abs() + B_ROPE * rms + 2.0 ** -30)).max().item()


def _rope64(x, S, inv, scale, backward):
    """float64 rotation of x [rows, nh, 128] (row position = row % S)."""
    ang = (torch.arange(x.shape[0], device=x.device) % S).double()[:, None] * inv.double()[None]
    cos, sin = torch.cat((ang, ang), -1).cos()[:, None] * scale, torch.cat((ang, ang), -1).sin()[:, None] * scale
    if backward:
        sin = -sin
    xd = x.double()
    return xd * cos + torch.cat((-xd[..., 64:], xd[..., :64]), -1) * sin


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("rope", list(ROPES))
def test_rope_table_vs_float64(rope, backward):
    from otter_b200 import functional as F
    from otter_b200.lm_llama import rope_table
    H, kv, B, S = 8, 2, 2, 2048
    inv, scale = rope_table(H * 128, H, ROPES[rope], max_position_embeddings=131072)
    inv_d = inv.to(DEV)
    g = torch.Generator().manual_seed(len(rope) + backward)
    width = (H + 2 * kv) * 128
    buf = torch.full((B * S, width + 16), float("nan"), dtype=BF16, device=DEV)
    src = _rnd(g, B * S, width).to(DEV)
    buf[:, :width] = src
    F.rope128_freqs_(buf[:, :H * 128], H, S, 1, inv_d, scale, backward=backward)
    F.rope128_freqs_(buf[:, H * 128:(H + kv) * 128], kv, S, 1, inv_d, scale, backward=backward)
    torch.cuda.synchronize()
    rq = _rope64(src[:, :H * 128].view(B * S, H, 128), S, inv_d, scale, backward)
    rk = _rope64(src[:, H * 128:(H + kv) * 128].view(B * S, kv, 128), S, inv_d, scale, backward)
    r1 = _rope_ratio(buf[:, :H * 128].view(B * S, H, 128), rq)
    r2 = _rope_ratio(buf[:, H * 128:(H + kv) * 128].view(B * S, kv, 128), rk)
    print(f"RATIO rope[{rope}-{backward}] q {r1:.4f} k {r2:.4f} (scale {scale:.4f})")
    assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
    assert torch.equal(buf[:, (H + kv) * 128:width].view(torch.int16), src[:, (H + kv) * 128:].view(torch.int16))
    assert torch.isnan(buf[:, width:].float()).all()


def test_rope_default_table_matches_theta_kernel():
    from otter_b200 import functional as F
    from otter_b200.lm_llama import rope_table
    H, S, theta = 4, 4096, 500000.0
    inv, scale = rope_table(H * 128, H, {"rope_type": "default", "rope_theta": theta})
    assert scale == 1.0
    g = torch.Generator().manual_seed(2)
    src = _rnd(g, S, 3 * H * 128).to(DEV)
    a, b = src.clone(), src.clone()
    F.rope128_(a, H, S, 2, theta)
    F.rope128_freqs_(b, H, S, 2, inv.to(DEV), 1.0)
    torch.cuda.synchronize()
    r = _rope_ratio(b[:, :2 * H * 128].view(S, 2 * H, 128), a[:, :2 * H * 128].view(S, 2 * H, 128))
    print(f"RATIO rope default table vs theta {r:.4f}")
    assert r <= 1.0
    assert torch.equal(a[:, 2 * H * 128:].view(torch.int16), b[:, 2 * H * 128:].view(torch.int16))


# ------------------------------------------------------------------------------------------------------------------
# the layer, an HF model, an Otter model
# ------------------------------------------------------------------------------------------------------------------
def _rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-20)).item()


@pytest.mark.parametrize("B,S,D,H,kv,rope", [(2, 100, 512, 4, 2, "llama3"), (1, 300, 1024, 8, 2, "yarn"),
                                              (1, 257, 1024, 8, 1, "llama3"), (1, 130, 512, 4, 4, "linear")])
def test_frozen_llama_gqa_layer_vs_oracle(B, S, D, H, kv, rope):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    torch.manual_seed(S)
    layer = FrozenLlamaDecoderLayer(D, H, 3 * D, num_key_value_heads=kv, rope_parameters=ROPES[rope],
                                    max_position_embeddings=131072)
    with torch.no_grad():
        layer.input_layernorm.weight.add_(0.1 * torch.randn(D))
        layer.post_attention_layernorm.weight.add_(0.1 * torch.randn(D))
    p_ref = {k: v.detach().clone() for k, v in layer.state_dict().items()}
    inv = layer.rope_inv_freq(torch.device("cpu"))
    layer.to(DEV)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, S, D, generator=g).to(BF16).float()
    w = torch.randn(B, S, D, generator=g).to(BF16).float()
    xg = x.to(DEV).requires_grad_(True)
    y = layer(xg, position_ids=torch.arange(S, device=DEV)[None])
    (y.float() * w.to(DEV)).sum().backward()
    xr = x.clone().requires_grad_(True)
    ref = llama_layer_gqa(xr, p_ref, H, num_kv_heads=kv, inv_freq=inv, attn_scale=layer.rope_attention_scaling)
    (ref * w).sum().backward()
    print(f"REL layer[{B}-{S}-{D}-{H}-{kv}-{rope}] y {_rel(y, ref):.2e} dx {_rel(xg.grad, xr.grad):.2e}")
    assert _rel(y, ref) <= 1.5e-2, _rel(y, ref)
    assert _rel(xg.grad, xr.grad) <= 3e-2, _rel(xg.grad, xr.grad)
    assert all(p.grad is None for p in layer.parameters())


def _llama3_text_config(vocab=64, layers=2):
    from transformers import LlamaConfig
    return LlamaConfig(vocab_size=vocab, hidden_size=512, intermediate_size=1024, num_hidden_layers=layers,
                       num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=512,
                       rope_parameters={"rope_type": "llama3", "rope_theta": 500000.0, "factor": 8.0,
                                        "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                        "original_max_position_embeddings": 64})


def test_swap_gqa_llama3_layers_in_an_hf_model():
    from transformers import LlamaForCausalLM
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer, swap_llama_layers, swappable
    cfg = _llama3_text_config()
    assert swappable(cfg)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).to(DEV)
    ids = torch.randint(0, 64, (2, 150), device=DEV)
    mask = torch.ones_like(ids)
    mask[1, 110:] = 0                                                                     # right padding
    with torch.no_grad():
        ref = model(input_ids=ids, attention_mask=mask, use_cache=False).logits.float()
    keys = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    swap_llama_layers(model)
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == keys
    assert all(isinstance(l, FrozenLlamaDecoderLayer) and l.num_key_value_heads == 2 for l in model.model.layers)
    with torch.no_grad():
        got = model(input_ids=ids, attention_mask=mask, use_cache=False).logits.float()
    valid = mask.bool()
    print(f"REL hf llama3 gqa logits {_rel(got[valid], ref[valid]):.2e}")
    assert _rel(got[valid], ref[valid]) <= 2e-2, _rel(got[valid], ref[valid])
    # incremental decoding with a KV cache is handed to the HF layer
    calls = []
    hook = model.model.layers[0]._hf_layer.register_forward_hook(lambda *a: calls.append(1))
    with torch.no_grad():
        out = model(input_ids=ids[:1], use_cache=True)
    hook.remove()
    assert calls and out.past_key_values is not None and _rel(out.logits, ref[:1]) <= 2e-2


def _otter(monkeypatch, swap):
    from otter_b200 import otter_hf
    monkeypatch.setattr(otter_hf, "AutoTokenizer", FakeTokenizer)
    monkeypatch.setenv("OTB_LLAMA_LAYERS", "1" if swap else "0")
    td = _llama3_text_config(vocab=68).to_dict()
    td["_name_or_path"] = "llama-tiny"
    td["architectures"] = ["LlamaForCausalLM"]
    vc = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=1, num_attention_heads=16, image_size=224,
              patch_size=14, hidden_act="quick_gelu")          # the CLIP-L width the perceiver is built for
    cfg = otter_hf.OtterConfig(vision_config=vc, text_config=td, cross_attn_every_n_layers=2)
    cfg.text_config._name_or_path = "llama-tiny"
    cfg.text_config.architectures = ["LlamaForCausalLM"]
    return otter_hf.OtterForConditionalGeneration(cfg)


def test_otter_over_a_gqa_llama3_lm(monkeypatch):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer
    torch.manual_seed(0)
    a = _otter(monkeypatch, True)
    b = _otter(monkeypatch, False)
    b.load_state_dict(a.state_dict(), strict=True)
    lang = [m for m in a.lang_encoder.modules()]
    assert sum(isinstance(m, FrozenLlamaDecoderLayer) for m in lang) == 2
    assert not any(isinstance(m, LlamaDecoderLayer) for m in lang)
    assert sum(isinstance(m, LlamaDecoderLayer) for m in b.lang_encoder.modules()) == 2
    a.to(DEV), b.to(DEV)
    g = torch.Generator().manual_seed(3)
    vision_x = torch.randn(2, 1, 1, 3, 224, 224, generator=g).to(DEV)
    lang_x = torch.randint(3, 60, (2, 40), generator=g)
    lang_x[:, 0] = a.media_token_id
    lang_x = lang_x.to(DEV)
    labels = lang_x.clone()
    outs = []
    for m in (a, b):
        o = m(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x), labels=labels)
        outs.append(o)
    la, lb = outs[0].loss.item(), outs[1].loss.item()
    print(f"otter gqa llama3: loss {la:.5f} vs {lb:.5f}, logits rel {_rel(outs[0].logits, outs[1].logits):.2e}")
    assert abs(la - lb) <= 2e-2 * abs(lb), (la, lb)
    assert _rel(outs[0].logits, outs[1].logits) <= 2e-2
    outs[0].loss.backward()
    grads = [p.grad for p in a.parameters() if p.requires_grad and p.grad is not None]
    assert grads and all(torch.isfinite(g_).all() for g_ in grads) and any(g_.abs().sum() > 0 for g_ in grads)
