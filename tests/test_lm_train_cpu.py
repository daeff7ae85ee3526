"""CPU: trainable MPT and LLaMA decoder layers (otter_b200/lm_mpt.py, otter_b200/lm_llama.py).

The CUDA entry points are replaced by plain torch formulas of what each computes (include/otter_b200.h), and every call
is recorded.  Against autograd through the reference-pinned oracles (oracle/restatement_lm.mpt_block,
oracle/restatement_llama.llama_layer and llama_layer_gqa of tests/test_llama_gqa_cpu.py):
- every parameter gradient of an unfrozen layer (MPT with and without biases; LLaMA multi-head, GQA, llama3 / yarn RoPE);
- partial unfreezing: only the parameters that require grad receive one, and a frozen weight costs no wgrad call;
- a frozen layer makes exactly the calls, with the same keyword arguments, it made before the layers could train;
- a tiny head-dim-128 MPTForCausalLM unfrozen: every parameter, norm_f and the tied wte included, gets a finite,
  non-zero gradient; left frozen, no decoder parameter gets one;
- the Otter freeze policy: train_lang_encoder=True leaves every decoder parameter trainable after init_weights.
The kernels themselves are checked on the GPU (tests/test_lm_train_gpu.py).
"""
import math

import pytest
import torch

from oracle import restatement_lm as RLM
from oracle import restatement_llama as RL
from oracle.ref_shims import FakeTokenizer
from test_llama_gqa_cpu import ROPES, llama_layer_gqa

F32 = torch.float32


def _gelu(v):
    return 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))


def _rot(x):
    return torch.cat((-x[..., 64:], x[..., :64]), -1)


@pytest.fixture
def kernels(monkeypatch):
    """Torch stand-ins for the kernels (fp32 arithmetic); returns the list of (name, sorted keyword names) calls."""
    from otter_b200 import functional as F
    from otter_b200 import lm_llama, lm_mpt
    from otter_b200 import params as P
    calls = []

    def rec(name, kw):
        calls.append((name, tuple(sorted(k for k, v in kw.items() if v is not None and v is not False))))

    def layernorm_fwd(x, g, b, eps=1e-5):
        rec("layernorm_fwd", {})
        x = x.float()
        mean = x.mean(-1)
        rstd = torch.rsqrt(x.var(-1, unbiased=False) + eps)
        return (x - mean[:, None]) * rstd[:, None] * g + b, mean, rstd

    def layernorm_bwd(dy, x, mean, rstd, g, *, add=None, want_dx=True, dgamma=None, dbeta=None, accumulate=False,
                      want_param_grads=True):
        rec("layernorm_bwd", dict(add=add, want_dx=not want_dx or None, dgamma=dgamma, dbeta=dbeta,
                                  accumulate=accumulate, want_param_grads=not want_param_grads or None))
        dy, x = dy.float(), x.float()
        xh = (x - mean[:, None]) * rstd[:, None]
        dx = None
        if want_dx:
            gy = dy * g
            dx = rstd[:, None] * (gy - gy.mean(-1, keepdim=True) - xh * (gy * xh).mean(-1, keepdim=True))
            dx = dx if add is None else dx + add.float()
        if want_param_grads:
            for t, v in ((dgamma, (dy * xh).sum(0)), (dbeta, dy.sum(0))):
                if t is not None:
                    t.copy_(t + v if accumulate else v)
        return dx, dgamma, dbeta

    def rmsnorm_fwd(x, w, eps, want_rstd=True):
        rec("rmsnorm_fwd", {})
        rstd = torch.rsqrt(x.float().pow(2).mean(-1) + eps)
        return x.float() * rstd[:, None] * w, rstd

    def rmsnorm_bwd(dy, x, rstd, w, add=None, *, dweight=None, accumulate=False):
        rec("rmsnorm_bwd", dict(add=add, dweight=dweight, accumulate=accumulate))
        xh = x.float() * rstd[:, None]
        gy = dy.float() * w
        dx = rstd[:, None] * (gy - xh * (gy * xh).mean(-1, keepdim=True))
        if dweight is not None:
            v = (dy.float() * xh).sum(0)
            dweight.copy_(dweight + v if accumulate else v)
        return dx if add is None else dx + add

    def linear_fwd(x, w, *, out=None, bias=None, act=0, aux_out=None, residual=None):
        rec("linear_fwd", dict(out=out, bias=bias, act=act or None, aux_out=aux_out, residual=residual))
        z = x.float() @ w.t() if bias is None else x.float() @ w.t() + bias
        if aux_out is not None:
            aux_out.copy_(z)
        y = _gelu(z) if act == 1 else z
        y = y if residual is None else y + residual
        if out is not None:
            out.copy_(y)
            return out
        return y

    def linear_dgrad(dy, w, *, aux_in=None, residual=None):
        rec("linear_dgrad", dict(aux_in=aux_in, residual=residual))
        dx = dy.float() @ w
        if aux_in is not None:                                        # epilogue: times gelu'(z)
            z = aux_in.detach().float().requires_grad_(True)
            with torch.enable_grad():
                dx = torch.autograd.grad(_gelu(z), z, dx)[0]
        return dx if residual is None else dx + residual

    def linear_wgrad(dy, x, *, out=None, accumulate=False):
        rec("linear_wgrad", dict(out=out, accumulate=accumulate))
        v = dy.float().t() @ x.float()
        out.copy_(out + v if accumulate else v)
        return out

    def grouped_colsum(x, div, mod, out=None, accumulate=False):
        rec("grouped_colsum", dict(out=out, accumulate=accumulate))
        assert div == 1 and mod == 1
        v = x.float().sum(0, keepdim=True)
        out.copy_(out + v if accumulate else v)
        return out

    def _attn(qkv, B, S, H, kv, slopes, scale):
        D, Dkv = H * 128, kv * 128
        sp = lambda t, n: t.reshape(B, S, n, 128).transpose(1, 2)
        q, k, v = sp(qkv[:, :D], H), sp(qkv[:, D:D + Dkv], kv), sp(qkv[:, D + Dkv:], kv)
        k, v = k.repeat_interleave(H // kv, 1), v.repeat_interleave(H // kv, 1)
        s = (q @ k.transpose(-1, -2)) * scale
        if slopes is not None:
            s = s + slopes.view(1, H, 1, 1) * torch.arange(1 - S, 1, dtype=F32).view(1, 1, 1, S)
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
        return (s.softmax(-1) @ v).transpose(1, 2).reshape(B * S, D)

    def lm_attn_fwd(qkv, B, S, H, *, slopes=None, causal=True, scale=None, kv_heads=None):
        rec("lm_attn_fwd", dict(slopes=slopes, kv_heads=kv_heads))
        return _attn(qkv.float(), B, S, H, kv_heads or H, slopes, scale), torch.zeros(B, H, S)

    def lm_attn_bwd(dout, qkv, out, lse, B, S, H, *, slopes=None, causal=True, scale=None, kv_heads=None):
        rec("lm_attn_bwd", dict(slopes=slopes, kv_heads=kv_heads))
        q = qkv.detach().float().clone().requires_grad_(True)
        with torch.enable_grad():
            return torch.autograd.grad(_attn(q, B, S, H, kv_heads or H, slopes, scale), q, dout.float())[0]

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
        rec("rope128_", dict(backward=backward))
        inv = 1.0 / (theta ** (torch.arange(0, 128, 2, dtype=F32) / 128))
        return _apply_rope(buf, H, S, nblk, inv, 1.0, backward)

    def rope128_freqs_(buf, H, S, nblk, inv_freq, attn_scale=1.0, backward=False):
        rec("rope128_freqs_", dict(backward=backward))
        return _apply_rope(buf, H, S, nblk, inv_freq, attn_scale, backward)

    def swiglu_fwd(g, u):
        rec("swiglu_fwd", {})
        return torch.nn.functional.silu(g) * u

    def swiglu_bwd(dh, g, u):
        rec("swiglu_bwd", {})
        gr, ur = g.detach().requires_grad_(True), u.detach().requires_grad_(True)
        with torch.enable_grad():
            return torch.autograd.grad(torch.nn.functional.silu(gr) * ur, (gr, ur), dh)

    for name, fn in dict(layernorm_fwd=layernorm_fwd, layernorm_bwd=layernorm_bwd, rmsnorm_fwd=rmsnorm_fwd,
                         rmsnorm_bwd=rmsnorm_bwd, linear_fwd=linear_fwd, linear_dgrad=linear_dgrad,
                         linear_wgrad=linear_wgrad, grouped_colsum=grouped_colsum, lm_attn_fwd=lm_attn_fwd,
                         lm_attn_bwd=lm_attn_bwd, rope128_=rope128_, rope128_freqs_=rope128_freqs_,
                         swiglu_fwd=swiglu_fwd, swiglu_bwd=swiglu_bwd).items():
        monkeypatch.setattr(F, name, fn)
    monkeypatch.setattr(P, "bf16_of", lambda p: p.detach().float())
    monkeypatch.setattr(P, "f32_of", lambda p: p.detach().float())
    monkeypatch.setattr(lm_llama, "BF16", F32)                        # keep the stand-in arithmetic in fp32
    real_empty = torch.empty                                          # MPT's GELU pre-activation buffer
    monkeypatch.setattr(lm_mpt.torch, "empty", lambda *a, **k: real_empty(*a, **{**k, "dtype": F32}))
    real_fn = lm_mpt._FrozenMPTBlockFn.apply
    monkeypatch.setattr(lm_mpt._FrozenMPTBlockFn, "apply", staticmethod(lambda x, *a: real_fn(x.float(), *a)))
    return calls


def _perturb_norms(module, seed):
    torch.manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))


def _check_grads(module, ref_params, names=None):
    """Every parameter that requires grad has the oracle's gradient (1e-3 rel / 1e-5 abs); the others have none."""
    seen = 0
    for n, p in module.named_parameters():
        if names is not None and n not in names:
            assert p.grad is None, n
            continue
        assert p.grad is not None, n
        ref = ref_params[n].grad
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-5), (n, (p.grad - ref).abs().max().item())
        seen += 1
    return seen


def _bf16_exact(*shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).bfloat16().float()


# ------------------------------------------------------------------------------------------------------------------
# MPT block
# ------------------------------------------------------------------------------------------------------------------
def _mpt_case(no_bias, trainable=None, seed=1):
    from otter_b200.lm_mpt import FrozenMPTBlock
    B, S, D, H = 2, 19, 256, 2
    blk = FrozenMPTBlock(D, H, no_bias=no_bias)
    _perturb_norms(blk, seed)
    for n, p in blk.named_parameters():
        p.requires_grad_(trainable is None or n in trainable)
    p_ref = {k: v.detach().clone().requires_grad_(True) for k, v in blk.named_parameters()}
    # bf16-representable input and upstream gradient: the module's bf16 casts are then lossless
    x, w = _bf16_exact(B, S, D, seed=seed), _bf16_exact(B, S, D, seed=seed + 1)
    ref = RLM.mpt_block(x, p_ref, H)
    (ref * w).sum().backward()
    y, _, _ = blk(x.clone())
    (y * w).sum().backward()
    assert torch.allclose(y, ref, rtol=1e-4, atol=1e-5)
    return blk, p_ref


@pytest.mark.parametrize("no_bias", [True, False])
def test_unfrozen_mpt_block_parameter_grads_match_the_oracle(kernels, no_bias):
    blk, p_ref = _mpt_case(no_bias)
    assert _check_grads(blk, p_ref) == (6 if no_bias else 12)


def test_partially_unfrozen_mpt_block(kernels):
    names = {"ffn.down_proj.weight", "norm_1.bias", "attn.Wqkv.bias"}
    blk, p_ref = _mpt_case(False, trainable=names)
    assert _check_grads(blk, p_ref, names) == 3
    assert [c[0] for c in kernels].count("linear_wgrad") == 1               # a frozen weight costs no wgrad launch
    assert [c[0] for c in kernels].count("grouped_colsum") == 1
    ln_param_calls = [c for c in kernels if c[0] == "layernorm_bwd" and "dgamma" in c[1]]
    assert len(ln_param_calls) == 1 and "dbeta" in ln_param_calls[0][1]      # norm_1 only


# the calls _FrozenMPTBlockFn made before its layers could train (one forward + backward, biases present)
MPT_FROZEN_CALLS = [
    ("layernorm_fwd", ()), ("linear_fwd", ("bias",)), ("lm_attn_fwd", ("slopes",)), ("linear_fwd", ("bias", "residual")),
    ("layernorm_fwd", ()), ("linear_fwd", ("act", "aux_out", "bias")), ("linear_fwd", ("bias", "residual")),
    ("linear_dgrad", ("aux_in",)), ("linear_dgrad", ()), ("layernorm_bwd", ("add", "want_param_grads")),
    ("linear_dgrad", ()), ("lm_attn_bwd", ("slopes",)), ("linear_dgrad", ()), ("layernorm_bwd", ("add", "want_param_grads")),
]


def test_frozen_mpt_block_makes_the_same_calls(kernels):
    from otter_b200.lm_mpt import FrozenMPTBlock
    blk = FrozenMPTBlock(256, 2, no_bias=False)
    x = torch.randn(1, 9, 256, requires_grad=True)
    y, _, _ = blk(x)
    y.sum().backward()
    assert kernels == MPT_FROZEN_CALLS
    assert x.grad is not None and all(p.grad is None for p in blk.parameters())


# ------------------------------------------------------------------------------------------------------------------
# LLaMA layer
# ------------------------------------------------------------------------------------------------------------------
def _llama_case(H, kv, rope, trainable=None, seed=2):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    B, S, D = 2, 21, H * 128
    kw = {} if (kv == H and rope == "default") else dict(num_key_value_heads=kv, rope_parameters=ROPES[rope],
                                                         max_position_embeddings=256)
    layer = FrozenLlamaDecoderLayer(D, H, 3 * D, **kw)
    _perturb_norms(layer, seed)
    torch.manual_seed(seed)
    with torch.no_grad():
        for p in layer.parameters():
            if p.dim() == 2:
                p.copy_(torch.randn_like(p) / math.sqrt(p.shape[1]))
    for n, p in layer.named_parameters():
        p.requires_grad_(trainable is None or n in trainable)
    p_ref = {k: v.detach().clone().requires_grad_(True) for k, v in layer.named_parameters()}
    x, w = _bf16_exact(B, S, D, seed=seed), _bf16_exact(B, S, D, seed=seed + 1)
    if kw:
        ref = llama_layer_gqa(x, p_ref, H, num_kv_heads=kv, inv_freq=layer.rope_inv_freq(torch.device("cpu")),
                              attn_scale=layer.rope_attention_scaling)
    else:
        ref = RL.llama_layer(x, p_ref, H)
    (ref * w).sum().backward()
    xg = x.clone().requires_grad_(True)
    y = layer(xg, position_ids=torch.arange(S)[None])
    (y * w).sum().backward()
    assert torch.allclose(y, ref, rtol=1e-4, atol=1e-5)
    return layer, p_ref


@pytest.mark.parametrize("H,kv,rope", [(2, 2, "default"), (4, 2, "llama3"), (4, 1, "yarn")])
def test_unfrozen_llama_layer_parameter_grads_match_the_oracle(kernels, H, kv, rope):
    layer, p_ref = _llama_case(H, kv, rope)
    assert _check_grads(layer, p_ref) == 9
    assert layer.self_attn.k_proj.weight.grad.shape == (kv * 128, H * 128)
    assert [c for c in kernels if c[0] == "rmsnorm_bwd"] == [("rmsnorm_bwd", ("add", "dweight"))] * 2


def test_partially_unfrozen_llama_layer(kernels):
    names = {"self_attn.k_proj.weight", "mlp.up_proj.weight", "post_attention_layernorm.weight"}
    layer, p_ref = _llama_case(4, 2, "llama3", trainable=names)
    assert _check_grads(layer, p_ref, names) == 3
    assert [c[0] for c in kernels].count("linear_wgrad") == 2
    assert [c for c in kernels if c[0] == "rmsnorm_bwd"] == [("rmsnorm_bwd", ("add", "dweight")), ("rmsnorm_bwd", ("add",))]


# the calls _FrozenLlamaLayerFn made before its layers could train (forward + backward)
def _llama_frozen_calls(gqa):
    rope, attn = ("rope128_freqs_", (("kv_heads",))) if gqa else ("rope128_", ())
    ropes = 2 if gqa else 1                                            # GQA: q block and k block apart
    return ([("rmsnorm_fwd", ())] + [("linear_fwd", ("out",))] * 3 + [(rope, ())] * ropes + [("lm_attn_fwd", attn)]
            + [("linear_fwd", ("residual",)), ("rmsnorm_fwd", ()), ("linear_fwd", ()), ("linear_fwd", ()),
               ("swiglu_fwd", ()), ("linear_fwd", ("residual",))]
            + [("linear_dgrad", ()), ("swiglu_bwd", ()), ("linear_dgrad", ()), ("linear_dgrad", ("residual",)),
               ("rmsnorm_bwd", ("add",)), ("linear_dgrad", ()), ("lm_attn_bwd", attn)] + [(rope, ("backward",))] * ropes
            + [("linear_dgrad", ()), ("linear_dgrad", ("residual",)), ("linear_dgrad", ("residual",)),
               ("rmsnorm_bwd", ("add",))])


@pytest.mark.parametrize("gqa", [False, True])
def test_frozen_llama_layer_makes_the_same_calls(kernels, gqa):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    kw = dict(num_key_value_heads=1, rope_parameters=ROPES["llama3"], max_position_embeddings=256) if gqa else {}
    layer = FrozenLlamaDecoderLayer(256, 2, 512, **kw)
    x = torch.randn(1, 9, 256, requires_grad=True)
    layer(x).sum().backward()
    assert kernels == _llama_frozen_calls(gqa)
    assert x.grad is not None and all(p.grad is None for p in layer.parameters())


def test_constructors_and_swap_still_freeze():
    from transformers import LlamaConfig, LlamaForCausalLM
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer, swap_llama_layers
    from otter_b200.lm_mpt import FrozenMPTBlock
    assert not any(p.requires_grad for p in FrozenMPTBlock(256, 2).parameters())
    assert not any(p.requires_grad for p in FrozenLlamaDecoderLayer(256, 2, 512).parameters())
    cfg = LlamaConfig(vocab_size=32, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2)
    model = swap_llama_layers(LlamaForCausalLM(cfg))
    assert not any(p.requires_grad for p in model.model.layers.parameters())


# ------------------------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------------------------
def _tiny_mpt(no_bias=True):
    from otter_b200.lm_mpt import MPTConfig, MPTForCausalLM
    cfg = MPTConfig(d_model=256, n_heads=2, n_layers=2, expansion_ratio=2, max_seq_len=64, vocab_size=64, no_bias=no_bias,
                    attn_config={"alibi": True, "attn_impl": "torch"})
    torch.manual_seed(4)
    return MPTForCausalLM(cfg)


@pytest.mark.parametrize("no_bias", [True, False])
def test_unfrozen_mpt_causal_lm_gets_every_gradient(kernels, no_bias):
    model = _tiny_mpt(no_bias)
    _perturb_norms(model, 5)
    model.requires_grad_(True)
    ids = torch.randint(0, 64, (2, 17))
    logits = model(input_ids=ids).logits
    torch.nn.functional.cross_entropy(logits[:, :-1].reshape(-1, 64).float(), ids[:, 1:].reshape(-1)).backward()
    names = [n for n, _ in model.named_parameters()]
    assert "transformer.norm_f.weight" in names and "transformer.wte.weight" in names
    for n, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0, n


def test_frozen_mpt_causal_lm_gives_no_decoder_gradient(kernels):
    model = _tiny_mpt(no_bias=False)
    model.requires_grad_(False)
    model.transformer.wte.requires_grad_(True)                          # as Otter's freeze policy leaves it
    ids = torch.randint(0, 64, (2, 17))
    model(input_ids=ids).logits.float().pow(2).mean().backward()
    assert model.transformer.wte.weight.grad is not None
    assert all(p.grad is None for n, p in model.named_parameters() if n != "transformer.wte.weight")
    assert [c[0] for c in kernels].count("linear_wgrad") == 1                      # the tied un-embedding's only
    assert not any(c[0] == "grouped_colsum" or "dgamma" in c[1] or "dweight" in c[1] for c in kernels)


# ------------------------------------------------------------------------------------------------------------------
# the Otter freeze policy (host logic only, no forward)
# ------------------------------------------------------------------------------------------------------------------
def _otter_cfg(text_config, **flags):
    from otter_b200 import otter_hf
    vc = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=1, num_attention_heads=16, image_size=224,
              patch_size=14, hidden_act="quick_gelu")          # the CLIP-L width the perceiver is built for
    cfg = otter_hf.OtterConfig(vision_config=vc, text_config=text_config, cross_attn_every_n_layers=1)
    for k, v in flags.items():
        setattr(cfg, k, v)
    return cfg


def _mpt_text_config():
    return dict(architectures=["MPTForCausalLM"], _name_or_path="mpt-tiny", d_model=256, n_heads=2, n_layers=2,
                expansion_ratio=2, max_seq_len=64, vocab_size=64, no_bias=True, attn_config={"alibi": True})


def _llama_text_config():
    from transformers import LlamaConfig
    td = LlamaConfig(vocab_size=64, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                     num_key_value_heads=1, max_position_embeddings=256).to_dict()
    td["_name_or_path"], td["architectures"] = "llama-tiny", ["LlamaForCausalLM"]
    return td


@pytest.mark.parametrize("lm", ["mpt", "llama"])
@pytest.mark.parametrize("train", [True, False])
def test_train_lang_encoder_unfreezes_the_swapped_decoder(monkeypatch, lm, train):
    from otter_b200 import otter_hf
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    from otter_b200.lm_mpt import FrozenMPTBlock
    monkeypatch.setattr(otter_hf, "AutoTokenizer", FakeTokenizer)
    monkeypatch.setenv("OTB_LLAMA_LAYERS", "1")
    td = _mpt_text_config() if lm == "mpt" else _llama_text_config()
    model = otter_hf.OtterForConditionalGeneration(_otter_cfg(td, train_lang_encoder=train))
    cls = FrozenMPTBlock if lm == "mpt" else FrozenLlamaDecoderLayer
    layers = [m for m in model.lang_encoder.modules() if isinstance(m, cls)]
    assert len(layers) == 2
    for layer in layers:
        assert all(p.requires_grad == train for p in layer.parameters())
    final_norm = model.lang_encoder.transformer.norm_f if lm == "mpt" else model.lang_encoder.model.norm
    assert final_norm.weight.requires_grad == train
