"""CPU: LoRA adapters (otter_b200/lora.py) on the MPT and LLaMA decoder layers.

- The numpy Philox4x32-10 mirror of csrc/otb_lora.cu passes the Random123 known-answer vectors, and the keep mask it
  derives follows the rule documented in include/otter_b200.h.
- float64 LoRA oracles (llama_layer_lora, mpt_block_lora, with explicit dropout masks) are pinned against HF's
  LlamaDecoderLayer with LoraLinear q / v projections (fixed masks substituted for the dropout modules) and against the
  reference-pinned MPT block with the adapter merged into Wqkv; "power" checks show the adapter-delta metric of
  tests/test_lora_gpu.py rejects a missing scaling, a q / v shared mask, a backward mask unlike the forward's and the
  adapter added after RoPE.
- The layers' kernel path with the CUDA entry points replaced by torch formulas (the `kernels` fixture of
  tests/test_lm_train_cpu.py, plus the dropout mirror) matches the oracles, masks and gradients included.
- Wrapping: tiny Otter-LLaMA (swapped layers, GQA) and Otter-MPT models with lora_config build without peft, with peft's
  state-dict layout, Otter's trainable set, the KV-cache HF layer sharing the adapters, the rank rule, and a
  save / load round trip of the trainable checkpoint.
"""
import math

import numpy as np
import pytest
import torch

from oracle import restatement_lm as RLM
from oracle import restatement_llama as RL
from oracle.ref_shims import FakeTokenizer
from test_llama_gqa_cpu import ROPES, _cfg
from test_lm_train_cpu import _bf16_exact, _llama_text_config, _mpt_text_config, _otter_cfg, _perturb_norms, kernels  # noqa: F401

F64 = torch.float64
_M32 = np.uint64(0xFFFFFFFF)
SEED = 0x0123456789ABCDEF


# ------------------------------------------------------------------------------------------------------------------
# Philox4x32-10 mirror and the keep rule
# ------------------------------------------------------------------------------------------------------------------
def philox4x32_10(ctr, key):
    """ctr uint [n, 4], key uint [n, 2] -> uint32 [n, 4] (Random123's philox4x32 with 10 rounds)."""
    c = [np.asarray(ctr[..., i], dtype=np.uint64) for i in range(4)]
    k0, k1 = np.asarray(key[..., 0], dtype=np.uint64), np.asarray(key[..., 1], dtype=np.uint64)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return np.stack(c, -1).astype(np.uint32)


def keep_threshold(p):
    """(uint32_t)floor((double)p * 2^32) with p an fp32 value, as the entry points compute it."""
    return int(float(np.float32(p)) * 2.0 ** 32)


def dropout_scale(p):
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def keep_mask(rows, cols, p, seed, stream_id):
    """bool [rows, cols]: element e = row * cols + col is kept iff word e % 4 of Philox(counter {lo(e/4), hi(e/4),
    stream_id, 0}, key {lo(seed), hi(seed)}) >= keep_threshold(p)."""
    e = np.arange(rows * cols, dtype=np.uint64)
    q = e >> np.uint64(2)
    ctr = np.stack([q & _M32, q >> np.uint64(32), np.full_like(q, stream_id), np.zeros_like(q)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64), (len(q), 2))
    words = philox4x32_10(ctr, key)[np.arange(len(q)), (e & np.uint64(3)).astype(np.int64)]
    return torch.from_numpy((words.astype(np.uint64) >= keep_threshold(p)).reshape(rows, cols))


@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_philox_known_answers(ctr, key, want):
    got = philox4x32_10(np.array([ctr], dtype=np.uint64), np.array([key], dtype=np.uint64))[0]
    assert [int(v) for v in got] == want


def test_keep_mask_follows_the_documented_rule():
    rows, cols, p, seed, sid = 3, 40, 0.3, 0xA409382229F31D0, 5
    m = keep_mask(rows, cols, p, seed, sid)
    thr = keep_threshold(p)
    for r, c in [(0, 0), (0, 3), (1, 7), (2, 39), (2, 17)]:
        e = r * cols + c
        ctr = np.array([[(e // 4) & 0xFFFFFFFF, e >> 34, sid, 0]], dtype=np.uint64)
        word = int(philox4x32_10(ctr, np.array([[seed & 0xFFFFFFFF, seed >> 32]], dtype=np.uint64))[0, e % 4])
        assert bool(m[r, c]) == (word >= thr)
    assert keep_mask(rows, cols, 0.0, seed, sid).all()                           # p = 0 keeps everything
    assert not torch.equal(m, keep_mask(rows, cols, p, seed, sid + 1))            # streams differ
    assert not torch.equal(m, keep_mask(rows, cols, p, seed + 1, sid))            # keys differ
    big = keep_mask(64, 1024, 0.25, seed, 0)
    assert abs(big.float().mean().item() - 0.75) < 4 * math.sqrt(0.25 * 0.75 / big.numel())


# ------------------------------------------------------------------------------------------------------------------
# float64 oracles
# ------------------------------------------------------------------------------------------------------------------
def _dropped(h, mask, p, bwd_mask=None):
    """h * mask / (1 - p); with bwd_mask, the gradient flows through bwd_mask instead (power check only)."""
    if mask is None:
        return h
    if bwd_mask is None:
        return h * mask.to(h.dtype) / (1 - p)
    return h * bwd_mask.to(h.dtype) / (1 - p) + (h * (mask.to(h.dtype) - bwd_mask.to(h.dtype)) / (1 - p)).detach()


def lora_delta(h, ad):
    """s (dropout(h) A^T) B^T.  ad: dict A [r, in], B [out, r], s, mask (bool [B*S, in] or None), p, bwd_mask."""
    hd = _dropped(h, None if ad.get("mask") is None else ad["mask"].view(h.shape), ad.get("p", 0.0),
                  None if ad.get("bwd_mask") is None else ad["bwd_mask"].view(h.shape))
    return ad["s"] * (hd @ ad["A"].t()) @ ad["B"].t()


def llama_layer_lora(x, p, num_heads, num_kv_heads=None, inv_freq=None, attn_scale=1.0, q=None, v=None, eps=1e-6,
                     rope_theta=10000.0, after_rope=False):
    """tests/test_llama_gqa_cpu.llama_layer_gqa with LoRA deltas (lora_delta dicts, or None) added to the q and v
    projections before the rotary embedding (after it with after_rope: power check only)."""
    B, S, D = x.shape
    hd = D // num_heads
    kvh = num_heads if num_kv_heads is None else num_kv_heads
    h = RL.rms_norm(x, p["input_layernorm.weight"], eps)
    sp = lambda t, n: t.view(B, S, n, hd).transpose(1, 2)
    qp = h @ p["self_attn.q_proj.weight"].t()
    if q is not None and not after_rope:
        qp = qp + lora_delta(h, q)
    vp = h @ p["self_attn.v_proj.weight"].t()
    if v is not None:
        vp = vp + lora_delta(h, v)
    qh, k, vh = sp(qp, num_heads), sp(h @ p["self_attn.k_proj.weight"].t(), kvh), sp(vp, kvh)
    if inv_freq is None:
        inv_freq = 1.0 / (rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
    fr = torch.arange(S, dtype=torch.float32)[:, None] * inv_freq[None].to(torch.float32)
    emb = torch.cat((fr, fr), -1)
    cos, sin = emb.cos()[None, None].to(x.dtype) * attn_scale, emb.sin()[None, None].to(x.dtype) * attn_scale
    qh, k = qh * cos + RL.rotate_half(qh) * sin, k * cos + RL.rotate_half(k) * sin
    if q is not None and after_rope:
        qh = qh + sp(lora_delta(h, q), num_heads)
    if kvh != num_heads:
        k, vh = k.repeat_interleave(num_heads // kvh, dim=1), vh.repeat_interleave(num_heads // kvh, dim=1)
    sim = (qh @ k.transpose(-1, -2)) / math.sqrt(hd)
    sim = sim.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
    o = (sim.softmax(-1) @ vh).transpose(1, 2).reshape(B, S, D)
    x1 = x + o @ p["self_attn.o_proj.weight"].t()
    h2 = RL.rms_norm(x1, p["post_attention_layernorm.weight"], eps)
    g, u = h2 @ p["mlp.gate_proj.weight"].t(), h2 @ p["mlp.up_proj.weight"].t()
    return x1 + (torch.nn.functional.silu(g) * u) @ p["mlp.down_proj.weight"].t()


def mpt_block_lora(x, p, n_heads, wqkv=None):
    """oracle/restatement_lm.mpt_block with a LoRA delta (lora_delta dict) added to the Wqkv projection."""
    TF = torch.nn.functional
    D = x.shape[-1]
    a = TF.layer_norm(x, (D,), p["norm_1.weight"], p.get("norm_1.bias"), 1e-5)
    b_qkv = p.get("attn.Wqkv.bias")
    if wqkv is not None:
        b_qkv = lora_delta(a, wqkv) + (0 if b_qkv is None else b_qkv)
    x = x + RLM.mpt_attention(a, p["attn.Wqkv.weight"], p["attn.out_proj.weight"], n_heads, True, 8, b_qkv,
                              p.get("attn.out_proj.bias"))
    m = TF.layer_norm(x, (D,), p["norm_2.weight"], p.get("norm_2.bias"), 1e-5)
    h = TF.gelu(TF.linear(m, p["ffn.up_proj.weight"], p.get("ffn.up_proj.bias")))
    return x + TF.linear(h, p["ffn.down_proj.weight"], p.get("ffn.down_proj.bias"))


def rel_fro(got, ref):
    return ((got.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-30)).item()


class _FixedMask(torch.nn.Module):
    def __init__(self, mask, p):
        super().__init__()
        self.mask, self.p = mask, p

    def forward(self, x):
        return x * self.mask.view(x.shape).to(x.dtype) / (1 - self.p)


def _adapter(out_f, in_f, r, g, alpha=32.0, p=0.0, mask=None):
    A = torch.randn(r, in_f, generator=g, dtype=F64) / math.sqrt(in_f)
    B = torch.randn(out_f, r, generator=g, dtype=F64) / math.sqrt(r)
    return {"A": A, "B": B, "s": alpha / r, "p": p, "mask": mask}


def _llama_params(D, kvd, I, g):
    p = {}
    for n, shp in (("self_attn.q_proj", (D, D)), ("self_attn.k_proj", (kvd, D)), ("self_attn.v_proj", (kvd, D)),
                   ("self_attn.o_proj", (D, D)), ("mlp.gate_proj", (I, D)), ("mlp.up_proj", (I, D)),
                   ("mlp.down_proj", (D, I))):
        p[n + ".weight"] = torch.randn(*shp, generator=g, dtype=F64) / math.sqrt(shp[1])
    for n in ("input_layernorm", "post_attention_layernorm"):
        p[n + ".weight"] = 1 + 0.1 * torch.randn(D, generator=g, dtype=F64)
    return p


@pytest.mark.parametrize("H,kv,rope", [(2, 2, "default"), (4, 2, "llama3")])
def test_llama_lora_oracle_matches_hf_layer_with_lora_linear(H, kv, rope):
    from transformers.models.llama import modeling_llama as M
    from otter_b200.lora import LoraLinear
    D, B, S, r, pdrop = H * 128, 2, 7, 8, 0.1
    cfg = _cfg(D, H, kv, rope)
    g = torch.Generator().manual_seed(H + kv)
    p = _llama_params(D, kv * 128, 3 * D, g)
    layer = M.LlamaDecoderLayer(cfg, layer_idx=0).double()
    layer.load_state_dict(p)
    ads = {}
    for i, name in enumerate(("q_proj", "v_proj")):
        base = getattr(layer.self_attn, name)
        lin = LoraLinear(base, r, 16.0, pdrop)
        ad = _adapter(base.out_features, D, r, g, alpha=16.0, p=pdrop, mask=keep_mask(B * S, D, pdrop, SEED, i))
        with torch.no_grad():
            lin.lora_A["default"].weight.copy_(ad["A"])
            lin.lora_B["default"].weight.copy_(ad["B"])
        lin.lora_dropout["default"] = _FixedMask(ad["mask"], pdrop)
        setattr(layer.self_attn, name, lin)
        ads[name] = ad
    rot = M.LlamaRotaryEmbedding(cfg)
    x = torch.randn(B, S, D, generator=g, dtype=F64)
    pos = torch.arange(S)[None].expand(B, S)
    mask = torch.full((S, S), float("-inf"), dtype=F64).triu(1)[None, None].expand(B, 1, S, S)
    cos, sin = rot(x.float(), pos)
    out = layer(x, attention_mask=mask, position_ids=pos, position_embeddings=(cos.double(), sin.double()))
    out = out[0] if isinstance(out, tuple) else out
    ref = llama_layer_lora(x, p, H, kv, rot.inv_freq, rot.attention_scaling, q=ads["q_proj"], v=ads["v_proj"])
    assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5)
    assert rel_fro(out - llama_layer_lora(x, p, H, kv, rot.inv_freq, rot.attention_scaling), ref - x) > 1e-3


def _mpt_params(D, g, bias):
    p = {"attn.Wqkv.weight": (3 * D, D), "attn.out_proj.weight": (D, D), "ffn.up_proj.weight": (4 * D, D),
         "ffn.down_proj.weight": (D, 4 * D)}
    p = {k: torch.randn(*s, generator=g, dtype=F64) / math.sqrt(s[1]) for k, s in p.items()}
    for n in ("norm_1", "norm_2"):
        p[n + ".weight"] = 1 + 0.1 * torch.randn(D, generator=g, dtype=F64)
    if bias:
        for n, w in list(p.items()):
            p[n.replace("weight", "bias")] = 0.1 * torch.randn(w.shape[0], generator=g, dtype=F64)
    return p


@pytest.mark.parametrize("bias", [False, True])
def test_mpt_lora_oracle_equals_the_merged_weight(bias):
    D, H, r = 256, 2, 16
    g = torch.Generator().manual_seed(7)
    p = _mpt_params(D, g, bias)
    ad = _adapter(3 * D, D, r, g)
    x = torch.randn(2, 9, D, generator=g, dtype=F64)
    merged = dict(p, **{"attn.Wqkv.weight": p["attn.Wqkv.weight"] + ad["s"] * ad["B"] @ ad["A"]})
    assert torch.allclose(mpt_block_lora(x, p, H, ad), RLM.mpt_block(x, merged, H), rtol=1e-10, atol=1e-10)


def _llama_deltas(x, p, H, kv, q, v, w, **kw):
    """(y - y_frozen, dx - dx_frozen) of the oracle under the upstream gradient w."""
    outs = []
    for qa, va in ((q, v), (None, None)):
        xx = x.clone().requires_grad_(True)
        y = llama_layer_lora(xx, p, H, kv, q=qa, v=va, **kw)
        (y * w).sum().backward()
        outs.append((y.detach(), xx.grad))
    return outs[0][0] - outs[1][0], outs[0][1] - outs[1][1]


def test_delta_metric_rejects_wrong_adapters():
    """The GPU tests' bounds (adapter delta within 1.5e-2 forward, 3e-2 input gradient) reject each of these bugs."""
    H, kv, D, B, S, r, pdrop = 4, 2, 512, 2, 16, 16, 0.05
    g = torch.Generator().manual_seed(11)
    p = _llama_params(D, kv * 128, 2 * D, g)
    x, w = torch.randn(B, S, D, generator=g, dtype=F64), torch.randn(B, S, D, generator=g, dtype=F64)
    q = _adapter(D, D, r, g, p=pdrop, mask=keep_mask(B * S, D, pdrop, SEED, 0))
    v = _adapter(kv * 128, D, r, g, p=pdrop, mask=keep_mask(B * S, D, pdrop, SEED, 1))
    dy, dx = _llama_deltas(x, p, H, kv, q, v, w)
    wrong = {
        "no scaling": (dict(q, s=1.0), dict(v, s=1.0), {}),
        "shared q / v mask": (q, dict(v, mask=q["mask"]), {}),
        "backward mask unlike the forward's": (dict(q, bwd_mask=keep_mask(B * S, D, pdrop, SEED + 1, 0)),
                                               dict(v, bwd_mask=keep_mask(B * S, D, pdrop, SEED + 1, 1)), {}),
        "adapter after RoPE": (q, v, {"after_rope": True}),
    }
    for name, (qw, vw, kw) in wrong.items():
        dy2, dx2 = _llama_deltas(x, p, H, kv, qw, vw, w, **kw)
        ry, rx = rel_fro(dy2, dy), rel_fro(dx2, dx)
        assert ry > 1.5e-2 or rx > 3e-2, (name, ry, rx)
        if name == "backward mask unlike the forward's":
            assert ry < 1e-12 and rx > 3e-2, (ry, rx)


# ------------------------------------------------------------------------------------------------------------------
# the layers' kernel path with torch stand-ins for the kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def lk(kernels, monkeypatch):
    """`kernels` plus the GEMM epilogue's alpha and the dropout entry points (the numpy mask mirror); seed fixed."""
    from otter_b200 import functional as F
    from otter_b200 import lora as L
    fwd, dgrad, wgrad = F.linear_fwd, F.linear_dgrad, F.linear_wgrad

    def linear_fwd(x, w, *, alpha=1.0, residual=None, out=None, **kw):
        if alpha == 1.0:
            return fwd(x, w, residual=residual, out=out, **kw)
        kernels.append(("linear_fwd", ("alpha",) + (("out",) if out is not None else ()) + (("residual",) if residual is not None else ())))
        y = alpha * (x.float() @ w.t()) + (0 if residual is None else residual)
        return out.copy_(y) if out is not None else y

    def linear_dgrad(dy, w, *, alpha=1.0, residual=None, **kw):
        if alpha == 1.0:
            return dgrad(dy, w, residual=residual, **kw)
        kernels.append(("linear_dgrad", ("alpha",)))
        return alpha * (dy.float() @ w) + (0 if residual is None else residual)

    def linear_wgrad(dy, x, *, out=None, accumulate=False, alpha=1.0):
        if alpha == 1.0:
            return wgrad(dy, x, out=out, accumulate=accumulate)
        kernels.append(("linear_wgrad", ("alpha", "out") + (("accumulate",) if accumulate else ())))
        v = alpha * (dy.float().t() @ x.float())
        return out.copy_(out + v if accumulate else v)

    def lora_dropout(x, p, seed, stream_id, out=None):
        kernels.append(("lora_dropout", (stream_id,)))
        m = keep_mask(x.shape[0], x.shape[1], p, seed, stream_id)
        return torch.where(m, x.float() * dropout_scale(p), torch.zeros((), dtype=torch.float32))

    def lora_dropout_bwd_add_(g, dx, p, seed, stream_id):
        kernels.append(("lora_dropout_bwd_add_", (stream_id,)))
        m = keep_mask(g.shape[0], g.shape[1], p, seed, stream_id)
        return dx.copy_(dx + torch.where(m, g.float() * dropout_scale(p), torch.zeros((), dtype=torch.float32)))

    for name, fn in dict(linear_fwd=linear_fwd, linear_dgrad=linear_dgrad, linear_wgrad=linear_wgrad,
                         lora_dropout=lora_dropout, lora_dropout_bwd_add_=lora_dropout_bwd_add_).items():
        monkeypatch.setattr(F, name, fn)
    monkeypatch.setattr(L, "draw_seed", lambda device: SEED)
    return kernels


def _set_adapter(lin, ad):
    with torch.no_grad():
        lin.lora_A["default"].weight.copy_(ad["A"])
        lin.lora_B["default"].weight.copy_(ad["B"])


def _lora_llama_layer(H, kv, r, pdrop, g):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    from otter_b200.lora import LoraLinear
    D = H * 128
    kw = {} if kv == H else dict(num_key_value_heads=kv, rope_parameters=ROPES["default"], max_position_embeddings=256)
    layer = FrozenLlamaDecoderLayer(D, H, 2 * D, **kw)
    p = _llama_params(D, kv * 128, 2 * D, g)
    layer.load_state_dict({k: v.float() for k, v in p.items()})
    ads = {}
    for name in ("q_proj", "v_proj"):
        base = getattr(layer.self_attn, name)
        lin = LoraLinear(base, r, 2.0 * r, pdrop)
        ads[name] = _adapter(base.out_features, D, r, g, alpha=2.0 * r, p=pdrop)
        ads[name] = {k: (v.float().double() if torch.is_tensor(v) else v) for k, v in ads[name].items()}
        _set_adapter(lin, ads[name])
        setattr(layer.self_attn, name, lin)
    for n, prm in layer.named_parameters():
        prm.requires_grad_("lora_" in n)
    return layer, {k: v.float().double() for k, v in p.items()}, ads


@pytest.mark.parametrize("H,kv,pdrop", [(2, 2, 0.0), (2, 2, 0.1), (4, 2, 0.1)])
def test_llama_layer_kernel_path_matches_the_oracle(lk, H, kv, pdrop):
    B, S, r = 2, 9, 8
    g = torch.Generator().manual_seed(3 + kv)
    layer, p, ads = _lora_llama_layer(H, kv, r, pdrop, g)
    D = H * 128
    x, w = _bf16_exact(B, S, D, seed=5), _bf16_exact(B, S, D, seed=6)
    xg = x.clone().requires_grad_(True)
    (layer(xg) * w).sum().backward()
    q, v = ads["q_proj"], ads["v_proj"]
    if pdrop:
        q["mask"], v["mask"] = keep_mask(B * S, D, pdrop, SEED, 0), keep_mask(B * S, D, pdrop, SEED, 1)
    ref_ad = {n: dict(a, A=a["A"].clone().requires_grad_(True), B=a["B"].clone().requires_grad_(True)) for n, a in ads.items()}
    xr = x.double().requires_grad_(True)
    ref = llama_layer_lora(xr, p, H, kv, q=ref_ad["q_proj"], v=ref_ad["v_proj"])
    (ref * w.double()).sum().backward()
    assert rel_fro(xg.grad, xr.grad) < 1e-4
    for name in ("q_proj", "v_proj"):
        lin = getattr(layer.self_attn, name)
        assert rel_fro(lin.lora_A["default"].weight.grad, ref_ad[name]["A"].grad) < 1e-4, name
        assert rel_fro(lin.lora_B["default"].weight.grad, ref_ad[name]["B"].grad) < 1e-4, name
        assert lin.base_layer.weight.grad is None
    names = [c[0] for c in lk]
    assert names.count("lora_dropout") == (4 if pdrop else 0)          # forward q, v; regenerated in backward q, v
    assert names.count("lora_dropout_bwd_add_") == (2 if pdrop else 0)
    if pdrop:
        assert [c[1] for c in lk if c[0] == "lora_dropout"] == [(0,), (1,), (0,), (1,)]


@pytest.mark.parametrize("pdrop", [0.0, 0.05])
def test_mpt_block_kernel_path_matches_the_oracle(lk, pdrop):
    from otter_b200.lm_mpt import FrozenMPTBlock
    from otter_b200.lora import LoraLinear
    B, S, D, H, r = 2, 11, 256, 2, 16
    g = torch.Generator().manual_seed(9)
    blk = FrozenMPTBlock(D, H, no_bias=False)
    p = _mpt_params(D, g, True)
    blk.load_state_dict({k: v.float() for k, v in p.items()})
    p = {k: v.float().double() for k, v in p.items()}
    lin = LoraLinear(blk.attn.Wqkv, r, 32.0, pdrop)
    ad = {k: (v.float().double() if torch.is_tensor(v) else v) for k, v in _adapter(3 * D, D, r, g, p=pdrop).items()}
    _set_adapter(lin, ad)
    blk.attn.Wqkv = lin
    for n, prm in blk.named_parameters():
        prm.requires_grad_("lora_" in n or n == "norm_1.weight")
    x, w = _bf16_exact(B, S, D, seed=7), _bf16_exact(B, S, D, seed=8)
    xg = x.clone().requires_grad_(True)
    (blk(xg)[0] * w).sum().backward()
    ad["mask"] = keep_mask(B * S, D, pdrop, SEED, 0) if pdrop else None
    ad = dict(ad, A=ad["A"].clone().requires_grad_(True), B=ad["B"].clone().requires_grad_(True))
    p["norm_1.weight"].requires_grad_(True)
    xr = x.double().requires_grad_(True)
    (mpt_block_lora(xr, p, H, ad) * w.double()).sum().backward()
    assert rel_fro(xg.grad, xr.grad) < 4e-3                  # the block's bf16 input cast rounds its input gradient
    assert rel_fro(lin.lora_A["default"].weight.grad, ad["A"].grad) < 1e-4
    assert rel_fro(lin.lora_B["default"].weight.grad, ad["B"].grad) < 1e-4
    assert rel_fro(blk.norm_1.weight.grad, p["norm_1.weight"].grad) < 1e-4
    assert blk.attn.Wqkv.base_layer.weight.grad is None


# ------------------------------------------------------------------------------------------------------------------
# wrapping, freeze policy, checkpoints
# ------------------------------------------------------------------------------------------------------------------
def _lora_otter(monkeypatch, lm, r=8, **flags):
    from otter_b200 import otter_hf
    monkeypatch.setattr(otter_hf, "AutoTokenizer", FakeTokenizer)
    monkeypatch.setenv("OTB_LLAMA_LAYERS", "1")
    td = _mpt_text_config() if lm == "mpt" else _llama_text_config()
    cfg = _otter_cfg(td, lora_config={"r": r, "lora_alpha": 16, "lora_dropout": 0.05}, **flags)
    return otter_hf.OtterForConditionalGeneration(cfg)


LLAMA_ADAPTER_KEYS = [
    f"lang_encoder.base_model.model.model.layers.{i}.decoder_layer.self_attn.{proj}.{leaf}"
    for i in range(2) for proj in ("q_proj", "v_proj")
    for leaf in ("base_layer.weight", "lora_A.default.weight", "lora_B.default.weight")]
MPT_ADAPTER_KEYS = [
    f"lang_encoder.base_model.model.transformer.blocks.{i}.decoder_layer.attn.Wqkv.{leaf}"
    for i in range(2) for leaf in ("base_layer.weight", "lora_A.default.weight", "lora_B.default.weight")]


@pytest.mark.parametrize("lm", ["llama", "mpt"])
def test_lora_config_builds_without_peft_in_peft_layout(monkeypatch, lm):
    import sys
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    from otter_b200.lm_mpt import FrozenMPTBlock
    from otter_b200.lora import LoraLinear
    model = _lora_otter(monkeypatch, lm)
    assert "peft" not in sys.modules
    le = model.lang_encoder
    arch = "LlamaForCausalLM" if lm == "llama" else "MPTForCausalLM"
    assert type(le).__name__ == f"{arch}LoRA"
    keys = list(model.state_dict())
    want = LLAMA_ADAPTER_KEYS if lm == "llama" else MPT_ADAPTER_KEYS
    assert sorted(k for k in keys if k.startswith("lang_encoder.") and (".q_proj." in k or ".v_proj." in k or ".Wqkv." in k)) == sorted(want)
    assert all(k.startswith("lang_encoder.base_model.model.") for k in keys if k.startswith("lang_encoder."))
    sd = model.state_dict()
    r = 8
    D = 256
    for k in want:
        if "lora_A" in k:
            assert tuple(sd[k].shape) == (r, D)
        if "lora_B" in k:
            assert sd[k].shape[1] == r and not sd[k].any()                    # peft's init: B = 0
    # attribute access reaches the language model as peft's __getattr__ chain does
    assert le.get_input_embeddings() is le.base_model.model.get_input_embeddings()
    assert len(le._get_decoder_layers()) == 2 and not le.is_conditioned()
    le.clear_conditioned_layers()
    cls = FrozenLlamaDecoderLayer if lm == "llama" else FrozenMPTBlock
    layers = [m for m in le.modules() if isinstance(m, cls)]
    assert len(layers) == 2
    # trainable set after init_weights: adapters, gated x-attn, perceiver, input embeddings (+ lm_head for LLaMA)
    trainable = {n for n, p_ in model.named_parameters() if p_.requires_grad}
    for n in trainable:
        assert ("lora_" in n or "gated_cross_attn_layer" in n or n.startswith("perceiver.")
                or "embed_tokens" in n or "wte" in n or "lm_head" in n), n
    assert sum("lora_A" in n for n in trainable) == len(want) // 3
    assert sum("lora_B" in n for n in trainable) == len(want) // 3
    assert any("gated_cross_attn_layer" in n for n in trainable) and any(n.startswith("perceiver.") for n in trainable)
    assert any("lm_head" in n for n in trainable) == (lm == "llama")
    assert not any("base_layer" in n for n in trainable)
    if lm == "llama":
        for layer in layers:                                              # the KV-cache HF layer shares the adapters
            hf = layer.__dict__["_hf_layer"]
            for proj in ("q_proj", "v_proj"):
                assert isinstance(getattr(layer.self_attn, proj), LoraLinear)
                assert getattr(hf.self_attn, proj) is getattr(layer.self_attn, proj)
            assert hf.self_attn.k_proj.weight is layer.self_attn.k_proj.weight


@pytest.mark.parametrize("lm", ["llama", "mpt"])
def test_rank_not_a_multiple_of_8_is_refused_on_kernel_layers(monkeypatch, lm):
    with pytest.raises(ValueError, match="multiple of 8"):
        _lora_otter(monkeypatch, lm, r=12)


def test_hf_layers_take_any_rank(monkeypatch):
    from transformers import LlamaConfig, LlamaForCausalLM
    from otter_b200.lora import LoraLinear, wrap_lora
    cfg = LlamaConfig(vocab_size=32, hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2)
    lm = LlamaForCausalLM(cfg)                                            # head dim 32: not swapped
    shell = wrap_lora(lm, r=3, lora_alpha=6, lora_dropout=0.0, target_modules=["q_proj", "v_proj"])
    assert isinstance(lm.model.layers[0].self_attn.q_proj, LoraLinear)
    ids = torch.randint(0, 32, (1, 5))
    y0 = shell(input_ids=ids).logits
    with torch.no_grad():
        lm.model.layers[0].self_attn.q_proj.lora_B["default"].weight.normal_()
    assert not torch.allclose(shell(input_ids=ids).logits, y0)


def test_lora_linear_forward_is_peft_formula():
    from otter_b200.lora import LoraLinear
    torch.manual_seed(0)
    base = torch.nn.Linear(24, 40)
    lin = LoraLinear(base, 4, 12.0, 0.0)
    assert lin.scaling == {"default": 3.0} and lin.weight is base.weight and lin.bias is base.bias
    assert not lin.lora_B["default"].weight.any()
    bound = 1 / math.sqrt(24)                                             # kaiming_uniform_(a=sqrt(5)) bound
    assert lin.lora_A["default"].weight.abs().max() <= bound and lin.lora_A["default"].weight.std() > bound / 4
    with torch.no_grad():
        lin.lora_B["default"].weight.normal_()
    x = torch.randn(5, 24)
    want = base(x) + x @ lin.lora_A["default"].weight.t() @ lin.lora_B["default"].weight.t() * 3.0
    assert torch.allclose(lin(x), want, atol=1e-5)


@pytest.mark.parametrize("lm", ["llama", "mpt"])
def test_trainable_checkpoint_round_trip(monkeypatch, tmp_path, lm):
    from otter_b200.checkpoint import load_trainable_checkpoint, save_final_weights
    model = _lora_otter(monkeypatch, lm)
    with torch.no_grad():
        for n, p_ in model.named_parameters():
            if "lora_B" in n:
                p_.normal_()
    path = save_final_weights(model, str(tmp_path))
    saved = torch.load(path, weights_only=True)
    assert any("lora_A.default" in k for k in saved) and not any("base_layer" in k for k in saved)
    other = _lora_otter(monkeypatch, lm)
    load_trainable_checkpoint(other, path)
    own = other.state_dict()
    for k, v in saved.items():
        assert torch.equal(own[k], v), k


def _fn_node(t, name):
    todo, seen = [t.grad_fn], set()
    while todo:
        n = todo.pop()
        if n is None or id(n) in seen:
            continue
        seen.add(id(n))
        if type(n).__name__ == name:
            return n
        todo.extend(f for f, _ in n.next_functions)
    raise AssertionError(f"{name} not in the graph")


def test_adapter_only_training_keeps_only_the_adapter_input(lk):
    """A layer that trains only its adapters keeps the norm output feeding them and none of the MLP activations."""
    from otter_b200.lm_mpt import FrozenMPTBlock
    from otter_b200.lora import LoraLinear
    layer, _, _ = _lora_llama_layer(2, 2, 8, 0.0, torch.Generator().manual_seed(1))
    y = layer(torch.randn(1, 9, 256, requires_grad=True))
    saved = _fn_node(y, "_FrozenLlamaLayerFnBackward").saved_tensors
    assert saved[9] is not None and saved[10] is None and saved[11] is None          # h1 kept; h2, SwiGLU out not
    layer.mlp.up_proj.weight.requires_grad_(True)
    y = layer(torch.randn(1, 9, 256, requires_grad=True))
    saved = _fn_node(y, "_FrozenLlamaLayerFnBackward").saved_tensors
    assert saved[9] is not None and saved[10] is not None and saved[11] is None
    blk = FrozenMPTBlock(256, 2)
    blk.attn.Wqkv = LoraLinear(blk.attn.Wqkv, 8, 16.0)
    for n, p in blk.named_parameters():
        p.requires_grad_("lora_" in n)
    y, _, _ = blk(torch.randn(1, 9, 256, requires_grad=True))
    saved = _fn_node(y, "_FrozenMPTBlockFnBackward").saved_tensors
    assert saved[10] is not None and saved[11] is None and saved[12] is None         # a kept; m, GELU out not
