"""CPU: KV-cache decoding of the MPT language model (otter_b200/lm_mpt.py) — the cached-step oracle against the reference
fixture, the host logic of MPTKVCache, what generate() is handed, each refusal, and the wiring of the decode step with the
CUDA entry points replaced by torch formulas of what each computes (the pattern of tests/test_mpt_wiring_cpu.py).  The
kernels themselves are checked on the GPU (tests/test_mpt_decode_gpu.py)."""
import ctypes as C
import math
import os

import pytest
import torch

from oracle import restatement_lm as RL
from oracle import restatement_mpt_decode as RD

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- the oracle of the cached step ----
@pytest.mark.parametrize("case", ["a", "b"])
def test_cached_oracle_matches_the_reference_block(case):
    g = torch.load(os.path.join(GOLDEN, "mpt_block_decode.pt"))[case]
    B, D, H = g["shape"]
    past, T = (), 0
    for n, y_ref in zip([g["prefill"]] + [1] * g["steps"], g["ys"]):
        y, past = RD.mpt_block_cached(g["x"][:, T:T + n], past, g["params"], H)
        T += n
        assert torch.allclose(y, y_ref, rtol=1e-3, atol=1e-5)
    assert torch.allclose(past[0], g["k"], rtol=1e-3, atol=1e-5) and torch.allclose(past[1], g["v"], rtol=1e-3, atol=1e-5)


def test_cached_oracle_steps_equal_the_uncached_oracle_on_the_grown_prefix():
    g = torch.load(os.path.join(GOLDEN, "mpt_block_decode.pt"))["b"]
    B, D, H = g["shape"]
    y, past = RD.mpt_block_cached(g["x"][:, :g["prefill"]], (), g["params"], H)
    assert torch.allclose(y, RL.mpt_block(g["x"][:, :g["prefill"]], g["params"], H), rtol=1e-5, atol=1e-6)
    for t in range(g["prefill"], g["prefill"] + g["steps"]):
        y, past = RD.mpt_block_cached(g["x"][:, t:t + 1], past, g["params"], H)
        full = RL.mpt_block(g["x"][:, :t + 1], g["params"], H)
        assert torch.allclose(y[:, 0], full[:, -1], rtol=1e-4, atol=1e-5)


# ---- MPTKVCache host logic ----
def test_cache_capacity_grows_geometrically():
    from otter_b200.lm_mpt import MPTKVCache
    g = MPTKVCache.grown_capacity
    assert g(0, 10) == 64 and g(64, 64) == 64 and g(64, 65) == 128 and g(128, 1000) == 1024 and g(128, 129) == 256
    cap, allocations = 0, 0
    for need in range(1, 5000):
        new = g(cap, need)
        assert new >= need and new % 64 == 0
        allocations += new != cap
        cap = new
    assert allocations <= 8                                            # doubling: O(log n) copies over n steps


def test_cache_prefill_reserve_and_reorder():
    from otter_b200.lm_mpt import MPTKVCache
    B, S, D = 3, 5, 16
    cache = MPTKVCache(2)
    assert len(cache) == 2 and cache.get_seq_length() == 0 and cache.is_compileable is False
    qkv = torch.randn(B * S, 3 * D)
    for i in range(2):
        cache.store_prefill(i, qkv + i, B, S)
    cache.seq_len = S
    assert cache.get_seq_length() == S and cache.layers[0].shape == (B, 64, 2 * D)      # S + 1 rows, in 64-row units
    want = qkv.view(B, S, 3 * D)[:, :, D:]
    assert torch.equal(cache.layers[0][:, :S], want) and torch.equal(cache.layers[1][:, :S], want + 1)
    old = cache.layers[0]
    cache.reserve(64)
    assert cache.layers[0] is old                                      # no copy while the capacity suffices
    cache.reserve(65)
    assert cache.layers[0].shape == (B, 128, 2 * D) and torch.equal(cache.layers[1][:, :S], want + 1)
    idx = torch.tensor([2, 2, 0])
    assert cache.reorder(idx) is cache
    assert torch.equal(cache.layers[0][:, :S], want[idx]) and cache.get_seq_length() == S


# ---- what generate() is handed ----
def _tiny_lm(**cfg):
    from otter_b200.lm_mpt import MPTConfig, MPTForCausalLM
    torch.manual_seed(3)
    config = MPTConfig(d_model=256, n_heads=2, n_layers=2, max_seq_len=64, vocab_size=72, no_bias=True,
                       attn_config=dict(alibi=True, attn_impl="torch"), **cfg)
    lm = MPTForCausalLM(config)
    with torch.no_grad():
        for p in lm.parameters():
            p.copy_(torch.randn_like(p) * (0.5 if p.dim() == 1 else 2.0 * p.shape[-1] ** -0.5))
            if p.dim() == 1:
                p.add_(1.0)
    return lm.eval()


def test_prepare_inputs_for_generation_follows_the_reference():
    from otter_b200.lm_mpt import MPTForCausalLM, MPTKVCache
    lm = _tiny_lm()
    ids, mask = torch.arange(10).view(2, 5), torch.ones(2, 5, dtype=torch.long)
    first = lm.prepare_inputs_for_generation(ids, attention_mask=mask)
    assert first["input_ids"] is ids and first["past_key_values"] is None and first["use_cache"] is True
    cache = MPTKVCache(2)
    step = lm.prepare_inputs_for_generation(ids, past_key_values=cache, attention_mask=mask, use_cache=True)
    assert step["input_ids"].tolist() == [[4], [9]] and step["past_key_values"] is cache and step["attention_mask"] is mask
    assert lm.prepare_inputs_for_generation(ids, attention_mask=mask, use_cache=False)["use_cache"] is False
    with pytest.raises(NotImplementedError):
        lm.prepare_inputs_for_generation(ids, inputs_embeds=torch.zeros(2, 5, 256))
    assert MPTForCausalLM._supports_default_dynamic_cache() is False
    for i in range(2):
        cache.store_prefill(i, torch.randn(2 * 5, 3 * 16), 2, 5)
    k0 = cache.layers[1][0, :5].clone()
    assert MPTForCausalLM._reorder_cache(cache, torch.tensor([0, 0])) is cache and torch.equal(cache.layers[1][1, :5], k0)


# ---- the kernels as torch formulas ----
def _gelu(v):
    return 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))


@pytest.fixture
def torch_kernels(monkeypatch):
    """fp32 stand-ins for the entry points the MPT layers call; `calls` counts them by name."""
    from otter_b200 import functional as F
    from otter_b200 import params as P
    calls = {}

    def counted(fn):
        def wrapped(*a, **k):
            calls[fn.__name__] = calls.get(fn.__name__, 0) + 1
            return fn(*a, **k)
        return wrapped

    def layernorm_fwd(x, g, b, eps=1e-5, want_stats=True, out=None):
        mean = x.mean(-1)
        rstd = torch.rsqrt(x.var(-1, unbiased=False) + eps)
        return (x - mean[:, None]) * rstd[:, None] * g + b, mean, rstd

    def _linear(x, w, *, alpha=1.0, bias=None, act=0, aux_out=None, residual=None, out=None):
        z = x @ w.t() if bias is None else x @ w.t() + bias
        if aux_out is not None:
            aux_out.copy_(z)
        y = (_gelu(z) if act == 1 else z) * alpha
        y = y if residual is None else y + residual
        if out is None:
            return y
        assert out.shape == y.shape
        out.copy_(y)
        return out

    def linear_fwd(x, w, **epi):
        return _linear(x, w, **epi)

    def linear_small_m(x, w, **epi):
        assert 1 <= x.shape[0] <= 8 and "aux_out" not in epi
        return _linear(x, w, **epi)

    def lm_attn_fwd(qkv, B, S, H, *, slopes=None, causal=True, scale=None):
        D = H * 128
        sp = lambda t: t.reshape(B, S, H, 128).transpose(1, 2)
        q, k, v = sp(qkv[:, :D]), sp(qkv[:, D:2 * D]), sp(qkv[:, 2 * D:])
        s = (q @ k.transpose(-1, -2)) * scale
        s = s + slopes.view(1, H, 1, 1) * torch.arange(1 - S, 1, dtype=torch.float32).view(1, 1, 1, S)
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
        return (s.softmax(-1) @ v).transpose(1, 2).reshape(B * S, D), torch.zeros(B, H, S)

    def lm_attn_decode(q, k, v, T, *, slopes=None, scale=None):
        B, D = q.shape
        H = D // 128
        assert k.shape == v.shape and k.shape[0] == B and k.shape[2] == D and T <= k.shape[1]
        qh = q.view(B, H, 1, 128)
        kh, vh = (t[:, :T].reshape(B, T, H, 128).transpose(1, 2) for t in (k, v))      # rows >= T are not touched
        s = (qh @ kh.transpose(-1, -2)) * scale
        s = s + slopes.view(1, H, 1, 1) * torch.arange(1 - T, 1, dtype=torch.float32).view(1, 1, 1, T)
        return (s.softmax(-1) @ vh).reshape(B, D)

    for fn in (layernorm_fwd, linear_fwd, linear_small_m, lm_attn_fwd, lm_attn_decode):
        monkeypatch.setattr(F, fn.__name__, counted(fn))
    monkeypatch.setattr(P, "bf16_of", lambda p: p.detach().float())
    monkeypatch.setattr(P, "f32_of", lambda p: p.detach().float())
    monkeypatch.setattr(torch, "bfloat16", torch.float32)         # the layers' storage type, for the stand-ins
    return calls


def _seeded_block(D, H, lora=False):
    from otter_b200 import lora as L
    from otter_b200.lm_mpt import FrozenMPTBlock
    torch.manual_seed(1)
    blk = FrozenMPTBlock(D, H, no_bias=True)
    with torch.no_grad():
        for p in blk.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    params = {k: v.detach().clone() for k, v in blk.state_dict().items()}
    if lora:
        blk.attn.Wqkv = L.LoraLinear(blk.attn.Wqkv, r=8, lora_alpha=16)
        with torch.no_grad():
            blk.attn.Wqkv.lora_B["default"].weight.normal_(0, 0.05)
        A, Bw = blk.attn.Wqkv.lora_A["default"].weight, blk.attn.Wqkv.lora_B["default"].weight
        params["attn.Wqkv.weight"] = params["attn.Wqkv.weight"] + 2.0 * (Bw @ A).detach()
        blk.requires_grad_(False)
    return blk.eval(), params


@pytest.mark.parametrize("lora", [False, True])
def test_cached_block_steps_match_the_oracle(torch_kernels, lora):
    from otter_b200.lm_mpt import MPTKVCache
    B, D, H, S0, steps = 2, 256, 2, 62, 5                        # 62 + 3 > 64: the cache grows on the way
    blk, params = _seeded_block(D, H, lora)
    x = torch.randn(B, S0 + steps, D)
    cache = MPTKVCache(1)
    with torch.no_grad():
        y, attn_w, past = blk(x[:, :S0], past_key_value=(cache, 0), attention_mask=torch.ones(B, S0))
        assert attn_w is None and past[0] is cache
        assert torch.allclose(y, RL.mpt_block(x[:, :S0], params, H), rtol=1e-4, atol=1e-5)
        cache.seq_len = S0
        capacities = set()
        for t in range(S0, S0 + steps):
            cache.reserve(t + 1)
            capacities.add(cache.layers[0].shape[1])
            y, _, _ = blk(x[:, t:t + 1], past_key_value=(cache, 0))
            cache.seq_len = t + 1
            assert torch.allclose(y[:, 0], RL.mpt_block(x[:, :t + 1], params, H)[:, -1], rtol=1e-4, atol=1e-5), t
    assert capacities == {64, 128}
    assert torch_kernels["lm_attn_decode"] == steps and torch_kernels["lm_attn_fwd"] == 1
    # Wq and Wkv apart, out_proj, up_proj, down_proj; with the adapter its A and two B products
    assert torch_kernels["linear_small_m"] == steps * (8 if lora else 5)


def test_cached_model_steps_match_the_uncached_forward(torch_kernels):
    lm = _tiny_lm()
    ids = torch.randint(0, 72, (2, 12))
    with torch.no_grad():
        full = lm(input_ids=ids).logits
        assert lm(input_ids=ids).past_key_values is None               # config.use_cache is False by default
        out = lm(input_ids=ids[:, :7], use_cache=True)
        assert torch.allclose(out.logits, full[:, :7], rtol=1e-4, atol=1e-5)
        cache = out.past_key_values
        for t in range(7, 12):
            assert cache.get_seq_length() == t
            out = lm(input_ids=ids[:, t:t + 1], past_key_values=cache, use_cache=True)
            assert out.past_key_values is cache
            assert torch.allclose(out.logits[:, 0], full[:, t], rtol=1e-4, atol=1e-4)
    assert _tiny_lm(use_cache=True).config.use_cache is True
    with torch.no_grad():
        assert _tiny_lm(use_cache=True)(input_ids=ids).past_key_values is not None


def test_generate_uses_the_cache_and_agrees_with_use_cache_false(torch_kernels):
    """Without the Otter layers the cached and the uncached arithmetic agree, so greedy tokens must be equal."""
    lm = _tiny_lm()
    lm.generation_config.pad_token_id = 0
    ids = torch.randint(1, 72, (2, 6))
    kw = dict(attention_mask=torch.ones_like(ids), max_new_tokens=5, do_sample=False)
    # MPTConfig.use_cache defaults to False (configuration_mpt.py) and transformers copies it into the generation
    # config, so the caller (or the config) asks for the cache
    assert lm.generation_config.use_cache is False
    cached = lm.generate(ids, use_cache=True, **kw)
    assert torch_kernels["lm_attn_decode"] == 4 * 2 and torch_kernels["lm_attn_fwd"] == 2      # 2 layers: 1 prefill + 4 steps
    uncached = lm.generate(ids, use_cache=False, **kw)
    assert torch_kernels["lm_attn_decode"] == 8 and torch_kernels["lm_attn_fwd"] == 2 + 5 * 2
    assert cached.shape == (2, 11) and torch.equal(cached, uncached)
    beams = lm.generate(ids, num_beams=2, num_return_sequences=2, use_cache=True, **kw)
    assert beams.shape == (4, 11) and torch_kernels["lm_attn_decode"] == 16
    torch.manual_seed(0)
    sampled = lm.generate(ids, attention_mask=kw["attention_mask"], max_new_tokens=5, do_sample=True, use_cache=True)
    assert sampled.shape == (2, 11) and torch_kernels["lm_attn_decode"] == 24
    by_config = _tiny_lm(use_cache=True)                                # config.use_cache = True: cached by default
    by_config.generation_config.pad_token_id = 0
    assert torch.equal(by_config.generate(ids, **kw), cached) and torch_kernels["lm_attn_decode"] == 32


# ---- refusals ----
def test_cache_refusals(torch_kernels):
    from otter_b200.lm_mpt import MPTKVCache
    lm = _tiny_lm()
    ids = torch.randint(0, 72, (2, 8))
    with torch.no_grad():
        cache = lm(input_ids=ids, use_cache=True).past_key_values
        with pytest.raises(NotImplementedError, match="one new token"):                 # chunked prefill
            lm(input_ids=ids[:, :2], past_key_values=cache, use_cache=True)
        with pytest.raises(NotImplementedError, match="MPTKVCache"):                    # a tuple / DynamicCache
            lm(input_ids=ids[:, :1], past_key_values=((ids, ids),) * 2, use_cache=True)
        mask = torch.ones(2, 9, dtype=torch.long)
        mask[1, 0] = 0
        with pytest.raises(NotImplementedError, match="one length"):                    # ragged batch with a cache
            lm(input_ids=ids[:, :1], past_key_values=cache, attention_mask=mask, use_cache=True)
        right = torch.ones(2, 8, dtype=torch.long)
        right[1, 6:] = 0
        with pytest.raises(NotImplementedError, match="one length"):
            lm(input_ids=ids, attention_mask=right, use_cache=True)
        assert lm(input_ids=ids, attention_mask=right).logits.shape == (2, 8, 72)      # uncached: right padding stays
        cache.seq_len = 64                                                              # max_seq_len reached
        with pytest.raises(AssertionError, match="seq_len"):
            lm(input_ids=ids[:, :1], past_key_values=cache, use_cache=True)
    lm.transformer.wte.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="inference"):                         # grad mode with a trainable weight
        lm(input_ids=ids, use_cache=True)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="inference"):        # training mode
        lm.train()(input_ids=ids, use_cache=True)
    blk = lm.eval().transformer.blocks[0]
    with pytest.raises(NotImplementedError, match="MPTKVCache"):
        blk(torch.zeros(2, 1, 256), past_key_value=(ids, ids))
    blk.norm_1.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="inference"):
        blk(torch.zeros(2, 1, 256), past_key_value=(MPTKVCache(1), 0))


# ---- C ABI ----
def test_decode_descriptor_layout_and_argument_checks():
    from otter_b200 import _lib
    lib = _lib.load()
    assert lib.otb_abi_sizeof(5) == C.sizeof(_lib.LmAttnDecodeDesc) == 6 * 8 + 4 * 8 + 4 * 4 + 4 + 4
    launches = lib.otb_launch_count()
    d = _lib.LmAttnDecodeDesc()
    assert lib.otb_lm_attn_decode(C.byref(d), None) == 1 and b"otb_lm_attn_decode" in lib.otb_last_error()
    d.q, d.k, d.v, d.out, d.ws = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    d.B, d.H, d.T, d.head_dim, d.ld_q, d.ld_out, d.ld_kv, d.kv_batch_stride = 1, 2, 5, 128, 256, 256, 512, 512 * 64
    d.k = 0x20002
    assert lib.otb_lm_attn_decode(C.byref(d), None) == 1 and b"aligned" in lib.otb_last_error()
    d.k, d.ld_kv = 0x20000, 130
    assert lib.otb_lm_attn_decode(C.byref(d), None) == 1 and b"multiples of 8" in lib.otb_last_error()
    d.ld_kv, d.head_dim = 512, 64
    assert lib.otb_lm_attn_decode(C.byref(d), None) == 1 and b"head_dim" in lib.otb_last_error()
    assert lib.otb_lm_attn_decode_ws_floats(0, 2, 5) == 0
    ws = [lib.otb_lm_attn_decode_ws_floats(1, 32, T) for T in (1, 64, 65, 1024, 4096)]
    assert ws[0] == ws[1] == 32 * 132 and ws == sorted(ws) and all(w % (32 * 132) == 0 for w in ws)

    def lin(M, N, K, x=0x10000, ldx=None, act=0):
        return lib.otb_linear_small_m(x, ldx or K, 0x20000, K, M, N, K, 1.0, None, act, None, 0, 0x30000, N, None)
    for bad in (lin(0, 64, 64), lin(9, 64, 64)):
        assert bad == 1 and b"1..8" in lib.otb_last_error()
    assert lin(4, 60, 64) == 1 and lin(4, 64, 60) == 1 and b"multiples of 8" in lib.otb_last_error()
    assert lin(4, 64, 64, x=0x10008) == 1 and b"aligned" in lib.otb_last_error()
    assert lin(4, 64, 64, ldx=32) == 1 and b"pitch" in lib.otb_last_error()
    assert lin(4, 64, 64, act=2) == 1 and b"act" in lib.otb_last_error()
    assert lib.otb_launch_count() == launches                          # every refusal came before a launch


def test_decode_wrappers_reject_cpu_tensors():
    from otter_b200 import _lib
    from otter_b200 import functional as F
    bf = torch.bfloat16
    with pytest.raises(_lib.OtbError, match="CUDA tensor"):
        F.linear_small_m(torch.zeros(2, 8, dtype=bf), torch.zeros(8, 8, dtype=bf))
    with pytest.raises(_lib.OtbError, match="CUDA tensor"):
        F.lm_attn_decode(torch.zeros(1, 128, dtype=bf), torch.zeros(1, 4, 128, dtype=bf), torch.zeros(1, 4, 128, dtype=bf), 2)
