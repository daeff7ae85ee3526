"""GPU: KV-cache decoding of the MPT language model — the two decode kernels against float64 references built from the
same bf16-rounded inputs, the cached block against the uncached block, and generate() on the tiny Otter-over-MPT model
against the reference's cached and uncached greedy sequences (tests/golden/tiny_mpt_generate.pt).

The metric.  Both kernels accumulate in fp32 from bf16 inputs the reference shares, and round once, to the bf16 output:
    |got - ref| <= A_REL |ref| + B_RMS rms(ref over the head / the output row) + FLOOR
A_REL = 2^-7 is twice the bf16 rounding error of an element (2^-8 relative); B_RMS = 2^-9 covers elements that are small
within their slice (fp32 accumulation over <= 16384 terms and exp2 / erf approximations stay below 2^-18 of the slice's
rms).  test_metric_rejects_a_shifted_key_and_a_dropped_split shows on the CPU that a value row paired with its
neighbour's key, an ALiBi bias one position off, or one split of nine left out of the combination exceed the bound.
"""
import os

import pytest
import torch

BF16 = torch.bfloat16
gpu = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
A_REL, B_RMS, FLOOR = 2.0 ** -7, 2.0 ** -9, 2.0 ** -16


def _ratio(got, ref, slice_len=None):
    got, ref = got.double(), ref.double()
    sl = ref if slice_len is None else ref.reshape(*ref.shape[:-1], -1, slice_len)
    rms = sl.pow(2).mean(-1, keepdim=True).sqrt().expand_as(sl).reshape(ref.shape)
    return ((got - ref).abs() / (A_REL * ref.abs() + B_RMS * rms + FLOOR)).max().item()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _decode_ref(q, k, v, T, slopes, scale, drop=None, v_shift=0, pos_shift=0):
    """float64 decode attention.  q [B, H*128]; k, v [B, >= T, H*128].  The keyword arguments mutate it the way a kernel
    bug would (power check): `drop` = slice of keys left out, `v_shift` = value rows rolled against the keys,
    `pos_shift` = ALiBi positions off by that many keys."""
    B, D = q.shape
    H = D // 128
    qh = q.double().view(B, H, 1, 128)
    kh, vh = (t[:, :T].double().reshape(B, T, H, 128).transpose(1, 2) for t in (k, v))
    s = (qh @ kh.transpose(-1, -2)) * scale
    if slopes is not None:
        pos = torch.arange(1 - T, 1, dtype=torch.float64, device=q.device) + pos_shift
        s = s + slopes.double().view(1, H, 1, 1) * pos.view(1, 1, 1, T)
    if drop is not None:
        s[..., drop] = float("-inf")
    return (s.softmax(-1) @ vh.roll(v_shift, dims=2)).reshape(B, D)


def test_metric_rejects_a_shifted_key_and_a_dropped_split():
    g = torch.Generator().manual_seed(0)
    B, H, T = 2, 2, 1000
    q, k, v = (torch.randn(s, generator=g).to(BF16) for s in ((B, H * 128), (B, T, H * 128), (B, T, H * 128)))
    slopes = torch.tensor([0.25, 0.0625])
    ref = _decode_ref(q, k, v, T, slopes, 128 ** -0.5)
    assert _ratio(ref.to(BF16), ref, 128) <= 0.6                       # the exact answer rounded to bf16 passes
    assert _ratio(_decode_ref(q, k, v, T, slopes, 128 ** -0.5, v_shift=1).to(BF16), ref, 128) > 1
    assert _ratio(_decode_ref(q, k, v, T, slopes, 128 ** -0.5, pos_shift=1).to(BF16), ref, 128) <= 0.6   # softmax shift invariance
    assert _ratio(_decode_ref(q, k, v, T - 1, slopes, 128 ** -0.5).to(BF16), ref, 128) > 1                 # the new token's key lost
    # a split left out of the combination; without ALiBi, under which keys that far back weigh nothing
    flat = _decode_ref(q, k, v, T, None, 128 ** -0.5)
    assert _ratio(_decode_ref(q, k, v, T, None, 128 ** -0.5, drop=slice(112, 224)).to(BF16), flat, 128) > 1


# ------------------------------------------------------------------------------------------------------------------
# otb_lm_attn_decode
# ------------------------------------------------------------------------------------------------------------------
def _split_boundaries(F, B, H, limit=4200):
    """Every T <= limit at which the kernel's split count changes (T-1 and T straddle a boundary)."""
    out, prev = set(), F.lm_attn_decode_splits(B, H, 1)
    for T in range(2, limit):
        n = F.lm_attn_decode_splits(B, H, T)
        if n != prev:
            out.update((T - 1, T))
        prev = n
    return out


def _decode_case(F, B, H, T, with_slopes, extra_cap, gen):
    from otter_b200.lm_mpt import alibi_slopes
    D, cap = H * 128, T + extra_cap
    cache = torch.full((B, cap, 2 * D), float("nan"), device=DEV, dtype=BF16)     # rows >= T: NaN, must not be read
    cache[:, :T] = torch.randn((B, T, 2 * D), device=DEV, generator=gen).to(BF16)
    q = torch.randn((B, D), device=DEV, generator=gen).to(BF16)
    slopes = alibi_slopes(H, device=DEV) if with_slopes else None
    need = int(F._lib.load().otb_lm_attn_decode_ws_floats(B, H, T))
    ws = torch.full((need + 64,), float("nan"), device=DEV)
    outbuf = torch.full((B + 2, D + 16), float("nan"), device=DEV, dtype=BF16)
    out = outbuf[1:B + 1, 8:8 + D]
    F.lm_attn_decode(q, cache[:, :, :D], cache[:, :, D:], T, slopes=slopes, out=out, ws=ws[:need])
    ref = _decode_ref(q, cache[:, :, :D], cache[:, :, D:], T, slopes, 128 ** -0.5)
    r = _ratio(out, ref, 128)
    assert r <= 1.0, f"B={B} H={H} T={T} slopes={with_slopes}: error / bound = {r:.3f}"
    assert torch.isnan(ws[need:]).all() and not torch.isnan(ws[:need].view(-1, 132)[:, [0, 1]]).any()
    border = outbuf.clone()
    border[1:B + 1, 8:8 + D] = float("nan")
    assert torch.isnan(border).all(), "written outside out"
    first = out.clone()
    ws.fill_(float("nan"))
    F.lm_attn_decode(q, cache[:, :, :D], cache[:, :, D:], T, slopes=slopes, out=out, ws=ws[:need])
    assert torch.equal(first, out), "two runs differ"
    return r


@gpu
def test_decode_attention_against_fp64():
    from otter_b200 import functional as F
    gen = torch.Generator(device=DEV).manual_seed(1)
    Ts = {1, 2, 63, 64, 65, 127, 128, 129, 1000, 2048, 4096}
    worst, cases = 0.0, 0
    for B, H in ((1, 1), (3, 2), (8, 32), (1, 32), (3, 32)):
        edges = _split_boundaries(F, B, H)
        assert edges or B * H >= 256, (B, H)
        ts = sorted(Ts | edges) if B * H <= 6 else sorted(Ts | set(sorted(edges)[:6]))
        if B * H >= 96:
            ts = [t for t in ts if t <= 2048]                           # 8 x 32 x 4096 x 512 B of cache is plenty at 2048
        for T in ts:
            worst = max(worst, _decode_case(F, B, H, T, with_slopes=(cases % 3 != 2), extra_cap=(0, 5, 64)[cases % 3], gen=gen))
            cases += 1
        print(f"lm_attn_decode B={B} H={H}: {len(ts)} values of T up to {ts[-1]}, worst error / bound so far {worst:.3f}",
              flush=True)
    print(f"RATIO lm_attn_decode: worst error / bound {worst:.3f} over {cases} cases")


@gpu
def test_decode_attention_equals_the_last_row_of_the_prefill_kernel():
    from otter_b200 import functional as F
    from otter_b200.lm_mpt import alibi_slopes
    gen = torch.Generator(device=DEV).manual_seed(2)
    for B, S, H in ((2, 130, 2), (1, 1000, 32)):
        D = H * 128
        qkv = torch.randn((B * S, 3 * D), device=DEV, generator=gen).to(BF16)
        slopes = alibi_slopes(H, device=DEV)
        o, _ = F.lm_attn_fwd(qkv, B, S, H, slopes=slopes, causal=True)
        v3 = qkv.view(B, S, 3 * D)
        got = F.lm_attn_decode(v3[:, -1, :D], v3[:, :, D:2 * D], v3[:, :, 2 * D:], S, slopes=slopes)
        last = o.view(B, S, D)[:, -1]
        # the prefill kernel rounds P to bf16 before its P V product, the decode kernel does not: the wider bound of
        # tests/test_attention_edges_gpu.py (B_RMS 2^-6) applies between the two
        r = ((got.double() - last.double()).abs() / (2.0 ** -7 * last.double().abs() + 2.0 ** -6 * last.double().pow(2).mean().sqrt())).max().item()
        assert r <= 1.0 and _rel(got, last) < 1e-2, (B, S, H, r)


@gpu
def test_decode_attention_refuses_bad_arguments():
    from otter_b200 import _lib
    from otter_b200 import functional as F
    q = torch.zeros((2, 256), device=DEV, dtype=BF16)
    kv = torch.zeros((2, 16, 512), device=DEV, dtype=BF16)
    n0 = F.launch_count()
    with pytest.raises(_lib.OtbError, match="does not hold"):
        F.lm_attn_decode(q, kv[:, :, :256], kv[:, :, 256:], 17)
    with pytest.raises(_lib.OtbError, match="bfloat16"):
        F.lm_attn_decode(q.float(), kv[:, :, :256], kv[:, :, 256:], 4)
    with pytest.raises(_lib.OtbError, match="aligned"):
        F.lm_attn_decode(q, kv[:, :, 4:260], kv[:, :, 256:], 4)
    with pytest.raises(_lib.OtbError, match="workspace"):
        F.lm_attn_decode(q, kv[:, :, :256], kv[:, :, 256:], 4, ws=torch.zeros(8, device=DEV))
    assert F.launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------
# otb_linear_small_m
# ------------------------------------------------------------------------------------------------------------------
def _gelu64(v):
    return 0.5 * v * (1 + torch.erf(v / 2 ** 0.5))


@gpu
@pytest.mark.parametrize("N,K", [(8, 8), (72, 256), (40, 4104), (4096, 4096), (12288, 4096), (4096, 16384), (16384, 4096)])
def test_linear_small_m_against_fp64(N, K):
    """(40, 4104): N is not a multiple of the 16 / 32 columns a CTA owns, K not of the 4096-element x chunk."""
    from otter_b200 import functional as F
    gen = torch.Generator(device=DEV).manual_seed(N + K)
    w_full = (torch.randn((N + 8, K + 8), device=DEV, generator=gen) * K ** -0.5).to(BF16)
    w = w_full[:N, :K] if N <= 72 else w_full[8:, :K]                   # a pitched row slice (ldw = K + 8)
    bias = torch.randn(N, device=DEV, generator=gen)
    worst = 0.0
    for M in (1, 2, 5, 8):
        x = torch.randn((M, K), device=DEV, generator=gen).to(BF16)
        res_full = torch.randn((M, N + 24), device=DEV, generator=gen).to(BF16)
        res = res_full[:, 8:8 + N]
        combos = [dict(), dict(bias=bias), dict(act=1), dict(bias=bias, act=1, residual=res, alpha=0.5),
                  dict(residual=res, alpha=2.0)] if (M in (1, 8) or N <= 72) else [dict(bias=bias, act=1, residual=res)]
        for epi in combos:
            outbuf = torch.full((M + 2, N + 16), float("nan"), device=DEV, dtype=BF16)
            out = outbuf[1:M + 1, 8:8 + N]                              # pitched, with canaries past N and past row M
            F.linear_small_m(x, w, out=out, **epi)
            z = x.double() @ w.double().t()
            if "bias" in epi:
                z = z + bias.double()
            if epi.get("act") == 1:
                z = _gelu64(z)
            z = z * epi.get("alpha", 1.0)
            if "residual" in epi:
                z = z + res.double()
            r = _ratio(out, z)
            assert r <= 1.0, f"M={M} N={N} K={K} {sorted(epi)}: error / bound = {r:.3f}"
            worst = max(worst, r)
            border = outbuf.clone()
            border[1:M + 1, 8:8 + N] = float("nan")
            assert torch.isnan(border).all(), "written outside out"
            if K >= 64:                                                  # the tensor-core GEMM on the same operands
                y = F.linear_fwd(x, w, **epi)
                assert _ratio(y, z) <= 1.0 and _rel(out, y) < 4e-3
            again = torch.empty_like(out)
            F.linear_small_m(x, w, out=again, **epi)
            assert torch.equal(again, out), "two runs differ"
    print(f"RATIO linear_small_m N={N} K={K}: worst error / bound {worst:.3f}")


@gpu
def test_linear_small_m_refuses_bad_arguments():
    from otter_b200 import _lib
    from otter_b200 import functional as F
    w = torch.zeros((64, 64), device=DEV, dtype=BF16)
    n0 = F.launch_count()
    for M in (0, 9):
        with pytest.raises(_lib.OtbError, match="1..8"):
            F.linear_small_m(torch.zeros((M, 64), device=DEV, dtype=BF16), w)
    with pytest.raises(_lib.OtbError, match="expected"):
        F.linear_small_m(torch.zeros((2, 32), device=DEV, dtype=BF16), w)
    with pytest.raises(_lib.OtbError, match="aligned"):
        F.linear_small_m(torch.zeros((2, 72), device=DEV, dtype=BF16)[:, 4:68], w)
    with pytest.raises(_lib.OtbError, match="multiples of 8"):
        F.linear_small_m(torch.zeros((2, 64), device=DEV, dtype=BF16), w[:60])
    assert F.launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------
# block level
# ------------------------------------------------------------------------------------------------------------------
def _block(D=256, H=2, lora=False, seed=1):
    from otter_b200 import lora as L
    from otter_b200.lm_mpt import FrozenMPTBlock
    torch.manual_seed(seed)
    blk = FrozenMPTBlock(D, H, no_bias=True)
    if lora:
        blk.attn.Wqkv = L.LoraLinear(blk.attn.Wqkv, r=8, lora_alpha=16)
        with torch.no_grad():
            blk.attn.Wqkv.lora_B["default"].weight.normal_(0, 0.05)
        blk.requires_grad_(False)
    return blk.to(DEV).eval()


def _cached_vs_uncached(blk, S0, steps, B=2):
    """-> (rel-Frobenius error of the cached steps' rows vs the uncached block's last rows, the cached rows, the cache)."""
    from otter_b200.lm_mpt import MPTKVCache
    x = torch.randn((B, S0 + steps, blk.d_model), device=DEV, generator=torch.Generator(device=DEV).manual_seed(S0)).to(BF16)
    cache = MPTKVCache(1)
    got, want = [], []
    with torch.no_grad():
        y, _, _ = blk(x[:, :S0], past_key_value=(cache, 0))
        assert torch.equal(y, blk(x[:, :S0])[0])                       # the prefill is the uncached forward, bit for bit
        cache.seq_len = S0
        for t in range(S0, S0 + steps):
            cache.reserve(t + 1)
            got.append(blk(x[:, t:t + 1], past_key_value=(cache, 0))[0][:, 0])
            cache.seq_len = t + 1
            want.append(blk(x[:, :t + 1])[0][:, -1])
    got, want = torch.stack(got), torch.stack(want)
    return _rel(got, want), got, cache


@gpu
@pytest.mark.parametrize("S0", [1, 9, 62, 64, 130])
def test_cached_block_steps_match_the_uncached_block(S0):
    """S0 = 62 and 64 cross a capacity growth (64 -> 128 rows) within the 5 steps."""
    blk = _block()
    r, _, cache = _cached_vs_uncached(blk, S0, 5)
    print(f"cached block S0={S0}: rel-Frobenius {r:.2e}, capacity {cache.layers[0].shape[1]}")
    assert r <= 1.5e-2
    assert cache.layers[0].shape[1] == (128 if S0 in (62, 64) else 64 if S0 < 62 else 192)


@gpu
def test_cached_block_steps_read_the_lora_adapter():
    blk = _block(lora=True)
    r, got, _ = _cached_vs_uncached(blk, 40, 5)
    with torch.no_grad():
        blk.attn.Wqkv.lora_B["default"].weight.zero_()
    _, zero, _ = _cached_vs_uncached(blk, 40, 5)
    moved = _rel(zero, got)
    print(f"cached LoRA block: parity {r:.2e}; lora_B = 0 moves the result by {moved:.2e}")
    assert r <= 1.5e-2 and moved > 5 * r


# ------------------------------------------------------------------------------------------------------------------
# model level: the tiny Otter over MPT
# ------------------------------------------------------------------------------------------------------------------
def _tiny_otter(monkeypatch):
    from oracle.ref_shims import FakeTokenizer
    from oracle.seeded import load_seeded_, seeded_tensor
    from otter_b200 import otter_hf
    from test_callers_gpu import EMB_KINDS, VKEYS, gold
    monkeypatch.setattr(otter_hf, "AutoTokenizer", FakeTokenizer)
    g = gold("tiny_mpt_generate.pt")
    cfg = otter_hf.OtterConfig(vision_config={k: v for k, v in g["vision_config"].items() if k in VKEYS},
                               text_config=dict(g["text_config"]), cross_attn_every_n_layers=2)
    model = otter_hf.OtterForConditionalGeneration(cfg)
    assert model.lang_encoder.__class__.__name__ == "MPTForCausalLM" and model.media_token_id == g["media_token_id"]
    load_seeded_(model, g["seed"], kinds=EMB_KINDS)
    model.to(DEV).eval()
    B = g["lang_x"].shape[0]
    vision_x = seeded_tensor("in.mptgen.vision_x", (B, 1, 1, 3, 224, 224), g["input_seed"], "randn").to(DEV)
    return model, g, vision_x, g["lang_x"].to(DEV)


def _follow(out, ref, L0, what):
    """Per-step logits vs the reference while the token ids agree; ids must agree wherever the reference's top-1 / top-2
    margin exceeds 10x the measured logit error (bf16 layers cannot decide a nearer tie).  -> qualifying steps."""
    B, steps = ref["margin"].shape
    qualified = 0
    for b in range(B):
        for t in range(steps):
            got, want = out.logits[t][b].float().cpu(), ref["logits"][b, t]
            err = (got - want).abs().max().item()
            assert _rel(got, want) <= 2e-2, (what, b, t, _rel(got, want))
            same = out.sequences[b, L0 + t].item() == ref["sequences"][b, L0 + t].item()
            if ref["margin"][b, t].item() > 10 * err:
                qualified += 1
                assert same, (what, b, t, err, ref["margin"][b, t].item())
            if not same:
                break                                                    # the prefixes differ from here on
    print(f"{what}: {qualified} of {B * steps} steps had a margin above 10x the logit error")
    return qualified


@gpu
def test_generate_follows_the_reference_cached_and_uncached(monkeypatch):
    from otter_b200 import functional as F
    model, g, vision_x, lang_x = _tiny_otter(monkeypatch)
    L0, n = lang_x.shape[1], g["new_tokens"]
    kw = dict(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x), max_new_tokens=n,
              do_sample=False, return_dict_in_generate=True, output_logits=True)
    cached = model.generate(use_cache=True, **kw)
    assert cached.sequences.shape == (lang_x.shape[0], L0 + n) and cached.past_key_values.get_seq_length() == L0 + n - 1
    assert not model.lang_encoder.is_conditioned()
    _follow(cached, g["cached"], L0, "generate(use_cache=True)")
    uncached = model.generate(use_cache=False, **kw)
    _follow(uncached, g["uncached"], L0, "generate(use_cache=False)")
    # use_cache=False is the uncached forward on the growing prefix, bit for bit
    ids = lang_x
    with torch.no_grad():
        model._encode_vision_x(vision_x=vision_x)
        for t in range(n):
            logits = model.lang_encoder(input_ids=ids, attention_mask=torch.ones_like(ids)).logits[:, -1]
            assert torch.equal(logits.float(), uncached.logits[t].float()), t
            ids = torch.cat([ids, logits.argmax(-1, keepdim=True)], dim=1)
        model.lang_encoder.clear_conditioned_layers()
    assert torch.equal(ids, uncached.sequences)
    # without use_cache the config decides, and MPT's default is False (transformers copies it to the generation config)
    default = model.generate(**kw)
    assert default.past_key_values is None and torch.equal(default.sequences, uncached.sequences)


@gpu
def test_generate_beams_sampling_and_launches_per_step(monkeypatch):
    from otter_b200 import functional as F
    model, g, vision_x, lang_x = _tiny_otter(monkeypatch)
    L0 = lang_x.shape[1]
    kw = dict(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x), use_cache=True)
    beams = model.generate(num_beams=2, max_new_tokens=4, do_sample=False, **kw)
    assert beams.shape[0] == lang_x.shape[0] and L0 < beams.shape[1] <= L0 + 4
    torch.manual_seed(0)
    sampled = model.generate(do_sample=True, max_new_tokens=4, **kw)
    assert sampled.shape[0] == lang_x.shape[0] and L0 < sampled.shape[1] <= L0 + 4
    assert not model.lang_encoder.is_conditioned()
    # kernel launches of one cached step of the language model do not depend on the prefix length
    lm = model.lang_encoder
    per_step = set()
    with torch.no_grad():
        for S0 in (5, 70):
            ids = torch.randint(3, 60, (2, S0 + 1), device=DEV)
            model._encode_vision_x(vision_x=vision_x)
            cache = lm(input_ids=ids[:, :S0], use_cache=True).past_key_values
            n0 = F.launch_count()
            lm(input_ids=ids[:, S0:], past_key_values=cache, use_cache=True)
            per_step.add(F.launch_count() - n0)
            lm.clear_conditioned_layers()
    assert len(per_step) == 1, per_step
    print(f"otter_b200 kernel launches per cached step (2 layers, 1 gated block): {per_step.pop()}")
