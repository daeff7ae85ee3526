"""TEST INFRASTRUCTURE — fixtures of KV-cache decoding on the UNMODIFIED reference MPT, on seeded inputs:

  block     tests/golden/mpt_block_decode.pt     MPTBlock (mpt/blocks.py:23-88, attn_impl "torch", alibi, no bias) called
                                                 with past_key_value: a prefill of 9 tokens, then 4 cached steps of one
                                                 token; outputs and the K / V the reference returns
  generate  tests/golden/tiny_mpt_generate.pt    the tiny Otter over the reference's MPTForCausalLM of
                                                 oracle/make_golden_r2.mpt_golden in eval mode: greedy decoding of 6 new
                                                 tokens with use_cache=True (the reference's default) and use_cache=False;
                                                 token ids, per-step logits and the top-1 / top-2 logit margin of each step.
                                                 The reference's MPTForCausalLM predates GenerationMixin being opt-in, so
                                                 under transformers 5 it has no generate(): the loop below is greedy search
                                                 over the reference's own prepare_inputs_for_generation
                                                 (modeling_mpt.py:460-492) and forward, conditioned as
                                                 OtterForConditionalGeneration.generate does (modeling_otter.py:1020-1042)

Run where the reference tree is available:  python oracle/make_golden_mpt_decode.py [block] [generate]
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shims  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
PREFILL, STEPS, NEW_TOKENS = 9, 4, 6


def block_decode_golden():
    from oracle.make_golden_lm import reference_block
    sys.path.insert(0, os.path.join(ref_shims.REF_ROOT, "src"))
    out = {}
    for name, (B, D, H) in {"a": (2, 64, 4), "b": (1, 96, 6)}.items():                # H=6: non-power-of-two slopes
        blk, _ = reference_block(D, H, no_bias=True, seed=5)
        from otter_ai.models.mpt.attention import build_attn_bias
        x = torch.randn(B, PREFILL + STEPS, D, generator=torch.Generator().manual_seed(21))
        ys, past, T = [], (), 0
        with torch.no_grad():
            for n in [PREFILL] + [1] * STEPS:
                T += n
                # modeling_mpt.py:131-151: the ALiBi bias of the whole context; the attention slices its last s_k keys
                bias = build_attn_bias("torch", torch.zeros(1, H, 1, T), H, T, causal=True, alibi=True, alibi_bias_max=8)
                y, _, past = blk(x[:, T - n:T], past_key_value=past, attn_bias=bias, is_causal=True)
                ys.append(y.clone())
        out[name] = {"shape": (B, D, H), "prefill": PREFILL, "steps": STEPS,
                     "params": {k: v.detach().clone() for k, v in blk.state_dict().items()},
                     "x": x, "ys": ys, "k": past[0].clone(), "v": past[1].clone()}
    path = os.path.join(GOLDEN, "mpt_block_decode.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


def mpt_generate_golden(seed_offset=6):      # the input seed whose greedy steps have the widest top-1 / top-2 margins
    from transformers import CLIPVisionConfig
    from oracle.make_golden import SEED
    from oracle.make_golden_r2 import EMB_KINDS, MPT_TINY, tiny_inputs
    from oracle.seeded import load_seeded_
    ref = ref_shims.load_reference_otter()
    vcfg = CLIPVisionConfig(hidden_size=1024, intermediate_size=4096, num_hidden_layers=1, num_attention_heads=16,
                            image_size=224, patch_size=14, hidden_act="quick_gelu")
    cfg = ref.OtterConfig(vision_config=vcfg.to_dict(), text_config=dict(MPT_TINY), cross_attn_every_n_layers=2)
    cfg.text_config.hidden_size = 256
    cfg.text_config.tie_word_embeddings = True
    model = ref.OtterForConditionalGeneration(cfg)
    load_seeded_(model, SEED, kinds=EMB_KINDS)
    model.eval()
    vision_x, lang_x, _ = tiny_inputs(model.media_token_id, L=12, seed=SEED + seed_offset, name="in.mptgen.vision_x")
    runs = {}
    lm = model.lang_encoder
    for use_cache in (True, False):
        ids, mask, past, steps = lang_x.clone(), torch.ones_like(lang_x), None, []
        with torch.no_grad():
            model._encode_vision_x(vision_x=vision_x)
            for _ in range(NEW_TOKENS):
                inputs = lm.prepare_inputs_for_generation(ids, past_key_values=past, attention_mask=mask,
                                                          use_cache=use_cache)
                o = lm(**inputs)
                past = o.past_key_values if use_cache else None
                steps.append(o.logits[:, -1].float())
                ids = torch.cat([ids, steps[-1].argmax(-1, keepdim=True)], dim=1)
                mask = torch.ones_like(ids)
            lm.clear_conditioned_layers()
        logits = torch.stack(steps, dim=1)                                             # [B, steps, V]
        top2 = logits.topk(2, dim=-1).values
        runs[use_cache] = dict(sequences=ids, logits=logits, margin=top2[..., 0] - top2[..., 1])
        print("use_cache", use_cache, ids[:, lang_x.shape[1]:].tolist(), "margins", runs[use_cache]["margin"])
        # generate() would stop a row there and pad it
        assert not (ids[:, lang_x.shape[1]:] == model.eoc_token_id).any(), "an end-of-chunk token: use another seed"
    path = os.path.join(GOLDEN, "tiny_mpt_generate.pt")
    torch.save(dict(seed=SEED, input_seed=SEED + seed_offset, media_token_id=model.media_token_id, lang_x=lang_x,
                    eoc_token_id=model.eoc_token_id, new_tokens=NEW_TOKENS, text_config=dict(MPT_TINY),
                    vision_config=vcfg.to_dict(), cached=runs[True], uncached=runs[False]), path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    which = sys.argv[1:] or ["block", "generate"]
    if "block" in which:
        block_decode_golden()
    if "generate" in which:
        mpt_generate_golden()
