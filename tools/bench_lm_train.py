"""Time one decoder layer's forward + backward, frozen and trainable, on one GPU (CUDA events after warm-up).

  python tools/bench_lm_train.py [--steps 20] [--warmup 5] [--tokens 1024,8192]

Layers (B * S tokens, S = min(tokens, 2048)):
  mpt7b      the MPT-7B block (D 4096, 32 heads, ALiBi, GELU MLP 16384, no biases) on FrozenMPTBlock
  llama7b    the LLaMA-7B layer (D 4096, 32 heads, I 11008, default RoPE) on FrozenLlamaDecoderLayer
  llama31_8b the Llama-3.1-8B layer (D 4096, 32 heads, 8 K/V heads, I 14336, llama3 RoPE) on FrozenLlamaDecoderLayer
Setups per layer:
  frozen     no parameter requires grad: the input gradient only
  trainable  every parameter requires grad: the input gradient and every weight gradient (fp32, fresh each step)
  hf         (LLaMA layers) HF's LlamaDecoderLayer under bf16 autocast, fp32 trainable weights, SDPA attention
Prints the card name and power limit first, then one JSON line per measurement: milliseconds per step (median) and the
peak allocated device memory during the timed steps (the layer's weights, its inputs and, when trainable, its fp32
weight gradients included).
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "tools"))

from bench_llama_layer import LLAMA3, _init_, card, timed  # noqa: E402


def measure(step, args):
    import torch
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    r = timed(step, args.steps, args.warmup)
    r["peak_mib"] = round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)
    return r


def layer_step(layer, call, x, dy):
    def step():
        x.grad = None
        for p in layer.parameters():
            p.grad = None
        call(x).backward(dy)
    return step


def _release(module):
    import torch
    for p in module.parameters():
        p.grad = None
    module.cpu()
    torch.cuda.empty_cache()


def bench_layer(name, layer, call, args, out, hf=None):
    """Each setup alone on the card, so that its peak memory counts only its own weights, gradients and activations."""
    import torch
    D = 4096
    for T in args.tokens:
        S = min(T, 2048)
        B = T // S
        x = (torch.randn(B, S, D, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
        dy = torch.randn(B, S, D, device="cuda").to(torch.bfloat16)
        layer.cuda()
        for setup in ("frozen", "trainable"):
            layer.requires_grad_(setup == "trainable")
            out(dict(layer=name, setup=setup, B=B, S=S, **measure(layer_step(layer, call, x, dy), args)))
        _release(layer)
        if hf is not None:
            step, module = hf(B, S, x.detach().float().requires_grad_(True), dy.float())
            out(dict(layer=name, setup="hf", B=B, S=S, **measure(step, args)))
            _release(module)


def hf_llama(mine, D, H, KV, I, rope):
    import torch
    from transformers import LlamaConfig
    from transformers.models.llama import modeling_llama as M
    cfg = LlamaConfig(hidden_size=D, num_attention_heads=H, num_key_value_heads=KV, intermediate_size=I,
                      num_hidden_layers=1, rms_norm_eps=1e-5, max_position_embeddings=131072, rope_parameters=dict(rope))
    cfg._attn_implementation = "sdpa"
    hf = M.LlamaDecoderLayer(cfg, layer_idx=0)
    hf.load_state_dict(mine.state_dict())
    rot = M.LlamaRotaryEmbedding(cfg)

    def make(B, S, x, dy):
        hf.cuda().requires_grad_(True)
        rot.cuda()
        pos = torch.arange(S, device="cuda")[None].expand(B, S)

        def step():
            x.grad = None
            for p in hf.parameters():
                p.grad = None
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = hf(x, attention_mask=None, position_ids=pos, position_embeddings=rot(x, pos))
                y = y[0] if isinstance(y, tuple) else y
            y.float().backward(dy)
        return step, hf
    return make


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tokens", default="1024,8192")
    ap.add_argument("--layers", default="mpt7b,llama7b,llama31_8b")
    args = ap.parse_args()
    args.tokens = [int(t) for t in args.tokens.split(",")]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lm_train: no GPU")
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    from otter_b200.lm_mpt import FrozenMPTBlock

    def out(rec):
        print(json.dumps(rec), flush=True)
    out({"card": card()})
    layers = args.layers.split(",")
    if "mpt7b" in layers:
        blk = FrozenMPTBlock(4096, 32, expansion_ratio=4, no_bias=True)
        _init_(blk, 0)
        bench_layer("mpt7b", blk, lambda x: blk(x)[0], args, out)
        del blk
    for name, (H, KV, I, rope) in (("llama7b", (32, 32, 11008, None)), ("llama31_8b", (32, 8, 14336, LLAMA3))):
        if name not in layers:
            continue
        kw = {} if rope is None else dict(num_key_value_heads=KV, rope_parameters=rope, max_position_embeddings=131072)
        layer = FrozenLlamaDecoderLayer(4096, H, I, 1e-5, **kw)
        _init_(layer, 1)
        hf = hf_llama(layer, 4096, H, KV, I, rope or {"rope_type": "default", "rope_theta": 10000.0})
        bench_layer(name, layer, lambda x, layer=layer: layer(x), args, out, hf=hf)
        del layer, hf


if __name__ == "__main__":
    main()
