"""Time one decoder layer's forward + backward with LoRA adapters, against the frozen and the fully trainable layer, on one
GPU (CUDA events after warm-up).

  python tools/bench_lora.py [--steps 20] [--warmup 5] [--tokens 1024,8192] [--r 16] [--p 0.05]

Layers (B * S tokens, S = min(tokens, 2048): 1x1024 and 4x2048 by default):
  mpt7b      the MPT-7B block (D 4096, 32 heads, GELU MLP 16384, no biases), adapter on Wqkv
  llama7b    the LLaMA-7B layer (D 4096, 32 heads, I 11008), adapters on q_proj / v_proj
  llama31_8b the Llama-3.1-8B layer (D 4096, 32 heads, 8 K/V heads, I 14336, llama3 RoPE), adapters on q_proj / v_proj
Setups per layer:
  frozen     no parameter requires grad: the input gradient only
  lora       LoRA r / lora_alpha = 2r / dropout p (training mode) as otter_b200.lora.wrap_lora builds it: only the adapters
             train (fp32 gradients, fresh each step); the base weights stay frozen
  trainable  no adapters, every parameter requires grad
Prints the card name and power limit first, then one JSON line per measurement: milliseconds per step (median) and the
peak allocated device memory during the timed steps.
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "tools"))

from bench_llama_layer import LLAMA3, _init_, card  # noqa: E402
from bench_lm_train import _release, layer_step, measure  # noqa: E402


def bench(name, make, targets, call, args, out):
    import torch
    from otter_b200.lora import wrap_lora
    D = 4096
    for T in args.tokens:
        S = min(T, 2048)
        B = T // S
        x = (torch.randn(B, S, D, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
        dy = torch.randn(B, S, D, device="cuda").to(torch.bfloat16)
        for setup in ("frozen", "lora", "trainable"):
            layer = make()
            if setup == "lora":
                wrap_lora(layer, r=args.r, lora_alpha=2 * args.r, lora_dropout=args.p, target_modules=targets)
                with torch.no_grad():                 # a trained adapter: B != 0 (the cost does not depend on it)
                    for n, p in layer.named_parameters():
                        if "lora_B" in n:
                            p.normal_(0, 0.02)
            layer.cuda().train()
            if setup == "trainable":
                layer.requires_grad_(True)
            rec = dict(layer=name, setup=setup, B=B, S=S, **measure(layer_step(layer, lambda x, m=layer: call(m, x), x, dy), args))
            if setup == "lora":
                rec.update(r=args.r, p=args.p)
            out(rec)
            _release(layer)
            del layer


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tokens", default="1024,8192")
    ap.add_argument("--layers", default="mpt7b,llama7b,llama31_8b")
    ap.add_argument("--r", type=int, default=16)
    ap.add_argument("--p", type=float, default=0.05)
    args = ap.parse_args()
    args.tokens = [int(t) for t in args.tokens.split(",")]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lora: no GPU")
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    from otter_b200.lm_mpt import FrozenMPTBlock

    def out(rec):
        print(json.dumps(rec), flush=True)
    out({"card": card()})
    layers = args.layers.split(",")
    if "mpt7b" in layers:
        def make_mpt():
            blk = FrozenMPTBlock(4096, 32, expansion_ratio=4, no_bias=True)
            _init_(blk, 0)
            return blk
        bench("mpt7b", make_mpt, ["Wqkv"], lambda m, x: m(x)[0], args, out)
    for name, (H, KV, I, rope) in (("llama7b", (32, 32, 11008, None)), ("llama31_8b", (32, 8, 14336, LLAMA3))):
        if name not in layers:
            continue
        kw = {} if rope is None else dict(num_key_value_heads=KV, rope_parameters=rope, max_position_embeddings=131072)

        def make_llama(kw=kw, H=H, I=I):
            layer = FrozenLlamaDecoderLayer(4096, H, I, 1e-5, **kw)
            _init_(layer, 1)
            return layer
        bench(name, make_llama, ["q_proj", "v_proj"], lambda m, x: m(x), args, out)


if __name__ == "__main__":
    main()
