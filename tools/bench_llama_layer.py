"""Time the frozen LLaMA decoder layer and its attention kernels on one GPU (CUDA events after warm-up).

  python tools/bench_llama_layer.py [--steps 20] [--warmup 5] [--parts gqa,attn,mha] [--parent DIR --rounds 3]

Parts (B = 4, S in {256, 2048}; forward + input gradient, the layer is frozen):
  gqa   one Llama-3.1-8B decoder layer (D 4096, 32 heads, 8 K/V heads, I 14336, llama3 RoPE theta 5e5, factor 8,
        low 1, high 4, original 8192) on FrozenLlamaDecoderLayer, and on HF's LlamaDecoderLayer under bf16 autocast
        (fp32 weights, SDPA attention) -- what such a config runs on without the swap
  attn  lm_attn_fwd + lm_attn_bwd alone, H = 32, kv_heads in {32, 8}
  mha   the LLaMA-7B layer (D 4096, 32 heads, I 11008, default RoPE) on FrozenLlamaDecoderLayer
--parent DIR: DIR is a built checkout of another commit; the mha part runs alternately from this tree and from DIR,
`--rounds` times each, in separate processes, so that both see the same card in the same state.
Prints the card name and power limit first, then one JSON line per measurement (milliseconds per step, median).
"""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return {"ms_median": ts[len(ts) // 2], "ms_min": ts[0], "ms_max": ts[-1], "steps": steps}


LLAMA3 = {"rope_type": "llama3", "rope_theta": 500000.0, "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
          "original_max_position_embeddings": 8192}


def _init_(module, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.02 if p.dim() == 2 else 0.1) + (1.0 if p.dim() == 1 else 0.0))


def layer_step(layer, B, S, D, dtype):
    import torch
    x = (torch.randn(B, S, D, device="cuda") * 0.5).to(dtype).requires_grad_(True)
    dy = torch.randn(B, S, D, device="cuda")        # fp32, as from a loss computed in fp32
    pos = torch.arange(S, device="cuda")[None]

    def step():
        x.grad = None
        layer(x, position_ids=pos).backward(dy)
    return step


def part_gqa(args, out):
    import torch
    from transformers import LlamaConfig
    from transformers.models.llama import modeling_llama as M
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    D, H, KV, I = 4096, 32, 8, 14336
    mine = FrozenLlamaDecoderLayer(D, H, I, 1e-5, num_key_value_heads=KV, rope_parameters=LLAMA3,
                                   max_position_embeddings=131072)
    _init_(mine, 0)
    mine.cuda()
    cfg = LlamaConfig(hidden_size=D, num_attention_heads=H, num_key_value_heads=KV, intermediate_size=I,
                      num_hidden_layers=1, rms_norm_eps=1e-5, max_position_embeddings=131072, rope_parameters=dict(LLAMA3))
    cfg._attn_implementation = "sdpa"
    hf = M.LlamaDecoderLayer(cfg, layer_idx=0)
    hf.load_state_dict(mine.state_dict())
    hf.cuda().requires_grad_(False)
    rot = M.LlamaRotaryEmbedding(cfg).cuda()
    for S in (256, 2048):
        B = 4
        out(dict(part="gqa", impl="otter_b200 FrozenLlamaDecoderLayer", B=B, S=S,
                 **timed(layer_step(mine, B, S, D, torch.bfloat16), args.steps, args.warmup)))
        x = torch.randn(B, S, D, device="cuda").mul_(0.5).requires_grad_(True)
        dy = torch.randn(B, S, D, device="cuda")
        pos = torch.arange(S, device="cuda")[None].expand(B, S)

        def hf_step():
            x.grad = None
            with torch.autocast("cuda", dtype=torch.bfloat16):
                pe = rot(x, pos)
                y = hf(x, attention_mask=None, position_ids=pos, position_embeddings=pe)
                y = y[0] if isinstance(y, tuple) else y
            y.float().backward(dy)
        out(dict(part="gqa", impl="HF LlamaDecoderLayer, bf16 autocast, sdpa", B=B, S=S,
                 **timed(hf_step, args.steps, args.warmup)))
    del mine, hf
    torch.cuda.empty_cache()


def part_attn(args, out):
    import torch
    from otter_b200 import functional as F
    H, B = 32, 4
    for kv in (32, 8):
        for S in (256, 2048):
            qkv = (torch.randn(B * S, (H + 2 * kv) * 128, device="cuda") * 0.8).to(torch.bfloat16)
            dout = (torch.randn(B * S, H * 128, device="cuda") * 0.5).to(torch.bfloat16)
            kw = {} if kv == H else {"kv_heads": kv}

            def step():
                o, lse = F.lm_attn_fwd(qkv, B, S, H, **kw)
                F.lm_attn_bwd(dout, qkv, o, lse, B, S, H, **kw)
            out(dict(part="attn", H=H, kv_heads=kv, B=B, S=S, **timed(step, args.steps, args.warmup)))


def part_mha(args, out, tree):
    import torch
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    D, H, I = 4096, 32, 11008
    layer = FrozenLlamaDecoderLayer(D, H, I)
    _init_(layer, 1)
    layer.cuda()
    for S in (256, 2048):
        out(dict(part="mha", tree=tree, B=4, S=S, **timed(layer_step(layer, 4, S, D, torch.bfloat16), args.steps, args.warmup)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--parts", default="gqa,attn,mha")
    ap.add_argument("--parent", default=None, help="built checkout of another commit (mha part, alternated)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--tree", default=HERE, help=argparse.SUPPRESS)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_llama_layer: no GPU")

    def out(rec):
        print(json.dumps(rec), flush=True)
    parts = args.parts.split(",")
    if args.tree == HERE:
        out({"card": card()})
    if "gqa" in parts:
        part_gqa(args, out)
    if "attn" in parts:
        part_attn(args, out)
    if "mha" in parts:
        if args.parent is None:
            part_mha(args, out, "this")
        else:                                   # alternate the two trees, one process per run
            for _ in range(args.rounds):
                for tree, name in ((HERE, "this"), (os.path.abspath(args.parent), "parent")):
                    cmd = [sys.executable, os.path.abspath(__file__), "--parts", "mha-only", "--tree", tree,
                           "--steps", str(args.steps), "--warmup", str(args.warmup)]
                    r = subprocess.run(cmd, capture_output=True, text=True, check=True)
                    for line in r.stdout.splitlines():
                        rec = json.loads(line)
                        rec["tree"] = name
                        out(rec)
    if "mha-only" in parts:
        part_mha(args, out, "this")


if __name__ == "__main__":
    main()
