"""KV-cache decode on one H100: the two decode kernels against their roofline, and the cached step against the uncached
full-prefix step that generate(use_cache=False) runs.  CUDA events after warm-up, medians; the card, its power limit and
its maximum SM clock are read in the same run and printed with the numbers.

    python tools/bench_mpt_decode.py [--layers 32] [--iters 30] [--profile DIR]

Bytes are counted from the shapes: a linear layer reads its N x K bf16 weight once (x and y are under 1 %); decode
attention reads T rows of K and of V, 128 bf16 each, per (sequence, head).  Kernel rows time the device work alone (a CUDA
graph of back-to-back calls); block and stack rows time the eager Python loop generate() runs, launch gaps included, and
the profile splits one such step into kernel families and gaps.  "roofline" is the H100 SXM data-sheet HBM3
bandwidth (3.35 TB/s); the share is bytes / time over that.  Weight sets rotate through more copies than the 50 MB L2 holds.
"""
import argparse
import json
import statistics
import subprocess
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from otter_b200 import functional as F  # noqa: E402
from otter_b200.lm_mpt import FrozenMPTBlock, MPTKVCache  # noqa: E402

DEV, BF16, HBM = "cuda:0", torch.bfloat16, 3.35e12
D, H = 4096, 32
SHAPES = {"Wqkv": (3 * D, D), "out_proj": (D, D), "up_proj": (4 * D, D), "down_proj": (D, 4 * D)}


def timed(fns, iters, warmup=3):
    """Median microseconds of one host call of each callable (enqueue + kernels), alternated within every repetition:
    what an eager decode loop pays."""
    for _ in range(warmup):
        for fn in fns:
            fn()
    ts = [[] for _ in fns]
    for _ in range(iters):
        for i, fn in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts[i].append(e0.elapsed_time(e1) * 1e3)
    return [statistics.median(t) for t in ts]


def timed_kernels(fns, iters, calls=12, warmup=3):
    """Median microseconds of the device work of one call: `calls` back-to-back calls are captured into a CUDA graph and
    the replay is timed, so the Python / launch overhead of a 10-100 us kernel is not in the number."""
    graphs = []
    for fn in fns:
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(calls):
                fn()
        graphs.append(g)
    return [t / calls for t in timed([g.replay for g in graphs], iters)]


def bench_linear(iters):
    rows = []
    for name, (N, K) in SHAPES.items():
        copies = max(2, int(200e6 // (N * K * 2)) + 1)                  # > 50 MB L2 between two uses of a copy
        ws = [(torch.randn((N, K), device=DEV) * K ** -0.5).to(BF16) for _ in range(copies)]
        for M in (1, 4, 8, 16):
            x = torch.randn((M, K), device=DEV).to(BF16)
            state = {"i": 0}

            def run(fn):
                def go():
                    state["i"] = (state["i"] + 1) % copies
                    fn(x, ws[state["i"]])
                return go
            fns = [run(F.linear_fwd)] + ([run(F.linear_small_m)] if M <= F.SMALL_M_MAX else [])
            t = timed_kernels(fns, iters)
            by = N * K * 2
            rows.append(dict(layer=name, M=M, N=N, K=K, linear_fwd_us=round(t[0], 1), linear_fwd_GBs=round(by / t[0] / 1e3),
                             small_m_us=round(t[1], 1) if len(t) > 1 else None,
                             small_m_GBs=round(by / t[1] / 1e3) if len(t) > 1 else None,
                             small_m_roofline=round(by / (t[1] * 1e-6) / HBM, 3) if len(t) > 1 else None))
            print(json.dumps(rows[-1]), flush=True)
        del ws
    return rows


def bench_attn(iters):
    rows = []
    for B in (1, 8):
        for T in (256, 1024, 2048):
            copies = max(2, int(200e6 // (B * T * 2 * D * 2)) + 1)
            caches = [torch.randn((B, T, 2 * D), device=DEV).to(BF16) for _ in range(copies)]
            q = torch.randn((B, D), device=DEV).to(BF16)
            state = {"i": 0}

            def go():
                state["i"] = (state["i"] + 1) % copies
                c = caches[state["i"]]
                F.lm_attn_decode(q, c[:, :, :D], c[:, :, D:], T)
            (t,) = timed_kernels([go], iters)
            by = B * H * T * 128 * 2 * 2
            rows.append(dict(kernel="lm_attn_decode", B=B, H=H, T=T, splits=F.lm_attn_decode_splits(B, H, T), us=round(t, 1),
                             GBs=round(by / t / 1e3), roofline=round(by / (t * 1e-6) / HBM, 3)))
            print(json.dumps(rows[-1]), flush=True)
    return rows


def make_stack(n_layers):
    torch.manual_seed(0)
    blocks = []
    for _ in range(n_layers):
        blk = FrozenMPTBlock(D, H, no_bias=True).to(DEV)
        with torch.no_grad():
            for p in blk.parameters():
                if p.dim() == 2:
                    p.normal_(0, p.shape[1] ** -0.5)
        blocks.append(blk.to(BF16).eval())
    return blocks


def bench_stack(n_layers, iters):
    """ms per token: one cached step of the stack at prefix T, and the uncached forward of the T + 1 tokens."""
    blocks = make_stack(n_layers)
    rows = []
    with torch.no_grad():
        for B in (1, 4):
            for T in (256, 1024, 2048):
                x = torch.randn((B, T + 1, D), device=DEV).to(BF16)
                cache = MPTKVCache(n_layers)
                h = x[:, :T]
                for i, blk in enumerate(blocks):
                    h = blk(h, past_key_value=(cache, i))[0]
                cache.seq_len = T
                cache.reserve(T + 1)

                def cached():
                    h = x[:, T:]
                    for i, blk in enumerate(blocks):
                        h = blk(h, past_key_value=(cache, i))[0]       # seq_len stays T: the step rewrites row T

                def uncached():
                    h = x
                    for blk in blocks:
                        h = blk(h)[0]
                t = timed([cached, uncached], max(5, iters // 3), warmup=2)       # eager, as generate() runs it
                rows.append(dict(layers=n_layers, B=B, prefix=T, cached_ms=round(t[0] / 1e3, 3),
                                 uncached_ms=round(t[1] / 1e3, 3), ratio=round(t[1] / t[0], 1)))
                print(json.dumps(rows[-1]), flush=True)
                del cache
    return rows, blocks


def profile_step(blocks, out_dir, T=1024, B=1):
    """Share of one cached step by kernel family and the launch gaps, from torch.profiler (a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        x = torch.randn((B, T + 1, D), device=DEV).to(BF16)
        cache = MPTKVCache(len(blocks))
        h = x[:, :T]
        for i, blk in enumerate(blocks):
            h = blk(h, past_key_value=(cache, i))[0]
        cache.seq_len = T
        cache.reserve(T + 1)

        def step():
            h = x[:, T:]
            for i, blk in enumerate(blocks):
                h = blk(h, past_key_value=(cache, i))[0]
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                step()
            torch.cuda.synchronize()
    fam = {"attention": 0.0, "small_m_linear": 0.0, "layernorm": 0.0, "other": 0.0}
    spans = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            n = e.name
            k = ("attention" if "attn_decode" in n else "small_m_linear" if "linear_small_m" in n
                 else "layernorm" if "layernorm" in n or "ln_" in n else "other")
            fam[k] += e.device_time if hasattr(e, "device_time") else e.cuda_time
            spans.append((e.time_range.start, e.time_range.end))
    spans.sort()
    busy = sum(b - a for a, b in spans)
    wall = spans[-1][1] - spans[0][0]
    res = dict(prefix=T, B=B, layers=len(blocks), us_per_step={k: round(v / 5, 1) for k, v in fam.items()},
               kernel_us_per_step=round(busy / 5, 1), launch_gap_us_per_step=round((wall - busy) / 5, 1))
    print(json.dumps(dict(profile=res)), flush=True)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "mpt_decode_profile.json"), "w") as f:
        json.dump(res, f)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--profile", default=None, help="directory for the torch.profiler summary (skipped when not given)")
    ap.add_argument("--out", default=None, help="write all rows as JSON to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mpt_decode.py needs a GPU: nothing here can be measured on the CPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(card=card, torch=torch.__version__)), flush=True)
    res = dict(card=card, linear=bench_linear(a.iters), attention=bench_attn(a.iters))
    res["block"], _ = bench_stack(1, a.iters)
    res["stack"], blocks = bench_stack(a.layers, a.iters)
    if a.profile:
        res["profile"] = profile_step(blocks, a.profile)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
