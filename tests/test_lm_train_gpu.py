"""GPU: weight gradients of the MPT and LLaMA decoder layers on the sm_90a kernels.

- otb_rmsnorm_bwd_params against float64 through the C ABI, in the style of tests/test_rowwise_edges_gpu.py: NaN-padded,
  offset canvases for every buffer (elements a kernel does not own keep their NaN bits), rows from 1 past the CTA cap
  (4 * SMs CTAs of 8 rows), ragged D from 8 to 8192, with and without `add` and `accumulate`.  dx must be bit-identical
  to otb_rmsnorm_bwd's, and a repeated run bit-identical to the first.
  Metric for dweight[j] = sum_r dy[r,j] x[r,j] rstd[r]: |got - ref| <= 2^-16 sum_r |dy x rstd| (+ 2^-23 |got| for the
  accumulate add).  Each term is two fp32 products of exact bf16 inputs and an fp32 rstd (3 roundings of 2^-24); a
  column's path through the sums is the rows of one CTA in order (<= 8 * ceil(groups / chunks)), the 8-way strided
  chunk sums and an 8-leaf tree: fewer than 2^8 fp32 additions for every shape here (recursive summation errs by < n u
  sum|terms|), so 2^-16 holds with room.  The CPU tests below show the bound rejects a dropped row and a bf16 rstd.
- The layers against float64 oracles (oracle/restatement_lm.mpt_block, oracle/restatement_llama.llama_layer,
  llama_layer_gqa of tests/test_llama_gqa_cpu.py) at tile-edge S and at 7B width: every parameter gradient within the
  bf16 parameter-gradient tolerance (rel-Frobenius <= 4e-2, DESIGN.md §2); y and dx bit-identical to the frozen layer's;
  a repeated backward bit-identical; two backward passes exactly twice one, through `.grad` and an fp32
  FlatGradBuffer; a direct bf16 wire sink holding the fp32 gradient rounded to bf16, and refusing a second write.
- Model level: MPTForCausalLM unfrozen against the oracle blocks composed in float64; Otter over a GQA LLaMA with
  train_lang_encoder=True against the same Otter with HF's fp32 layers (OTB_LLAMA_LAYERS=0): loss, every LM gradient and
  three SGD steps (the forward after a step reads the refreshed bf16 weight copies).
- A fresh process whose first backward reaches the library through a bf16, contiguous gradient.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import restatement_lm as RLM
from oracle import restatement_llama as RL
from oracle.ref_shims import FakeTokenizer
from test_llama_gqa_cpu import ROPES, llama_layer_gqa
from test_rowwise_edges_gpu import _Canvas, _geom, _in, _lib, _ok, _rnd, _sms, _stream, rms_ref

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda:0"
gpu = pytest.mark.gpu
REL_PARAM = 4e-2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------
# the RMSNorm weight-gradient metric, and its power on the CPU
# ------------------------------------------------------------------------------------------------------------------
def dw_terms(x, dy, rstd):
    """float64 [rows, D] terms dy * x * rstd."""
    return dy.double() * x.double() * rstd.double()[:, None]


def dw_ratio(got, ref, absum, prior=None):
    bound = 2.0 ** -16 * absum + (2.0 ** -23 * got.double().abs() if prior is not None else 0.0) + 1e-30
    return ((got.double() - ref).abs() / bound).max().item()


def _power_case(rows=1024, D=1024):
    g = torch.Generator().manual_seed(5)
    x, dy = _rnd(g, rows, D, scale=2.0), _rnd(g, rows, D)
    rstd = (x.double().pow(2).mean(-1) + 1e-6).rsqrt()
    t = dw_terms(x, dy, rstd)
    return x, dy, rstd, t.sum(0), t.abs().sum(0)


def test_dw_bound_rejects_a_dropped_row():
    x, dy, rstd, ref, absum = _power_case()
    mut = ref - dw_terms(x[7:8], dy[7:8], rstd[7:8])[0]
    r = dw_ratio(mut, ref, absum)
    print(f"POWER dropped row: {r:.1f} x bound")
    assert r > 4.0


def test_dw_bound_rejects_a_bf16_rstd():
    x, dy, rstd, ref, absum = _power_case()
    mut = dw_terms(x, dy, rstd.to(BF16).double()).sum(0)
    r = dw_ratio(mut, ref, absum)
    print(f"POWER bf16 rstd: {r:.1f} x bound")
    assert r > 2.0


def test_dw_bound_accepts_the_fp32_rounded_answer():
    x, dy, rstd, ref, absum = _power_case()
    assert dw_ratio(ref.float(), ref, absum) <= 0.01


# ------------------------------------------------------------------------------------------------------------------
# GPU: otb_rmsnorm_bwd_params
# ------------------------------------------------------------------------------------------------------------------
def _rows(spec):
    """An int, or 'k*cap+c': k times the row count that fills the kernel's CTA cap (4 * SMs CTAs of 8 rows), plus c."""
    if isinstance(spec, int):
        return spec
    k, c = spec.split("*cap")
    return int(k) * 32 * _sms() + int(c or 0)


def _run_rms_params(tag, rows, D, *, add, acc, pad, eps=1e-6):
    lib = _lib()
    g = torch.Generator().manual_seed(rows * 31 + D)
    x = _rnd(g, rows, D, scale=2.0)
    if rows >= 3:
        x[2] = 0.0                                                     # all-zero row: rstd = eps^-1/2, zero terms
    w = (1 + 0.2 * torch.randn(D, generator=g)).to(DEV)
    dy, a = _rnd(g, rows, D), _rnd(g, rows, D)
    r = rms_ref(x.to(DEV), w, eps, dy.to(DEV))
    rs32 = r["rstd"].float()
    cx, c0x = _in(x, pad)
    cdy, c0dy = _in(dy, 3 * pad)
    ca, c0a = _in(a, pad) if add else (None, 0)
    pdx, c0dx = _geom(D, pad)
    prior = torch.randn(D, generator=g).to(DEV) * 4 if acc else None
    chunks = lib.otb_rmsnorm_bwd_chunks(rows, D)
    assert 1 <= chunks <= 4 * _sms()

    def run():
        cdx = _Canvas(rows, pdx)
        cdx.own(rows, c0dx, c0dx + D)
        cdw = _Canvas(1, D + 2 * pad + 4, F32, extra=0)
        cdw.own(1, pad, pad + D, prior[None] if acc else None)
        ws = torch.full((chunks * D,), float("nan"), device=DEV)
        _ok(lib.otb_rmsnorm_bwd_params(cdy.ptr(c0dy), cdy.pitch, cx.ptr(c0x), cx.pitch, C.c_void_p(rs32.data_ptr()),
                                       C.c_void_p(w.data_ptr()), ca.ptr(c0a) if add else None, ca.pitch if add else 0,
                                       cdx.ptr(c0dx), cdx.pitch, cdw.ptr(pad), int(acc), C.c_void_p(ws.data_ptr()),
                                       rows, D, _stream()), "otb_rmsnorm_bwd_params")
        return cdx, cdw

    cdx, cdw = run()
    cref = _Canvas(rows, pdx)
    cref.own(rows, c0dx, c0dx + D)
    _ok(lib.otb_rmsnorm_bwd(cdy.ptr(c0dy), cdy.pitch, cx.ptr(c0x), cx.pitch, C.c_void_p(rs32.data_ptr()),
                            C.c_void_p(w.data_ptr()), ca.ptr(c0a) if add else None, ca.pitch if add else 0,
                            cref.ptr(c0dx), cref.pitch, rows, D, _stream()), "otb_rmsnorm_bwd")
    cdx2, cdw2 = run()
    torch.cuda.synchronize()
    cdx.check(f"{tag} dx")
    cdw.check(f"{tag} dweight")
    assert torch.equal(cdx.bits(), cref.bits()), f"{tag}: dx differs from otb_rmsnorm_bwd's"
    assert torch.equal(cdx.bits(), cdx2.bits()) and torch.equal(cdw.bits(), cdw2.bits()), f"{tag}: not bit-repeatable"
    t = dw_terms(x.to(DEV), dy.to(DEV), rs32)
    ref = t.sum(0) + (prior.double() if acc else 0.0)
    got = cdw.t[0, pad:pad + D]
    ratio = dw_ratio(got, ref, t.abs().sum(0), prior)
    print(f"RATIO {tag} dweight {ratio:.4f} (chunks {chunks})")
    assert ratio <= 1.0, ratio


@gpu
@pytest.mark.parametrize("rows,D,add,acc,pad", [
    (1, 8, False, False, 0), (7, 264, True, True, 16), (9, 1032, True, False, 32), (300, 5128, False, True, 0),
    ("1*cap-1", 4096, True, True, 0), ("1*cap", 2056, False, False, 16), ("1*cap+1", 4104, True, True, 16),
    ("2*cap+5", 8192, True, False, 0), (8192, 4096, True, True, 32),
])
def test_rmsnorm_bwd_params(rows, D, add, acc, pad):
    n = _rows(rows)
    _run_rms_params(f"rms_params[{rows}={n}-{D}-add{int(add)}-acc{int(acc)}-{pad}]", n, D, add=add, acc=acc, pad=pad)


@gpu
def test_rmsnorm_bwd_params_rejects_bad_arguments():
    lib = _lib()
    n0 = lib.otb_launch_count()
    p = C.c_void_p(0x10000)
    assert lib.otb_rmsnorm_bwd_params(p, 8, p, 8, p, p, None, 0, p, 8, None, 0, p, 4, 8, None) == 1      # no dweight
    assert lib.otb_rmsnorm_bwd_params(p, 8, p, 8, p, p, None, 0, p, 8, p, 0, C.c_void_p(0x10004), 4, 8, None) == 1
    assert b"aligned" in lib.otb_last_error()
    assert lib.otb_rmsnorm_bwd_params(p, 16392, p, 16392, p, p, None, 0, p, 16392, p, 0, p, 4, 16392, None) == 1
    assert lib.otb_launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------
# GPU: the layers
# ------------------------------------------------------------------------------------------------------------------
def _rel(got, ref):
    got, ref = got.detach().double(), ref.detach().to(got.device).double()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-30)).item()


def _init(module, seed):
    torch.manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            if p.dim() == 2:
                p.copy_(torch.randn_like(p) / math.sqrt(p.shape[1]))
            else:
                p.add_(0.1 * torch.randn_like(p))


def _mpt(D, H, no_bias):
    from otter_b200.lm_mpt import FrozenMPTBlock
    blk = FrozenMPTBlock(D, H, no_bias=no_bias)
    _init(blk, D + H)

    def oracle(x, p):
        return RLM.mpt_block(x, p, H)
    return blk, oracle, lambda m, x: m(x)[0]


def _llama(D, H, kv, rope, inter):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    kw = {} if rope == "default" and kv == H else dict(num_key_value_heads=kv, rope_parameters=ROPES[rope],
                                                         max_position_embeddings=131072)
    layer = FrozenLlamaDecoderLayer(D, H, inter, **kw)
    _init(layer, D + kv)
    inv = layer.rope_inv_freq(torch.device("cpu")).to(DEV) if kw else None
    sc = layer.rope_attention_scaling

    def oracle(x, p):
        if not kw:
            return RL.llama_layer(x, p, H)
        return llama_layer_gqa(x, p, H, num_kv_heads=kv, inv_freq=inv, attn_scale=sc)
    return layer, oracle, lambda m, x: m(x)


def _fwd_bwd(module, call, x, w):
    xg = x.clone().requires_grad_(True)
    y = call(module, xg)
    (y.float() * w).sum().backward()
    return y.detach(), xg.grad


def _grads(module):
    return {n: p.grad.detach().clone() for n, p in module.named_parameters()}


LAYER_CASES = {
    "mpt-s127-bias": lambda: _mpt(256, 2, False),
    "mpt-s129": lambda: _mpt(256, 2, True),
    "mpt7b-s128": lambda: _mpt(4096, 32, True),
    "llama-mha-s127": lambda: _llama(512, 4, 4, "default", 1024),
    "llama-gqa-llama3-s193": lambda: _llama(1024, 8, 2, "llama3", 2048),
    "llama7b-s128": lambda: _llama(4096, 32, 32, "default", 11008),
    "llama31-8b-gqa-s128": lambda: _llama(4096, 32, 8, "llama3", 14336),
}
SEQ = {"mpt-s127-bias": (2, 127), "mpt-s129": (1, 129), "mpt7b-s128": (1, 128), "llama-mha-s127": (2, 127),
       "llama-gqa-llama3-s193": (1, 193), "llama7b-s128": (1, 128), "llama31-8b-gqa-s128": (1, 128)}


@gpu
@pytest.mark.parametrize("case", list(LAYER_CASES))
def test_trainable_layer(case):
    from otter_b200.dp import FlatGradBuffer
    module, oracle, call = LAYER_CASES[case]()
    B, S = SEQ[case]
    D = module.d_model if hasattr(module, "d_model") else module.hidden_size
    p64 = {k: v.detach().to(DEV, F64).requires_grad_(True) for k, v in module.named_parameters()}
    module.to(DEV)
    g = torch.Generator().manual_seed(S)
    x = torch.randn(B, S, D, generator=g).to(BF16).to(DEV)
    w = torch.randn(B, S, D, generator=g).to(BF16).to(DEV).float()

    y0, dx0 = _fwd_bwd(module, call, x, w)                                   # frozen
    assert all(p.grad is None for p in module.parameters())
    module.requires_grad_(True)
    y1, dx1 = _fwd_bwd(module, call, x, w)
    assert torch.equal(y0.view(torch.int16), y1.view(torch.int16)), "y differs from the frozen layer's"
    assert torch.equal(dx0.view(torch.int16), dx1.view(torch.int16)), "dx differs from the frozen layer's"
    g1 = _grads(module)

    with torch.device(DEV):
        ref = oracle(x.double(), p64)
    (ref * w.double()).sum().backward()
    worst = 0.0
    for n, gr in g1.items():
        r = _rel(gr, p64[n].grad)
        worst = max(worst, r)
        assert r <= REL_PARAM, (n, r)
    print(f"REL {case}: worst parameter gradient {worst:.2e}, y {_rel(y1, ref):.2e}")

    for p in module.parameters():                                               # repeated backward: same bits
        p.grad = None
    _fwd_bwd(module, call, x, w)
    assert all(torch.equal(p.grad, g1[n]) for n, p in module.named_parameters()), "backward is not bit-repeatable"
    _fwd_bwd(module, call, x, w)                                                # accumulation into .grad
    assert all(torch.equal(p.grad, 2 * g1[n]) for n, p in module.named_parameters())

    params = list(module.parameters())
    fb = FlatGradBuffer(params)                                                 # fp32 sinks, accumulated by the kernels
    fb.begin_step()
    _fwd_bwd(module, call, x, w)
    _fwd_bwd(module, call, x, w)
    fb.finish_step()
    assert all(torch.equal(p.grad, 2 * g1[n]) for n, p in module.named_parameters())

    weights = [p for n, p in module.named_parameters() if p.dim() == 2]         # one wgrad GEMM each per step
    fb = FlatGradBuffer(params, comm_dtype=BF16, direct_params=weights)
    fb.begin_step()
    _fwd_bwd(module, call, x, w)
    fb.finish_step()
    for n, p in module.named_parameters():
        if p.dim() == 2:
            assert p._otb_grad.dtype == BF16 and torch.equal(p._otb_grad, g1[n].to(BF16)), n
        else:
            assert torch.equal(p.grad, g1[n]), n
    with pytest.raises(RuntimeError, match="one write per step"):
        _fwd_bwd(module, call, x, w)


# ------------------------------------------------------------------------------------------------------------------
# GPU: model level
# ------------------------------------------------------------------------------------------------------------------
def _mpt_lm_ref(ids, p, n_layers, H):
    x = p["transformer.wte.weight"][ids]
    for i in range(n_layers):
        pre = f"transformer.blocks.{i}."
        x = RLM.mpt_block(x, {k[len(pre):]: v for k, v in p.items() if k.startswith(pre)}, H)
    D = x.shape[-1]
    x = torch.nn.functional.layer_norm(x, (D,), p["transformer.norm_f.weight"], p.get("transformer.norm_f.bias"), 1e-5)
    logits = x @ p["transformer.wte.weight"].t()
    V = logits.shape[-1]
    return torch.nn.functional.cross_entropy(logits[:, :-1].reshape(-1, V), ids[:, 1:].reshape(-1))


@gpu
@pytest.mark.parametrize("no_bias", [True, False])
def test_unfrozen_mpt_lm_vs_the_oracle_blocks(no_bias):
    from otter_b200.lm_mpt import MPTConfig, MPTForCausalLM
    cfg = MPTConfig(d_model=256, n_heads=2, n_layers=2, expansion_ratio=4, max_seq_len=256, vocab_size=128,
                    no_bias=no_bias, attn_config={"alibi": True, "attn_impl": "torch"})
    model = MPTForCausalLM(cfg)
    _init(model, 11)
    model.requires_grad_(True)
    p64 = {k: v.detach().to(DEV, F64).requires_grad_(True) for k, v in model.named_parameters()}
    model.to(DEV)
    ids = torch.randint(0, 128, (2, 150), generator=torch.Generator().manual_seed(1)).to(DEV)
    opt = torch.optim.SGD(model.parameters(), lr=0.5)
    losses = []
    for step in range(3):
        opt.zero_grad()
        loss = model(input_ids=ids, labels=ids).loss
        loss.backward()
        with torch.device(DEV):
            ref = _mpt_lm_ref(ids, p64, 2, 2)
        ref.backward()
        print(f"mpt lm step {step}: loss {loss.item():.5f} vs {ref.item():.5f}")
        losses.append(loss.item())
        assert abs(loss.item() - ref.item()) <= 1e-2 * abs(ref.item())
        for n, p in model.named_parameters():
            assert _rel(p.grad, p64[n].grad) <= REL_PARAM, (step, n, _rel(p.grad, p64[n].grad))
        opt.step()
        with torch.no_grad():
            for p in p64.values():
                p -= 0.5 * p.grad
                p.grad = None
    assert losses[-1] < losses[0]


def _otter_llama(monkeypatch, swap):
    from transformers import LlamaConfig
    from otter_b200 import otter_hf
    monkeypatch.setattr(otter_hf, "AutoTokenizer", FakeTokenizer)
    monkeypatch.setenv("OTB_LLAMA_LAYERS", "1" if swap else "0")
    td = LlamaConfig(vocab_size=68, hidden_size=512, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4,
                     num_key_value_heads=2, max_position_embeddings=512,
                     rope_parameters=dict(ROPES["llama3"])).to_dict()
    td["_name_or_path"], td["architectures"] = "llama-tiny", ["LlamaForCausalLM"]
    vc = dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=1, num_attention_heads=16, image_size=224,
              patch_size=14, hidden_act="quick_gelu")
    cfg = otter_hf.OtterConfig(vision_config=vc, text_config=td, cross_attn_every_n_layers=2)
    cfg.train_lang_encoder = True
    cfg.text_config._name_or_path = "llama-tiny"
    cfg.text_config.architectures = ["LlamaForCausalLM"]
    return otter_hf.OtterForConditionalGeneration(cfg)


@gpu
def test_otter_gqa_llama_train_lang_encoder(monkeypatch):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    torch.manual_seed(0)
    a = _otter_llama(monkeypatch, True)
    b = _otter_llama(monkeypatch, False)
    b.load_state_dict(a.state_dict(), strict=True)
    layers = [m for m in a.lang_encoder.modules() if isinstance(m, FrozenLlamaDecoderLayer)]
    assert len(layers) == 2 and all(p.requires_grad for l in layers for p in l.parameters())
    a.to(DEV), b.to(DEV)
    g = torch.Generator().manual_seed(3)
    vision_x = torch.randn(2, 1, 1, 3, 224, 224, generator=g).to(DEV)
    lang_x = torch.randint(3, 60, (2, 130), generator=g)
    lang_x[:, 0] = a.media_token_id
    lang_x = lang_x.to(DEV)
    opts = [torch.optim.SGD([p for p in m.parameters() if p.requires_grad], lr=0.2) for m in (a, b)]
    losses = []
    for step in range(3):
        out = []
        for m, opt in zip((a, b), opts):
            opt.zero_grad()
            loss = m(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x), labels=lang_x).loss
            loss.backward()
            out.append(loss.item())
        print(f"otter gqa llama step {step}: loss {out[0]:.5f} vs fp32 HF layers {out[1]:.5f}")
        assert abs(out[0] - out[1]) <= 2e-2 * abs(out[1])
        # every LM parameter.  The gated cross-attention layers' are left out: with their tanh gates at the initial 0,
        # the gate gradients are near-cancelling sums, and the gated block has parity tests of its own.
        gb = dict(b.lang_encoder.named_parameters())
        lm = [n for n, p in a.lang_encoder.named_parameters() if p.requires_grad and "gated_cross_attn" not in n]
        assert len(lm) == 2 * 9 + 3
        for n in lm:
            p = dict(a.lang_encoder.named_parameters())[n]
            assert p.grad is not None and _rel(p.grad, gb[n].grad) <= REL_PARAM, (step, n, _rel(p.grad, gb[n].grad))
        for opt in opts:
            opt.step()
        losses.append(out)
    assert losses[-1][0] < losses[0][0]


# ------------------------------------------------------------------------------------------------------------------
# GPU: a fresh process
# ------------------------------------------------------------------------------------------------------------------
FRESH = r"""
import torch
from otter_b200.lm_llama import FrozenLlamaDecoderLayer
layer = FrozenLlamaDecoderLayer(512, 4, 1024, num_key_value_heads=2).to("cuda")
layer.requires_grad_(True)
x = torch.randn(1, 64, 512, device="cuda", dtype=torch.bfloat16, requires_grad=True)
y = layer(x)
y.backward(torch.randn_like(y))              # bf16, contiguous: the first backward goes straight to the library
torch.cuda.synchronize()
assert torch.isfinite(x.grad.float()).all() and layer.self_attn.q_proj.weight.grad is not None
print("FRESH ok")
"""


@gpu
def test_first_backward_in_a_fresh_process():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", FRESH], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "FRESH ok" in r.stdout, r.stderr[-3000:]
