"""GPU: frozen LLaMA decoder layer (SURVEY.md §8f rank 1, config c3's LM) — the whole layer (forward + input gradient)
against the CPU oracle pinned to HF's LlamaDecoderLayer.  The RMSNorm / rotary / SwiGLU kernels are tested against
float64 in tests/test_rowwise_edges_gpu.py."""
import pytest
import torch

from oracle import restatement_llama as RL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16


def _rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-20)).item()


@pytest.mark.parametrize("B,S,D,H", [(2, 100, 256, 2), (1, 300, 512, 4)])
def test_frozen_llama_layer_vs_oracle(B, S, D, H):
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer
    torch.manual_seed(S)
    layer = FrozenLlamaDecoderLayer(D, H, 3 * D)
    with torch.no_grad():
        layer.input_layernorm.weight.add_(0.1 * torch.randn(D))
        layer.post_attention_layernorm.weight.add_(0.1 * torch.randn(D))
    p_ref = {k: v.detach().clone() for k, v in layer.state_dict().items()}
    layer.to(DEV)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, S, D, generator=g).to(BF16).float()
    w = torch.randn(B, S, D, generator=g).to(BF16).float()
    xg = x.to(DEV).requires_grad_(True)
    y = layer(xg, position_ids=torch.arange(S, device=DEV)[None])
    (y.float() * w.to(DEV)).sum().backward()
    xr = x.clone().requires_grad_(True)
    ref = RL.llama_layer(xr, p_ref, H)
    (ref * w).sum().backward()
    assert _rel(y, ref) <= 1.5e-2, _rel(y, ref)
    assert _rel(xg.grad, xr.grad) <= 3e-2, _rel(xg.grad, xr.grad)
    assert all(p.grad is None for p in layer.parameters())                                # frozen: activation grads only


def test_swap_llama_layers_in_an_hf_model():
    from transformers import LlamaConfig, LlamaForCausalLM
    from otter_b200.lm_llama import FrozenLlamaDecoderLayer, swap_llama_layers
    cfg = LlamaConfig(vocab_size=64, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                      num_key_value_heads=2, max_position_embeddings=128)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).to(DEV)
    ids = torch.randint(0, 64, (2, 40), device=DEV)
    mask = torch.ones_like(ids)
    mask[1, 30:] = 0                                                                      # right padding
    with torch.no_grad():
        ref = model(input_ids=ids, attention_mask=mask, use_cache=False).logits.float()
    keys = set(model.state_dict().keys())
    swap_llama_layers(model)
    assert set(model.state_dict().keys()) == keys                                         # checkpoint-compatible
    assert all(isinstance(l, FrozenLlamaDecoderLayer) for l in model.model.layers)
    with torch.no_grad():
        got = model(input_ids=ids, attention_mask=mask, use_cache=False).logits.float()
    valid = mask.bool()
    assert _rel(got[valid], ref[valid]) <= 2e-2, _rel(got[valid], ref[valid])
    # incremental decoding with a KV cache is handed to the HF layer the reference itself runs
    with torch.no_grad():
        out = model(input_ids=ids[:1], use_cache=True)
    assert out.past_key_values is not None and _rel(out.logits, ref[:1]) <= 2e-2
    left = mask.flip(1)
    with pytest.raises(NotImplementedError):
        model(input_ids=ids, attention_mask=left, use_cache=False)
