"""GPU: Persimmon decoder layer (SURVEY.md §8f rank 3) — the whole layer fwd + bwd (every parameter gradient) against
the CPU oracle pinned to HF Persimmon.  The causal mode of the head-64 attention kernels is tested in
tests/test_attention_edges_gpu.py, the qk-LayerNorm + partial-RoPE kernels in tests/test_rowwise_edges_gpu.py.
Production numerics (bf16 operands): tolerances of tests/test_modules_gpu.py."""
import pytest
import torch

from oracle import restatement_persimmon as RP

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16


def _rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-20)).item()


@pytest.mark.parametrize("B,S,D,H", [(2, 100, 256, 4), (1, 300, 512, 8)])
def test_persimmon_layer_fwd_bwd_vs_oracle(B, S, D, H):
    from otter_b200.lm_persimmon import PersimmonDecoderLayer
    torch.manual_seed(S)
    layer = PersimmonDecoderLayer(hidden_size=D, num_attention_heads=H, intermediate_size=4 * D)
    with torch.no_grad():
        for n, p in layer.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    p_ref = {k: v.detach().clone().requires_grad_(True) for k, v in layer.state_dict().items()}
    layer.to(DEV)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, S, D, generator=g).to(BF16).float()
    w = torch.randn(B, S, D, generator=g).to(BF16).float()
    xg = x.to(DEV).requires_grad_(True)
    (y,) = layer(xg, position_ids=torch.arange(S, device=DEV)[None])
    (y.float() * w.to(DEV)).sum().backward()
    xr = x.clone().requires_grad_(True)
    ref = RP.persimmon_layer(xr, p_ref, H, rotary_ndims=32)
    (ref * w).sum().backward()
    assert _rel(y, ref) <= 1.5e-2, _rel(y, ref)
    assert _rel(xg.grad, xr.grad) <= 3e-2, _rel(xg.grad, xr.grad)
    named = dict(layer.named_parameters())
    for k, pr in p_ref.items():
        assert named[k].grad is not None, k
        assert _rel(named[k].grad, pr.grad) <= 4e-2, (k, _rel(named[k].grad, pr.grad))
    # frozen input: parameter gradients must still arrive (autograd tracks the parameters, not only x)
    layer.zero_grad()
    (y2,) = layer(x.to(DEV))
    (y2.float() * w.to(DEV)).sum().backward()
    assert _rel(named["mlp.dense_h_to_4h.weight"].grad, p_ref["mlp.dense_h_to_4h.weight"].grad) <= 4e-2
    with pytest.raises(NotImplementedError):
        layer(x.to(DEV), position_ids=torch.arange(1, S + 1, device=DEV)[None])
