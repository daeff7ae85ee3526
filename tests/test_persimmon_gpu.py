"""GPU: Persimmon decoder layer (SURVEY.md §8f rank 3) — the qk-LayerNorm + partial-RoPE kernels against plain torch,
and the whole layer fwd + bwd (every parameter gradient) against the CPU oracle pinned to HF Persimmon.  The causal
mode of the head-64 attention kernels is tested in tests/test_attention_edges_gpu.py.
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


@pytest.mark.parametrize("rows_S,H,rot", [((2, 37), 4, 32), ((1, 300), 2, 16), ((3, 8), 64, 32)])
def test_qkln_rope_fwd_bwd_vs_torch(rows_S, H, rot):
    from otter_b200 import functional as F
    B, S = rows_S
    rows = B * S
    g = torch.Generator().manual_seed(rows + H)
    fused = (torch.randn(rows, H * 192, generator=g) * 1.5).to(BF16)
    par = [(1 + 0.2 * torch.randn(64, generator=g)), 0.2 * torch.randn(64, generator=g),
           (1 + 0.2 * torch.randn(64, generator=g)), 0.2 * torch.randn(64, generator=g)]
    qkv, stats = F.qkln_rope_fwd(fused.to(DEV), H, S, *[t.to(DEV) for t in par], rot, 25000.0, 1e-5)
    # torch reference on the bf16-rounded input
    x = fused.float().view(B, S, H, 3, 64).requires_grad_(True)
    pr = [t.clone().requires_grad_(True) for t in par]
    qs = RP.layer_norm(x[..., 0, :], pr[0], pr[1], 1e-5)
    ks = RP.layer_norm(x[..., 1, :], pr[2], pr[3], 1e-5)
    inv = 1.0 / (25000.0 ** (torch.arange(0, rot, 2, dtype=torch.float32) / rot))
    fr = torch.arange(S, dtype=torch.float32)[:, None] * inv[None]
    emb = torch.cat((fr, fr), -1)
    cos, sin = emb.cos()[None, :, None, :], emb.sin()[None, :, None, :]
    rope = lambda t: torch.cat((t[..., :rot] * cos + RP.rotate_half(t[..., :rot]) * sin, t[..., rot:]), -1)
    ref = torch.cat([rope(qs).reshape(rows, H * 64), rope(ks).reshape(rows, H * 64), x[..., 2, :].reshape(rows, H * 64)], 1)
    err = (qkv.float().cpu() - ref.detach()).abs()
    assert (err > 2e-2 + 1e-2 * ref.detach().abs()).sum().item() == 0, err.max().item()
    assert torch.equal(qkv[:, 2 * H * 64:].cpu(), fused.view(rows, H, 3, 64)[:, :, 2].reshape(rows, H * 64))   # v: copy
    dq = torch.randn(rows, 3 * H * 64, generator=g).to(BF16)
    ref.backward(dq.float())
    grads = [torch.empty(64, device=DEV) for _ in range(4)]
    dfused = F.qkln_rope_bwd(dq.to(DEV), fused.to(DEV), stats, H, S, par[0].to(DEV), par[2].to(DEV), rot, 25000.0, *grads)
    assert _rel(dfused, x.grad.reshape(rows, H * 192)) <= 1e-2
    for got, want in zip(grads, pr):
        assert _rel(got, want.grad) <= 1e-2, (_rel(got, want.grad))


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
