"""GPU parity of §8f rank 1: the frozen MPT block built on the causal / ALiBi head-dim-128 attention, against the
reference-pinned oracle (oracle/restatement_lm.py).  The attention kernels themselves (otb_lm_attn_fwd / _bwd) are
tested against a float64 reference in tests/test_attention_edges_gpu.py.
Tolerances are bf16-storage tolerances (inputs, P and outputs are rounded to bf16 in the kernels)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda", 0)


def test_frozen_mpt_block_matches_oracle():
    from oracle import restatement_lm as R
    from otter_b200.lm_mpt import FrozenMPTBlock
    torch.manual_seed(0)
    B, S, D, H = 2, 150, 256, 2
    blk = FrozenMPTBlock(D, H).to(dev())
    with torch.no_grad():
        for prm in blk.parameters():
            prm.copy_(torch.randn_like(prm) * (0.3 if prm.ndim == 1 else prm.shape[-1] ** -0.5))
            if prm.ndim == 1:
                prm.add_(1.0)
    x = torch.randn(B, S, D, device=dev()).to(torch.bfloat16).requires_grad_(True)
    y, _, _ = blk(x)
    gy = torch.randn(B, S, D, device=dev()).to(torch.bfloat16)
    (gx,) = torch.autograd.grad(y, x, gy)
    params = {k: v.detach().float().cpu() for k, v in blk.state_dict().items()}
    xr = x.detach().float().cpu().requires_grad_(True)
    yr = R.mpt_block(xr, params, H)
    (gxr,) = torch.autograd.grad(yr, xr, gy.float().cpu())
    rel_y = (y.float().cpu() - yr).abs().max().item() / yr.abs().max().item()
    rel_g = (gx.float().cpu() - gxr).abs().max().item() / gxr.abs().max().item()
    assert rel_y < 3e-2, rel_y
    assert rel_g < 5e-2, rel_g
    assert all(p.grad is None for p in blk.parameters())          # frozen: no weight gradients are produced


def test_golden_key_names_match_reference_block():
    from otter_b200.lm_mpt import FrozenMPTBlock
    gold = torch.load(os.path.join(os.path.dirname(__file__), "golden", "mpt_block_tiny.pt"))
    assert set(FrozenMPTBlock(256, 2).state_dict().keys()) == set(gold["a"]["params"].keys())
