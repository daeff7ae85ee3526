"""GPU: BASELINE.json full-size shapes, checked through size-independent properties and (where the CPU oracle
finishes in seconds) directly against oracle/restatement.py.  c2: D=4096, L=256, batch 8; c3: video F=8
(2048+64 keys = 17 key tiles of the attention kernels); c5: Fuyu patch-linear 1225 x 2700 -> 4096 + scatter."""
import pytest
import torch

from oracle import restatement as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _gated(D=4096, Dv=1024, gate=0.5, seed=0):
    from otter_b200.modeling_otter import OtterGatedCrossAttentionBlock
    torch.manual_seed(seed)
    gb = OtterGatedCrossAttentionBlock(dim=D, dim_visual=Dv).to(DEV)
    with torch.no_grad():
        gb.attn_gate.fill_(gate), gb.ff_gate.fill_(gate)
    return gb


@torch.no_grad()
def test_c2_gated_block_properties():
    B, L, D = 8, 256, 4096
    g = torch.Generator(device="cpu").manual_seed(0)
    x = torch.randn(B, L, D, generator=g).to(DEV).to(torch.bfloat16)
    media = torch.randn(B, 1, 64, 1024, generator=g).to(DEV).to(torch.bfloat16)
    loc = torch.zeros(B, L, dtype=torch.bool, device=DEV)
    loc[:, 3] = True                              # tokens 0..2 precede the first <image>
    # (1) gates at 0 -> exact identity (tanh(0) = 0), reference :362,371
    assert torch.equal(_gated(gate=0.0)(x, media, media_locations=loc), x)
    gb = _gated(gate=0.5)
    y = gb(x, media, media_locations=loc)
    assert torch.isfinite(y.float()).all()
    # (2) batch-sharding invariance (what data parallelism relies on): halves == whole, bit for bit
    y0 = gb(x[:4].contiguous(), media[:4].contiguous(), media_locations=loc[:4].contiguous())
    y1 = gb(x[4:].contiguous(), media[4:].contiguous(), media_locations=loc[4:].contiguous())
    assert torch.equal(torch.cat([y0, y1]), y)
    # (3) rows before the first <image> get no attention contribution: masked x-attn output rows are exactly 0
    a = gb.attn(x, media, media_locations=loc)
    assert a[:, :3].abs().max().item() == 0.0 and a[:, 3:].abs().max().item() > 0
    # (4) sample 0 against the CPU oracle (fp32), bf16 tolerance of tests/test_modules_gpu.py
    p = {k: v.detach().float().cpu() for k, v in gb.state_dict().items()}
    ref = R.gated_cross_attention_block(x[:1].float().cpu(), media[:1].float().cpu(), loc[:1].cpu(), p)
    rel = (y[:1].float().cpu() - ref).norm() / ref.norm()
    assert rel < 1.5e-2, rel


def test_c3_video_perceiver_streaming_attention():
    """F=8 frames -> 2048 media keys + 64 latents = 17 key tiles streamed through the double-buffered TMA ring: the
    two-sweep forward and the dQ workspace of the backward, fwd + bwd."""
    from otter_b200.modeling_otter import OtterPerceiverResampler
    torch.manual_seed(1)
    rs = OtterPerceiverResampler(dim=1024, depth=2, max_num_frames=16).to(DEV)
    x = torch.randn(1, 1, 8, 256, 1024, device=DEV)
    out = rs(x)
    # mean(LN(x)^2) is constant for a default-initialised final LayerNorm (zero gradient): use a random linear
    # functional of the output as the loss instead
    wgt = torch.randn(out.shape, device=DEV)
    (out.float() * wgt).mean().backward()
    p = {k: v.detach().float().cpu().requires_grad_(True) for k, v in rs.state_dict().items()}
    ref = R.perceiver_resampler(x.cpu(), p)
    (ref * wgt.cpu()).mean().backward()
    rel = (out.detach().float().cpu() - ref.detach()).norm() / ref.detach().norm()
    assert rel < 1.5e-2, rel
    for k in ("latents", "frame_embs", "layers.0.to_kv.weight", "layers.1.norm_media.weight", "layers.0.feed_forward.1.weight"):
        got, want = dict(rs.named_parameters())[k].grad.float().cpu(), p[k].grad
        assert (got - want).norm() <= 4e-2 * want.norm() + 1e-7, (k, (got - want).norm().item(), want.norm().item())
    assert rs.frame_embs.grad[8:].abs().max().item() == 0.0        # unused frame slots get zero gradient


@torch.no_grad()
def test_c5_fuyu_patch_linear_and_scatter():
    """OtterHD/Fuyu path (fuyu/modeling_fuyu.py:126-131): Linear(2700 -> 4096, bias) on 1225 patches of a
    1024x1024 image (35x35 patches of 30x30x3), scattered into the word embeddings."""
    from otter_b200 import functional as F
    g = torch.Generator().manual_seed(0)
    n_p, K, D, S = 1225, 2700, 4096, 1300
    patches = torch.randn(n_p, K, generator=g).to(torch.bfloat16)
    w = (torch.randn(D, K, generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(D, generator=g) * 0.1
    word = torch.randn(1, S, D, generator=g).to(torch.bfloat16)
    idx = torch.full((1, S), -1, dtype=torch.int64)
    idx[0, 5:5 + n_p] = torch.arange(n_p)
    Kp = (K + 7) // 8 * 8                                             # 2704: row pitch multiple of 8 elements
    pp = torch.zeros(n_p, Kp, dtype=torch.bfloat16); pp[:, :K] = patches
    wp = torch.zeros(D, Kp, dtype=torch.bfloat16); wp[:, :K] = w
    emb = F.linear_fwd(pp.to(DEV), wp.to(DEV), bias=bias.to(DEV))
    out = F.fuyu_scatter(word.to(DEV), emb, idx.to(DEV), torch.tensor([0, n_p], dtype=torch.int64, device=DEV))
    ref = R.fuyu_patch_embed([patches.float()], w.float(), bias, word.float(), idx, q=R.bf16_round)
    err = (out.float().cpu() - ref).abs()
    assert err.max().item() <= 2e-2 + 1e-2 * ref.abs().max().item()
    assert torch.equal(out[0, :5].cpu(), word[0, :5]) and torch.equal(out[0, 5 + n_p:].cpu(), word[0, 5 + n_p:])


# ---------------------------------------------------------------------------------------------------------------
# ragged / degenerate shapes against the CPU oracle (production bf16 mode and the fp32-grade forward mode)
# ---------------------------------------------------------------------------------------------------------------
def _rel(a, b):
    return ((a.detach().float().cpu() - b).norm() / b.norm().clamp_min(1e-12)).item()


@torch.no_grad()
@pytest.mark.parametrize("B,L,T,n,locs,attend_previous", [
    (1, 1, 1, 64, [[]], True),                         # cached decode step: one token, no <image> (reference quirk §3.3)
    (3, 77, 3, 32, [[0, 30, 60], [5], []], True),      # ragged <image> counts per row, 32 latents per media, odd L
    (2, 130, 2, 64, [[0, 1], [128, 129]], False),      # adjacent <image> tokens, tile-boundary positions, attend_previous=False
    (1, 9, 5, 8, [[0, 2, 4, 6, 8]], True),             # 5 media x 8 latents = 40 keys (partial key tile)
])
def test_gated_block_ragged_shapes_vs_oracle(B, L, T, n, locs, attend_previous):
    import otter_b200
    from otter_b200.modeling_otter import OtterGatedCrossAttentionBlock
    torch.manual_seed(3)
    D, Dv = 256, 128
    gb = OtterGatedCrossAttentionBlock(dim=D, dim_visual=Dv).to(DEV)
    gb.attn_gate.fill_(0.8), gb.ff_gate.fill_(-0.6)
    x = torch.randn(B, L, D, device=DEV)
    media = torch.randn(B, T, n, Dv, device=DEV)
    loc = torch.zeros(B, L, dtype=torch.bool)
    for b, ps in enumerate(locs):
        loc[b, ps] = True
    p = {k: v.detach().float().cpu() for k, v in gb.state_dict().items()}
    ref = R.gated_cross_attention_block(x.cpu(), media.cpu(), loc, p, attend_previous=attend_previous)
    out = gb(x, media, media_locations=loc.to(DEV), attend_previous=attend_previous)
    assert _rel(out, ref) < 1.5e-2
    with otter_b200.precision("fp32"):
        out32 = gb(x, media, media_locations=loc.to(DEV), attend_previous=attend_previous)
    err = (out32.float().cpu() - ref).abs()
    assert (err > 1e-5 + 1e-3 * ref.abs()).sum().item() == 0, err.max().item()


@pytest.mark.parametrize("b,T,Fr,v,n_lat", [(1, 1, 1, 1, 64), (2, 3, 2, 50, 32), (1, 1, 1, 257, 128)])
def test_resampler_odd_shapes_vs_oracle(b, T, Fr, v, n_lat):
    """1 media token, non-multiple-of-64 token counts, 32 / 128 latents, T > 1 with frame embeddings."""
    import otter_b200
    from otter_b200.modeling_otter import OtterPerceiverResampler
    torch.manual_seed(4)
    rs = OtterPerceiverResampler(dim=128, depth=2, num_latents=n_lat, max_num_frames=4).to(DEV)
    x = torch.randn(b, T, Fr, v, 128, device=DEV)
    wgt = torch.randn(b, T, n_lat, 128, device=DEV)
    out = rs(x)
    (out.float() * wgt).mean().backward()
    p = {k: v_.detach().float().cpu().requires_grad_(True) for k, v_ in rs.state_dict().items()}
    ref = R.perceiver_resampler(x.cpu(), p)
    (ref * wgt.cpu()).mean().backward()
    assert _rel(out, ref.detach()) < 1.5e-2
    for k in ("latents", "frame_embs", "layers.1.to_q.weight", "layers.0.norm_media.bias"):
        got, want = dict(rs.named_parameters())[k].grad.float().cpu(), p[k].grad
        assert (got - want).norm() <= 5e-2 * want.norm() + 1e-7, (k, (got - want).norm().item(), want.norm().item())
    with torch.no_grad(), otter_b200.precision("fp32"):
        out32 = rs(x)
    err = (out32.float().cpu() - ref.detach()).abs()
    assert (err > 1e-5 + 1e-3 * ref.detach().abs()).sum().item() == 0, err.max().item()


@torch.no_grad()
def test_c5_fuyu_module_entry_reference_signature_and_errors():
    """otter_b200.modeling_fuyu with the reference's argument names, shapes (K = 2700, no caller-side padding) and
    errors (modeling_fuyu.py:61-62,73-76), two samples with different patch counts, against the oracle."""
    from otter_b200 import modeling_fuyu as MF
    g = torch.Generator().manual_seed(2)
    K, D, S = 2700, 4096, 700
    lin = torch.nn.Linear(K, D).to(DEV)
    emb_tok = torch.nn.Embedding(100, D).to(DEV).to(torch.bfloat16)
    counts = [300, 525]
    patches = [torch.randn(1, n, K, generator=g).to(torch.bfloat16).to(DEV) for n in counts]
    ids = torch.randint(0, 100, (2, S), generator=g).to(DEV)
    idx = torch.full((2, S), -1, dtype=torch.int64)
    idx[0, 10:10 + 300] = torch.arange(300)
    idx[1, 3:3 + 525] = torch.arange(525)
    out = MF.embed_inputs(emb_tok, lin, ids, image_patches=patches, image_patches_indices=idx.to(DEV))
    w = lin.weight.detach().to(torch.bfloat16).float().cpu()
    ref = R.fuyu_patch_embed([p_[0].float().cpu() for p_ in patches], w, lin.bias.detach().float().cpu(),
                             emb_tok(ids).float().cpu(), idx, q=R.bf16_round)
    err = (out.float().cpu() - ref).abs()
    assert err.max().item() <= 2e-2 + 1e-2 * ref.abs().max().item()
    # cached decode step: patches ignored (modeling_fuyu.py:124)
    o2 = MF.embed_inputs(emb_tok, lin, ids, image_patches=patches, image_patches_indices=idx.to(DEV), past_key_values=((),))
    assert torch.equal(o2, emb_tok(ids))
    word = emb_tok(ids)
    with pytest.raises(ValueError, match="Batch sizes must match"):
        MF.gather_continuous_embeddings(word, [torch.zeros(3, D, device=DEV)], idx.to(DEV))
    with pytest.raises(ValueError, match="does not match number of continuous token ids"):
        MF.gather_continuous_embeddings(word, [torch.zeros(299, D, device=DEV, dtype=torch.bfloat16),
                                               torch.zeros(525, D, device=DEV, dtype=torch.bfloat16)], idx.to(DEV))
