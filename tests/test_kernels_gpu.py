"""GPU parity tests of the individual kernels, called through the C ABI (ctypes).

Reference for each op = the same op in plain torch fp32 on the bf16-rounded inputs (a floating-point
kernel: tolerance written at each assert; integer/index outputs are compared bit-exact against the
numpy oracle).
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev()).to(torch.bfloat16)


def assert_close(got, ref, rtol, atol, what=""):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} outside tol, max err {err.max().item():.4e}, max ref {ref.abs().max().item():.3f}"


def test_text_time_bit_exact():
    from oracle.restatement import text_time_np
    from otter_b200 import functional as F
    rng = np.random.RandomState(0)
    for L in (1, 7, 32, 257, 2048):
        loc = rng.rand(5, L) < 0.1
        loc[0, :] = False
        if L > 3:
            loc[1, 0] = True
        for ap in (True, False):
            got = F.text_time(torch.from_numpy(loc).to(dev()), ap).cpu().numpy()
            ref = text_time_np(loc, ap)
            assert got.dtype == np.int32 and np.array_equal(got.astype(np.int64), ref), (L, ap)


def test_small_passes():
    from otter_b200 import functional as F
    src = torch.randn(64, 1024, device=dev())
    out = F.bcast_rows(src, 64 * 5, 1, 64)
    assert torch.equal(out.view(5, 64, 1024), src.to(torch.bfloat16).expand(5, 64, 1024))
    x = rnd(5 * 64, 1024)
    cs = F.grouped_colsum(x, 1, 64)
    assert_close(cs, x.float().view(5, 64, 1024).sum(0), 1e-5, 1e-4, "grouped colsum latents")
    xf = rnd(2 * 3 * 16, 128)  # (img=6 -> F=3) x v=16
    cs = F.grouped_colsum(xf, 16, 3)
    assert_close(cs, xf.float().view(2, 3, 16, 128).sum((0, 2)), 1e-5, 1e-4, "grouped colsum frames")
    a, dy = rnd(1000, 512, seed=1), rnd(1000, 512, seed=2)
    gate = torch.tensor([0.3], device=dev())
    dg = F.gate_grad(dy, a, gate)
    ref = (1 - math.tanh(0.3) ** 2) * (dy.float() * a.float()).sum()
    assert abs(dg.item() - ref.item()) <= 1e-3 * abs(ref.item()) + 1e-2
    loss, dx = F.sqmean_loss(a)
    assert abs(loss.item() - a.float().pow(2).mean().item()) < 1e-4
    assert_close(dx, 2 * a.float() / a.numel(), 1e-2, 1e-9, "sqmean grad")
    w = torch.randn(1000, 333, device=dev())
    assert torch.equal(F.cast_bf16(w), w.to(torch.bfloat16))
    assert torch.equal(F.cast_f32(a), a.float())
    # CLIP embedding pieces
    px = torch.randn(2, 3, 56, 56, device=dev())
    cols = F.im2col_patches(px, 14, 592)
    ref = torch.nn.functional.unfold(px, 14, stride=14).transpose(1, 2).reshape(-1, 588)
    assert torch.equal(cols[:, :588], ref.to(torch.bfloat16)) and cols[:, 588:].abs().max().item() == 0
    pe = rnd(2 * 16, 256)
    cls, pos = torch.randn(256, device=dev()), torch.randn(17, 256, device=dev())
    h = F.clip_assemble(pe, cls, pos, 2, 16)
    ref = torch.cat([cls.expand(2, 1, 256), pe.float().view(2, 16, 256)], 1) + pos[None]
    assert_close(h, ref, 1e-2, 1e-2, "clip assemble")
    fe = torch.randn(4, 256, device=dev())
    hid = rnd(6, 17, 256)
    m = F.media_from_clip(hid, fe, 3)
    ref = hid.float()[:, 1:] + fe[:3].repeat(2, 1)[:, None, :]
    assert_close(m.view(6, 16, 256), ref, 1e-2, 1e-2, "media_from_clip")
    # fuyu scatter
    from oracle.restatement import fuyu_gather_continuous_embeddings
    word = rnd(2, 10, 64)
    cont = [rnd(3, 64, seed=1), rnd(4, 64, seed=2)]
    idx = torch.full((2, 10), -1, dtype=torch.int64)
    idx[0, 2:5] = torch.arange(3)
    idx[1, 1:5] = torch.tensor([3, 2, 1, 0])
    ref = fuyu_gather_continuous_embeddings(word.cpu().float(), [c.cpu().float() for c in cont], idx)
    got = F.fuyu_scatter(word, torch.cat(cont), idx.to(dev()), torch.tensor([0, 3, 7], device=dev()))
    assert torch.equal(got.cpu().float(), ref)
    idx[1, 9] = 4                                   # id == n_1: out of range -> never read out of bounds, word row kept
    got = F.fuyu_scatter(word, torch.cat(cont), idx.to(dev()), torch.tensor([0, 3, 7], device=dev()))
    assert torch.equal(got[1, 9], word[1, 9])


def test_label_mask_bit_exact():
    """SURVEY.md §8f row 2: device label masking == the reference's masking() (golden, bit-exact).  The fused shifted
    cross-entropy is tested in tests/test_rowwise_edges_gpu.py."""
    import os
    from otter_b200 import losses
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "label_mask.pt"), weights_only=False)
    for name, c in g["cases"].items():
        got = losses.label_mask(c["input_ids"].to(dev()), g["eos"], g["answer"], g["eoc"])
        assert got.dtype == torch.int64 and torch.equal(got.cpu(), c["labels"]), name


def test_multi_tensor_cast_matches_per_tensor_cast():
    """params.refresh(): one launch for a list of fp32 weights == torch round-to-nearest-even bf16, bit for bit."""
    from otter_b200 import params as P
    torch.manual_seed(5)
    shapes = [(1,), (7,), (4096,), (4097,), (33, 129), (1024, 1024), (3, 5, 7), (2048, 4096)]
    ps = [torch.nn.Parameter(torch.randn(*s, device=dev()) * 3) for s in shapes]
    P.refresh(ps)
    for p in ps:
        got = P.bf16_of(p)
        assert got.shape == p.shape
        assert torch.equal(got, p.detach().to(torch.bfloat16)), p.shape
    with torch.no_grad():
        for p in ps:
            p.mul_(1.5)                                  # version bump: shadows stale
    P.refresh(ps)                                        # second call reuses the pointer table and the shadow buffers
    for p in ps:
        assert torch.equal(P.bf16_of(p), p.detach().to(torch.bfloat16)), p.shape


def test_upcast_with_folded_scale():
    """otb_cast_bf16_f32_scale: the up-cast after the bf16 all-reduce(SUM) with 1/world_size folded in (dp.py)."""
    from otter_b200 import functional as F
    g = torch.Generator().manual_seed(5)
    for n in (8, 4099, 1 << 20):
        src = torch.randn(n, generator=g).to(torch.bfloat16)
        out = torch.full((n,), 7.0, device=dev())
        F.cast_f32_scaled(src.to(dev()), out, 1.0 / 3.0)
        assert torch.equal(out.cpu(), src.float() * torch.tensor(1.0 / 3.0, dtype=torch.float32))
