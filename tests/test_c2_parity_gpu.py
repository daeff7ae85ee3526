"""GPU: forward AND backward of the headline configuration (BASELINE.json configs[1]: D=4096, L=256, per-GPU batch 8)
against the CPU oracle, plus the GEMM kernel (`gemm_bf16_kernel`) called directly
through the C ABI at the shapes / layouts / epilogues it runs with in the timed step.

Tolerances are the production-mode (bf16 operands, fp32 accumulate) bounds of tests/test_modules_gpu.py, restated
at each assert: outputs rel-Frobenius <= 1.5e-2, activation gradients <= 3e-2 and parameter gradients <= 4e-2 (rel-Frobenius
of the whole tensor, which is stricter than the norm pins of the golden tests), the two scalar gate gradients 12 %.
Reference lines: modeling_otter.py:373-395 (block), :262-340 (masked cross-attention).
"""
import math

import pytest
import torch

from oracle import restatement as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BF16 = torch.bfloat16


def _rel(got, ref):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-20)).item()


def test_c2_gated_block_fwd_bwd_all_samples_vs_oracle():
    """All 8 samples of the c2 batch through one gated block, fwd + bwd: y, dx, dmedia and every parameter gradient
    (both tanh gates included) against oracle.restatement in fp32."""
    from otter_b200.modeling_otter import OtterGatedCrossAttentionBlock
    B, L, D, Dv, n = 8, 256, 4096, 1024, 64
    torch.manual_seed(11)
    gb = OtterGatedCrossAttentionBlock(dim=D, dim_visual=Dv)
    with torch.no_grad():
        gb.attn_gate.fill_(0.5), gb.ff_gate.fill_(-0.4)
        gb.attn.norm.weight.add_(0.1 * torch.randn(D)), gb.attn.norm.bias.add_(0.1 * torch.randn(D))
        gb.feed_forward[0].weight.add_(0.1 * torch.randn(D)), gb.feed_forward[0].bias.add_(0.1 * torch.randn(D))
    p_ref = {k: v.detach().clone().float().requires_grad_(True) for k, v in gb.state_dict().items()}
    gb.to(DEV)
    g = torch.Generator().manual_seed(5)
    # operands are bf16-representable so that both sides see identical inputs
    x = torch.randn(B, L, D, generator=g).to(BF16).float()
    media = torch.randn(B, 1, n, Dv, generator=g).to(BF16).float()
    wgt = torch.randn(B, L, D, generator=g).to(BF16).float()      # random linear functional as the loss
    loc = torch.zeros(B, L, dtype=torch.bool)
    loc[:, 0] = True
    loc[3, 0], loc[3, 7] = False, True                            # one sample with rows before the first <image>
    loc[5, 100] = True                                            # one sample with more <image> tokens than media

    xg = x.to(DEV).requires_grad_(True)
    mg = media.to(DEV).requires_grad_(True)
    y = gb(xg, mg, media_locations=loc.to(DEV))
    (y.float() * wgt.to(DEV)).sum().backward()

    xr, mr = x.clone().requires_grad_(True), media.clone().requires_grad_(True)
    yr = R.gated_cross_attention_block(xr, mr, loc, p_ref)
    (yr * wgt).sum().backward()

    assert _rel(y, yr) <= 1.5e-2, ("y", _rel(y, yr))
    for b in range(B):                                            # per sample, so one bad sample cannot hide
        assert _rel(y[b], yr[b]) <= 1.5e-2, ("y", b, _rel(y[b], yr[b]))
        assert _rel(xg.grad[b], xr.grad[b]) <= 3e-2, ("dx", b, _rel(xg.grad[b], xr.grad[b]))
        assert _rel(mg.grad[b], mr.grad[b]) <= 3e-2, ("dmedia", b, _rel(mg.grad[b], mr.grad[b]))
    named = dict(gb.named_parameters())
    for k, pr in p_ref.items():
        got = named[k].grad
        assert got is not None, k
        if k.endswith("_gate"):
            assert abs(got.item() - pr.grad.item()) <= 0.12 * abs(pr.grad.item()) + 1e-6, (k, got.item(), pr.grad.item())
        else:
            assert _rel(got, pr.grad) <= 4e-2, (k, _rel(got, pr.grad))      # same bound as the c3 test


# ---------------------------------------------------------------------------------------------------------------
# gemm_bf16_kernel at the step's own shapes (M = B*L = 2048 tokens, D = 4096, 4D = 16384), every FFN launch class
# ---------------------------------------------------------------------------------------------------------------
def _rn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(BF16).to(DEV)


def _close(got, ref, rtol, atol, what):
    err = (got.float() - ref.float()).abs()
    bad = (err > atol + rtol * ref.float().abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{err.numel()} outside tol, max err {err.max().item():.3e}"


def _gelu_grad(z):
    return 0.5 * (1 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)


@pytest.fixture(scope="module")
def ffn_operands():
    g = torch.Generator().manual_seed(21)
    M, D = 2048, 4096
    ops = dict(M=M, D=D,
               x=_rn(g, M, D), h=_rn(g, M, 4 * D), dy=_rn(g, M, D), dz=_rn(g, M, 4 * D),
               w1=_rn(g, 4 * D, D, scale=D ** -0.5), w2=_rn(g, D, 4 * D, scale=(4 * D) ** -0.5),
               gate=torch.tensor([0.7], device=DEV))
    return ops


def test_gemm2_forward_classes(ffn_operands):
    """K-major x K-major (layout 0,0): FFN up with GELU + pre-activation side output; FFN down with side output,
    tanh-gate and residual (modeling_otter.py:390-393)."""
    from otter_b200 import functional as F
    o = ffn_operands
    z = torch.empty(o["M"], 4 * o["D"], device=DEV, dtype=BF16)
    hh = F.linear_fwd(o["x"], o["w1"], act=1, aux_out=z)
    zr = o["x"].float() @ o["w1"].float().t()
    _close(z, zr, 1e-2, 2e-2, "up: pre-activation")
    _close(hh, torch.nn.functional.gelu(z.float()), 1e-2, 1e-2, "up: gelu(z)")       # GELU of the value it stored
    a2 = torch.empty(o["M"], o["D"], device=DEV, dtype=BF16)
    y = F.linear_fwd(o["h"], o["w2"], aux_out=a2, scale_ptr=o["gate"], scale_tanh=True, residual=o["x"])
    ar = o["h"].float() @ o["w2"].float().t()
    _close(a2, ar, 1e-2, 2e-2, "down: branch output")
    _close(y, ar * math.tanh(0.7) + o["x"].float(), 1e-2, 2e-2, "down: gate + residual")


def test_gemm2_dgrad_classes(ffn_operands):
    """K-major x MN-major (layout 0,1): dz = (dy W2) * gelu'(z) * tanh(g); dh0 = dz W1."""
    from otter_b200 import functional as F
    o = ffn_operands
    g = torch.Generator().manual_seed(22)
    z = _rn(g, o["M"], 4 * o["D"])
    dz = F.linear_dgrad(o["dy"], o["w2"], aux_in=z, scale_ptr=o["gate"], scale_tanh=True)
    ref = (o["dy"].float() @ o["w2"].float()) * _gelu_grad(z.float()) * math.tanh(0.7)
    _close(dz, ref, 1e-2, 2e-2, "dgrad down (dGELU, gate)")
    dh = F.linear_dgrad(o["dz"], o["w1"])
    _close(dh, o["dz"].float() @ o["w1"].float(), 1e-2, 4e-2, "dgrad up")


def test_gemm2_wgrad_classes(ffn_operands):
    """MN-major x MN-major (layout 1,1), fp32 output: dW2 = tanh(g) dy^T h (store, then accumulate); dW1 = dz^T x."""
    from otter_b200 import functional as F
    o = ffn_operands
    gw2 = torch.empty(o["D"], 4 * o["D"], device=DEV)
    F.linear_wgrad(o["dy"], o["h"], out=gw2, accumulate=False, scale_ptr=o["gate"], scale_tanh=True)
    ref2 = (o["dy"].float().t() @ o["h"].float()) * math.tanh(0.7)
    _close(gw2, ref2, 2e-3, 2e-2, "wgrad down (store)")
    F.linear_wgrad(o["dy"], o["h"], out=gw2, accumulate=True, scale_ptr=o["gate"], scale_tanh=True)
    _close(gw2, 2 * ref2, 2e-3, 4e-2, "wgrad down (accumulate)")
    gw1 = torch.full((4 * o["D"], o["D"]), 3.0, device=DEV)
    F.linear_wgrad(o["dz"], o["x"], out=gw1, accumulate=True)
    _close(gw1, o["dz"].float().t() @ o["x"].float() + 3.0, 2e-3, 2e-2, "wgrad up (accumulate onto 3.0)")


@pytest.mark.parametrize("rows,D", [(2048, 4096), (512, 1024)])
def test_gate_grad_and_layernorm_bwd_at_step_shapes(rows, D):
    """gate_grad / LayerNorm backward at the step's row counts (2048 x 4096 gated, 512 x 1024 perceiver)."""
    from otter_b200 import functional as F
    g = torch.Generator().manual_seed(rows)
    dy, a = _rn(g, rows, D), _rn(g, rows, D)
    gate = torch.tensor([0.5], device=DEV)
    dg = F.gate_grad(dy, a, gate)
    want = (1 - math.tanh(0.5) ** 2) * (dy.double() * a.double()).sum().item()
    scale = (dy.double() * a.double()).abs().sum().item()
    assert abs(dg.item() - want) <= 2e-6 * scale, (dg.item(), want)                  # fp32 two-stage reduction
    x = _rn(g, rows, D, scale=2.0)
    gam = (1 + 0.1 * torch.randn(D, generator=g)).to(DEV)
    bet = (0.1 * torch.randn(D, generator=g)).to(DEV)
    add = _rn(g, rows, D)
    y, mean, rstd = F.layernorm_fwd(x, gam, bet)
    dx, dgam, dbet = F.layernorm_bwd(dy, x, mean, rstd, gam, add=add)
    xr = x.float().requires_grad_(True)
    gr, br = gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
    torch.nn.functional.layer_norm(xr, (D,), gr, br, 1e-5).backward(dy.float())
    _close(dx, xr.grad + add.float(), 1e-2, 2e-2, "ln dx + add")
    assert _rel(dgam, gr.grad) <= 2e-3 and _rel(dbet, br.grad) <= 2e-3, (_rel(dgam, gr.grad), _rel(dbet, br.grad))


def test_direct_wire_format_sinks_match_fp32_sinks():
    """FlatGradBuffer(direct_params=...): the wgrad epilogues write bf16 straight into the all-reduce's wire buffer
    (the N > 1 default of bench.py).  Single rank: after all_reduce() the fp32 `.grad` views must equal the fp32-sink
    gradients up to one bf16 rounding (rel-Frobenius <= 4e-3), and a second write in the same step is refused."""
    from otter_b200.dp import FlatGradBuffer
    from otter_b200.modeling_otter import OtterGatedCrossAttentionBlock
    B, L, D, Dv, n = 2, 128, 1024, 256, 64
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B, L, D, generator=g).to(BF16).to(DEV)
    media = torch.randn(B, 1, n, Dv, generator=g).to(BF16).to(DEV)
    w = torch.randn(B, L, D, generator=g).to(BF16).to(DEV)
    loc = torch.zeros(B, L, dtype=torch.bool, device=DEV)
    loc[:, 0] = True
    grads = {}
    for mode in ("fp32", "direct"):
        torch.manual_seed(4)
        gb = OtterGatedCrossAttentionBlock(dim=D, dim_visual=Dv).to(DEV)
        with torch.no_grad():
            gb.attn_gate.fill_(0.5), gb.ff_gate.fill_(0.5)
        params = list(gb.parameters())
        direct = [m.weight for m in gb.modules() if isinstance(m, torch.nn.Linear)] if mode == "direct" else None
        flat = FlatGradBuffer(params, device=DEV, comm_dtype=torch.bfloat16 if direct else None, direct_params=direct)
        for _ in range(2):                                  # second step: the sinks are reused
            flat.begin_step()
            y = gb(x.clone().requires_grad_(True), media, media_locations=loc)
            (y.float() * w).sum().backward()
            flat.finish_step()
            flat.all_reduce()
        torch.cuda.synchronize()
        grads[mode] = {k: p.grad.detach().float().clone() for k, p in gb.named_parameters()}
        if direct:
            assert all(p._otb_grad.dtype == BF16 for p in direct)
    for k, ref in grads["fp32"].items():
        got = grads["direct"][k]
        tol = 4e-3 if ref.dim() == 2 else 1e-6
        assert _rel(got, ref) <= tol, (k, _rel(got, ref))
