"""Row-wise kernels against a float64 reference at the edges of their launch and vector structure.

Kernels under test (bf16 activations, fp32 parameters, statistics and parameter gradients):
  otb_layernorm_fwd           one warp per row, lane-strided 16 B vectors
  otb_layernorm_bwd           five routes: ln_bwd_fused_kernel<1> (D <= 2048) and <2> (D <= 4096) with dx and the gamma /
                              beta partials; the same kernel with dx == nullptr; ln_bwd_dx_kernel alone (no parameter
                              gradients); for D > 4096 ln_bwd_dx_kernel + ln_bwd_param_kernel + ln_bwd_finalize_kernel.
                              The one-pass kernel walks 4-row batches with stride gridDim.x = min(batches, SMs), so row
                              counts around 4 * SMs decide how many batches (and which smem parity) a CTA sees.
  otb_rmsnorm_fwd / _bwd      one warp per row
  otb_rope128                 in place, grid-stride over (row, block, head, pair), grid capped at 8 * SMs blocks
  otb_swiglu_fwd / _bwd       grid-stride over 16 B vectors, same cap
  otb_qkln_rope_fwd / _bwd    one warp per (row, head), grid capped at min(592, 4 * SMs) blocks of 8 warps; partial
                              rotary through a lane shuffle at distance rot / 4; fixed-order two-stage parameter sums
  otb_shifted_cross_entropy   one CTA per row; the row in shared memory (fp32 V <= 51200, bf16 V <= 102400, the bf16
                              exponentials kept there in bf16) or re-read from global memory; 16 B vectors where the row
                              start is 16 B aligned, scalar loads otherwise
  otb_gate_grad, otb_sqmean_loss, otb_grouped_colsum   the small fp32 reductions used next to them

Reference: float64 on the device from the same bf16-rounded inputs (fp32 parameters as given), gradients by autograd in
float64.  A backward kernel is handed the reference's forward statistics rounded to fp32, so it is measured on its own;
the forward statistics are checked separately.  The tests without the `gpu` mark show on the CPU that the metric
rejects float64 references mutated the way a kernel bug would mutate them.

Every GPU case of the row-wise kernels goes through the C ABI with NaN-filled, padded, offset output buffers and
NaN-padded inputs (`_Canvas`): every element a kernel owns must be finite and within the bound, every other element must
keep its NaN bits, and a read outside an input's rows or columns shows up as NaN in an output.  gate_grad, sqmean_loss,
grouped_colsum and the cross-entropy autograd function are called through their Python entry points.
"""
import ctypes as C
import math
import re

import numpy as np
import pytest
import torch

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
gpu = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------------------------
# The metric.
#
# bf16 outputs, per slice s (one row for LayerNorm, RMSNorm, SwiGLU and cross-entropy; one head of one row for RoPE
# and qk-LayerNorm):      |got - ref| <= A_REL * |ref| + B * rms(ref_s) + FLOOR  (+ a CE term, below)
#
# Where the kernels round and the reference does not.  bf16 keeps 8 significant bits: rounding to nearest has a
# relative error below u = 2^-8.
#   - Every output element is rounded to bf16 once: < 2^-8 |ref|.  A_REL = 2^-7, so output rounding alone uses at
#     most 0.5 of the bound (derived, not measured).
#   - Everything before that rounding is fp32 (u32 = 2^-24) and is charged to B:
#     * LayerNorm / RMSNorm forward: the row statistics are lane-strided sums of D/32 terms plus a 5-level shuffle
#       tree, so mean and variance carry < (D/32 + 5) u32 <= 2^-16.4 of sum|terms| (D = 6144).  x - mean then errs by
#       < 2^-16.4 mean|x| * rstd, which is 2^-11.4 of the row's scale for the largest common offset tested
#       (mean / std = 32).  B_NORM = 2^-10.
#     * LayerNorm / RMSNorm backward: dx = rstd (g - mean(g) - xhat mean(g xhat)) [+ add].  The fp32 error is a few
#       u32 of rstd (|g| + |mean g| + |xhat mean(g xhat)|); with random dy these terms are of the size of rms(dx), so
#       B_NORM = 2^-10 leaves > 2^10 before cancellation in the bracket could matter.  The statistics handed to the
#       kernel are the reference's rounded to fp32: 2^-24 relative, plus 2^-24 |mean| rstd <= 2^-19 in xhat.
#     * RoPE (rope128 and qk-LayerNorm): the kernel's angle is pos * inv_freq in fp32 with inv_freq = exp2f(-log2(theta)
#       * 2i / rot).  The exponent e carries ~2 u32 of |e|, exp2f ~2 u32, the product u32 and sincosf ~1 u32, so the
#       angle errs by < pos (0.37 * 2^-23 + 2^-22 + 2^-24) < pos * 2^-21.2 (the first term peaks at 2^e |e| = 0.53).
#       At pos = 4095 that is 2^-9.2 rad.  The error of a rotated pair is angle error * |pair|, and the largest pair
#       of a 128-value head is ~2.9 rms: < 2^-7.7 rms.  B_ROPE = 2^-7.  The LayerNorm of the qk kernels adds
#       B_NORM-sized terms.
#     * SwiGLU: sigmoid uses __expf, whose error is (2 + 1.17 |x|) ulp: < 2^-16 relative for |g| <= 100 (the largest
#       tested).  dg = dh u (s + g s (1 - s)) cancels near g = -1.28; the fp32 error there is ~2^-16 of dh u s, of the
#       size of rms(dg).  B_SWIGLU = 2^-10.
#   - FLOOR = 2^-60: SwiGLU at g <= -88, where the exact output is ~1e-37 and __expf overflows to give 0.
#
# Cross-entropy dlogits, per row: d_c = (p_c - [c = t]) / count.  Besides the output rounding, p carries a relative
# error that the subtraction of 1 at the target does not shrink, so the bound adds A_P * p / count:
#   - fp32 logits, row in shared memory: p = __expf(x - M) / S.  x - M is exact or rounded relative to itself;
#     __expf errs by (2 + 1.17 |x - M|) ulp, < 2^-16.3 down to the underflow at x - M = -87; S and 1/S a few u32.
#     A_P = 2^-15.  Output rounding (fp32): A_OUT = 2^-20.
#   - bf16 logits, row in shared memory: the exponentials are stored back into the row as bf16, so p carries another
#     2^-8: A_P = 2^-7.  The output is bf16: A_OUT = A_REL.
#   - row re-read from global memory: p = __expf(x - lse) with lse = M + log S in fp32, which is off by up to
#     2^-24 |lse| + the error of S: A_P += 2^-22 |lse|.
#   No error scales with the row's rms; B_CE = 0 and FLOOR = 2^-60 (p below 1e-38 is a denormal for __expf).
#
# fp32 outputs that are sums over many rows (dgamma, dbeta, the qk parameter gradients, mean / rstd, the CE loss,
# gate_grad, sqmean_loss, grouped_colsum):   |got - ref| <= C_SUM * sum|terms| + FLOOR
# Such sums can nearly cancel, so the bound scales with the sum of the absolute terms, not with |ref|.  The deepest
# sequential fp32 chain here is < 200 additions (the one-pass LN backward: rows / grid per thread, then grid / 8 + 8
# in the finalize; the D > 4096 route: rows / chunks / 8 + 8 + chunks), each adding < u32 of the running sum, plus
# ~4 u32 per term from products and the rounded statistics: < 2^-16.3.  C_SUM = 2^-16.  A dgamma term is
# |dy| (|xhat| + |mean| rstd): the mean handed to the kernel is rounded to fp32, which moves xhat by 2^-24 |mean| rstd
# however small xhat is (left out at first; a 3-row case with a mean / std = 32 row then used 0.60 of the bound, the
# exact answer rounded to fp32 0.004).  For `accumulate`, |old|
# is one more term; for rstd the "sum" is rstd itself (half the variance's relative error plus 2 ulp of rsqrtf); for
# the CE loss it is sum over counted rows of (|lse| + |x_t| + 1) / count.
#
# The constants above were fixed before the first GPU run.  Every RATIO line also prints the same ratio for the exact
# answer rounded to the output type, the part no kernel of that output type can avoid.  Measured on an H100 80GB HBM3
# (700 W limit): bf16 outputs 0.33 - 0.49 of the bound, the same as the exact answer rounded to bf16 (CE dlogits 0.46
# against 0.28); fp32 sums <= 0.024.  The power checks below exceed the bound by 1.9x (RMSNorm rstd x (1 + 2^-6)) to
# > 1e7x.
# ------------------------------------------------------------------------------------------------------------------
A_REL = 2.0 ** -7
B_NORM = 2.0 ** -10
B_ROPE = 2.0 ** -7
B_SWIGLU = 2.0 ** -10
FLOOR = 2.0 ** -60
A_P = {F32: 2.0 ** -15, BF16: 2.0 ** -7}
A_OUT = {F32: 2.0 ** -20, BF16: A_REL}
A_P_LSE = 2.0 ** -22
C_SUM = 2.0 ** -16
EPS = 1e-5


def _ratio(got, ref, A, B, extra=None):
    """max over elements of |got - ref| / bound; <= 1 passes.  Slices are the last dimension.  NaN in got -> NaN."""
    got, ref = got.double(), ref.double()
    bound = A * ref.abs() + B * ref.pow(2).mean(-1, keepdim=True).sqrt() + FLOOR
    if extra is not None:
        bound = bound + extra
    return ((got - ref).abs() / bound).max().item()


def _sum_ratio(got, ref, absum):
    got, ref = got.double(), ref.double()
    return ((got - ref).abs() / (C_SUM * absum.double() + FLOOR)).max().item()


def _fail_report(what, q):
    q = torch.nan_to_num(q, nan=math.inf)
    i = np.unravel_index(int(q.argmax()), tuple(q.shape))
    print(f"WORST {what} at {i}: error / bound {q[i].item():.4g}; elements over the bound: {(q > 1).sum().item()}")


def _check(what, got, ref, A, B, extra=None, out=BF16):
    r = _ratio(got, ref, A, B, extra)
    print(f"RATIO {what} {r:.4f} (exact answer rounded to {str(out)[6:]}: {_ratio(ref.to(out), ref, A, B, extra):.4f})")
    if not r <= 1.0:
        got, ref = got.double(), ref.double()
        bound = A * ref.abs() + B * ref.pow(2).mean(-1, keepdim=True).sqrt() + FLOOR + (0 if extra is None else extra)
        _fail_report(what, (got - ref).abs() / bound)
    assert r <= 1.0, f"{what}: error / bound = {r:.3f}"


def _check_sum(what, got, ref, absum):
    r = _sum_ratio(got, ref, absum)
    print(f"RATIO {what} {r:.4f} (exact answer rounded to float32: {_sum_ratio(ref.float(), ref, absum):.4f})")
    if not r <= 1.0:
        _fail_report(what, (got.double() - ref.double()).abs() / (C_SUM * absum.double() + FLOOR))
    assert r <= 1.0, f"{what}: error / bound = {r:.3f}"


# ------------------------------------------------------------------------------------------------------------------
# float64 references (any device)
# ------------------------------------------------------------------------------------------------------------------
def ln_ref(x, gamma, beta, dy=None):
    """-> y, mean, rstd and, with dy, dx, dgamma, dbeta and the sums of |terms| of dgamma / dbeta."""
    D = x.shape[-1]
    grad = dy is not None
    x64, g64, b64 = (t.detach().double().requires_grad_(grad) for t in (x, gamma, beta))
    y = torch.nn.functional.layer_norm(x64, (D,), g64, b64, EPS)
    mean = x64.detach().mean(-1)
    rstd = (x64.detach().var(-1, unbiased=False) + EPS).rsqrt()
    r = {"y": y.detach(), "mean": mean, "rstd": rstd}
    if grad:
        dy64 = dy.double()
        r["dx"], r["dgamma"], r["dbeta"] = torch.autograd.grad(y, (x64, g64, b64), dy64)
        xhat = (x64.detach() - mean[:, None]) * rstd[:, None]
        # the kernel gets mean rounded to fp32, which moves xhat by 2^-24 |mean| rstd however small xhat is
        r["abs_dgamma"] = (dy64.abs() * (xhat.abs() + (mean * rstd).abs()[:, None])).sum(0)
        r["abs_dbeta"] = dy64.abs().sum(0)
    return r


def rms_ref(x, w, eps, dy=None):
    x64 = x.detach().double().requires_grad_(dy is not None)
    rstd = (x64.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    y = x64 * rstd * w.double()
    r = {"y": y.detach(), "rstd": rstd.detach()[:, 0]}
    if dy is not None:
        r["dx"] = torch.autograd.grad(y, x64, dy.double())[0]
    return r


def rope_ref(x, pos, rot, theta, partner_shift=0, dim0=0):
    """rotate_half RoPE of dims [dim0, dim0 + rot) of the last axis of x [rows, heads, d]; angle = pos * theta^(-2j/rot),
    j = i mod rot/2.  partner_shift != 0 pairs i with i + rot/2 + shift (a mutation; 0 is the real operation)."""
    half = rot // 2
    inv = theta ** (-2.0 * torch.arange(half, dtype=F64, device=x.device) / rot)
    ang = pos.to(x.device).double()[:, None] * inv[None]
    cos, sin = torch.cat([ang.cos(), ang.cos()], -1)[:, None], torch.cat([ang.sin(), ang.sin()], -1)[:, None]
    xr = x[..., dim0:dim0 + rot]
    i = torch.arange(rot, device=x.device)
    partner = torch.where(i < half, half + (i + partner_shift) % half, (i - half + partner_shift) % half)
    sign = torch.where(i < half, -1.0, 1.0).to(x.device, F64)
    rh = xr[..., partner] * sign
    return torch.cat([x[..., :dim0], xr * cos + rh * sin, x[..., dim0 + rot:]], -1)


def swiglu_ref(g, u, dh=None):
    g64, u64 = (t.detach().double().requires_grad_(dh is not None) for t in (g, u))
    h = torch.nn.functional.silu(g64) * u64
    r = {"h": h.detach()}
    if dh is not None:
        r["dg"], r["du"] = torch.autograd.grad(h, (g64, u64), dh.double())
    return r


def qkln_ref(fused, row0, H, S, par, rot, theta, dqkv=None):
    """fused [n, H*192] = rows row0.. of [rows][H][q | k | v][64].  -> qkv [n, 3H, 64], stats [n, H, 4] and, with dqkv,
    dfused [n, H, 3, 64], the four parameter gradients and the sums of |terms| of each."""
    n = fused.shape[0]
    grad = dqkv is not None
    x = fused.detach().double().view(n, H, 3, 64).requires_grad_(grad)
    pr = [p.detach().double().requires_grad_(grad) for p in par]
    q, k = x[:, :, 0], x[:, :, 1]
    qs = torch.nn.functional.layer_norm(q, (64,), pr[0], pr[1], EPS)
    ks = torch.nn.functional.layer_norm(k, (64,), pr[2], pr[3], EPS)
    pos = torch.arange(row0, row0 + n, device=fused.device) % S
    qr, kr = (rope_ref(t, pos, rot, theta) if rot else t for t in (qs, ks))
    out = torch.cat([qr, kr, x[:, :, 2]], 1)
    st = []
    for t in (q.detach(), k.detach()):
        st += [t.mean(-1), (t.var(-1, unbiased=False) + EPS).rsqrt()]
    r = {"qkv": out.detach(), "stats": torch.stack(st, -1)}
    if grad:
        gr = torch.autograd.grad(out, [x, *pr, qs, ks], dqkv.double().view(n, 3 * H, 64))
        r["dfused"], r["dpar"] = gr[0], list(gr[1:5])
        absum = []
        for w, dys in ((0, gr[5]), (1, gr[6])):
            xh = (x.detach()[:, :, w] - st[2 * w][..., None]) * st[2 * w + 1][..., None]
            xh = xh.abs() + (st[2 * w] * st[2 * w + 1]).abs()[..., None]           # as ln_ref: rounded mean
            absum += [(dys.abs() * xh).sum((0, 1)), dys.abs().sum((0, 1))]
        r["abs"] = absum
    return r


def ce_ref(logits, labels, tgt_shift=0, no_minus_one=False, count_delta=0, drop_last=False):
    """Shifted cross-entropy (target of row (b, t) = labels[b, t + 1], last position ignored, mean over counted rows)
    in float64.  The keyword arguments are mutations for the power checks; the defaults are the real operation."""
    x = logits.double()
    V = x.shape[-1]
    tgt = torch.roll(labels, -1, 1)
    tgt[:, -1] = -100
    tgt = tgt.reshape(-1).to(x.device)
    ign = tgt == -100
    t = (tgt.clamp_min(0) + tgt_shift).clamp(0, V - 1)
    lse = torch.logsumexp(x[:, :-1] if drop_last else x, -1)
    p = torch.exp(x - lse[:, None])
    count = int((~ign).sum()) + count_delta
    inv = 1.0 / max(count, 1)
    xt = x.gather(1, t[:, None])[:, 0]
    loss = ((lse - xt) * ~ign).sum() * inv
    onehot = torch.zeros_like(x).scatter_(1, t[:, None], 0.0 if no_minus_one else 1.0)
    d = ((p - onehot) * inv).masked_fill(ign[:, None], 0.0)
    return {"loss": loss, "d": d, "p": p.masked_fill(ign[:, None], 0.0), "lse": lse, "ign": ign, "inv": inv,
            "abs_loss": ((lse.abs() + xt.abs() + 1) * ~ign).sum() * inv}


def _ce_extra(r, dtype, in_smem):
    a_p = A_P[dtype] + (0.0 if in_smem else A_P_LSE * r["lse"].abs()[:, None])
    return a_p * r["p"] * r["inv"]


def _ce_ratio(got_loss, got_d, r, dtype, in_smem):
    return max(_sum_ratio(got_loss, r["loss"], r["abs_loss"]),
               _ratio(got_d, r["d"], A_OUT[dtype], 0.0, _ce_extra(r, dtype, in_smem)))


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(BF16)


def _param(g, n, spread=0.2):
    return 1 + spread * torch.randn(n, generator=g), spread * torch.randn(n, generator=g)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the metric rejects plausible kernel bugs.  Each mutation is applied to the float64 reference.
# ------------------------------------------------------------------------------------------------------------------
def _mutant(r):
    print(f"MUTANT ratio {r:.3f}")
    return r


def _norm_case(kind, rows, D, seed=0):
    g = torch.Generator().manual_seed(seed)
    x, dy = _rnd(g, rows, D, scale=2.0), _rnd(g, rows, D)
    gamma, beta = _param(g, D)
    if kind == "ln":
        return x, gamma, beta, ln_ref(x, gamma, beta, dy), dy
    return x, gamma, beta, rms_ref(x, gamma, 1e-6, dy), dy


@pytest.mark.parametrize("kind", ["ln", "rms"])
def test_metric_rejects_rstd_of_one_row_off_by_2_pow_minus_6(kind):
    x, gamma, beta, r, _ = _norm_case(kind, 9, 264)
    x64 = x.double()
    if kind == "ln":
        xhat = (x64 - r["mean"][:, None]) * r["rstd"][:, None]
        xhat[4] *= 1 + 2.0 ** -6
        y = xhat * gamma.double() + beta.double()
    else:
        y = x64 * (r["rstd"][:, None] * torch.tensor([1 + 2.0 ** -6 if i == 4 else 1.0 for i in range(9)],
                                                     dtype=F64)[:, None]) * gamma.double()
    assert _mutant(_ratio(y, r["y"], A_REL, B_NORM)) > 1.0


@pytest.mark.parametrize("kind", ["ln", "rms"])
@pytest.mark.parametrize("tensor", ["y", "dx"])
def test_metric_rejects_one_vector_from_the_neighbouring_row(kind, tensor):
    *_, r, _ = _norm_case(kind, 9, 264, seed=1)
    t = r[tensor].clone()
    t[3, 136:144] = r[tensor][4, 136:144]
    assert _mutant(_ratio(t, r[tensor], A_REL, B_NORM)) > 1.0


@pytest.mark.parametrize("tensor", ["y", "dx"])
def test_metric_rejects_last_vector_of_ragged_row_left_at_zero(tensor):
    """D = 264 = 256 + 8: lane 0 owns the 33rd vector; a loop bound of D / 256 vectors per lane would skip it."""
    *_, r, _ = _norm_case("ln", 7, 264, seed=2)
    t = r[tensor].clone()
    t[:, 256:] = 0.0
    assert _mutant(_ratio(t, r[tensor], A_REL, B_NORM)) > 1.0


@pytest.mark.parametrize("missing", ["one_row", "one_4_row_batch"])
def test_metric_rejects_dgamma_missing_rows(missing):
    rows = 2048
    x, gamma, beta, r, dy = _norm_case("ln", rows, 256, seed=3)
    lost = [1029] if missing == "one_row" else [1028, 1029, 1030, 1031]
    xhat = (x.double() - r["mean"][:, None]) * r["rstd"][:, None]
    dg = r["dgamma"] - (dy.double()[lost] * xhat[lost]).sum(0)
    db = r["dbeta"] - dy.double()[lost].sum(0)
    assert _mutant(_sum_ratio(dg, r["dgamma"], r["abs_dgamma"])) > 1.0
    assert _mutant(_sum_ratio(db, r["dbeta"], r["abs_dbeta"])) > 1.0


def test_metric_rejects_accumulate_ignored():
    x, gamma, beta, r, dy = _norm_case("ln", 300, 264, seed=4)
    old = torch.randn(264, generator=torch.Generator().manual_seed(5)).double()
    assert _mutant(_sum_ratio(r["dgamma"], old + r["dgamma"], r["abs_dgamma"] + old.abs())) > 1.0


def _rope_case(S=2048, H=2, seed=6):
    g = torch.Generator().manual_seed(seed)
    return _rnd(g, S, H, 128).double(), torch.arange(S)


@pytest.mark.parametrize("delta", [-1, 1])
def test_metric_rejects_rope_angle_of_one_row_from_neighbouring_position(delta):
    x, pos = _rope_case()
    ref = rope_ref(x, pos, 128, 10000.0)
    pos_m = pos.clone()
    pos_m[1500] += delta
    assert _mutant(_ratio(rope_ref(x, pos_m, 128, 10000.0), ref, A_REL, B_ROPE)) > 1.0


@pytest.mark.parametrize("rot,d", [(128, 128), (64, 64), (4, 64)])
@pytest.mark.parametrize("shift", [-1, 1])
def test_metric_rejects_rotate_half_partner_off_by_one(rot, d, shift):
    """rope128 (rot = d = 128) and the qk-LN partial rotary at both ends of its lane shuffle (rot 64 and 4)."""
    x, pos = _rope_case(S=300)
    x = x[..., :d]
    ref = rope_ref(x, pos, rot, 10000.0)
    assert _mutant(_ratio(rope_ref(x, pos, rot, 10000.0, partner_shift=shift), ref, A_REL, B_ROPE)) > 1.0


@pytest.mark.parametrize("rot", [4, 32])
def test_metric_rejects_rotation_of_the_wrong_dims(rot):
    """Partial rotary applied to dims [rot, 2 rot) instead of [0, rot)."""
    x, pos = _rope_case(S=300)
    x = x[..., :64]
    ref = rope_ref(x, pos, rot, 25000.0)
    assert _mutant(_ratio(rope_ref(x, pos, rot, 25000.0, dim0=rot), ref, A_REL, B_ROPE)) > 1.0


@pytest.mark.parametrize("rot,d", [(128, 128), (32, 64)])
def test_metric_rejects_backward_with_the_forward_rotation(rot, d):
    x, pos = _rope_case(S=300)
    x, dy = x[..., :d].clone().requires_grad_(True), _rope_case(S=300, seed=7)[0][..., :d]
    ref = torch.autograd.grad(rope_ref(x, pos, rot, 10000.0), x, dy)[0]
    assert _mutant(_ratio(rope_ref(dy, pos, rot, 10000.0), ref, A_REL, B_ROPE)) > 1.0


def _ce_case(dtype, V=1000, B=3, L=37, seed=8):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(B * L, V, generator=g) * 2).to(dtype)
    labels = torch.randint(0, V, (B, L), generator=g)
    labels[labels % 5 == 0] = -100
    return logits, labels


@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("mutation", ["target+1", "target-1", "no_minus_one", "count+1", "count-1", "drop_last_logit"])
def test_metric_rejects_cross_entropy_mutations(dtype, mutation):
    logits, labels = _ce_case(dtype)
    r = ce_ref(logits, labels)
    kw = {"target+1": {"tgt_shift": 1}, "target-1": {"tgt_shift": -1}, "no_minus_one": {"no_minus_one": True},
          "count+1": {"count_delta": 1}, "count-1": {"count_delta": -1}, "drop_last_logit": {"drop_last": True}}[mutation]
    m = ce_ref(logits, labels, **kw)
    assert _mutant(_ce_ratio(m["loss"], m["d"], r, dtype, True)) > 1.0


def test_metric_accepts_bf16_output_rounding():
    """The other side: rounding the exact answer to bf16 stays below 0.5 of each bf16 bound (derived at the constants)."""
    _, _, _, r, _ = _norm_case("ln", 64, 264)
    assert _mutant(_ratio(r["y"].to(BF16), r["y"], A_REL, B_NORM)) < 0.5
    assert _mutant(_ratio(r["dx"].to(BF16), r["dx"], A_REL, B_NORM)) < 0.5
    x, pos = _rope_case(S=64)
    y = rope_ref(x, pos, 128, 10000.0)
    assert _mutant(_ratio(y.to(BF16), y, A_REL, B_ROPE)) < 0.5
    logits, labels = _ce_case(BF16)
    c = ce_ref(logits, labels)
    assert _mutant(_ratio(c["d"].to(BF16), c["d"], A_REL, 0.0, _ce_extra(c, BF16, True))) < 0.5


def test_rope_reference_matches_the_rotate_half_formula():
    """rope_ref (index-built partner) equals the textbook x cos + rotate_half(x) sin with emb = cat(freqs, freqs)."""
    x, pos = _rope_case(S=40)
    inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2, dtype=F64) / 128))
    emb = torch.cat([pos.double()[:, None] * inv] * 2, -1)[:, None]
    rh = torch.cat([-x[..., 64:], x[..., :64]], -1)
    assert torch.allclose(rope_ref(x, pos, 128, 10000.0), x * emb.cos() + rh * emb.sin(), rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------
# GPU harness: the C ABI with NaN-filled canvases.
# ------------------------------------------------------------------------------------------------------------------
DEV = "cuda:0"


def _lib():
    from otter_b200 import _lib as L
    return L.load()


def _ok(rc, what):
    from otter_b200 import _lib as L
    L.check(rc, what)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rows(spec):
    """An int, or 'k*4sm+c': k one-pass-kernel waves of 4-row batches (4 * SMs rows) plus c."""
    if isinstance(spec, int):
        return spec
    k, c = re.fullmatch(r"(\d+)\*4sm([+-]\d+)?", spec).groups()
    return int(k) * 4 * _sms() + int(c or 0)


class _Canvas:
    """A NaN-filled [rows + extra, pitch] buffer with owned rectangles."""

    def __init__(self, rows, pitch, dtype=BF16, extra=2):
        self.t = torch.full((rows + extra, pitch), float("nan"), dtype=dtype, device=DEV)
        self.owned = torch.zeros(rows + extra, pitch, dtype=torch.bool, device=DEV)
        self.pitch = pitch

    def own(self, r1, c0, c1, init=None):
        self.owned[:r1, c0:c1] = True
        if init is not None:
            self.t[:r1, c0:c1] = init.to(DEV, self.t.dtype)
        return self.t[:r1, c0:c1]

    def put(self, src, c0=0):
        self.t[:src.shape[0], c0:c0 + src.shape[1]] = src.to(DEV, self.t.dtype)
        return self

    def ptr(self, c0=0):
        return C.c_void_p(self.t.data_ptr() + c0 * self.t.element_size())

    def bits(self):
        return self.t.view({2: torch.int16, 4: torch.int32}[self.t.element_size()])

    def check(self, what):
        nan = torch.full((1,), float("nan"), dtype=self.t.dtype, device=DEV).view(self.bits().dtype)
        assert torch.isfinite(self.t[self.owned].float()).all(), f"{what}: an owned element was not written"
        assert (self.bits()[~self.owned] == nan).all(), f"{what}: an element outside the output was written"


def _geom(D, pad):
    """(row pitch, first column) of a D-wide operand: tight, or `pad` extra columns around it (16 B aligned)."""
    return (D, 0) if not pad else (D + pad, pad // 2)


def _vec(v, pad=0):
    """An fp32 vector in a NaN canvas, starting `pad` floats in (0 keeps the 16 B alignment float4 loads need)."""
    c = _Canvas(1, v.numel() + pad + 3, F32, extra=0)
    c.own(1, pad, pad + v.numel(), v[None])
    return c


def _in(x, pad):
    p, c0 = _geom(x.shape[1], pad)
    cv = _Canvas(x.shape[0], p).put(x, c0)
    return cv, c0


# ------------------------------------------------------------------------------------------------------------------
# GPU: LayerNorm
# ------------------------------------------------------------------------------------------------------------------
def _ln_inputs(rows, D, seed, special=False):
    g = torch.Generator().manual_seed(seed * 7919 + rows * 31 + D)
    x = _rnd(g, rows, D, scale=2.0)
    if special and rows >= 2:
        x[1] = 0.75                                            # constant row: variance 0, rstd = eps^-1/2, y = beta
    if special and rows >= 3:
        x[2] = (64.0 + 2.0 * torch.randn(D, generator=g)).to(BF16)   # common offset: mean / std = 32
    gamma, beta = _param(g, D)
    return g, x, gamma, beta


def _run_ln_fwd(tag, rows, D, pad=0, special=False, seed=0):
    lib = _lib()
    _, x, gamma, beta = _ln_inputs(rows, D, seed, special)
    cx, cx0 = _in(x, pad)
    py, cy0 = _geom(D, 2 * pad)
    cy = _Canvas(rows, py)
    y = cy.own(rows, cy0, cy0 + D)
    cm, cr = _Canvas(1, rows + 4, F32, 0), _Canvas(1, rows + 4, F32, 0)
    mean, rstd = cm.own(1, 1, rows + 1)[0], cr.own(1, 1, rows + 1)[0]
    gd, bd = gamma.to(DEV), beta.to(DEV)
    _ok(lib.otb_layernorm_fwd(cx.ptr(cx0), cx.pitch, C.c_void_p(gd.data_ptr()), C.c_void_p(bd.data_ptr()),
                              cy.ptr(cy0), cy.pitch, cm.ptr(1), cr.ptr(1), rows, D, EPS, _stream()), "otb_layernorm_fwd")
    torch.cuda.synchronize()
    for cv, what in ((cy, "y"), (cm, "mean"), (cr, "rstd")):
        cv.check(f"{tag} {what}")
    r = ln_ref(x.to(DEV), gd, bd)
    _check(f"{tag} y", y, r["y"], A_REL, B_NORM)
    _check_sum(f"{tag} mean", mean, r["mean"], x.to(DEV).double().abs().mean(-1))
    _check_sum(f"{tag} rstd", rstd, r["rstd"], r["rstd"])
    if special and rows >= 2:
        assert rstd[1].item() == pytest.approx(EPS ** -0.5, rel=2.0 ** -20)


def _run_ln_bwd(tag, rows, D, *, add=True, dx=True, params=True, accumulate=False, pad=0, seed=0):
    """otb_layernorm_bwd given the reference's statistics rounded to fp32.  dx / params / accumulate select the route."""
    lib = _lib()
    g, x, gamma, beta = _ln_inputs(rows, D, seed, special=True)
    dy, a = _rnd(g, rows, D), _rnd(g, rows, D)
    xd, gd, bd = x.to(DEV), gamma.to(DEV), beta.to(DEV)
    r = ln_ref(xd, gd, bd, dy.to(DEV))
    mean, rstd = r["mean"].float(), r["rstd"].float()
    cdy, c0dy = _in(dy, pad)
    cx, c0x = _in(x, 2 * pad)
    ca, c0a = _in(a, 3 * pad) if add else (None, 0)
    cdx = None
    if dx:
        p, c0dx = _geom(D, pad + 16 if pad else 0)
        cdx = _Canvas(rows, p)
        dxv = cdx.own(rows, c0dx, c0dx + D)
    outs = []
    if params:
        old = [torch.randn(D, generator=g) * 3 for _ in range(2)] if accumulate else [None, None]
        outs = [_Canvas(1, D + 8, F32, 0) for _ in range(2)]
        views = [cv.own(1, 4, 4 + D, o[None] if o is not None else None)[0] for cv, o in zip(outs, old)]
        ws = torch.full((2 * lib.otb_ln_chunks(rows, D) * D,), float("nan"), device=DEV)     # scratch
    _ok(lib.otb_layernorm_bwd(cdy.ptr(c0dy), cdy.pitch, cx.ptr(c0x), cx.pitch, C.c_void_p(mean.data_ptr()),
                              C.c_void_p(rstd.data_ptr()), C.c_void_p(gd.data_ptr()), ca.ptr(c0a) if add else None,
                              ca.pitch if add else 0, cdx.ptr(c0dx) if dx else None, cdx.pitch if dx else 0,
                              outs[0].ptr(4) if params else None, outs[1].ptr(4) if params else None, int(accumulate),
                              C.c_void_p(ws.data_ptr()) if params else None, rows, D, _stream()), "otb_layernorm_bwd")
    torch.cuda.synchronize()
    if dx:
        cdx.check(f"{tag} dx")
        _check(f"{tag} dx", dxv, r["dx"] + (a.to(DEV).double() if add else 0), A_REL, B_NORM)
    if params:
        for cv, v, o, key in zip(outs, views, old, ("dgamma", "dbeta")):
            cv.check(f"{tag} {key}")
            o = torch.zeros(D, dtype=F64) if o is None else o.double()
            _check_sum(f"{tag} {key}", v, r[key] + o.to(DEV), r["abs_" + key] + o.abs().to(DEV))


@gpu
@pytest.mark.parametrize("rows,D", [(37, 256), (512, 1024), (300, 4096), (101, 3072), (2, 2048), (64, 6144)])
def test_layernorm_fwd_bwd(rows, D):
    _run_ln_fwd(f"ln[{rows}-{D}] fwd", rows, D)
    _run_ln_bwd(f"ln[{rows}-{D}] bwd", rows, D)


@gpu
@pytest.mark.parametrize("D,rows,pad", [
    (8, 1, 0), (256, 7, 16), (264, 8, 0), (1024, 9, 32), (2048, 7, 0), (2056, 9, 16), (4096, 8, 64), (4104, 1, 16),
    (6144, 9, 0), (264, 300, 16),
])
def test_layernorm_fwd_edges(D, rows, pad):
    """D around the 256-column lane stride, rows around one 8-warp CTA; rows 1 / 2 of every case with rows >= 3 are a
    constant row and a row with a large common offset."""
    _run_ln_fwd(f"ln_fwd[{D}-{rows}-{pad}]", rows, D, pad=pad, special=True)


@gpu
@pytest.mark.parametrize("rows,D,add,dx,params,acc,pad", [
    # one-pass kernel <1> / <2>: batches per CTA 1 .. 4, with and without the smem parity flipping
    (1, 2048, True, True, True, False, 0), (3, 2056, True, True, True, True, 16), (4, 4096, False, True, True, False, 0),
    (5, 2048, True, True, True, True, 32), ("1*4sm-1", 2056, True, True, True, False, 16),
    ("1*4sm", 4096, True, True, True, True, 0), ("1*4sm+1", 2048, False, True, True, False, 16),
    ("3*4sm+5", 2056, True, True, True, True, 16), (2048, 4096, True, True, True, True, 0),
    (2048, 2048, False, True, True, False, 64),
    # one-pass kernel without dx (perceiver norm_media)
    ("3*4sm+5", 2048, False, False, True, False, 16), (7, 4096, False, False, True, True, 0),
    # ln_bwd_dx_kernel alone (frozen MPT / Persimmon layers)
    (2048, 4096, True, True, False, False, 16), (5, 2056, False, True, False, False, 0),
    (300, 6144, True, True, False, False, 32),
    # D > 4096: dx + param + finalize; last chunk short (2048 / 9 chunks, 2049 / 6), rows < 8 * chunks (1, 13, 47)
    (1, 4104, True, True, True, False, 0), (13, 6144, True, True, True, True, 16), (47, 6144, False, True, True, False, 0),
    (2048, 4104, True, True, True, True, 32), (2049, 6144, True, True, True, False, 0),
    (300, 6144, False, False, True, True, 16),
])
def test_layernorm_bwd_routes(rows, D, add, dx, params, acc, pad):
    n = _rows(rows)
    _run_ln_bwd(f"ln_bwd[{rows}={n}-{D}-add{int(add)}-dx{int(dx)}-p{int(params)}-acc{int(acc)}-{pad}]", n, D, add=add,
                dx=dx, params=params, accumulate=acc, pad=pad)


# ------------------------------------------------------------------------------------------------------------------
# GPU: RMSNorm
# ------------------------------------------------------------------------------------------------------------------
def _run_rms(tag, rows, D, *, add=True, pad=0, eps=1e-6, seed=0):
    lib = _lib()
    g = torch.Generator().manual_seed(seed * 7919 + rows * 31 + D)
    x = _rnd(g, rows, D, scale=2.0)
    if rows >= 3:
        x[2] = 0.0                                             # all-zero row: rstd = eps^-1/2, y = 0
    w = (1 + 0.2 * torch.randn(D, generator=g)).to(DEV)
    dy, a = _rnd(g, rows, D), _rnd(g, rows, D)
    r = rms_ref(x.to(DEV), w, eps, dy.to(DEV))
    cx, c0x = _in(x, pad)
    py, c0y = _geom(D, 2 * pad)
    cy, cr = _Canvas(rows, py), _Canvas(1, rows + 4, F32, 0)
    y, rstd = cy.own(rows, c0y, c0y + D), cr.own(1, 1, rows + 1)[0]
    _ok(lib.otb_rmsnorm_fwd(cx.ptr(c0x), cx.pitch, C.c_void_p(w.data_ptr()), cy.ptr(c0y), cy.pitch, cr.ptr(1), rows, D,
                            eps, _stream()), "otb_rmsnorm_fwd")
    cdy, c0dy = _in(dy, 3 * pad)
    ca, c0a = _in(a, pad) if add else (None, 0)
    pdx, c0dx = _geom(D, pad)
    cdx = _Canvas(rows, pdx)
    dx = cdx.own(rows, c0dx, c0dx + D)
    rs32 = r["rstd"].float()
    _ok(lib.otb_rmsnorm_bwd(cdy.ptr(c0dy), cdy.pitch, cx.ptr(c0x), cx.pitch, C.c_void_p(rs32.data_ptr()),
                            C.c_void_p(w.data_ptr()), ca.ptr(c0a) if add else None, ca.pitch if add else 0,
                            cdx.ptr(c0dx), cdx.pitch, rows, D, _stream()), "otb_rmsnorm_bwd")
    torch.cuda.synchronize()
    for cv, what in ((cy, "y"), (cr, "rstd"), (cdx, "dx")):
        cv.check(f"{tag} {what}")
    _check(f"{tag} y", y, r["y"], A_REL, B_NORM)
    _check_sum(f"{tag} rstd", rstd, r["rstd"], r["rstd"])
    _check(f"{tag} dx", dx, r["dx"] + (a.to(DEV).double() if add else 0), A_REL, B_NORM)
    if rows >= 3:
        assert y[2].abs().max().item() == 0.0


@gpu
@pytest.mark.parametrize("rows,D,add,pad", [(13, 8, True, 16), (7, 264, False, 32), (301, 4096, True, 0),
                                            (2049, 5120, True, 16)])
def test_rmsnorm_fwd_bwd(rows, D, add, pad):
    _run_rms(f"rms[{rows}-{D}-{int(add)}-{pad}]", rows, D, add=add, pad=pad)


# ------------------------------------------------------------------------------------------------------------------
# GPU: rope128 (in place)
# ------------------------------------------------------------------------------------------------------------------
def _run_rope(tag, B, S, H, nblk, theta, pad=0, seed=0):
    """Forward, then backward on fresh data.  The buffer holds nblk rotated blocks, one more block (v) and `pad` NaN
    columns; everything but the rotated blocks must stay bit-identical."""
    lib = _lib()
    rows, width = B * S, nblk * H * 128
    full = width + H * 128
    g = torch.Generator().manual_seed(seed * 7919 + S * 31 + H)
    pos = (torch.arange(rows) % S).to(DEV)
    for backward in (False, True):
        src = _rnd(g, rows, full)
        cv = _Canvas(rows, full + pad).put(src)
        before = cv.bits().clone()
        _ok(lib.otb_rope128(cv.ptr(), cv.pitch, rows, H, S, nblk, float(theta), int(backward), _stream()),
            "otb_rope128")
        torch.cuda.synchronize()
        rest = torch.ones_like(cv.owned)
        rest[:rows, :width] = False
        assert torch.equal(cv.bits()[rest], before[rest]), f"{tag}: an element outside the rotated blocks changed"
        x = src[:, :width].to(DEV).double().view(rows, nblk * H, 128)
        if backward:          # the transpose, from autograd of the forward
            x0 = _rnd(g, rows, width).to(DEV).double().view(rows, nblk * H, 128).requires_grad_(True)
            ref = torch.autograd.grad(rope_ref(x0, pos, 128, theta), x0, x)[0]
        else:
            ref = rope_ref(x, pos, 128, theta)
        _check(f"{tag} {'dx' if backward else 'y'}", cv.t[:rows, :width].reshape(rows, nblk * H, 128), ref, A_REL, B_ROPE)


@gpu
@pytest.mark.parametrize("B,S,H,nblk,theta,pad", [
    (2, 1, 32, 2, 10000.0, 64), (4, 25, 1, 1, 500000.0, 16),
    (1, 2048, 32, 2, 10000.0, 0),                 # LLaMA-7B: 8.4 M pairs, ~31 grid-stride passes
    (2, 2048, 1, 1, 500000.0, 128), (1, 4096, 2, 2, 500000.0, 32),
])
def test_rope128_fwd_bwd(B, S, H, nblk, theta, pad):
    _run_rope(f"rope[{B}-{S}-{H}-{nblk}-{theta:g}-{pad}]", B, S, H, nblk, theta, pad)


# ------------------------------------------------------------------------------------------------------------------
# GPU: SwiGLU
# ------------------------------------------------------------------------------------------------------------------
def _run_swiglu(tag, rows, I, pad=0, big=False, seed=0):
    """g and u are the two halves of one [rows][2I] buffer; dg and du the two halves of another."""
    lib = _lib()
    g = torch.Generator().manual_seed(seed * 7919 + rows + I)
    gv = torch.randn(rows, I, generator=g) * 2
    if big:                                     # |g| up to ~100: sigmoid saturates, __expf(-g) overflows at g < -88
        gv[:, ::7] *= 12
    gu = torch.cat([gv.to(BF16), _rnd(g, rows, I)], 1)
    dh = _rnd(g, rows, I)
    cgu, c0 = _in(gu, pad)
    cdh, c0dh = _in(dh, 2 * pad)
    ph, c0h = _geom(I, pad)
    ch = _Canvas(rows, ph)
    h = ch.own(rows, c0h, c0h + I)
    pd, c0d = _geom(2 * I, 2 * pad)
    cd = _Canvas(rows, pd)
    dg, du = cd.own(rows, c0d, c0d + I), cd.own(rows, c0d + I, c0d + 2 * I)
    _ok(lib.otb_swiglu_fwd(cgu.ptr(c0), cgu.pitch, cgu.ptr(c0 + I), cgu.pitch, ch.ptr(c0h), ch.pitch, rows, I,
                           _stream()), "otb_swiglu_fwd")
    _ok(lib.otb_swiglu_bwd(cdh.ptr(c0dh), cdh.pitch, cgu.ptr(c0), cgu.pitch, cgu.ptr(c0 + I), cgu.pitch, cd.ptr(c0d),
                           cd.pitch, cd.ptr(c0d + I), cd.pitch, rows, I, _stream()), "otb_swiglu_bwd")
    torch.cuda.synchronize()
    ch.check(f"{tag} h")
    cd.check(f"{tag} dg|du")
    gud = gu.to(DEV)
    r = swiglu_ref(gud[:, :I], gud[:, I:], dh.to(DEV))
    _check(f"{tag} h", h, r["h"], A_REL, B_SWIGLU)
    _check(f"{tag} dg", dg, r["dg"], A_REL, B_SWIGLU)
    _check(f"{tag} du", du, r["du"], A_REL, B_SWIGLU)


@gpu
@pytest.mark.parametrize("rows,I,pad,big", [
    ("2cap+77", 8, 16, True),                     # one vector per row, > 2 grid-stride passes
    (600, 11008, 32, True),                       # LLaMA-7B intermediate size, ~3 passes
    (9, 11008, 0, False),
])
def test_swiglu_fwd_bwd(rows, I, pad, big):
    n = 2 * 8 * _sms() * 256 + 77 if rows == "2cap+77" else rows
    _run_swiglu(f"swiglu[{n}-{I}-{pad}-{int(big)}]", n, I, pad, big)


# ------------------------------------------------------------------------------------------------------------------
# GPU: qk-LayerNorm + partial RoPE (Persimmon)
# ------------------------------------------------------------------------------------------------------------------
QK_BLOCK_ROWS = 256                               # float64 reference built per row block


def _run_qkln(tag, B, S, H, rot, theta, *, accumulate=False, pad=0, seed=0):
    lib = _lib()
    rows = B * S
    g = torch.Generator().manual_seed(seed * 7919 + rows * 31 + H * 7 + rot)
    fused = (torch.randn(rows, H * 192, generator=g) * 1.5).to(BF16)
    par = [t.to(DEV) for t in (*_param(g, 64), *_param(g, 64))]
    dqkv = _rnd(g, rows, 3 * H * 64)
    cf, c0f = _in(fused, pad)
    pq, c0q = _geom(3 * H * 64, 2 * pad)
    cq, cs = _Canvas(rows, pq), _Canvas(1, rows * H * 4 + 6, F32, 0)
    qkv, stats = cq.own(rows, c0q, c0q + 3 * H * 64), cs.own(1, 2, 2 + rows * H * 4)[0]
    pp = [C.c_void_p(t.data_ptr()) for t in par]
    _ok(lib.otb_qkln_rope_fwd(cf.ptr(c0f), cf.pitch, *pp, cq.ptr(c0q), cq.pitch, cs.ptr(2), rows, H, S, rot,
                              float(theta), EPS, _stream()), "otb_qkln_rope_fwd")
    torch.cuda.synchronize()
    cq.check(f"{tag} qkv")
    cs.check(f"{tag} stats")

    refs = [qkln_ref(fused[r0:r0 + QK_BLOCK_ROWS].to(DEV), r0, H, S, par, rot, theta,
                     dqkv[r0:r0 + QK_BLOCK_ROWS].to(DEV)) for r0 in range(0, rows, QK_BLOCK_ROWS)]
    cat = lambda key: torch.cat([r[key] for r in refs])
    ref_stats = cat("stats")
    q3 = qkv.reshape(rows, 3 * H, 64)
    _check(f"{tag} q|k", q3[:, :2 * H], cat("qkv")[:, :2 * H], A_REL, B_ROPE)
    assert torch.equal(q3[:, 2 * H:].cpu(), fused.view(rows, H, 3, 64)[:, :, 2]), f"{tag}: v is a copy"
    st = stats.view(rows, H, 4)
    absx = [fused.to(DEV).double().view(rows, H, 3, 64)[:, :, w].abs().mean(-1) for w in (0, 1)]
    for w, name in ((0, "q"), (1, "k")):
        _check_sum(f"{tag} mean_{name}", st[..., 2 * w], ref_stats[..., 2 * w], absx[w])
        _check_sum(f"{tag} rstd_{name}", st[..., 2 * w + 1], ref_stats[..., 2 * w + 1], ref_stats[..., 2 * w + 1])

    stats32 = ref_stats.float().contiguous()       # the backward is handed the reference's statistics
    cdq, c0dq = _in(dqkv, pad)
    cdf = _Canvas(rows, cf.pitch + 16)
    dfused = cdf.own(rows, c0f + 8, c0f + 8 + H * 192)
    old = [torch.randn(64, generator=g) if accumulate else None for _ in range(4)]
    outs = [_vec(o if o is not None else torch.full((64,), float("nan"))) for o in old]
    ws = torch.full((lib.otb_qkln_rope_ws_floats(),), float("nan"), device=DEV)
    _ok(lib.otb_qkln_rope_bwd(cdq.ptr(c0dq), cdq.pitch, cf.ptr(c0f), cf.pitch, C.c_void_p(stats32.data_ptr()), pp[0],
                              pp[2], cdf.ptr(c0f + 8), cdf.pitch, *(o.ptr() for o in outs), int(accumulate),
                              C.c_void_p(ws.data_ptr()), rows, H, S, rot, float(theta), _stream()), "otb_qkln_rope_bwd")
    torch.cuda.synchronize()
    cdf.check(f"{tag} dfused")
    df = dfused.reshape(rows, H, 3, 64)
    _check(f"{tag} dq|dk", df[:, :, :2], cat("dfused")[:, :, :2], A_REL, B_ROPE)
    assert torch.equal(df[:, :, 2].cpu(), dqkv[:, 2 * H * 64:].view(rows, H, 64)), f"{tag}: dv is a copy"
    for j, name in enumerate(("dq_gamma", "dq_beta", "dk_gamma", "dk_beta")):
        outs[j].check(f"{tag} {name}")
        o = torch.zeros(64, dtype=F64) if old[j] is None else old[j].double()
        want = sum(r["dpar"][j] for r in refs) + o.to(DEV)
        absum = sum(r["abs"][j] for r in refs) + o.abs().to(DEV)
        _check_sum(f"{tag} {name}", outs[j].t[0, :64], want, absum)


@gpu
@pytest.mark.parametrize("rows_S,H,rot", [((2, 37), 4, 32), ((1, 300), 2, 16), ((3, 8), 64, 32)])
def test_qkln_rope_fwd_bwd_vs_torch(rows_S, H, rot):
    B, S = rows_S
    _run_qkln(f"qkln[{B}x{S}-{H}-{rot}]", B, S, H, rot, 25000.0)


@gpu
@pytest.mark.parametrize("B,S,H,rot,theta,acc,pad", [
    (2, 5, 3, 0, 25000.0, False, 16),             # no rotary
    (3, 7, 2, 4, 10000.0, True, 0),               # shuffle distance 1
    (1, 50, 4, 64, 25000.0, True, 64),            # shuffle distance 16: the whole head rotates
    (2, 2048, 64, 32, 25000.0, True, 0),          # Persimmon-8B: 262 144 (row, head) items, ~62 per warp
])
def test_qkln_rope_edges(B, S, H, rot, theta, acc, pad):
    _run_qkln(f"qkln[{B}x{S}-{H}-{rot}-{theta:g}-acc{int(acc)}-{pad}]", B, S, H, rot, theta, accumulate=acc, pad=pad)


# ------------------------------------------------------------------------------------------------------------------
# GPU: shifted cross-entropy
# ------------------------------------------------------------------------------------------------------------------
def _ce_inputs(dtype, V, B, L, offset=0.0, seed=0, ignore_all=False):
    """Logits [B*L, V] and labels [B, L] (every fifth class id ignored, the second sequence fully ignored).  Row 0
    targets class 0, row 1 class V - 1, and row 2 (target V // 2) has p_target ~ 1."""
    rows = B * L
    g = torch.Generator().manual_seed(seed * 7919 + V + rows)
    x = torch.randn(rows, V, generator=g) * 2 + offset
    labels = torch.randint(0, V, (B, L), generator=g)
    labels[labels % 5 == 0] = -100
    if L >= 4:
        labels[0, 1], labels[0, 2], labels[0, 3] = 0, V - 1, V // 2
        x[2, V // 2] = x[2].max() + 25
    if B >= 2 and L >= 2:
        labels[1, :] = -100                       # a fully ignored sequence
    if ignore_all:
        labels[:] = -100
    return x.to(dtype), labels


def _run_ce(tag, dtype, V, B, L, *, pad=8, offset=0.0, seed=0, ignore_all=False):
    """`pad` extra columns in both the logits and the dlogits row pitch.  A row takes the 16 B-vector body only if both
    its logits and its dlogits start 16 B aligned.  pad a multiple of the vector width (16 B / element size): dlogits
    start one vector in, so every row is aligned when V is a multiple of the vector width, and alternate rows are for
    V = 32002 (fp32).  Other pad: dlogits start one element in, so rows are misaligned and take the scalar loop.
    pad = 0: tight rows, ld = ldd = V (bf16 V = 32002: one row start in four is aligned)."""
    lib = _lib()
    rows = B * L
    logits, labels = _ce_inputs(dtype, V, B, L, offset, seed, ignore_all)
    vec = 16 // logits.element_size()
    d0 = (vec if pad else 0) if pad % vec == 0 else 1
    cl = _Canvas(rows, V + pad, dtype).put(logits)
    cd = _Canvas(rows, V + 2 * pad + d0, dtype)
    d = cd.own(rows, d0, d0 + V)
    closs = _Canvas(1, 4, F32, 0)
    loss = closs.own(1, 1, 2)
    ws = torch.full((1 + rows,), float("nan"), device=DEV)
    lab = labels.to(DEV)
    _ok(lib.otb_shifted_cross_entropy(cl.ptr(), int(dtype == F32), cl.pitch, C.c_void_p(lab.data_ptr()), B, L, V,
                                      closs.ptr(1), cd.ptr(d0), cd.pitch, C.c_void_p(ws.data_ptr()), _stream()),
        "otb_shifted_cross_entropy")
    torch.cuda.synchronize()
    closs.check(f"{tag} loss")
    cd.check(f"{tag} dlogits")
    r = ce_ref(logits.to(DEV), lab)
    in_smem = V * (4 if dtype == F32 else 2) <= 200 * 1024
    _check_sum(f"{tag} loss", loss[0, 0], r["loss"], r["abs_loss"])
    _check(f"{tag} dlogits", d, r["d"], A_OUT[dtype], 0.0, _ce_extra(r, dtype, in_smem), out=dtype)
    assert (d[r["ign"]] == 0).all(), f"{tag}: ignored rows must have an exactly zero gradient"
    if bool(r["ign"].all()):
        assert loss.item() == 0.0


@gpu
@pytest.mark.parametrize("dtype,V,B,L,pad,offset", [
    (F32, 1000, 3, 37, 0, 0.0), (BF16, 50432, 3, 37, 0, 0.0),              # the earlier cases
    (F32, 8, 2, 5, 8, 0.0), (F32, 1000, 2, 6, 3, 0.0), (F32, 32002, 2, 5, 8, 0.0), (F32, 50432, 2, 4, 16, 0.0),
    (F32, 51201, 2, 4, 8, 0.0),                                             # 200 KB + 4 B: global-memory path
    (F32, 51208, 2, 4, 8, 0.0),                                             # global memory, 16 B vectors
    (F32, 4096, 2, 6, 8, 1.0e4),                                            # logits ~1e4
    (BF16, 8, 2, 5, 8, 0.0), (BF16, 1000, 2, 6, 3, 0.0), (BF16, 32002, 2, 5, 0, 0.0),
    (BF16, 50432, 2, 4, 16, 0.0), (BF16, 102401, 2, 4, 8, 0.0), (BF16, 102408, 2, 4, 8, 0.0),
])
def test_shifted_cross_entropy(dtype, V, B, L, pad, offset):
    _run_ce(f"ce[{str(dtype)[6:]}-{V}-{B}x{L}-{pad}-{offset:g}]", dtype, V, B, L, pad=pad, offset=offset)


@gpu
@pytest.mark.parametrize("dtype,V,B,L,ignore_all", [(F32, 100, 3, 1, False), (BF16, 64, 2, 4, True)])
def test_shifted_cross_entropy_nothing_supervised(dtype, V, B, L, ignore_all):
    """L = 1 (the only position is the last one) and an all-ignored batch: loss exactly 0, gradient exactly 0."""
    _run_ce(f"ce_none[{str(dtype)[6:]}-{V}-{B}x{L}]", dtype, V, B, L, ignore_all=ignore_all)


@gpu
@pytest.mark.parametrize("dtype,V,B,L,ignore_all", [
    (F32, 1000, 3, 37, False), (BF16, 50432, 3, 37, False),                 # the earlier cases
    (F32, 16000, 3, 37, False),                                             # ~3 grid-stride passes of the scale
    (F32, 64, 2, 4, True),                                                  # nothing supervised
])
def test_shifted_cross_entropy_autograd(dtype, V, B, L, ignore_all):
    """losses.shifted_cross_entropy, the autograd function the LM heads call: forward, then (loss * c).backward() with
    c != 1, so the backward's otb_scale_by_scalar multiplies every dlogit by c (bf16 [3, 37, 50432]: ~10 grid-stride
    passes of its 132 * 16 blocks).  x.grad is compared with c times the float64 gradient.  The scale rounds the output
    a second time, so the bf16 relative term doubles to 2 A_OUT (two roundings, each < 2^-8)."""
    from otter_b200 import losses
    c = 0.37
    logits, labels = _ce_inputs(dtype, V, B, L, ignore_all=ignore_all)
    x = logits.view(B, L, V).to(DEV).requires_grad_(True)
    lab = labels.to(DEV)
    loss = losses.shifted_cross_entropy(x, lab)
    (loss * c).backward()
    torch.cuda.synchronize()
    r = ce_ref(logits.to(DEV), lab)
    tag = f"ce_autograd[{str(dtype)[6:]}-{V}-{B}x{L}]"
    _check_sum(f"{tag} loss", loss.detach(), r["loss"], r["abs_loss"])
    _check(f"{tag} grad", x.grad.view(B * L, V), c * r["d"], 2 * A_OUT[dtype], 0.0,
           c * _ce_extra(r, dtype, V * x.element_size() <= 200 * 1024), out=dtype)
    assert (x.grad.view(B * L, V)[r["ign"]] == 0).all(), f"{tag}: ignored rows must have an exactly zero gradient"
    if ignore_all:
        assert loss.item() == 0.0


def test_cross_entropy_reference_matches_the_oracle():
    """ce_ref (float64) against oracle.restatement.shifted_cross_entropy (F.cross_entropy on rolled labels) and its
    autograd gradient, in fp32."""
    from oracle import restatement as R
    logits, labels = _ce_inputs(F32, 300, 3, 37)
    xr = logits.view(3, 37, 300).clone().requires_grad_(True)
    want = R.shifted_cross_entropy(xr, labels.clone())
    want.backward()
    r = ce_ref(logits, labels)
    assert abs(r["loss"].item() - want.item()) <= 1e-5 * abs(want.item())
    assert torch.allclose(r["d"], xr.grad.view(-1, 300).double(), rtol=1e-4, atol=1e-8)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the small reductions next to them
# ------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [1, 8, 13, 8 * 592 * 256 + 8])
def test_gate_grad(n):
    """otb_gate_grad: 592 blocks grid-stride over 16 B vectors (two passes for the largest n), block 0 adds the
    scalar tail; then accumulate onto the result."""
    from otter_b200 import functional as F
    g = torch.Generator().manual_seed(n % 1000)
    dy, a = _rnd(g, n).to(DEV), _rnd(g, n).to(DEV)
    gate = torch.tensor([0.3], device=DEV)
    th = 1 - math.tanh(0.3) ** 2
    prod = dy.double() * a.double()
    want, absum = th * prod.sum(), th * prod.abs().sum()
    dg = F.gate_grad(dy, a, gate)
    _check_sum(f"gate_grad[{n}]", dg[0], want, absum)
    dg2 = F.gate_grad(dy, a, gate, dgate=dg.clone(), accumulate=True)
    _check_sum(f"gate_grad[{n}] accumulate", dg2[0], 2 * want, 2 * absum)


@gpu
@pytest.mark.parametrize("n", [8, 8 * 592 * 256 + 8])
def test_sqmean_loss(n):
    from otter_b200 import functional as F
    x = _rnd(torch.Generator().manual_seed(n % 1000), n).to(DEV)
    loss, dx = F.sqmean_loss(x)
    x64 = x.double()
    _check_sum(f"sqmean[{n}] loss", loss[0], x64.pow(2).mean(), x64.pow(2).mean())
    _check(f"sqmean[{n}] dx", dx, 2 * x64 / n, A_REL, 0.0)


@gpu
@pytest.mark.parametrize("rows,D,div,mod", [(5 * 64, 1024, 1, 64), (96, 128, 16, 3), (101, 200, 3, 4), (7, 62, 2, 5)])
def test_grouped_colsum(rows, D, div, mod):
    """out[g] (+)= sum of rows r with (r // div) % mod == g; x is a column slice of a wider buffer."""
    from otter_b200 import functional as F
    g = torch.Generator().manual_seed(rows + D)
    big = _rnd(g, rows, D + 40).to(DEV)
    x = big[:, 24:24 + D]
    grp = (torch.arange(rows, device=DEV) // div) % mod
    x64 = x.double()
    want = torch.zeros(mod, D, dtype=F64, device=DEV).index_add_(0, grp, x64)
    absum = torch.zeros(mod, D, dtype=F64, device=DEV).index_add_(0, grp, x64.abs())
    out = F.grouped_colsum(x, div, mod)
    _check_sum(f"colsum[{rows}-{D}-{div}-{mod}]", out, want, absum)
    old = torch.randn(mod, D, generator=g).to(DEV)
    out2 = F.grouped_colsum(x, div, mod, out=old.clone(), accumulate=True)
    _check_sum(f"colsum[{rows}-{D}-{div}-{mod}] accumulate", out2, want + old.double(), absum + old.double().abs())


# ------------------------------------------------------------------------------------------------------------------
# GPU: the earlier LLaMA kernel test, now through the metric above
# ------------------------------------------------------------------------------------------------------------------
@gpu
def test_rmsnorm_rope_swiglu_kernels():
    _run_rms("llama rms", 75, 512, add=True)
    _run_rope("llama rope", 3, 25, 2, 2, 10000.0)
    _run_swiglu("llama swiglu", 75, 384)
