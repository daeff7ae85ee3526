"""Attention kernels against a float64 reference at the boundaries of their tile structure.

Kernels under test (all bf16 in, fp32 softmax, bf16 out):
  otb_attn_fwd / otb_attn_bwd     head dim 64: 128-key forward tiles (one pass when there is a single key tile),
                                  128-key backward tiles walked in 64-key halves, an fp32 dQ workspace when there is more
                                  than one key tile; one or two key sources, eq / ge media masks, causal
  otb_lm_attn_fwd / _bwd          head dim 128: causal and / or ALiBi; 128-key forward tiles, 64-key backward tiles,
                                  dQ workspace once a query row sees more than one backward key tile
  otb_xattn_out_fused             media-masked attention (<= 64 keys, <= 8 heads) + output projection + tanh gate
                                  + residual in one kernel

Reference: plain float64 attention on the device, from the same bf16-rounded inputs, gradients from autograd, one head
at a time.  Every floating-point output goes through one metric (`_ratio`); the tests without the `gpu` mark show, on
the CPU, that the metric rejects float64 references mutated the way a kernel bug would mutate them.

Outputs are pre-filled with NaN wherever the test owns the buffer, so an owned element a kernel never writes fails the
comparison.  The canary tests call the C ABI directly with padded, offset buffers and check that a kernel writes every
element it owns and nothing else.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

BF16 = torch.bfloat16
gpu = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------------------------
# The metric.
#
# For each slice s (one head's 64 / 128 values of one query row for O and dQ, of one key row for dK and dV, of one
# output row for the fused kernel's y and aux):     |got - ref| <= A_REL * |ref| + B_RMS * rms(ref_s) + FLOOR
#
# Where the kernels round (the reference does not).  bf16 has 8 significant bits, so rounding to nearest has a relative
# error below 2^-8 (half of the spacing 2^-7 at 1.0):
#   - every output element is rounded to bf16 once: error < 2^-8 |ref|.  A_REL = 2^-7 leaves a factor 2, so output
#     rounding alone can use up to 0.5 of the bound on an element that is large within its slice;
#   - P (forward and backward) and dS are rounded to bf16 before their MMAs.  Each term of a sum over keys (O, dQ) or
#     query rows (dK, dV) then carries an independent relative error < 2^-8 (rms 2^-8 / sqrt(3)).  For sums of terms
#     of random sign the result is of the size of sqrt(sum of squared terms), so the error has a standard deviation of
#     ~2^-8 / sqrt(3) = 0.0023 of the slice's rms; B_RMS = 2^-6 is about 7 standard deviations.  The largest of the
#     10^5 - 10^7 elements of a case lies 4-5 standard deviations out, so this term too can use most of its share;
#   - inputs are bf16 for both sides, and the fp32 accumulations (<= 2112 terms) and ex2.approx are below 2^-20 relative;
#   - the backward's delta = rowsum(dO . O) is taken from the bf16 O it is given, and so is the reference's
#     (ref_attention, o_given): that rounding belongs to the forward, whose O is checked on its own.
# Measured on an H100, the largest error / bound per case family and tensor is 0.30 - 0.72 (0.27 - 0.33 for the exact
# answer rounded to bf16): the bound is about 1.4x the worst element, while each of the mutations in the power checks below exceeds it (dK x 1.02, the smallest, by 1.7x).  Every
# RATIO line also prints the same ratio for the exact answer rounded to bf16, the part no bf16-output kernel can avoid.
# FLOOR covers one case where the exact answer is 0 but fp32 is not: with a single visible key dS = P (dP - delta) is
# exactly 0, while the kernel's dP (MMA) and delta (row sum) differ by fp32 rounding, ~2^-21 for unit-scale inputs.
# Rows that must be exactly zero (text_time == 0 under the eq mask) are asserted exactly, not through the metric.
#
# lse (natural log, 0 for zeroed and uniform rows):  |got - ref| <= 1e-4 * (1 + |ref|).
# ------------------------------------------------------------------------------------------------------------------
A_REL = 2.0 ** -7
B_RMS = 2.0 ** -6
FLOOR = 2.0 ** -16
LSE_TOL = 1e-4


def _ratio(got, ref):
    """max over elements of |got - ref| / bound; <= 1 passes.  Slices are the last dimension.  NaN in got -> NaN."""
    got, ref = got.double(), ref.double()
    rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    bound = A_REL * ref.abs() + B_RMS * rms + FLOOR
    return ((got - ref).abs() / bound).max().item()


def _lse_ratio(got, ref):
    got, ref = got.double(), ref.double()
    return ((got - ref).abs() / (LSE_TOL * (1.0 + ref.abs()))).max().item()


def _check(what, got, ref, lse=False):
    r = _lse_ratio(got, ref) if lse else _ratio(got, ref)
    print(f"RATIO {what} {r:.4f}" + ("" if lse else f" (exact answer rounded to bf16: {_ratio(ref.to(BF16), ref):.4f})"))
    if not r <= 1.0 and not lse:              # where it fails: index of the worst element, its slice's rms
        got, ref = got.double(), ref.double()
        rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
        q = (got - ref).abs() / (A_REL * ref.abs() + B_RMS * rms + FLOOR)
        i = np.unravel_index(int(torch.nan_to_num(q, nan=math.inf).argmax()), tuple(q.shape))
        bad = (q > 1).nonzero()[:, -2].unique() if q.dim() > 1 else None
        print(f"WORST {what} at {i}: got {got[i].item():.6g} ref {ref[i].item():.6g} slice rms "
              f"{rms[i[:-1]].item():.4g}; slices over the bound: {bad.numel()} (first {bad[:12].tolist()})")
    assert r <= 1.0, f"{what}: error / bound = {r:.3f}"


# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------
def _mask64(P, Sq, Sk, device, tt=None, n=0, ge=False, causal=False):
    """-> (allowed [P,Sq,Sk], zero [P,Sq,1]) with the kernels' mask semantics (csrc/otb_attn_common.cuh row_class):
    eq: key j (media slot j // n + 1) is visible iff slot == tt; tt == 0 rows are zeroed after the softmax.
    ge: visible iff slot <= tt; tt == 0 rows see no key and are uniform, not zeroed.
    A row that sees no key and is not zeroed is uniform over all keys (the reference's -FLT_MAX fill)."""
    allowed = torch.ones(P, Sq, Sk, dtype=torch.bool, device=device)
    zero = torch.zeros(P, Sq, 1, dtype=torch.bool, device=device)
    if tt is not None:
        slot = torch.arange(Sk, device=device) // n + 1
        t = tt.to(device).long().view(P, Sq, 1)
        allowed = (slot <= t) if ge else (slot == t)
        if not ge:
            zero = t == 0
    if causal:
        allowed = allowed & (torch.arange(Sk, device=device)[None, None, :] <= torch.arange(Sq, device=device)[None, :, None])
    return allowed, zero


def ref_attention(q, k, v, scale, allowed, zero=None, bias=None, dout=None, o_given=None):
    """One head, float64.  q [P,Sq,d], k / v [P,Sk,d], allowed [P,Sq,Sk], zero [P,Sq,1] or None, bias [Sk] or None
    (added to the scaled scores).  -> dict o, lse (0 for zeroed and uniform rows), p, and dq, dk, dv if dout is given.

    o_given: the bf16 forward output a backward kernel is handed.  The backward kernels take O as an input and form
    delta = rowsum(dO . O) from it, so dS = P (dP - delta) is defined by that O.  Where attention sits on a few keys,
    dS nearly cancels while the (< 2^-8) rounding of O moves delta by up to ~2^-8 |dP|: a test that ignored this would
    measure the forward's rounding, not the backward.  Autograd's gradients are corrected to that delta exactly:
    dS += P * (delta_exact - delta_given)."""
    q, k, v = (t.detach().double().requires_grad_(dout is not None) for t in (q, k, v))
    s = scale * (q @ k.transpose(-1, -2))
    if bias is not None:
        s = s + bias.double()
    if zero is None:
        zero = torch.zeros_like(allowed[..., :1])
    flat = zero | ~allowed.any(-1, keepdim=True)               # zeroed or uniform: constant scores, no gradient
    s = torch.where(flat, torch.zeros_like(s), s.masked_fill(~allowed, -math.inf))
    p = torch.softmax(s, -1).masked_fill(zero, 0.0)
    o = p @ v
    lse = torch.logsumexp(s, -1).masked_fill(flat[..., 0], 0.0)
    r = {"o": o.detach(), "lse": lse.detach(), "p": p.detach()}
    if dout is not None:
        r["dq"], r["dk"], r["dv"] = torch.autograd.grad(o, (q, k, v), dout.double())
        if o_given is not None:
            dd = (dout.double() * (r["o"] - o_given.double())).sum(-1, keepdim=True).masked_fill(flat, 0.0).detach()
            r["dq"] = r["dq"] + scale * dd * (r["p"] @ k.detach())
            r["dk"] = r["dk"] + scale * (r["p"] * dd).transpose(-1, -2) @ q.detach()
    return r


def _heads(t, P, S, col0, H, d):
    """[P*S, cols] -> [P, H, S, d] view of the heads at columns col0 + h*d."""
    return t[:, col0:col0 + H * d].reshape(P, S, H, d).permute(0, 2, 1, 3)


def _stack(refs, key):
    return torch.stack([r[key] for r in refs], 1)               # per-head [P, S, d] -> [P, H, S, d]


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(BF16)


def _media_tt(P, Sq, T):
    """text_time [P, Sq] covering 0 .. T + 1 in every problem: every row class of both masks."""
    r = torch.arange(P * Sq).view(P, Sq)
    return ((r * 7 + 3 + r // Sq) % (T + 2)).to(torch.int32)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the metric rejects plausible kernel bugs.  Each mutation below is applied to the float64 reference.
# ------------------------------------------------------------------------------------------------------------------
def _mutant_ratio(got, ref, lse=False):
    r = _lse_ratio(got, ref) if lse else _ratio(got, ref)
    print(f"MUTANT ratio {r:.3f}")
    return r


def _inputs64(P, H, Sq, Sk, seed):
    g = torch.Generator().manual_seed(seed)
    return [_rnd(g, P, H, S, 64).double() for S in (Sq, Sk, Sk, Sq)]       # q, k, v, dout


def _mutant64(P, H, Sq, Sk, mutate, tt=None, n=0, causal=False, seed=0):
    """(ref, mutant) over all heads; `mutate(allowed)` edits the mask of the mutant."""
    q, k, v, do = _inputs64(P, H, Sq, Sk, seed)
    refs, muts = [], []
    for h in range(H):
        allowed, zero = _mask64(P, Sq, Sk, "cpu", tt, n, False, causal)
        refs.append(ref_attention(q[:, h], k[:, h], v[:, h], 0.125, allowed, zero, dout=do[:, h]))
        allowed = allowed.clone()
        mutate(allowed)
        muts.append(ref_attention(q[:, h], k[:, h], v[:, h], 0.125, allowed, zero, dout=do[:, h]))
    return refs, muts


def _drop_keys(keys):
    def f(allowed):
        allowed[..., keys] = False
    return f


def test_metric_rejects_one_dropped_key_of_2112():
    # the old test_attention_fwd_bwd_unmasked[2-2-64-2048-64] passed this mutation
    refs, muts = _mutant64(2, 2, 64, 2112, _drop_keys([2047]))
    assert _mutant_ratio(_stack(muts, "o"), _stack(refs, "o")) > 1.0


@pytest.mark.parametrize("Sk", [65, 129])
def test_metric_rejects_dropped_last_key_of_a_ragged_tile(Sk):
    refs, muts = _mutant64(1, 2, 128, Sk, _drop_keys([Sk - 1]))
    assert _mutant_ratio(_stack(muts, "o"), _stack(refs, "o")) > 1.0


def _diag_plus_one(rows):
    def f(allowed):
        for i in rows:
            if i + 1 < allowed.shape[-1]:
                allowed[:, i, i + 1] = True
    return f


def test_metric_rejects_causal_diagonal_off_by_one_head64():
    refs, muts = _mutant64(2, 2, 257, 257, _diag_plus_one(range(128, 256)), causal=True)
    assert _mutant_ratio(_stack(muts, "o"), _stack(refs, "o")) > 1.0


def _lm_inputs(B, S, H, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = _rnd(g, B * S, 3 * H * 128, scale=0.8).double()
    dout = _rnd(g, B * S, H * 128, scale=0.5).double()
    return qkv, dout


def _lm_ref(qkv, dout, B, S, H, slopes, causal, scale, mutate=None):
    D = H * 128
    out = []
    for h in range(H):
        q, k, v = (qkv[:, c * D + h * 128:c * D + (h + 1) * 128].reshape(B, S, 128) for c in range(3))
        allowed, _ = _mask64(B, S, S, qkv.device, causal=causal)
        if mutate is not None:
            allowed = allowed.clone()
            mutate(allowed)
        bias = None if slopes is None else slopes[h].double() * (torch.arange(S, device=qkv.device) - (S - 1)).double()
        out.append(ref_attention(q, k, v, scale, allowed, bias=bias, dout=dout[:, h * 128:(h + 1) * 128].reshape(B, S, 128)))
    return out


@pytest.mark.parametrize("alibi", [True, False])
def test_metric_rejects_causal_diagonal_off_by_one_lm(alibi):
    # LLaMA (no ALiBi) at S = 384: the old max-abs 3e-2 limit was only just above this mutation
    B, S, H = 1, 384, 2
    qkv, dout = _lm_inputs(B, S, H, 1)
    slopes = 2.0 ** (-8.0 * torch.arange(1, H + 1) / H) if alibi else None      # MPT's slopes for a power-of-two H
    refs = _lm_ref(qkv, dout, B, S, H, slopes, True, 128 ** -0.5)
    muts = _lm_ref(qkv, dout, B, S, H, slopes, True, 128 ** -0.5, _diag_plus_one(range(128, 256)))
    assert _mutant_ratio(_stack(muts, "o"), _stack(refs, "o")) > 1.0


@pytest.mark.parametrize("shift", ["slot", "key"])
def test_metric_rejects_media_slot_off_by_one_for_one_row(shift):
    """One text row (tt = 2, T = 3, n = 64: slot 2 = keys 64..127) attends the wrong keys: the next slot, or the slot
    window moved by one key."""
    P, H, Sq, T, n = 1, 2, 130, 3, 64
    tt = _media_tt(P, Sq, T)
    row = int((tt[0] == 2).nonzero()[0])

    def f(allowed):
        allowed[0, row] = False
        lo = (3 if shift == "slot" else 2) * n - n + (0 if shift == "slot" else 1)
        allowed[0, row, lo:lo + n] = True
    refs, muts = _mutant64(P, H, Sq, T * n, f, tt=tt, n=n)
    assert _mutant_ratio(_stack(muts, "o"), _stack(refs, "o")) > 1.0


@pytest.mark.parametrize("case", ["head64", "lm"])
def test_metric_rejects_dk_scaled_by_1_02(case):
    # the old LM test normalised by the global max of the gradient and passed this (LM case: its S = 200 shape)
    if case == "head64":
        q, k, v, do = _inputs64(2, 2, 200, 200, 3)
        refs = [ref_attention(q[:, h], k[:, h], v[:, h], 0.125, *_mask64(2, 200, 200, "cpu", causal=True),
                              dout=do[:, h]) for h in range(2)]
    else:
        qkv, dout = _lm_inputs(2, 200, 2, 3)
        refs = _lm_ref(qkv, dout, 2, 200, 2, 2.0 ** (-8.0 * torch.arange(1, 3) / 2), True, 128 ** -0.5)
    dk = _stack(refs, "dk")
    assert _mutant_ratio(dk * 1.02, dk) > 1.0


@pytest.mark.parametrize("case", ["head64", "lm"])
def test_metric_rejects_dq_missing_one_key_tile(case):
    """dQ without one key tile's dS K, as if the workspace add had been skipped: the last 128-key tile of source 1 in
    the 2048 + 64 key case (head 64), the 64-key backward tile 128..191 of the LM at S = 200."""
    if case == "head64":
        q, k, v, do = _inputs64(2, 2, 64, 2112, 0)
        scale, tile = 0.125, slice(1920, 2048)
        allowed = torch.ones(2, 64, 2112, dtype=torch.bool)
    else:
        qkv, do = _lm_inputs(1, 200, 2, 2)
        q, k, v = (qkv[:, c * 256:(c + 1) * 256].reshape(1, 200, 2, 128).permute(0, 2, 1, 3) for c in range(3))
        do = do.reshape(1, 200, 2, 128).permute(0, 2, 1, 3)
        scale, tile = 128 ** -0.5, slice(128, 192)
        allowed = _mask64(1, 200, 200, "cpu", causal=True)[0]
    got, want = [], []
    for h in range(q.shape[1]):
        r = ref_attention(q[:, h], k[:, h], v[:, h], scale, allowed, dout=do[:, h])
        ds = r["p"] * ((do[:, h] @ v[:, h].transpose(-1, -2)) - (do[:, h] * r["o"]).sum(-1, keepdim=True)) * scale
        got.append(r["dq"] - ds[..., tile] @ k[:, h, tile])
        want.append(r["dq"])
    assert _mutant_ratio(torch.stack(got, 1), torch.stack(want, 1)) > 1.0


@pytest.mark.parametrize("case", ["Sk129", "media", "lm_causal"])
def test_metric_rejects_lse_shifted(case):
    """lse + log(1 + 1/n), n = the number of keys the row sees: as if one more key of average weight had been counted."""
    if case == "Sk129":
        q, k, v, _ = _inputs64(1, 2, 128, 129, 4)
        allowed, zero = _mask64(1, 128, 129, "cpu")
    elif case == "media":
        q, k, v, _ = _inputs64(2, 2, 130, 192, 5)
        allowed, zero = _mask64(2, 130, 192, "cpu", _media_tt(2, 130, 3), 64)
    else:
        q, k, v, _ = _inputs64(1, 2, 192, 192, 6)
        allowed, zero = _mask64(1, 192, 192, "cpu", causal=True)
    lse = torch.stack([ref_attention(q[:, h], k[:, h], v[:, h], 0.125, allowed, zero)["lse"] for h in range(2)], 1)
    nvis = allowed.sum(-1).double()[:, None]
    normal = (nvis > 0) & ~zero[..., 0][:, None]
    shifted = torch.where(normal, lse + torch.log1p(1.0 / nvis.clamp_min(1)), lse)
    assert _mutant_ratio(shifted, lse, lse=True) > 1.0


def test_reference_backward_with_given_o():
    """ref_attention's o_given correction equals the backward written out: dS = P (dO V^T - rowsum(dO . O_given))."""
    q, k, v, do = (t[:, 0] for t in _inputs64(1, 1, 70, 90, 8))
    allowed, zero = _mask64(1, 70, 90, "cpu", _media_tt(1, 70, 3), 30)
    o_given = ref_attention(q, k, v, 0.125, allowed, zero)["o"].to(BF16)
    r = ref_attention(q, k, v, 0.125, allowed, zero, dout=do, o_given=o_given)
    normal = ~(zero | ~allowed.any(-1, keepdim=True))
    ds = r["p"] * (do @ v.transpose(-1, -2) - (do * o_given.double()).sum(-1, keepdim=True)) * normal
    assert torch.allclose(r["dq"], 0.125 * ds @ k, rtol=1e-10, atol=1e-12)
    assert torch.allclose(r["dk"], 0.125 * ds.transpose(-1, -2) @ q, rtol=1e-10, atol=1e-12)
    assert torch.allclose(r["dv"], r["p"].transpose(-1, -2) @ do, rtol=1e-10, atol=1e-12)


def test_metric_accepts_bf16_output_rounding():
    """The other side: rounding the exact answer to bf16 (what every kernel does last) stays below 0.5 of the bound,
    the cap derived at the constants (error < 2^-8 |ref| against A_REL |ref| = 2^-7 |ref|)."""
    q, k, v, do = _inputs64(2, 2, 129, 257, 7)
    refs = [ref_attention(q[:, h], k[:, h], v[:, h], 0.125, *_mask64(2, 129, 257, "cpu"), dout=do[:, h]) for h in range(2)]
    for key in ("o", "dq", "dk", "dv"):
        t = _stack(refs, key)
        assert _mutant_ratio(t.to(BF16), t) < 0.5


# ------------------------------------------------------------------------------------------------------------------
# GPU: otb_attn_fwd / otb_attn_bwd (head dim 64)
# ------------------------------------------------------------------------------------------------------------------
DEV = "cuda:0"


def _nan(rows, cols, dtype=BF16):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device=DEV)


def _run_attn64(tag, P, H, Sq, Sk1, Sk2=0, *, tt=None, n=0, T=0, ge=False, causal=False, scale=0.125, seed=0):
    """Forward + backward of one head-64 problem through otter_b200.functional, every output compared with the
    float64 reference.  Outputs the test allocates are NaN-filled first."""
    from otter_b200 import functional as F
    g = torch.Generator().manual_seed(seed * 1000 + P * 131 + H * 17 + Sq * 7 + Sk1 * 3 + Sk2)
    inner = H * 64
    if causal:                                    # q | k | v in one buffer (the Persimmon / CLIP-style qkv layout)
        qkv = _rnd(g, P * Sq, 3 * inner).to(DEV)
        q, q0, kv1, k0, v0 = qkv, 0, qkv, inner, 2 * inner
    else:
        q, q0 = _rnd(g, P * Sq, inner).to(DEV), 0
        kv1, k0, v0 = _rnd(g, P * Sk1, 2 * inner).to(DEV), 0, inner
    kv2 = _rnd(g, P * Sk2, 2 * inner).to(DEV) if Sk2 else None
    dout = _rnd(g, P * Sq, inner).to(DEV)
    ttd = tt.to(DEV).contiguous() if tt is not None else None
    spec = F.AttnSpec(q, q0, kv1, k0, v0, P, H, Sq, Sk1, scale, kv2=kv2, k2_col0=0, v2_col0=inner, Sk2=Sk2,
                      text_time=ttd, n_per_media=n, T_img=T, mask_ge=ge, causal=causal)
    out, lse = F.attn_fwd(spec, out=_nan(P * Sq, inner))
    dq = _nan(P * Sq, q.shape[1])
    dkv1 = dq if causal else _nan(P * Sk1, 2 * inner)
    dkv2 = _nan(P * Sk2, 2 * inner) if Sk2 else None
    F.attn_bwd(spec, out, 0, lse, dout, 0, dq, q0, dkv1, k0, v0, dkv2, 0, inner)
    torch.cuda.synchronize()

    Sk = Sk1 + Sk2
    allowed, zero = _mask64(P, Sq, Sk, DEV, ttd, n, ge, causal)
    hq, hdo = _heads(q, P, Sq, q0, H, 64), _heads(dout, P, Sq, 0, H, 64)
    hk, hv = _heads(kv1, P, Sk1, k0, H, 64), _heads(kv1, P, Sk1, v0, H, 64)
    if Sk2:
        hk = torch.cat([hk, _heads(kv2, P, Sk2, 0, H, 64)], 2)
        hv = torch.cat([hv, _heads(kv2, P, Sk2, inner, H, 64)], 2)
    ho = _heads(out, P, Sq, 0, H, 64)
    refs = [ref_attention(hq[:, h], hk[:, h], hv[:, h], scale, allowed, zero, dout=hdo[:, h], o_given=ho[:, h])
            for h in range(H)]
    _check(f"{tag} O", ho, _stack(refs, "o"))
    _check(f"{tag} lse", lse, _stack(refs, "lse"), lse=True)
    _check(f"{tag} dQ", _heads(dq, P, Sq, q0, H, 64), _stack(refs, "dq"))
    dk, dv = _stack(refs, "dk"), _stack(refs, "dv")
    _check(f"{tag} dK", _heads(dkv1, P, Sk1, k0, H, 64), dk[:, :, :Sk1])
    _check(f"{tag} dV", _heads(dkv1, P, Sk1, v0, H, 64), dv[:, :, :Sk1])
    if Sk2:
        _check(f"{tag} dK2", _heads(dkv2, P, Sk2, 0, H, 64), dk[:, :, Sk1:])
        _check(f"{tag} dV2", _heads(dkv2, P, Sk2, inner, H, 64), dv[:, :, Sk1:])
    if zero.any():                                # eq mask, text_time == 0: exactly zero output and dQ
        rows = zero.view(-1)
        assert out[rows].abs().max().item() == 0.0
        assert _heads(dq, P, Sq, q0, H, 64).permute(0, 2, 1, 3).reshape(P * Sq, -1)[rows].abs().max().item() == 0.0
        assert (_stack(refs, "lse").permute(0, 2, 1)[zero[..., 0]] == 0).all() and (lse.permute(0, 2, 1)[zero[..., 0]] == 0).all()


@gpu
@pytest.mark.parametrize("P,H,Sq,Sk1,Sk2", [
    # the earlier cases: perceiver (Sk2 = 64 latents), CLIP, c3 video (2048 + 64 keys), gated x-attn with n = 64,
    # and enough (problem, head) pairs to fill the GPU several times over
    (2, 8, 64, 256, 64), (1, 2, 64, 96, 64), (3, 4, 257, 257, 0), (2, 2, 64, 2048, 64), (2, 8, 300, 64, 0),
    (8, 16, 257, 257, 0), (16, 8, 300, 64, 0), (15, 8, 700, 130, 64),
    # Sq at 1 and around one 128-row query tile x Sk1 around the 64-key backward halves and the 128-key tiles
    # (Sk1 <= 128: one key tile, single-pass forward, no dQ workspace)
    (1, 2, 1, 1, 0), (3, 2, 127, 63, 0), (1, 2, 128, 64, 0), (3, 2, 129, 65, 0), (1, 2, 1, 127, 0),
    (3, 2, 128, 128, 0), (1, 2, 129, 129, 0), (3, 2, 127, 255, 0), (1, 2, 128, 257, 0), (3, 2, 1, 257, 0),
    (1, 2, 129, 1, 0),
    # two key sources: ragged first source, second source of 1 / 64 / 129 keys
    (2, 2, 129, 65, 1), (2, 2, 127, 257, 64), (1, 3, 128, 129, 129),
    # perceiver: 64 latent queries over 257 vision keys + 64 latents
    (2, 8, 64, 257, 64),
])
def test_attention_fwd_bwd_unmasked(P, H, Sq, Sk1, Sk2):
    _run_attn64(f"unmasked[{P}-{H}-{Sq}-{Sk1}-{Sk2}]", P, H, Sq, Sk1, Sk2)


@gpu
@pytest.mark.parametrize("P,H,S", [
    (2, 4, 100), (1, 2, 300), (2, 3, 520),                  # earlier cases: 1, 3 and 5 key tiles
    (2, 2, 1), (2, 2, 64), (2, 2, 65), (2, 2, 128), (2, 2, 129), (2, 2, 257),
    (2, 16, 257),                                           # CLIP-L shape with a causal mask
    (1, 64, 300),                                           # Persimmon: 64 heads
])
def test_causal_attention_fwd_bwd(P, H, S):
    _run_attn64(f"causal[{P}-{H}-{S}]", P, H, S, S, causal=True)


@gpu
@pytest.mark.parametrize("ge,T,n,P,Sq", [
    (False, 1, 64, 2, 130), (False, 2, 32, 2, 129), (False, 3, 64, 2, 130), (False, 5, 32, 1, 257),
    (False, 5, 64, 1, 200),                       # 320 keys: slot 2 straddles the 128-key tile boundary
    (True, 1, 32, 2, 64), (True, 2, 64, 2, 129), (True, 3, 64, 2, 130), (True, 5, 32, 1, 257),
])
def test_attention_media_mask_classes(ge, T, n, P, Sq):
    """text_time covering 0 .. T + 1, so every row class of the mask (zeroed / one slot or a prefix of slots / uniform)
    appears; with T * n > 128 the slots and the uniform rows span more than one key tile."""
    _run_attn64(f"mask[{'ge' if ge else 'eq'}-T{T}-n{n}-{P}-{Sq}]", P, 2, Sq, T * n, tt=_media_tt(P, Sq, T), n=n, T=T,
                ge=ge)


@gpu
def test_attention_c2_gated_xattn_shape():
    """c2 gated cross-attention: 8 samples x 256 text rows x 8 heads over 64 media latents, <image> at position 3."""
    from otter_b200 import functional as F
    loc = torch.zeros(8, 256, dtype=torch.bool)
    loc[:, 3] = True
    tt = F.text_time(loc.to(DEV), True).cpu()
    _run_attn64("c2", 8, 8, 256, 64, tt=tt, n=64, T=1)


@gpu
@pytest.mark.parametrize("T,L,pos,attend_previous", [
    (1, 256, [[0], [5]], True),
    (2, 160, [[0, 40], [3, 90]], True),
    (1, 64, [[0, 8, 16], [2, 9]], True),          # more <image> tokens than media -> uniform rows
    (3, 300, [[0, 100, 200], [10, 20, 290]], False),
    (2, 40, [[], [7]], True),                      # a sample without any <image>
])
def test_attention_media_mask(T, L, pos, attend_previous):
    from oracle.restatement import text_time_np
    from otter_b200 import functional as F
    P, n = 2, 64
    loc = np.zeros((P, L), dtype=bool)
    for b, ps in enumerate(pos):
        loc[b, ps] = True
    tt = F.text_time(torch.from_numpy(loc).to(DEV), attend_previous)
    assert np.array_equal(tt.cpu().numpy().astype(np.int64), text_time_np(loc, attend_previous))
    _run_attn64(f"media[{T}-{L}]", P, 8, L, T * n, tt=tt.cpu(), n=n, T=T)


# ------------------------------------------------------------------------------------------------------------------
# GPU: otb_lm_attn_fwd / otb_lm_attn_bwd (head dim 128)
# ------------------------------------------------------------------------------------------------------------------
def _run_lm(tag, B, S, H, alibi, causal, scale=None):
    from otter_b200 import functional as F
    from otter_b200.lm_mpt import alibi_slopes
    qkv, dout = _lm_inputs(B, S, H, S * 10 + H + B)
    qkv, dout = qkv.to(BF16).to(DEV), dout.to(BF16).to(DEV)
    slopes = alibi_slopes(H, device=DEV) if alibi else None
    sc = 128 ** -0.5 if scale is None else scale
    out, lse = F.lm_attn_fwd(qkv, B, S, H, slopes=slopes, causal=causal, scale=scale)
    dqkv = F.lm_attn_bwd(dout, qkv, out, lse, B, S, H, slopes=slopes, causal=causal, scale=scale)
    torch.cuda.synchronize()
    D = H * 128
    hdo, ho = _heads(dout, B, S, 0, H, 128), _heads(out, B, S, 0, H, 128)
    pos = (torch.arange(S, device=DEV) - (S - 1)).double()
    allowed, _ = _mask64(B, S, S, DEV, causal=causal)
    refs = []
    for h in range(H):                            # one head at a time: S = 2048 x 32 heads stays small
        q, k, v = (_heads(qkv, B, S, c * D, H, 128)[:, h] for c in range(3))
        bias = slopes[h].double() * pos if alibi else None
        refs.append(ref_attention(q, k, v, sc, allowed, bias=bias, dout=hdo[:, h], o_given=ho[:, h]))
    _check(f"{tag} O", _heads(out, B, S, 0, H, 128), _stack(refs, "o"))
    _check(f"{tag} lse", lse, _stack(refs, "lse"), lse=True)
    for c, key in enumerate(("dq", "dk", "dv")):
        _check(f"{tag} {key}", _heads(dqkv, B, S, c * D, H, 128), _stack(refs, key))


@gpu
@pytest.mark.parametrize("B,S,H,alibi,causal,scale", [
    # earlier cases
    (2, 200, 2, True, True, None), (1, 256, 3, True, True, None), (1, 77, 1, False, True, None),
    (1, 384, 2, True, True, None), (2, 130, 1, True, False, None),
    # S around the 64-key backward tiles and the 128-key forward tiles; S <= 64 runs without the dQ workspace
    (1, 1, 2, True, True, None), (2, 2, 2, False, False, None), (1, 63, 2, True, False, None),
    (2, 64, 2, False, True, None), (1, 65, 2, True, True, 0.05), (2, 127, 2, False, False, None),
    (1, 128, 2, True, False, None), (2, 129, 2, False, True, None), (1, 191, 2, True, True, None),
    (2, 192, 2, False, False, 0.1), (1, 193, 2, False, True, None), (2, 320, 3, True, False, None),
])
def test_lm_attention_fwd_bwd(B, S, H, alibi, causal, scale):
    _run_lm(f"lm[{B}-{S}-{H}-{alibi}-{causal}-{scale}]", B, S, H, alibi, causal, scale)


@gpu
@pytest.mark.parametrize("model", ["mpt7b", "llama7b"])
def test_lm_attention_7b_shape(model):
    """S = 2048, 32 heads: MPT-7B (ALiBi + causal; the key bias reaches -slope * 2047) and LLaMA-7B (causal only)."""
    _run_lm(model, 1, 2048, 32, model == "mpt7b", True)


# ------------------------------------------------------------------------------------------------------------------
# GPU: otb_xattn_out_fused
# ------------------------------------------------------------------------------------------------------------------
GATE = 0.6


def _fused_ref(q, kv, wo, x, P, H, Sq, T, n, tt, ge):
    inner = H * 64
    allowed, zero = _mask64(P, Sq, T * n, q.device, tt, n, ge)
    refs = [ref_attention(_heads(q, P, Sq, 0, H, 64)[:, h], _heads(kv, P, T * n, 0, H, 64)[:, h],
                          _heads(kv, P, T * n, inner, H, 64)[:, h], 0.125, allowed, zero) for h in range(H)]
    o = _stack(refs, "o")
    a = o.permute(0, 2, 1, 3).reshape(P * Sq, inner) @ wo.double().t()
    return o, _stack(refs, "lse"), a, a * math.tanh(GATE) + x.double(), zero


@gpu
@pytest.mark.parametrize("H,T,n,ge,D,P,Sq", [
    (1, 1, 64, False, 512, 2, 77), (4, 2, 32, True, 4096, 2, 130), (8, 1, 16, False, 512, 3, 129),
    (8, 2, 32, False, 4096, 1, 200), (4, 1, 16, True, 512, 2, 1), (8, 1, 64, True, 1024, 2, 127),
])
def test_xattn_out_fused_vs_reference(H, T, n, ge, D, P, Sq):
    from otter_b200 import functional as F
    g = torch.Generator().manual_seed(H * 100 + D + Sq)
    inner = H * 64
    q = _rnd(g, P * Sq, inner).to(DEV)
    kv = _rnd(g, P * T * n, 2 * inner).to(DEV)
    wo = _rnd(g, D, inner, scale=inner ** -0.5).to(DEV)
    x = _rnd(g, P * Sq, D).to(DEV)
    tt = _media_tt(P, Sq, T)
    spec = F.AttnSpec(q, 0, kv, 0, inner, P, H, Sq, T * n, 0.125, text_time=tt.to(DEV), n_per_media=n, T_img=T,
                      mask_ge=ge)
    y, aux, o, lse = F.xattn_out_fused(spec, wo, torch.tensor([GATE], device=DEV), x)
    torch.cuda.synchronize()
    o_r, lse_r, a_r, y_r, zero = _fused_ref(q, kv, wo, x, P, H, Sq, T, n, tt, ge)
    tag = f"fused[{H}-{T}-{n}-{ge}-{D}-{P}-{Sq}]"
    _check(f"{tag} O", _heads(o, P, Sq, 0, H, 64), o_r)
    _check(f"{tag} lse", lse, lse_r, lse=True)
    _check(f"{tag} aux", aux.view(P * Sq, D // 64, 64), a_r.view(P * Sq, D // 64, 64))
    _check(f"{tag} y", y.view(P * Sq, D // 64, 64), y_r.view(P * Sq, D // 64, 64))
    if zero.any():                                # zeroed rows: O = 0, aux = 0, y = x exactly
        rows = zero.view(-1)
        assert o[rows].abs().max().item() == 0.0 and aux[rows].abs().max().item() == 0.0
        assert torch.equal(y[rows], x[rows])


# ------------------------------------------------------------------------------------------------------------------
# GPU canaries: the C ABI with descriptors built here, padded / offset buffers pre-filled with NaN.  Afterwards every
# element a kernel owns is finite (and matches the reference), every other element still holds the NaN bit pattern.
# Inputs sit in NaN-padded buffers too, so a read outside a tensor map's logical rows / columns would show up as NaN.
# ------------------------------------------------------------------------------------------------------------------
class _Canvas:
    """A NaN-filled [rows, pitch] buffer with owned rectangles."""

    def __init__(self, rows, pitch, dtype=BF16):
        self.t = torch.full((rows, pitch), float("nan"), dtype=dtype, device=DEV)
        self.owned = torch.zeros(rows, pitch, dtype=torch.bool, device=DEV)

    def own(self, r1, c0, c1):
        self.owned[:r1, c0:c1] = True
        return self.t[:r1, c0:c1]

    def put(self, src, c0):
        self.t[:src.shape[0], c0:c0 + src.shape[1]] = src
        return self

    def ptr(self, c0=0):
        return C.c_void_p(self.t.data_ptr() + c0 * self.t.element_size())

    def check(self, what):
        ints = {2: torch.int16, 4: torch.int32}[self.t.element_size()]
        nan = torch.full((1,), float("nan"), dtype=self.t.dtype, device=DEV).view(ints)
        assert torch.isfinite(self.t[self.owned].float()).all(), f"{what}: an owned element was not written"
        assert (self.t.view(ints)[~self.owned] == nan).all(), f"{what}: an element outside the output was written"


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc, what):
    from otter_b200 import _lib
    _lib.check(rc, what)


@gpu
def test_canary_attn_fwd_bwd():
    from otter_b200 import _lib
    lib = _lib.load()
    P, H, Sq, Sk1, Sk2 = 2, 3, 130, 129, 65
    inner = H * 64
    g = torch.Generator().manual_seed(11)
    q, kv1, kv2, dout = (_rnd(g, r, c).to(DEV) for r, c in
                         ((P * Sq, inner), (P * Sk1, 2 * inner), (P * Sk2, 2 * inner), (P * Sq, inner)))
    # inputs: logical columns [8, ...) of a wider matrix, NaN around them and in 3 rows past the last one
    cq = _Canvas(P * Sq + 3, inner + 32).put(q, 16)
    ck1 = _Canvas(P * Sk1 + 3, 2 * inner + 48).put(kv1[:, :inner], 8).put(kv1[:, inner:], inner + 24)
    ck2 = _Canvas(P * Sk2 + 3, 2 * inner + 48).put(kv2[:, :inner], 40).put(kv2[:, inner:], inner + 40)
    cdo = _Canvas(P * Sq + 2, inner + 24).put(dout, 8)
    co, clse = _Canvas(P * Sq + 4, inner + 64), _Canvas(1, P * H * Sq + 7, torch.float32)
    o_view, lse_view = co.own(P * Sq, 40, 40 + inner), clse.own(1, 0, P * H * Sq)
    d = _lib.AttnDesc()
    d.q, d.kv1, d.kv2, d.out, d.lse, d.text_time = cq.ptr(), ck1.ptr(), ck2.ptr(), co.ptr(), clse.ptr(), None
    d.ldq, d.ldkv1, d.ldkv2, d.ld_out = cq.t.stride(0), ck1.t.stride(0), ck2.t.stride(0), co.t.stride(0)
    d.q_cols, d.kv1_cols, d.kv2_cols = 16 + inner + 8, 2 * inner + 32, 2 * inner + 40   # logical widths < pitch
    d.q_col0, d.k1_col0, d.v1_col0, d.k2_col0, d.v2_col0, d.out_col0 = 16, 8, inner + 24, 40, inner + 40, 40
    d.n_per_media, d.T_img = 0, 0
    d.P, d.H, d.Sq, d.Sk1, d.Sk2, d.head_dim = P, H, Sq, Sk1, Sk2, 64
    d.scale, d.mask_ge, d.causal = 0.125, 0, 0
    _ok(lib.otb_attn_fwd(C.byref(d), _stream()), "otb_attn_fwd")
    torch.cuda.synchronize()
    co.check("otb_attn_fwd out")
    clse.check("otb_attn_fwd lse")

    cdq = _Canvas(P * Sq + 2, inner + 64)
    cd1, cd2 = _Canvas(P * Sk1 + 2, 2 * inner + 64), _Canvas(P * Sk2 + 2, 2 * inner + 64)
    dq_view = cdq.own(P * Sq, 56, 56 + inner)
    dk1_view, dv1_view = cd1.own(P * Sk1, 8, 8 + inner), cd1.own(P * Sk1, inner + 16, 2 * inner + 16)
    dk2_view, dv2_view = cd2.own(P * Sk2, inner + 32, 2 * inner + 32), cd2.own(P * Sk2, 0, inner)
    ws = torch.full((P * Sq, H * 64), float("nan"), dtype=torch.float32, device=DEV)   # scratch: no initialisation
    gr = _lib.AttnGrads()
    gr.dout, gr.dq, gr.dkv1, gr.dkv2, gr.dq_ws = cdo.ptr(), cdq.ptr(), cd1.ptr(), cd2.ptr(), C.c_void_p(ws.data_ptr())
    gr.ld_dout, gr.ld_dq, gr.ld_dkv1, gr.ld_dkv2 = cdo.t.stride(0), cdq.t.stride(0), cd1.t.stride(0), cd2.t.stride(0)
    gr.dout_cols, gr.dout_col0, gr.dq_col0 = 8 + inner, 8, 56
    gr.dk1_col0, gr.dv1_col0, gr.dk2_col0, gr.dv2_col0 = 8, inner + 16, inner + 32, 0
    _ok(lib.otb_attn_bwd(C.byref(d), C.byref(gr), _stream()), "otb_attn_bwd")
    torch.cuda.synchronize()
    for cv, what in ((cdq, "dq"), (cd1, "dkv1"), (cd2, "dkv2")):
        cv.check(f"otb_attn_bwd {what}")

    allowed, zero = _mask64(P, Sq, Sk1 + Sk2, DEV)
    hk = torch.cat([_heads(kv1, P, Sk1, 0, H, 64), _heads(kv2, P, Sk2, 0, H, 64)], 2)
    hv = torch.cat([_heads(kv1, P, Sk1, inner, H, 64), _heads(kv2, P, Sk2, inner, H, 64)], 2)
    hq, hdo, ho = _heads(q, P, Sq, 0, H, 64), _heads(dout, P, Sq, 0, H, 64), _heads(o_view, P, Sq, 0, H, 64)
    refs = [ref_attention(hq[:, h], hk[:, h], hv[:, h], 0.125, allowed, zero, dout=hdo[:, h], o_given=ho[:, h])
            for h in range(H)]
    _check("canary attn O", ho, _stack(refs, "o"))
    _check("canary attn lse", lse_view.reshape(P, H, Sq), _stack(refs, "lse"), lse=True)
    _check("canary attn dQ", _heads(dq_view, P, Sq, 0, H, 64), _stack(refs, "dq"))
    dk, dv = _stack(refs, "dk"), _stack(refs, "dv")
    _check("canary attn dK1", _heads(dk1_view, P, Sk1, 0, H, 64), dk[:, :, :Sk1])
    _check("canary attn dV1", _heads(dv1_view, P, Sk1, 0, H, 64), dv[:, :, :Sk1])
    _check("canary attn dK2", _heads(dk2_view, P, Sk2, 0, H, 64), dk[:, :, Sk1:])
    _check("canary attn dV2", _heads(dv2_view, P, Sk2, 0, H, 64), dv[:, :, Sk1:])


@gpu
@pytest.mark.parametrize("B,S,H,alibi,causal", [(2, 130, 2, True, True), (1, 64, 3, False, False)])
def test_canary_lm_attn_fwd_bwd(B, S, H, alibi, causal):
    """Column offsets other than the 0 / D / 2D of functional.lm_attn_*: K first, then V, then Q."""
    from otter_b200 import _lib
    from otter_b200.lm_mpt import alibi_slopes
    lib = _lib.load()
    D = H * 128
    qkv, dout = _lm_inputs(B, S, H, 5 + S)
    qkv, dout = qkv.to(BF16).to(DEV), dout.to(BF16).to(DEV)
    slopes = alibi_slopes(H, device=DEV) if alibi else None
    k0, v0, q0 = 8, D + 24, 2 * D + 40
    cqkv = _Canvas(B * S + 3, 3 * D + 64).put(qkv[:, D:2 * D], k0).put(qkv[:, 2 * D:], v0).put(qkv[:, :D], q0)
    co, clse = _Canvas(B * S + 2, D + 64), _Canvas(1, B * H * S + 5, torch.float32)
    o_view, lse_view = co.own(B * S, 24, 24 + D), clse.own(1, 0, B * H * S)
    d = _lib.LmAttnDesc()
    d.qkv, d.out, d.lse = cqkv.ptr(), co.ptr(), clse.ptr()
    d.alibi_slopes = C.c_void_p(slopes.data_ptr()) if alibi else None
    d.ld_qkv, d.ld_out = cqkv.t.stride(0), co.t.stride(0)
    d.qkv_cols, d.q_col0, d.k_col0, d.v_col0, d.out_col0 = 3 * D + 48, q0, k0, v0, 24
    d.B, d.H, d.S, d.head_dim, d.causal, d.scale = B, H, S, 128, int(causal), 128 ** -0.5
    _ok(lib.otb_lm_attn_fwd(C.byref(d), _stream()), "otb_lm_attn_fwd")
    torch.cuda.synchronize()
    co.check("otb_lm_attn_fwd out")
    clse.check("otb_lm_attn_fwd lse")

    cdo = _Canvas(B * S + 2, D + 32).put(dout, 16)
    cdqkv = _Canvas(B * S + 3, 3 * D + 64)
    dk_view, dv_view, dq_view = cdqkv.own(B * S, 8, 8 + D), cdqkv.own(B * S, D + 16, 2 * D + 16), \
        cdqkv.own(B * S, 2 * D + 24, 3 * D + 24)
    ws = torch.full((B * S, H * 128), float("nan"), dtype=torch.float32, device=DEV)
    gr = _lib.LmAttnGrads()
    gr.dout, gr.dqkv, gr.dq_ws = cdo.ptr(), cdqkv.ptr(), C.c_void_p(ws.data_ptr())
    gr.ld_dout, gr.ld_dqkv = cdo.t.stride(0), cdqkv.t.stride(0)
    gr.dout_cols, gr.dout_col0, gr.dq_col0, gr.dk_col0, gr.dv_col0 = D + 24, 16, 2 * D + 24, 8, D + 16
    _ok(lib.otb_lm_attn_bwd(C.byref(d), C.byref(gr), _stream()), "otb_lm_attn_bwd")
    torch.cuda.synchronize()
    cdqkv.check("otb_lm_attn_bwd dqkv")

    pos = (torch.arange(S, device=DEV) - (S - 1)).double()
    allowed, _ = _mask64(B, S, S, DEV, causal=causal)
    hdo, ho = _heads(dout, B, S, 0, H, 128), _heads(o_view, B, S, 0, H, 128)
    refs = [ref_attention(*(_heads(qkv, B, S, c * D, H, 128)[:, h] for c in range(3)), 128 ** -0.5, allowed,
                          bias=slopes[h].double() * pos if alibi else None, dout=hdo[:, h], o_given=ho[:, h])
            for h in range(H)]
    _check("canary lm O", _heads(o_view, B, S, 0, H, 128), _stack(refs, "o"))
    _check("canary lm lse", lse_view.reshape(B, H, S), _stack(refs, "lse"), lse=True)
    for view, key in ((dq_view, "dq"), (dk_view, "dk"), (dv_view, "dv")):
        _check(f"canary lm {key}", _heads(view, B, S, 0, H, 128), _stack(refs, key))


@gpu
def test_canary_xattn_out_fused():
    from otter_b200 import _lib
    lib = _lib.load()
    P, H, Sq, T, n, D, ge = 2, 4, 130, 2, 32, 1024, True
    inner = H * 64
    g = torch.Generator().manual_seed(13)
    q, kv = _rnd(g, P * Sq, inner).to(DEV), _rnd(g, P * T * n, 2 * inner).to(DEV)
    wo, x = _rnd(g, D, inner, scale=inner ** -0.5).to(DEV), _rnd(g, P * Sq, D).to(DEV)
    tt = _media_tt(P, Sq, T)
    gate = torch.tensor([GATE], device=DEV)
    cq = _Canvas(P * Sq + 3, inner + 32).put(q, 24)
    ckv = _Canvas(P * T * n + 3, 2 * inner + 48).put(kv[:, :inner], 8).put(kv[:, inner:], inner + 16)
    cwo = _Canvas(D + 3, inner + 32).put(wo, 0)
    cx = _Canvas(P * Sq + 2, D + 64).put(x, 24)
    co, clse = _Canvas(P * Sq + 4, inner + 64), _Canvas(1, P * H * Sq + 7, torch.float32)
    caux, cy = _Canvas(P * Sq + 3, D + 64), _Canvas(P * Sq + 3, D + 32)
    o_view, lse_view = co.own(P * Sq, 24, 24 + inner), clse.own(1, 0, P * H * Sq)
    aux_view, y_view = caux.own(P * Sq, 16, 16 + D), cy.own(P * Sq, 8, 8 + D)
    ttd = tt.to(DEV).contiguous()
    d = _lib.AttnDesc()
    d.q, d.kv1, d.kv2, d.out, d.lse, d.text_time = cq.ptr(), ckv.ptr(), None, co.ptr(), clse.ptr(), C.c_void_p(ttd.data_ptr())
    d.ldq, d.ldkv1, d.ldkv2, d.ld_out = cq.t.stride(0), ckv.t.stride(0), 0, co.t.stride(0)
    d.q_cols, d.kv1_cols, d.kv2_cols = 24 + inner, 2 * inner + 16, 0
    d.q_col0, d.k1_col0, d.v1_col0, d.k2_col0, d.v2_col0, d.out_col0 = 24, 8, inner + 16, 0, 0, 24
    d.n_per_media, d.T_img = n, T
    d.P, d.H, d.Sq, d.Sk1, d.Sk2, d.head_dim = P, H, Sq, T * n, 0, 64
    d.scale, d.mask_ge, d.causal = 0.125, int(ge), 0
    _ok(lib.otb_xattn_out_fused(C.byref(d), cwo.ptr(), cwo.t.stride(0), C.c_void_p(gate.data_ptr()), cx.ptr(24),
                                cx.t.stride(0), caux.ptr(16), caux.t.stride(0), cy.ptr(8), cy.t.stride(0), D, _stream()),
        "otb_xattn_out_fused")
    torch.cuda.synchronize()
    for cv, what in ((co, "O"), (clse, "lse"), (caux, "aux"), (cy, "y")):
        cv.check(f"otb_xattn_out_fused {what}")
    o_r, lse_r, a_r, y_r, _ = _fused_ref(q, kv, wo, x, P, H, Sq, T, n, tt, ge)
    _check("canary fused O", _heads(o_view, P, Sq, 0, H, 64), o_r)
    _check("canary fused lse", lse_view.reshape(P, H, Sq), lse_r, lse=True)
    _check("canary fused aux", aux_view.reshape(P * Sq, D // 64, 64), a_r.view(P * Sq, D // 64, 64))
    _check("canary fused y", y_view.reshape(P * Sq, D // 64, 64), y_r.view(P * Sq, D // 64, 64))
