"""The GEMM (otb_gemm_bf16, csrc/otb_gemm.cu) against a float64 reference at the edges of its tile structure.

Under test:
  - the three instantiated operand layouts: (K, K) forward, (K, MN) dgrad, (MN, MN) wgrad;
  - 128 x 128 output tiles with 64-deep k-blocks, ragged in M, N and K; TMA loads that must stop at the extents, not
    at the row pitch; TMA stores (and the fp32 reduce-add of `accumulate`) clipped to M x N;
  - the persistent ping-pong schedule: CTAs with one, two or an odd number of tiles, alternate tiles on the two MMA
    warpgroups, the grouped tile walk (32 M-tiles per group, a ragged last group);
  - every compiled epilogue class (kEpiCls) and the run-time epilogue, against the order include/otter_b200.h
    documents: bias, aux_out, act or act'(aux_in), alpha * scale, residual, accumulate;
  - the fp32-grade route functional.linear_f32 (split-3 operands, chunked accumulate, fp32 epilogue).

Reference: float64 on the device from the same bf16 operands (fp32 bias, gate and fp32 residual).  The tests without
the `gpu` mark show on the CPU that the metric rejects float64 references mutated the way a GEMM bug would mutate them.

Every otb_gemm_bf16 case here is launched through the C ABI with operands and outputs placed inside NaN-filled canvases
with a larger row pitch and extra rows (`Canvas`): every element a launch owns must be finite and within the bound,
every other element must keep its bits, and a load past an operand's extent shows up as NaN in an owned output.
"""
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
gpu = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------------------------
# The metric, per output element:
#
#     |got - ref| <= A_OUT * |ref| + E + FLOOR
#
# E is a bound on the fp32 error before the output is rounded, carried through the epilogue in float64 next to the
# reference (epi_ref).  It starts from the accumulator:
#
#   - Accumulator.  The products of two bf16 values are exact in fp32.  The tensor core adds each k16 step (16
#     products) into its fp32 accumulator and TRUNCATES (functional.linear_f32 records this): the error of a step does
#     not average out with the next one, it has one sign, so the accumulated error grows with the number of k16 steps,
#     not with its square root.  A step's error is below a few fp32 ulps (2^-23 relative) of the larger of the running
#     sum and the step's products, both <= the partial sum of |a_k b_k| <= S = sum_k |a_k b_k|.  We allow 4 ulps per step:
#         e_acc = C_STEP * ceil(K / 16) * S,   C_STEP = 2^-21.
#     Zero-filled steps past a ragged K add exact zeros and cost nothing.  The bound is linear in K, so it holds at the
#     largest K tested (16384: 1024 steps, 2^-11 S) by construction; a constant sized for small K would not.  For
#     random-sign operands the exact sum is ~sqrt(K) smaller than S, so at large K and fp32 output this term is loose.
#   - Epilogue (fp32, U32 = 2^-24 per rounding).  Each fp32 operation adds a rounding of its result's magnitude; we
#     charge U = 2^-21 (8 roundings) of |z| after the bias, of |v| after act and scale, of |v| after the residual and of
#     |v| after the accumulate: the residual and the accumulated old value enter through these terms, so a result that
#     cancels is still bounded by the magnitudes that were added.  The accumulator error is multiplied by |act'(z)| (or
#     by |act'(aux_in)| for the backward) and by |scale|; a curved activation adds E^2 (|act''| <= 2 for relu^2, < 1
#     for GELU and quick-GELU).
#   - Fast math.  The epilogue's erf (otb_common.cuh erf_exp_half, Abramowitz-Stegun 7.1.26) errs by <= 1.5e-7
#     absolute, plus ~1 fp32 rounding of a value near 1 and exp2f's error: ERF_ERR = 2^-22 absolute in erf and in gelu'.
#     That is 0.5 |z| ERF_ERR in GELU and |z| ERF_ERR in v * gelu'(aux) (the argument rounding of gelu'(aux), |act''| |aux|
#     U32, is < 2^-25 and inside it).  quick-GELU: __expf errs by (2 + 1.17 |x|) ulp, rcp.approx by 1 ulp, so
#     sigmoid(1.702 z) errs by < (4 + 4 |z|) 2^-23 relative.  The gate's tanhf (2 ulp) is inside U.
#   - accumulate: the TMA reduce-add at L2 is one fp32 rounding of old + v (the last U term).
#
# Output rounding: bf16 keeps 8 significant bits, rounding to nearest errs by < 2^-8 |ref|; A_OUT = 2^-7 leaves a
# factor 2 (as in the attention and row-wise edge tests).  fp32 outputs: < 2^-24 |ref|, A_OUT = 2^-23.
# FLOOR = 2^-60: quick-GELU at z < -52, where __expf overflows and the exact answer is < 1e-37.
#
# The fp32-grade route (linear_f32) starts from fp32 x and W split into three bf16 terms each; the six kept cross
# products leave out x1 y2, x2 y1, x2 y2 and the split residuals, each < 2^-26 |x| |y|: SPLIT = 2^-24 of S.  Each
# accumulator run is at most F32_KCHUNK = 512 columns of the 6K-long operand (32 k16 steps, C_STEP each) and every
# chunk is added to the running fp32 sum by one rounded add (U32 per chunk), so
#     e_acc = (SPLIT + C_STEP * ceil(min(6K, 512) / 16) * 1.02 + U32 * chunks) * S       (S of the fp32 x and W;
# the six products of one pair sum to < 1.02 |x| |y|).  The epilogue terms are the same as above.
#
# The constants were fixed before the first GPU run and no run has forced a change.  Every RATIO line also prints the
# same ratio for the exact answer rounded to the output type, the part no kernel with that output type can avoid.
# Measured on an H100 80GB HBM3 (400 W power limit), worst error / bound per family:
#   - bf16 outputs (layouts, tile counts, depths, ragged edges, epilogue classes and sweep, hot-path shapes, canaries):
#     0.43 - 0.50, each equal to the exact answer rounded to bf16 (output rounding dominates);
#   - fp32 outputs with GELU (epilogue class gelu_f32, the sweep, the fp32-grade route): 0.42 - 0.62 against 0.03 - 0.08
#     for the exact answer rounded to fp32: the fast erf's 1.5e-7 is the largest error there;
#   - fp32 outputs of plain GEMMs and wgrad: 0.006 - 0.08.  Here the accumulator term C_STEP ceil(K/16) S is loose for
#     random-sign operands (the running sum is ~sqrt(K) below S); it is the worst case of truncation, not a typical one.
# The power checks below exceed the bound by 3.7x (one k16 step missing at K = 16384, bf16 out: the tightest) to > 1e5x.
# ------------------------------------------------------------------------------------------------------------------
C_STEP = 2.0 ** -21
U = 2.0 ** -21
U32 = 2.0 ** -24
ERF_ERR = 2.0 ** -22
SPLIT = 2.0 ** -24
A_OUT = {BF16: 2.0 ** -7, F32: 2.0 ** -23}
FLOOR = 2.0 ** -60
F32_KCHUNK = 512


def c_acc(K):
    return C_STEP * math.ceil(K / 16)


def c_acc_f32grade(K):
    K6 = 6 * K
    return SPLIT + C_STEP * math.ceil(min(K6, F32_KCHUNK) / 16) * 1.02 + U32 * math.ceil(K6 / F32_KCHUNK)


def _gelu(z):
    return 0.5 * z * (1.0 + torch.erf(z / math.sqrt(2.0)))


def _gelu_grad(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def epi_ref(acc, S, c, *, bias=None, aux_out=False, act=0, aux_in=None, alpha=1.0, gate=None, tanh=False,
            residual=None, old=None, mut=()):
    """The epilogue of include/otter_b200.h in float64 on acc = A B^T, with its error bound E (see above).
    c: accumulator error per unit of S.  `mut` names mutations for the power checks; () is the real operation.
    -> dict out, E and, with aux_out, aux / E_aux."""
    e = c * S
    z = acc if bias is None else acc + (bias.roll(8) if "bias_shift8" in mut else bias)
    e = e + U * z.abs()
    r = {}
    if aux_out:
        r["aux"], r["E_aux"] = z, e
    if aux_in is None:
        if act == 0:
            y, d, extra = z, 1.0, 0.0
        elif act == 1:
            y, d, extra = _gelu(z), _gelu_grad(z).abs(), 0.5 * z.abs() * ERF_ERR + e * e
        elif act == 2:
            sg = torch.sigmoid(1.702 * z)
            y = z * sg
            d = (sg + 1.702 * z * sg * (1 - sg)).abs()
            extra = y.abs() * (4 + 4 * z.abs()) * 2.0 ** -23 + e * e
        else:
            rl = z.clamp_min(0)
            y, d, extra = rl * rl, 2 * rl, e * e
        if aux_out and "aux_after_act" in mut:
            r["aux"] = y
    else:
        at = z if "grad_at_acc" in mut else aux_in
        if act == 3 and "gelu_grad_for_relu2" not in mut:
            f, extra = 2 * at.clamp_min(0), 0.0
        else:
            f, extra = _gelu_grad(at), z.abs() * ERF_ERR
        y, d = z * f, f.abs()
    e = d * e + extra
    s = alpha
    if gate is not None:
        s = alpha * (math.tanh(gate) if tanh and "gate_untanhed" not in mut else gate)
    if residual is not None and "residual_before_scale" in mut:
        y = y + residual
    y = y * s
    e = abs(s) * e + U * y.abs()
    if residual is not None:
        if "residual_before_scale" not in mut:
            y = y + (residual.roll(1, 0) if "residual_next_row" in mut else residual)
        e = e + U * y.abs()
    if old is not None:
        if "accumulate_stores" not in mut:
            y = old + y
        e = e + U * y.abs()
    r["out"], r["E"] = y, e
    return r


def _ratio(got, ref, E, out):
    got, ref = got.double(), ref.double()
    return ((got - ref).abs() / (A_OUT[out] * ref.abs() + E + FLOOR)).max().item()


def _check(what, got, ref, E, out):
    r = _ratio(got, ref, E, out)
    print(f"RATIO {what} {r:.4g} (exact answer rounded to {str(out)[6:]}: {_ratio(ref.to(out), ref, E, out):.4g})")
    if not r <= 1.0:
        q = (got.double() - ref).abs() / (A_OUT[out] * ref.abs() + E + FLOOR)
        q = torch.nan_to_num(q, nan=math.inf)
        i = np.unravel_index(int(q.argmax()), tuple(q.shape))
        print(f"WORST {what} at {i}: got {got[i].item():.6g} ref {ref[i].item():.6g}; over the bound: "
              f"{(q > 1).sum().item()}")
    assert r <= 1.0, f"{what}: error / bound = {r:.3f}"


# the compiled epilogue classes of otb_gemm.cu (kEpiCls): bias, aux_out, act, aux_in, scale, residual, fp32 out, acc
EPI_CLS = [
    (0, 0, 0, 0, 0, 0, 0, 0), (0, 0, 0, 0, 1, 0, 0, 0), (1, 0, 0, 0, 0, 0, 0, 0), (1, 0, 2, 0, 0, 0, 0, 0),
    (1, 0, 0, 0, 0, 1, 0, 0), (0, 0, 0, 0, 0, 1, 0, 0), (0, 1, 1, 0, 0, 0, 0, 0), (0, 1, 0, 0, 1, 1, 0, 0),
    (0, 0, 0, 1, 1, 0, 0, 0), (0, 0, 0, 1, 0, 0, 0, 0), (0, 0, 0, 0, 0, 0, 1, 0), (0, 0, 0, 0, 1, 0, 1, 0),
    (0, 0, 0, 0, 0, 0, 1, 1), (0, 0, 0, 0, 1, 0, 1, 1),
]


def epi_class_of(o):
    """The launch class otb_gemm_bf16 picks for options `o` (as _run takes them); -1 = run-time epilogue."""
    if o.get("res") == "f32":
        return -1
    aux_in, act = bool(o.get("aux_in")), o.get("act", 0)
    if aux_in and act == 3:
        return -1
    key = (int(bool(o.get("bias"))), int(bool(o.get("aux_out"))), 0 if aux_in else act, int(aux_in),
           int(o.get("gate") is not None or o.get("alpha", 1.0) != 1.0), int(o.get("res") is not None),
           int(o.get("out", BF16) == F32), int(bool(o.get("acc"))))
    return EPI_CLS.index(key) if key in EPI_CLS else -1


# ------------------------------------------------------------------------------------------------------------------
# CPU: the metric rejects plausible GEMM bugs.  Each mutation is applied to the float64 reference.
# ------------------------------------------------------------------------------------------------------------------
def _mutant(name, r):
    print(f"MUTANT {name} ratio {r:.3f}")
    return r


def _cpu_operands(M, N, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(BF16).double()
    b = (torch.randn(N, K, generator=g) * K ** -0.5).to(BF16).double()
    return a, b, a @ b.t(), a.abs() @ b.abs().t()


@pytest.mark.parametrize("K", [16384, 72])
@pytest.mark.parametrize("out", [BF16, F32])
def test_metric_rejects_one_missing_k16_step(K, out):
    """16 terms of one k16 step missing from one tile; at K = 72 the step of the ragged last k-block (8 real terms)."""
    a, b, acc, S = _cpu_operands(256, 256, K, seed=1)
    k0 = K - 8 if K == 72 else 4096
    m = acc.clone()
    m[128:, :128] -= a[128:, k0:k0 + 16] @ b[:128, k0:k0 + 16].t()
    r = epi_ref(acc, S, c_acc(K))
    assert _mutant(f"k16 step missing K={K} {out}", _ratio(m, r["out"], r["E"], out)) > 1.0


def test_metric_rejects_k_block_from_the_neighbouring_tile():
    """A stale ring slot: one 64-deep k-block of tile (1, 0) computed with the A rows of tile (0, 0)."""
    a, b, acc, S = _cpu_operands(256, 256, 512, seed=2)
    k0 = 192
    m = acc.clone()
    m[128:, :128] += (a[:128, k0:k0 + 64] - a[128:, k0:k0 + 64]) @ b[:128, k0:k0 + 64].t()
    r = epi_ref(acc, S, c_acc(512))
    assert _mutant("stale k-block", _ratio(m, r["out"], r["E"], BF16)) > 1.0


@pytest.mark.parametrize("mutation", ["swap_16B_units", "swap_rows_r_r^1", "ragged_last_8_cols_zero"])
@pytest.mark.parametrize("out", [BF16, F32])
def test_metric_rejects_store_layout_mutations(mutation, out):
    a, b, acc, S = _cpu_operands(200, 136, 136, seed=3)
    r = epi_ref(acc, S, c_acc(136))
    m = r["out"].clone()
    w = 16 // (2 if out == BF16 else 4)                        # elements per 16 B unit
    if mutation == "swap_16B_units":                          # units 1 and 2 of row 37 inside one store box
        m[37, w:2 * w], m[37, 2 * w:3 * w] = r["out"][37, 2 * w:3 * w], r["out"][37, w:2 * w]
    elif mutation == "swap_rows_r_r^1":                       # rows 36 and 37 of the second 32-row quarter
        m[36], m[37] = r["out"][37], r["out"][36]
    else:                                                     # N = 136: columns 128..135 of the second N tile
        m[128:, 128:] = 0.0
    assert _mutant(f"{mutation} {out}", _ratio(m, r["out"], r["E"], out)) > 1.0


_EPI_MUTATIONS = {
    "bias_shift8": dict(bias=True),
    "residual_next_row": dict(res=True),
    "gate_untanhed": dict(gate=0.5, tanh=True),
    "residual_before_scale": dict(gate=0.5, tanh=True, res=True),
    "grad_at_acc": dict(aux_in=True, act=1),
    "gelu_grad_for_relu2": dict(aux_in=True, act=3),
    "accumulate_stores": dict(old=True),
    "aux_after_act": dict(aux_out=True, act=1),
}


@pytest.mark.parametrize("mutation", list(_EPI_MUTATIONS) + ["f32_through_bf16"])
def test_metric_rejects_epilogue_mutations(mutation):
    M, N, K = 200, 136, 136
    a, b, acc, S = _cpu_operands(M, N, K, seed=4)
    g = torch.Generator().manual_seed(5)
    o = _EPI_MUTATIONS.get(mutation, {})
    kw = {}
    if o.get("bias"):
        kw["bias"] = torch.randn(N, generator=g).float().double()
    if o.get("res"):
        kw["residual"] = torch.randn(M, N, generator=g).to(BF16).double()
    if o.get("aux_in"):
        kw["aux_in"] = (torch.randn(M, N, generator=g) * 1.5).to(BF16).double()
    if o.get("old"):
        kw["old"] = torch.randn(M, N, generator=g).float().double()
    for k in ("gate", "tanh", "act", "aux_out"):
        if k in o:
            kw[k] = o[k]
    out = F32 if mutation in ("accumulate_stores", "f32_through_bf16") else BF16
    r = epi_ref(acc, S, c_acc(K), **kw)
    if mutation == "f32_through_bf16":
        got, ref, E = r["out"].to(BF16).double(), r["out"], r["E"]
    elif mutation == "aux_after_act":
        got, ref, E = epi_ref(acc, S, c_acc(K), mut=(mutation,), **kw)["aux"], r["aux"], r["E_aux"]
    else:
        got, ref, E = epi_ref(acc, S, c_acc(K), mut=(mutation,), **kw)["out"], r["out"], r["E"]
    assert _mutant(mutation, _ratio(got, ref, E, out)) > 1.0


def test_metric_accepts_output_rounding():
    """The other side: the exact answer rounded to the output type stays below 0.5 of the bound."""
    for K in (72, 16384):
        _, _, acc, S = _cpu_operands(128, 136, K, seed=6)
        r = epi_ref(acc, S, c_acc(K))
        for out in (BF16, F32):
            assert _mutant(f"rounded K={K} {out}", _ratio(r["out"].to(out), r["out"], r["E"], out)) < 0.5


def test_epi_class_mirror_covers_every_compiled_class():
    opts = [dict(), dict(gate=0.5), dict(bias=1), dict(bias=1, act=2), dict(bias=1, res="bf16"), dict(res="bf16"),
            dict(aux_out=1, act=1), dict(aux_out=1, gate=0.5, res="bf16"), dict(aux_in=1, gate=0.5), dict(aux_in=1),
            dict(out=F32), dict(out=F32, alpha=0.5), dict(out=F32, acc=1), dict(out=F32, acc=1, gate=0.5)]
    assert [epi_class_of(o) for o in opts] == list(range(14))
    assert epi_class_of(dict(out=F32, res="f32")) == -1 and epi_class_of(dict(aux_in=1, act=3)) == -1


# ------------------------------------------------------------------------------------------------------------------
# GPU harness: the C ABI with NaN-filled canvases.
# ------------------------------------------------------------------------------------------------------------------
DEV = "cuda:0"
LAYOUTS = {"fwd": (0, 0), "dgrad": (0, 1), "wgrad": (1, 1)}


def _lib():
    from otter_b200 import _lib as L
    return L.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class Canvas:
    """A [rows, cols] view at (row0, col0) inside a [rows + row0 + 2, pitch] buffer filled with `fill`."""

    def __init__(self, rows, cols, dtype, fill=float("nan"), row0=1, col0=8, pitch=None):
        pitch = pitch or -(-(col0 + cols + 16) // 8) * 8
        self.t = torch.full((rows + row0 + 2, pitch), fill, dtype=dtype, device=DEV)
        self.v = self.t[row0:row0 + rows, col0:col0 + cols]
        self.owned = torch.zeros(self.t.shape, dtype=torch.bool, device=DEV)
        self.owned[row0:row0 + rows, col0:col0 + cols] = True
        self.fill = torch.full((1,), fill, dtype=dtype, device=DEV)

    def bits(self, t):
        return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])

    def check(self, what):
        assert torch.isfinite(self.t[self.owned].float()).all(), f"{what}: an owned element is not finite"
        assert (self.bits(self.t)[~self.owned] == self.bits(self.fill)).all(), \
            f"{what}: an element outside the output changed"


def _put(x, **kw):
    cv = Canvas(x.shape[0], x.shape[1], x.dtype, **kw)
    cv.v.copy_(x)
    return cv


def _randn(g, *shape, scale=1.0, dtype=BF16):
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


class Operands:
    """A [M,K] and B [N,K] (logical, bf16) in the storage order of `layout`, inside NaN canvases."""

    def __init__(self, layout, M, N, K, seed=0, a_kw=None, b_kw=None):
        self.layout, self.M, self.N, self.K = layout, M, N, K
        g = torch.Generator(device=DEV).manual_seed(seed * 1000003 + M * 7919 + N * 31 + K)
        self.a = _randn(g, M, K)
        self.b = _randn(g, N, K, scale=K ** -0.5)
        a_mn, b_mn = LAYOUTS[layout]
        self.ca = _put(self.a.t() if a_mn else self.a, **(a_kw or {}))
        self.cb = _put(self.b.t() if b_mn else self.b, **(b_kw or {}))
        self.g = g

    def ref(self, rows=None):
        a = self.a if rows is None else self.a[rows]
        a64, b64 = a.double(), self.b.double()
        return a64 @ b64.t(), a64.abs() @ b64.abs().t()


def _launch(layout, A, B, M, N, K, out, *, bias=None, aux_in=None, aux_out=None, gate=None, tanh=False, alpha=1.0,
            residual=None, res_fp32=False, accumulate=False, act=0):
    """otb_gemm_bf16 on tensor views (their data pointer and row pitch)."""
    from otter_b200 import _lib as L
    e = L.GemmEpilogue()
    e.bias, e.aux_in, e.aux_out, e.scale_ptr, e.residual, e.out = (_p(t) for t in (bias, aux_in, aux_out, gate,
                                                                                    residual, out))
    e.ld_out = out.stride(0)
    e.ld_aux_in = aux_in.stride(0) if aux_in is not None else 0
    e.ld_aux_out = aux_out.stride(0) if aux_out is not None else 0
    e.ld_res = residual.stride(0) if residual is not None else 0
    e.act, e.scale_tanh, e.out_fp32, e.accumulate = act, int(tanh), int(out.dtype == F32), int(accumulate)
    e.alpha, e.res_fp32 = alpha, int(res_fp32)
    a_mn, b_mn = LAYOUTS[layout]
    L.check(_lib().otb_gemm_bf16(_p(A), a_mn, A.stride(0), _p(B), b_mn, B.stride(0), M, N, K, C.byref(e),
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream)), "otb_gemm_bf16")


SENTINEL = -1234.5                      # finite padding of accumulate outputs: a stray reduce-add changes its bits


class EpiInputs:
    """The epilogue's input tensors for one operand set, NaN past N and past M (made once, shared by many launches)."""

    def __init__(self, ops):
        M, N, g = ops.M, ops.N, ops.g
        self.bias = Canvas(1, N, F32, row0=0, col0=4)
        self.bias.v.copy_(_randn(g, 1, N, dtype=F32))
        self.res = _put(_randn(g, M, N), col0=16)
        self.res32 = _put(_randn(g, M, N, dtype=F32), col0=8)
        self.aux_in = _put(_randn(g, M, N, scale=1.5), col0=24)
        self.old = _randn(g, M, N, dtype=F32)
        self.gate = torch.empty(4, device=DEV)


def _run(tag, ops, o, *, epi=None, rows=None, acc_S=None, out_kw=None):
    """One launch with epilogue options `o` (keys: bias, aux_out, act, aux_in, alpha, gate, tanh, res ('bf16' | 'f32'),
    out (BF16 | F32), acc), its canary checks and its metric checks.  rows: output rows the float64 reference covers
    (default all).  -> the output view."""
    M, N, K = ops.M, ops.N, ops.K
    epi = epi or EpiInputs(ops)
    out_dt = o.get("out", BF16)
    acc = bool(o.get("acc"))
    cout = Canvas(M, N, out_dt, fill=SENTINEL if acc else float("nan"), **(out_kw or {"col0": 8}))
    if acc:
        cout.v.copy_(epi.old)
    caux = Canvas(M, N, BF16, col0=40) if o.get("aux_out") else None
    gate = o.get("gate")
    if gate is not None:
        epi.gate.fill_(gate)
    res = o.get("res")
    _launch(ops.layout, ops.ca.v, ops.cb.v, M, N, K, cout.v, bias=epi.bias.v[0] if o.get("bias") else None,
            aux_in=epi.aux_in.v if o.get("aux_in") else None, aux_out=caux.v if caux else None,
            gate=epi.gate[:1] if gate is not None else None, tanh=bool(o.get("tanh")), alpha=o.get("alpha", 1.0),
            residual={None: None, "bf16": epi.res.v, "f32": epi.res32.v}[res], res_fp32=res == "f32",
            accumulate=acc, act=o.get("act", 0))
    torch.cuda.synchronize()
    cout.check(f"{tag} out")
    if caux:
        caux.check(f"{tag} aux_out")
    a64, S = acc_S if acc_S is not None else ops.ref(rows)
    sel = (lambda t: t) if rows is None else (lambda t: t[rows])
    r = epi_ref(a64, S, c_acc(K), bias=epi.bias.v[0].double() if o.get("bias") else None,
                aux_out=bool(caux), act=o.get("act", 0), aux_in=sel(epi.aux_in.v).double() if o.get("aux_in") else None,
                alpha=o.get("alpha", 1.0), gate=gate, tanh=bool(o.get("tanh")),
                residual=None if res is None else sel({"bf16": epi.res.v, "f32": epi.res32.v}[res]).double(),
                old=sel(epi.old).double() if acc else None)
    _check(f"{tag} out", sel(cout.v), r["out"], r["E"], out_dt)
    if caux:
        _check(f"{tag} aux_out", sel(caux.v), r["aux"], r["E_aux"], BF16)
    return cout.v


def _opts(spec):
    """'bias+gelu+aux_out+f32' -> option dict."""
    o = {}
    for w in filter(None, spec.split("+")):
        if w in ("bias", "aux_out", "aux_in", "acc"):
            o[w] = True
        elif w in ("gelu", "qgelu", "relu2"):
            o["act"] = {"gelu": 1, "qgelu": 2, "relu2": 3}[w]
        elif w == "gate":
            o.update(gate=0.5, tanh=True)
        elif w == "raw_scale":
            o["gate"] = -0.8
        elif w == "alpha":
            o["alpha"] = 0.375
        elif w in ("res", "res32"):
            o["res"] = "bf16" if w == "res" else "f32"
        elif w == "f32":
            o["out"] = F32
        else:
            raise ValueError(w)
    return o


# ------------------------------------------------------------------------------------------------------------------
# GPU: layouts, tile counts, depths, ragged edges
# ------------------------------------------------------------------------------------------------------------------
@gpu
def test_gemm_layouts_and_epilogues():
    """The functional entry points (linear_fwd / _dgrad / _wgrad) with a few epilogues and a column-sliced A."""
    from otter_b200 import functional as F
    g = torch.Generator(device=DEV).manual_seed(0)
    x, w, dy = _randn(g, 300, 256), _randn(g, 520, 256, scale=0.1), _randn(g, 300, 520)
    x64, w64, dy64 = x.double(), w.double(), dy.double()

    def chk(what, got, a, b, out=BF16, **kw):
        r = epi_ref(a @ b.t(), a.abs() @ b.abs().t(), c_acc(a.shape[1]), **kw)
        _check(f"layouts {what}", got, r["out"], r["E"], out)
        return r

    chk("linear_fwd", F.linear_fwd(x, w), x64, w64)
    chk("linear_dgrad", F.linear_dgrad(dy, w), dy64, w64.t())
    dw = F.linear_wgrad(dy, x)
    assert dw.dtype == F32
    chk("linear_wgrad", dw, dy64.t(), x64.t(), F32)
    dw2 = F.linear_wgrad(dy, x, out=dw.clone(), accumulate=True)
    chk("linear_wgrad accumulate", dw2, dy64.t(), x64.t(), F32, old=dw.double())
    z = torch.empty(300, 520, device=DEV, dtype=BF16)
    h = F.linear_fwd(x, w, act=1, aux_out=z)
    r = chk("gelu", h, x64, w64, act=1, aux_out=True)
    _check("layouts aux_out", z, r["aux"], r["E_aux"], BF16)
    gate = torch.tensor([0.5], device=DEV)
    res = _randn(g, 300, 520)
    chk("gate+residual", F.linear_fwd(x, w, scale_ptr=gate, scale_tanh=True, residual=res), x64, w64, gate=0.5,
        tanh=True, residual=res.double())
    bias = _randn(g, 520, dtype=F32)
    chk("bias+quick_gelu", F.linear_fwd(x, w, bias=bias, act=2), x64, w64, bias=bias.double(), act=2)
    big = _randn(g, 300, 1024)
    chk("strided A", F.linear_fwd(big[:, 256:512], w), big[:, 256:512].double(), w64)


# (M, N) multiples of 128: tile count = M/128 * N/128, around 132 and 264 on a 132-SM H100
@gpu
@pytest.mark.parametrize("tm,tn", [(1, 1), (1, 131), (12, 11), (7, 19), (1, 263), (12, 22), (5, 53)])
def test_tile_counts(tm, tn):
    _run(f"tiles[{tm}x{tn}]", Operands("fwd", 128 * tm, 128 * tn, 256), {})


@gpu
@pytest.mark.parametrize("spec", ["sm-1", "sm", "sm+1", "2sm-1", "2sm", "2sm+1", "3sm+3"])
@pytest.mark.parametrize("layout", ["fwd", "wgrad"])
def test_tile_counts_around_sm_count(spec, layout):
    """Tile counts from the device's SM count: one tile per CTA, one CTA with two, two per CTA, odd counts per CTA."""
    k, c = (spec.split("sm") + [""])[:2]
    tiles = int(k or 1) * _sms() + int(c or 0)
    tm = next(d for d in (7, 5, 3, 2, 1) if tiles % d == 0)
    M, N = 128 * tm - 8, 128 * (tiles // tm) - 8               # ragged on both sides, tile count unchanged
    _run(f"sm_tiles[{layout}-{spec}={tiles}]", Operands(layout, M, N, 200, seed=1), {"out": F32} if layout == "wgrad"
         else {})


# K = 16 / 64 / 72: one (partial) k-block, far shorter than the other warpgroup's epilogue; K = 16384: 256 k-blocks
@gpu
@pytest.mark.parametrize("K", [16, 64, 72, 16384])
def test_depths(K):
    _run(f"depth[{K}]", Operands("fwd", 2048, 4096, K), {"act": 1, "aux_out": True}, rows=_sample_rows(2048))


@gpu
def test_ragged_edges():
    M, N, K = 2056, 1032, 1024                                 # M = 16 * 128 + 8, N = 8 * 128 + 8
    _run("ragged fwd", Operands("fwd", M, N, K), {})
    _run("ragged dgrad", Operands("dgrad", M, K, N), {})
    _run("ragged wgrad", Operands("wgrad", N, K, M), {"out": F32})


# M = 16520: 130 M-tiles = 4 full groups of 32 and a last group of 2, the last M-tile itself partial
@gpu
@pytest.mark.parametrize("layout", ["fwd", "dgrad", "wgrad"])
def test_grouped_walk_ragged_last_group(layout):
    _run(f"grouped[{layout}]", Operands(layout, 16520, 384, 256), {"out": F32} if layout == "wgrad" else {})


# Each boundary of M, N and K once per layout, with an epilogue input at the edge.  MN-major A needs M % 8 == 0.
EDGE_CASES = [
    ("fwd", 1, 8, 8, "bias"), ("fwd", 8, 56, 16, "res"), ("fwd", 63, 64, 56, "aux_in+gate"),
    ("fwd", 64, 72, 64, "bias+gelu+aux_out"), ("fwd", 65, 120, 72, "res+f32"), ("fwd", 127, 128, 120, "f32+acc"),
    ("fwd", 128, 136, 136, "bias+res"), ("fwd", 129, 264, 8, "bias+qgelu"), ("fwd", 2056, 1032, 72, "aux_out+gate+res"),
    ("fwd", 65, 136, 16384, "f32"), ("fwd", 129, 136, 16384, ""),
    ("fwd", 4096, 264, 64, "bias"), ("dgrad", 4216, 136, 72, "res"),       # tiles_m = 32 (one full group), 33
    ("dgrad", 1, 136, 72, "aux_in"), ("dgrad", 63, 8, 8, "f32+acc+gate"), ("dgrad", 65, 56, 120, "aux_in+relu2"),
    ("dgrad", 129, 72, 16, "res32+f32"), ("dgrad", 127, 120, 136, "alpha+raw_scale"),
    ("dgrad", 2056, 264, 56, "aux_in+gate"), ("dgrad", 64, 128, 16384, ""),
    ("wgrad", 8, 8, 8, "f32"), ("wgrad", 64, 56, 72, "f32+acc"), ("wgrad", 128, 136, 120, "f32+acc+gate"),
    ("wgrad", 2056, 72, 136, "f32"), ("wgrad", 136, 120, 16, "f32+acc"), ("wgrad", 8, 1032, 16384, "f32+acc"),
    ("wgrad", 1024, 128, 16520, "f32+acc"), ("wgrad", 72, 64, 56, "bias"),
]


@gpu
@pytest.mark.parametrize("layout,M,N,K,spec", EDGE_CASES)
def test_edges(layout, M, N, K, spec):
    _run(f"edge[{layout}-{M}-{N}-{K}-{spec}]", Operands(layout, M, N, K, seed=2), _opts(spec))


# every compiled epilogue class (kEpiCls in otb_gemm.cu), and the run-time epilogue options with each combination the
# hot path uses outside those classes: fp32 residual (fp32-grade forward), bias + relu^2 + pre-activation (Persimmon
# up-projection), relu^2'(aux) (Persimmon dgrad), bias + GELU into fp32 (fp32-grade forward); at 8 x 64 = 512 tiles
CLASS_SPECS = ["", "gate", "bias", "bias+qgelu", "bias+res", "res", "gelu+aux_out", "aux_out+gate+res", "aux_in+gate",
               "aux_in", "f32", "f32+gate", "f32+acc", "f32+acc+gate"]
RUNTIME_SPECS = {"res_fp32": "res32+f32", "relu2_aux_out": "bias+relu2+aux_out", "relu2_grad": "aux_in+relu2",
                 "gelu_f32": "bias+gelu+f32"}


@gpu
@pytest.mark.parametrize("cls", list(range(14)) + list(RUNTIME_SPECS))
def test_epilogue_classes(cls):
    o = _opts(CLASS_SPECS[cls] if isinstance(cls, int) else RUNTIME_SPECS[cls])
    assert epi_class_of(o) == (cls if isinstance(cls, int) else -1)
    _run(f"class[{cls}]", Operands("fwd", 1024, 8192, 128), o)


@gpu
def test_bit_identical_runs_and_accumulate_twice():
    from otter_b200 import functional as F
    g = torch.Generator(device=DEV).manual_seed(3)
    x, w = _randn(g, 2048, 4096), _randn(g, 16384, 4096, scale=4096 ** -0.5)
    z1 = torch.empty(2048, 16384, device=DEV, dtype=BF16)
    z2 = torch.empty_like(z1)
    h1 = F.linear_fwd(x, w, act=1, aux_out=z1)
    h2 = F.linear_fwd(x, w, act=1, aux_out=z2)
    assert torch.equal(h1, h2) and torch.equal(z1, z2)
    dz, xa = _randn(g, 2048, 16384), _randn(g, 2048, 4096)
    gw = torch.zeros(16384, 4096, device=DEV)
    F.linear_wgrad(dz, xa, out=gw, accumulate=True)
    once = gw.clone()
    F.linear_wgrad(dz, xa, out=gw, accumulate=True)
    rows = _sample_rows(16384)
    a, b = dz.t()[rows].double(), xa.t().double()
    r = epi_ref(a @ b.t(), a.abs() @ b.abs().t(), c_acc(2048), old=torch.zeros_like(once[rows], dtype=F64))
    _check("wgrad_up accumulate once", once[rows], r["out"], r["E"], F32)
    # 0 + v is v exactly, and the second launch computes the same v bit for bit: v + v = 2 v exactly
    assert torch.equal(gw, 2 * once), "accumulate twice is not exactly twice"


def _sample_rows(M):
    """Output rows the float64 reference of a large launch covers: both ends of every 32-row quarter and the middle
    of each tile, and the last rows."""
    idx = torch.arange(M, device=DEV)
    keep = torch.isin(idx % 128, torch.tensor([0, 1, 30, 31, 32, 33, 62, 63, 64, 65, 94, 95, 96, 97, 126, 127],
                                              device=DEV)) | (idx >= M - 3)
    return idx[keep]


# ------------------------------------------------------------------------------------------------------------------
# GPU: the epilogue specification sweep
# ------------------------------------------------------------------------------------------------------------------
SCALES = {"none": {}, "alpha": {"alpha": -1.625}, "raw": {"gate": 0.6}, "tanh": {"gate": 0.6, "tanh": True},
          "alpha_tanh": {"alpha": 1.5, "gate": -0.7, "tanh": True}}


@gpu
@pytest.mark.parametrize("out", ["bf16", "f32"])
@pytest.mark.parametrize("layout", ["fwd", "dgrad", "wgrad"])
def test_epilogue_sweep(layout, out):
    """Every option combination otb_gemm_bf16 accepts, at one ragged shape: every compiled class and the run-time path
    against the documented order."""
    M, N, K = 200, 136, 136
    ops = Operands(layout, M, N, K, seed=4)
    epi = EpiInputs(ops)
    acc_S = ops.ref()
    outs = [dict(out=BF16, res=None), dict(out=BF16, res="bf16")] if out == "bf16" else \
        [dict(out=F32, res=r, acc=a) for r in (None, "bf16", "f32") for a in (False, True)]
    per_cls = {}
    n = 0
    for bias in (False, True):
        for aux_out in (False, True):
            for act in range(4):
                for aux_in in (False, True):
                    for sc in SCALES.values():
                        for ot in outs:
                            o = dict(bias=bias, aux_out=aux_out, act=act, aux_in=aux_in, **sc, **ot)
                            tag = f"sweep[{layout}-{o}]"
                            _run(tag, ops, o, epi=epi, acc_S=acc_S)
                            c = epi_class_of(o)
                            per_cls[c] = per_cls.get(c, 0) + 1
                            n += 1
    print(f"SWEEP {layout} {out}: {n} combinations; per class {dict(sorted(per_cls.items()))}")
    assert n == 160 * len(outs)


# ------------------------------------------------------------------------------------------------------------------
# GPU: canaries of column-sliced outputs and padded inputs
# ------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("layout,M,N,K,spec", [
    ("fwd", 200, 136, 72, "bias+gelu+aux_out"), ("fwd", 129, 264, 136, "aux_out+gate+res"),
    ("dgrad", 65, 120, 200, "aux_in+alpha+raw_scale"), ("dgrad", 200, 72, 8, "res32+f32+aux_out"),
    ("wgrad", 136, 200, 72, "f32+acc"), ("wgrad", 64, 8, 129, "f32+acc+gate"), ("fwd", 63, 56, 16, "f32+acc+bias"),
])
def test_canaries_column_slices(layout, M, N, K, spec):
    """Outputs are offset column slices (col0 = 24 / 40, row 1 of a wider buffer); operands sit at odd 8-column
    offsets with pitches far above their extents and NaN past K and past M / N.  `_run` checks that the owned elements
    are finite and within the bound and that every other element kept its bits (a finite sentinel for accumulate)."""
    a_kw = dict(col0=56, pitch=-(-(K + M + 200) // 8) * 8)
    b_kw = dict(col0=120, pitch=-(-(K + N + 304) // 8) * 8, row0=3)
    ops = Operands(layout, M, N, K, seed=5, a_kw=a_kw, b_kw=b_kw)
    _run(f"canary[{layout}-{M}-{N}-{K}-{spec}]", ops, _opts(spec), out_kw=dict(col0=24, pitch=N + 64, row0=2))


# ------------------------------------------------------------------------------------------------------------------
# GPU: schedule invariance (bitwise)
# ------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("layout", ["fwd", "dgrad", "wgrad"])
def test_schedule_invariance(layout):
    """Rows of a launch with many tiles per CTA equal, bit for bit, the same rows computed by a launch of one M-tile
    (a different CTA and warpgroup) and by a launch of one N window: the k order of a tile does not depend on where
    the tile runs.  M = 16520: 130 M-tiles, a ragged last group of 2, the last tile 8 rows."""
    M, N, K = 16520, 384, 256
    ops = Operands(layout, M, N, K, seed=6)
    out_dt = F32 if layout == "wgrad" else BF16
    epi = dict(act=1) if layout == "fwd" else {}
    full = _run(f"invariance[{layout}] full", ops, dict(out=out_dt, **epi), rows=_sample_rows(M))
    a_mn, b_mn = LAYOUTS[layout]
    for t in (0, 31, 32, 67, 129):
        m0, mw = 128 * t, min(128, M - 128 * t)
        A = ops.ca.v[:, m0:m0 + mw] if a_mn else ops.ca.v[m0:m0 + mw]
        out = torch.full((mw, N), float("nan"), dtype=out_dt, device=DEV)
        _launch(layout, A, ops.cb.v, mw, N, K, out, **epi)
        torch.cuda.synchronize()
        assert torch.equal(out, full[m0:m0 + mw]), f"{layout}: M-tile {t} differs from the full launch"
    B = ops.cb.v[:, 128:256] if b_mn else ops.cb.v[128:256]
    out = torch.full((M, 128), float("nan"), dtype=out_dt, device=DEV)
    _launch(layout, ops.ca.v, B, M, 128, K, out, **epi)
    torch.cuda.synchronize()
    assert torch.equal(out, full[:, 128:256]), f"{layout}: the N window differs from the full launch"


# ------------------------------------------------------------------------------------------------------------------
# GPU: hot-path shapes at full size (the float64 reference covers _sample_rows of each output)
# ------------------------------------------------------------------------------------------------------------------
HOT = {
    # bench c2 gated FFN (D 4096, 4 x D): up-projection + GELU, down-projection * tanh gate + residual, and backward
    "ffn_up_fwd": ("fwd", 2048, 16384, 4096, "gelu+aux_out", {}),
    "ffn_down_fwd": ("fwd", 2048, 4096, 16384, "gate+res", {}),
    "ffn_down_dgrad": ("dgrad", 2048, 16384, 4096, "aux_in+gate", {}),
    "ffn_up_dgrad": ("dgrad", 2048, 4096, 16384, "", {}),
    "ffn_up_wgrad": ("wgrad", 16384, 4096, 2048, "f32+acc", {}),
    # CLIP ViT-L/14 at 8 images x 257 tokens
    "clip_qkv": ("fwd", 2056, 3072, 1024, "bias", {}),
    "clip_fc1": ("fwd", 2056, 4096, 1024, "bias+qgelu", {}),
    "clip_fc2": ("fwd", 2056, 1024, 4096, "bias+res", {}),
    "clip_fc1_wgrad": ("wgrad", 4096, 1024, 2056, "f32+acc", {}),
    # LLaMA-7B layer at S = 2048: k written into qkv[:, D:2D]; dgrad reading dqkv[:, D:2D] as a strided A
    "llama_k_slice": ("fwd", 2048, 4096, 4096, "", dict(out_kw=dict(col0=4096, pitch=3 * 4096, row0=0))),
    "llama_k_dgrad_strided": ("dgrad", 2048, 4096, 4096, "res", dict(a_kw=dict(col0=4096, pitch=3 * 4096, row0=0))),
    "llama_down": ("fwd", 2048, 4096, 11008, "res", {}),
}


@gpu
@pytest.mark.parametrize("name", list(HOT))
def test_hot_path_shapes(name):
    layout, M, N, K, spec, kw = HOT[name]
    ops = Operands(layout, M, N, K, seed=7, a_kw=kw.get("a_kw"))
    _run(f"hot[{name}]", ops, _opts(spec), rows=_sample_rows(M), out_kw=kw.get("out_kw"))


# ------------------------------------------------------------------------------------------------------------------
# GPU: the fp32-grade route
# ------------------------------------------------------------------------------------------------------------------
# 6K around F32_KCHUNK = 512: 480 and 504 (one fused launch), 528 (two chunks), 1032, 3096 (2 and 6 full chunks + a
# short one).  The split operand [rows][6K] bf16 needs a 16-byte row pitch, so K is a multiple of 4.
@gpu
@pytest.mark.parametrize("K", [80, 84, 88, 172, 516])
@pytest.mark.parametrize("spec", ["", "bias", "bias+gelu", "bias+qgelu", "gate+res", "bias+gelu+gate+res",
                                  "raw_scale+res"])
def test_linear_f32_grade(K, spec):
    from otter_b200 import functional as F
    M, N = 136, 72
    o = _opts(spec)
    g = torch.Generator(device=DEV).manual_seed(8 * K + len(spec))
    x, w = _randn(g, M, K, dtype=F32), _randn(g, N, K, scale=K ** -0.5, dtype=F32)
    bias = _randn(g, N, dtype=F32) if o.get("bias") else None
    res = _randn(g, M, N, dtype=F32) if o.get("res") else None
    gate = torch.tensor([o["gate"]], device=DEV) if "gate" in o else None
    got = F.linear_f32(x, F.split3_concat(w, 1), N, bias=bias, act=o.get("act", 0), scale_ptr=gate,
                       scale_tanh=bool(o.get("tanh")), residual=res)
    x64, w64 = x.double(), w.double()
    r = epi_ref(x64 @ w64.t(), x64.abs() @ w64.abs().t(), c_acc_f32grade(K),
                bias=None if bias is None else bias.double(), act=o.get("act", 0), gate=o.get("gate"),
                tanh=bool(o.get("tanh")), residual=None if res is None else res.double())
    _check(f"f32grade[{K}-{spec}]", got, r["out"], r["E"], F32)
