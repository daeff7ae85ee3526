"""CPU: the ALGORITHM csrc/otb_attn_lm.cu implements (log2-domain two-sweep softmax with the ALiBi key bias folded into
the exponent, causal per-row key ranges per key tile (128 keys forward, 64 backward), LSE hand-over to the backward,
dS = P (dP - delta) scale, dQ accumulated across key tiles) restated in numpy and checked against autograd of the
reference-pinned oracle.  It validates the formulas of the kernel — tile loop bounds, bias offsets, log domains — not the
wgmma plumbing."""
import math

import numpy as np
import torch

from oracle import restatement_lm as R

LOG2E = 1.4426950408889634


def _row_hi(S, causal, row, k0, tk=128):
    valid = min(tk, S - k0)
    return max(0, min(valid, row - k0 + 1)) if causal else valid


def kernel_algorithm(q, k, v, dout, slope, causal):
    """q,k,v,dout: [S,128] float32 of one (batch, head).  Returns out, lse, dq, dk, dv following the kernel loops."""
    S = q.shape[0]
    scale = 1.0 / math.sqrt(128)
    scale_log2, slope2 = np.float32(scale * LOG2E), np.float32(slope * LOG2E)
    nt_all = (S + 127) // 128
    out, lse = np.zeros((S, 128), np.float32), np.zeros(S, np.float32)
    for qt in range(nt_all):
        nt = min(nt_all, qt + 1) if causal else nt_all
        rows = range(qt * 128, min(S, qt * 128 + 128))
        for row in rows:
            m, l, acc = -np.inf, np.float32(0), np.zeros(128, np.float32)
            for sweep in (0, 1):
                for j in range(nt):
                    hi = _row_hi(S, causal, row, j * 128)
                    kf0 = np.float32(j * 128 - (S - 1))
                    for cc in range(hi):
                        s = np.float32(q[row] @ k[j * 128 + cc])
                        t = s * scale_log2 + slope2 * (kf0 + np.float32(cc))
                        if sweep == 0:
                            m = max(m, t)
                        else:
                            p = np.float32(2.0 ** (t - m))
                            l += p
                            acc += p * v[j * 128 + cc]
            out[row] = acc / l
            lse[row] = (m + math.log2(l)) * 0.6931471805599453
    dq, dk, dv = np.zeros_like(q), np.zeros_like(k), np.zeros_like(v)
    delta = (dout * out).sum(1)
    for j in range((S + 63) // 64):                      # backward: 64-key tiles, query tiles of 128 rows
        k0 = j * 64
        for i in range(k0 // 128 if causal else 0, nt_all):
            for row in range(i * 128, min(S, i * 128 + 128)):
                hi = _row_hi(S, causal, row, k0, 64)
                kf0 = np.float32(k0 - (S - 1))
                for cc in range(hi):
                    key = k0 + cc
                    t = np.float32(q[row] @ k[key]) * scale_log2 + slope2 * (kf0 + np.float32(cc))
                    pr = np.float32(2.0 ** (t - lse[row] * LOG2E))
                    dp = np.float32(dout[row] @ v[key])
                    ds = pr * (dp - delta[row]) * scale
                    dv[key] += pr * dout[row]
                    dk[key] += ds * q[row]
                    dq[row] += ds * k[key]
    return out, lse, dq, dk, dv


def _oracle(q, k, v, dout, slope, causal):
    S = q.shape[0]
    tq, tk, tv = (torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (q, k, v))
    w = tq @ tk.T / math.sqrt(128)
    w = w + slope * torch.arange(1 - S, 1, dtype=torch.float64)[None, :]      # == R.alibi_key_bias row for this head
    if causal:
        w = w.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
    o = torch.softmax(w, -1) @ tv
    o.backward(torch.tensor(dout, dtype=torch.float64))
    return o.detach().numpy(), tq.grad.numpy(), tk.grad.numpy(), tv.grad.numpy()


def test_kernel_algorithm_matches_autograd():
    rng = np.random.RandomState(0)
    slope = float(R.alibi_slopes(8)[2])
    for S, causal, sl in ((150, True, slope), (70, True, 0.0), (140, False, slope)):
        q, k, v, dout = (rng.randn(S, 128).astype(np.float32) * 0.5 for _ in range(4))
        out, lse, dq, dk, dv = kernel_algorithm(q, k, v, dout, sl, causal)
        o, gq, gk, gv = _oracle(q, k, v, dout, sl, causal)
        assert np.abs(out - o).max() < 1e-4
        for got, want in ((dq, gq), (dk, gk), (dv, gv)):
            assert np.abs(got - want).max() < 1e-3 * max(1.0, np.abs(want).max())


def test_oracle_bias_is_what_the_kernel_adds():
    b = R.alibi_key_bias(8, 150)
    s = R.alibi_slopes(8)
    assert torch.allclose(b[2], s[2] * torch.arange(1 - 150, 1, dtype=torch.float32))
