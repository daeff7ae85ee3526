"""CPU model of the TMA-store epilogue's addressing (csrc/otb_gemm.cu epilogue_tile): every lane writes its 16 B
units into the warp's SWIZZLE_128B stage exactly as the kernel does; a model of the TMA engine (de-swizzle by
unit ^ (row & 7), clip the 32-row x 128-byte box against the tensor) stores it.  The result must equal the plain
tile for bf16 and fp32 outputs, full and ragged M / N, BN = 128 and 256."""
import numpy as np


def run_tile(acc, M, N, m0, n0, BN, out_fp32):
    """acc: [128, BN] float32 accumulator tile of one CTA.  Returns the [M, N] output it would produce."""
    esz = 4 if out_fp32 else 2
    cols_per_box = 128 // esz
    out = np.full((M, N), np.nan, np.float32)
    for warp in range(8):
        q, half = warp & 3, warp >> 2
        row0 = m0 + q * 32
        if row0 >= M:
            continue
        stage = np.full((32, 8, 16 // esz), np.nan, np.float32)      # [row][physical 16 B unit][elements]
        for c in range(half * (BN // 64), (half + 1) * (BN // 64)):
            colbase = n0 + c * 32
            if colbase >= N:
                break
            last_of_box = out_fp32 or (c & 1) == 1 or colbase + 32 >= N
            for lane in range(32):
                xr = lane & 7
                for g in range(4):
                    v = acc[q * 32 + lane, c * 32 + g * 8: c * 32 + g * 8 + 8]
                    if out_fp32:
                        stage[lane, (2 * g) ^ xr] = v[:4]
                        stage[lane, (2 * g + 1) ^ xr] = v[4:]
                    else:
                        stage[lane, ((c & 1) * 4 + g) ^ xr] = v
            if last_of_box:
                box_col = colbase if out_fp32 else (colbase & ~63)
                for r in range(32):                                  # the TMA engine: de-swizzle + clip
                    for u in range(8):
                        data = stage[r, u ^ (r & 7)]
                        for e in range(16 // esz):
                            col = box_col + u * (16 // esz) + e
                            if row0 + r < M and col < N and col < box_col + cols_per_box:
                                out[row0 + r, col] = data[e]
    return out


def test_staging_layout_roundtrip():
    rng = np.random.RandomState(0)
    for BN in (128, 256):
        for out_fp32 in (False, True):
            for (M, N, m0, n0) in ((128, BN, 0, 0), (200, BN + 40, 128, 0), (200, BN + 40, 128, BN), (300, 40, 256, 0),
                                   (520, 3 * BN - 24, 512, 2 * BN)):
                acc = rng.randn(128, BN).astype(np.float32)
                got = run_tile(acc, M, N, m0, n0, BN, out_fp32)
                want = np.full((M, N), np.nan, np.float32)
                rows, cols = min(128, M - m0), min(BN, N - n0)
                if rows > 0 and cols > 0:
                    want[m0:m0 + rows, n0:n0 + cols] = acc[:rows, :cols]
                assert np.array_equal(np.isnan(got), np.isnan(want)), (BN, out_fp32, M, N, m0, n0)
                assert np.array_equal(np.nan_to_num(got), np.nan_to_num(want)), (BN, out_fp32, M, N, m0, n0)
