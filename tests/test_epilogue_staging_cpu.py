"""CPU model of the TMA-store epilogue's addressing (csrc/otb_gemm.cu epilogue_tile): every lane writes its 16 B
units into its warp's SWIZZLE_128B stage exactly as the kernel does; a model of the TMA engine (de-swizzle by
unit ^ (row & 7), clip the 32-row x 128-byte box against the tensor) stores it.

The walk is the kernel's: MMA warpgroup wg (warps 4 wg .. 4 wg + 3) owns a whole 128 x 128 tile and runs the epilogue
on its two 64-row halves h in turn.  Warp w takes the 32-row quarter q = w & 1 of the half and the column half
half = (w >> 1) & 1, and reuses its own 4 KB stage for every box of both halves.  The result must equal the plain tile
for bf16 and fp32 outputs, full and ragged M / N, from either warpgroup."""
import numpy as np

BM, BN = 128, 128


def run_tile(acc, M, N, m0, n0, out_fp32, wg=0):
    """acc: [128, 128] float32 accumulator tile (the park tile).  Returns the [M, N] output it would produce."""
    esz = 4 if out_fp32 else 2
    cols_per_box = 128 // esz
    out = np.full((M, N), np.nan, np.float32)
    for warp in range(4 * wg, 4 * wg + 4):
        q, half = warp & 1, (warp >> 1) & 1
        stage = np.full((32, 8, 16 // esz), np.nan, np.float32)      # [row][physical 16 B unit][elements], per warp
        for h in range(2):
            row0 = m0 + 64 * h + q * 32
            if row0 >= M:
                continue
            for c in range(half * (BN // 64), (half + 1) * (BN // 64)):
                colbase = n0 + c * 32
                if colbase >= N:
                    break
                last_of_box = out_fp32 or (c & 1) == 1 or colbase + 32 >= N
                for lane in range(32):
                    xr = lane & 7
                    for g in range(4):
                        v = acc[64 * h + q * 32 + lane, c * 32 + g * 8: c * 32 + g * 8 + 8]
                        if out_fp32:
                            stage[lane, (2 * g) ^ xr] = v[:4]
                            stage[lane, (2 * g + 1) ^ xr] = v[4:]
                        else:
                            stage[lane, ((c & 1) * 4 + g) ^ xr] = v
                if last_of_box:
                    box_col = colbase if out_fp32 else (colbase & ~63)
                    for r in range(32):                              # the TMA engine: de-swizzle + clip
                        for u in range(8):
                            data = stage[r, u ^ (r & 7)]
                            for e in range(16 // esz):
                                col = box_col + u * (16 // esz) + e
                                if row0 + r < M and col < N and col < box_col + cols_per_box:
                                    out[row0 + r, col] = data[e]
    return out


def test_staging_layout_roundtrip():
    rng = np.random.RandomState(0)
    for out_fp32 in (False, True):
        for wg in (0, 1):
            for (M, N, m0, n0) in ((128, 128, 0, 0), (200, 168, 128, 0), (200, 168, 128, 128), (300, 40, 256, 0),
                                   (520, 360, 512, 256), (63, 8, 0, 0), (65, 136, 0, 128), (129, 72, 128, 0),
                                   (100, 128, 0, 0)):
                acc = rng.randn(BM, BN).astype(np.float32)
                got = run_tile(acc, M, N, m0, n0, out_fp32, wg)
                want = np.full((M, N), np.nan, np.float32)
                rows, cols = min(BM, M - m0), min(BN, N - n0)
                if rows > 0 and cols > 0:
                    want[m0:m0 + rows, n0:n0 + cols] = acc[:rows, :cols]
                what = (out_fp32, wg, M, N, m0, n0)
                assert np.array_equal(np.isnan(got), np.isnan(want)), what
                assert np.array_equal(np.nan_to_num(got), np.nan_to_num(want)), what
