// otter_b200 — HBM-bound passes of the hot path: LayerNorm fwd/bwd, mask index construction,
// casts, broadcast / grouped reductions, tanh-gate gradient, CLIP embedding assembly, Fuyu scatter.
// All are plain coalesced, 16-byte-vectorised CUDA kernels (no tensor cores: byte/element work).
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

// ------------------------------------------------------------------------------------------------
// LayerNorm forward: one warp per row, 3 sweeps over the row (2nd/3rd hit L1), fp32 statistics.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const bf16* __restrict__ x, long long ldx, const float* __restrict__ gamma,
              const float* __restrict__ beta, bf16* __restrict__ y, long long ldy, float* __restrict__ mean_out,
              float* __restrict__ rstd_out, int rows, int D, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= rows) return;
  const bf16* xr = x + static_cast<long long>(row) * ldx;
  const int nvec = D >> 3;
  float s = 0.f;
  for (int v = lane; v < nvec; v += 32) {
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(xr) + v), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) s += f[i];
  }
  const float mean = warp_sum(s) / D;
  float ss = 0.f;
  for (int v = lane; v < nvec; v += 32) {
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(xr) + v), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float d = f[i] - mean; ss += d * d; }
  }
  const float rstd = rsqrtf(warp_sum(ss) / D + eps);
  bf16* yr = y + static_cast<long long>(row) * ldy;
  for (int v = lane; v < nvec; v += 32) {
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(xr) + v), f);
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v + 1);
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * v), b1 = __ldg(reinterpret_cast<const float4*>(beta) + 2 * v + 1);
    f[0] = (f[0] - mean) * rstd * g0.x + b0.x; f[1] = (f[1] - mean) * rstd * g0.y + b0.y;
    f[2] = (f[2] - mean) * rstd * g0.z + b0.z; f[3] = (f[3] - mean) * rstd * g0.w + b0.w;
    f[4] = (f[4] - mean) * rstd * g1.x + b1.x; f[5] = (f[5] - mean) * rstd * g1.y + b1.y;
    f[6] = (f[6] - mean) * rstd * g1.z + b1.z; f[7] = (f[7] - mean) * rstd * g1.w + b1.w;
    reinterpret_cast<uint4*>(yr)[v] = pack8(f);
  }
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
}

// LayerNorm backward, input gradient: dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma
__global__ void __launch_bounds__(256)
ln_bwd_dx_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x, long long ldx,
                 const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                 const bf16* __restrict__ add, long long ldadd, bf16* __restrict__ dx, long long lddx, int rows,
                 int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= rows) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + static_cast<long long>(row) * ldx);
  const uint4* dr = reinterpret_cast<const uint4*>(dy + static_cast<long long>(row) * lddy);
  const float mu = mean[row], rs = rstd[row];
  const int nvec = D >> 3;
  float s1 = 0.f, s2 = 0.f;
  for (int v = lane; v < nvec; v += 32) {
    float fx[8], fd[8];
    unpack8(__ldg(xr + v), fx);
    unpack8(__ldg(dr + v), fd);
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v + 1);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float g = fd[i] * gg[i];
      s1 += g;
      s2 += g * (fx[i] - mu) * rs;
    }
  }
  s1 = warp_sum(s1) / D;
  s2 = warp_sum(s2) / D;
  uint4* outr = reinterpret_cast<uint4*>(dx + static_cast<long long>(row) * lddx);
  const uint4* addr = add ? reinterpret_cast<const uint4*>(add + static_cast<long long>(row) * ldadd) : nullptr;
  for (int v = lane; v < nvec; v += 32) {
    float fx[8], fd[8], fa[8];
    unpack8(__ldg(xr + v), fx);
    unpack8(__ldg(dr + v), fd);
    if (addr) unpack8(__ldg(addr + v), fa);
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v + 1);
    const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float xh = (fx[i] - mu) * rs;
      o[i] = rs * (fd[i] * gg[i] - s1 - xh * s2) + (addr ? fa[i] : 0.f);
    }
    outr[v] = pack8(o);
  }
}

// LayerNorm backward, parameter gradients: column partial sums over a chunk of rows.
// block (32, 8): x -> column pair, y -> row lane.  ws layout: [2][chunks][D] (0: dgamma, 1: dbeta)
__global__ void __launch_bounds__(256)
ln_bwd_param_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x, long long ldx,
                    const float* __restrict__ mean, const float* __restrict__ rstd, float* __restrict__ ws, int rows,
                    int D, int chunks) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sg[8][64], sb[8][64];
  const int col = blockIdx.x * 64 + threadIdx.x * 2;
  const int chunk = blockIdx.y;
  const int rows_per = (rows + chunks - 1) / chunks;
  const int r0 = chunk * rows_per, r1 = min(rows, r0 + rows_per);
  float g0 = 0.f, g1 = 0.f, b0 = 0.f, b1 = 0.f;
  if (col < D) {
    for (int r = r0 + threadIdx.y; r < r1; r += 8) {
      const float2 d = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dy + static_cast<long long>(r) * lddy + col));
      const float2 xv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + static_cast<long long>(r) * ldx + col));
      const float mu = mean[r], rs = rstd[r];
      g0 += d.x * (xv.x - mu) * rs; g1 += d.y * (xv.y - mu) * rs;
      b0 += d.x; b1 += d.y;
    }
  }
  sg[threadIdx.y][threadIdx.x * 2] = g0; sg[threadIdx.y][threadIdx.x * 2 + 1] = g1;
  sb[threadIdx.y][threadIdx.x * 2] = b0; sb[threadIdx.y][threadIdx.x * 2 + 1] = b1;
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  if (t < 128) {
    const int c = t & 63, which = t >> 6;
    float acc = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) acc += which ? sb[y][c] : sg[y][c];
    const int gc = blockIdx.x * 64 + c;
    if (gc < D) ws[(static_cast<long long>(which) * chunks + chunk) * D + gc] = acc;
  }
}
// One-pass LayerNorm backward (D <= 4096): dx AND the gamma/beta column partials from a single read of
// x / dy.  A CTA walks its rows in batches of kLnR; thread t owns the 16 B column vectors t, t+256, ... (VPT of them) of
// every row, so the parameter partials stay in its registers across all rows of the CTA (deterministic: fixed order,
// no atomics) and the two row statistics of a batch take one block reduction (double-buffered smem, one barrier).
// ws layout is the one ln_bwd_finalize_kernel reads: [2][gridDim.x][D].
constexpr int kLnR = 4;
template <int VPT>
__global__ void __launch_bounds__(256)
ln_bwd_fused_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x, long long ldx,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                    const bf16* __restrict__ add, long long ldadd, bf16* __restrict__ dx, long long lddx,
                    float* __restrict__ ws, int rows, int D) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[2][8][2 * kLnR];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nvec = D >> 3;
  float gam[VPT][8], pg[VPT][8], pb[VPT][8];
#pragma unroll
  for (int j = 0; j < VPT; ++j) {
    const int v = threadIdx.x + j * 256;
#pragma unroll
    for (int i = 0; i < 8; ++i) { pg[j][i] = 0.f; pb[j][i] = 0.f; gam[j][i] = 0.f; }
    if (v < nvec) {
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * v + 1);
      gam[j][0] = g0.x; gam[j][1] = g0.y; gam[j][2] = g0.z; gam[j][3] = g0.w;
      gam[j][4] = g1.x; gam[j][5] = g1.y; gam[j][6] = g1.z; gam[j][7] = g1.w;
    }
  }
  const int nbatch = (rows + kLnR - 1) / kLnR;
  int parity = 0;
  for (int b = blockIdx.x; b < nbatch; b += gridDim.x, parity ^= 1) {
    const int r0 = b * kLnR;
    uint4 ux[kLnR][VPT], ud[kLnR][VPT];
    float mu[kLnR], rs[kLnR];
#pragma unroll
    for (int r = 0; r < kLnR; ++r) {
      const int row = r0 + r;
      const bool ok = row < rows;
      mu[r] = ok ? __ldg(mean + row) : 0.f;
      rs[r] = ok ? __ldg(rstd + row) : 0.f;
#pragma unroll
      for (int j = 0; j < VPT; ++j) {
        const int v = threadIdx.x + j * 256;
        ux[r][j] = make_uint4(0u, 0u, 0u, 0u);
        ud[r][j] = make_uint4(0u, 0u, 0u, 0u);
        if (ok && v < nvec) {
          ux[r][j] = __ldg(reinterpret_cast<const uint4*>(x + static_cast<long long>(row) * ldx) + v);
          ud[r][j] = __ldg(reinterpret_cast<const uint4*>(dy + static_cast<long long>(row) * lddy) + v);
        }
      }
    }
    // per-row sums of g = dy*gamma and g*xhat, and the column partials (dgamma += dy*xhat, dbeta += dy)
    float s[2 * kLnR];
#pragma unroll
    for (int r = 0; r < kLnR; ++r) {
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int j = 0; j < VPT; ++j) {
        float fx[8], fd[8];
        unpack8(ux[r][j], fx);
        unpack8(ud[r][j], fd);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float xh = (fx[i] - mu[r]) * rs[r];         // rows >= `rows` and vectors >= nvec hold zeros (rs = 0)
          const float g = fd[i] * gam[j][i];
          s1 += g;
          s2 += g * xh;
          pg[j][i] += fd[i] * xh;
          pb[j][i] += fd[i];
        }
      }
      s[2 * r] = warp_sum(s1);
      s[2 * r + 1] = warp_sum(s2);
    }
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 2 * kLnR; ++k) red[parity][warp][k] = s[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2 * kLnR; ++k) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += red[parity][w][k];
      s[k] = t / D;
    }
    if (dx != nullptr) {
#pragma unroll
      for (int r = 0; r < kLnR; ++r) {
        const int row = r0 + r;
        if (row >= rows) break;
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
          const int v = threadIdx.x + j * 256;
          if (v >= nvec) continue;
          float fx[8], fd[8], fa[8], o[8];
          unpack8(ux[r][j], fx);
          unpack8(ud[r][j], fd);
          if (add != nullptr) unpack8(__ldg(reinterpret_cast<const uint4*>(add + static_cast<long long>(row) * ldadd) + v), fa);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float xh = (fx[i] - mu[r]) * rs[r];
            o[i] = rs[r] * (fd[i] * gam[j][i] - s[2 * r] - xh * s[2 * r + 1]) + (add != nullptr ? fa[i] : 0.f);
          }
          reinterpret_cast<uint4*>(dx + static_cast<long long>(row) * lddx)[v] = pack8(o);
        }
      }
    }
  }
  if (ws != nullptr) {
    const long long chunks = gridDim.x;
#pragma unroll
    for (int j = 0; j < VPT; ++j) {
      const int v = threadIdx.x + j * 256;
      if (v >= nvec) continue;
      float* wg = ws + (0 * chunks + blockIdx.x) * D + v * 8;
      float* wb = ws + (1 * chunks + blockIdx.x) * D + v * 8;
      *reinterpret_cast<float4*>(wg) = make_float4(pg[j][0], pg[j][1], pg[j][2], pg[j][3]);
      *reinterpret_cast<float4*>(wg + 4) = make_float4(pg[j][4], pg[j][5], pg[j][6], pg[j][7]);
      *reinterpret_cast<float4*>(wb) = make_float4(pb[j][0], pb[j][1], pb[j][2], pb[j][3]);
      *reinterpret_cast<float4*>(wb + 4) = make_float4(pb[j][4], pb[j][5], pb[j][6], pb[j][7]);
    }
  }
}

__global__ void ln_bwd_finalize_kernel(const float* __restrict__ ws, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, int D, int chunks, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= D) return;
  float g = 0.f, b = 0.f;
  for (int k = 0; k < chunks; ++k) {
    g += ws[static_cast<long long>(k) * D + c];
    b += ws[(static_cast<long long>(chunks) + k) * D + c];
  }
  if (dgamma) dgamma[c] = (accumulate ? dgamma[c] : 0.f) + g;
  if (dbeta) dbeta[c] = (accumulate ? dbeta[c] : 0.f) + b;
}

// Wide finalize for the one-pass kernel's [2][chunks][D] partials (chunks up to one per SM): a CTA owns 32 columns,
// its 8 thread rows stride over the chunks (coalesced 128 B reads), then a fixed-order smem reduction (deterministic).
__global__ void __launch_bounds__(256)
ln_bwd_finalize_wide_kernel(const float* __restrict__ ws, float* __restrict__ dgamma, float* __restrict__ dbeta, int D,
                            int chunks, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sg[8][32], sb[8][32];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float g = 0.f, b = 0.f;
  if (c < D) {
    for (int k = threadIdx.y; k < chunks; k += 8) {
      g += ws[static_cast<long long>(k) * D + c];
      b += ws[(static_cast<long long>(chunks) + k) * D + c];
    }
  }
  sg[threadIdx.y][threadIdx.x] = g;
  sb[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < D) {
    float tg = 0.f, tb = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) { tg += sg[y][threadIdx.x]; tb += sb[y][threadIdx.x]; }
    if (dgamma) dgamma[c] = (accumulate ? dgamma[c] : 0.f) + tg;
    if (dbeta) dbeta[c] = (accumulate ? dbeta[c] : 0.f) + tb;
  }
}

// ------------------------------------------------------------------------------------------------
// text_time (integer, bit-exact)  modeling_otter.py:296-311 — one thread per batch row (L <= few K)
// ------------------------------------------------------------------------------------------------
__global__ void text_time_kernel(const uint8_t* __restrict__ loc, int B, int L, int attend_previous,
                                 int* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const uint8_t* l = loc + static_cast<long long>(b) * L;
  int* o = out + static_cast<long long>(b) * L;
  int total = 0;
  if (!attend_previous)
    for (int i = 0; i < L; ++i) total += l[i] ? 1 : 0;
  int run = 0;
  for (int i = 0; i < L; ++i) {
    const bool m = l[i] != 0;
    run += m ? 1 : 0;
    int t = run;
    if (!attend_previous) {
      if (!m) t += 1;
      if (t > total) t = 0;
    }
    o[i] = t;
  }
}

// ------------------------------------------------------------------------------------------------
// casts / broadcasts / reductions
// ------------------------------------------------------------------------------------------------
__global__ void cast_f32_bf16_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long n) {
  pdl_launch_dependents();
  pdl_wait();
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 8;
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src + i)), b = __ldg(reinterpret_cast<const float4*>(src + i + 4));
      const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      *reinterpret_cast<uint4*>(dst + i) = pack8(f);
    } else {
      for (long long k = i; k < n; ++k) dst[k] = __float2bfloat16(src[k]);
    }
  }
}
// Multi-tensor cast: one launch re-derives the bf16 copies of a whole list of fp32 tensors.  The device table holds one
// {src, dst, n, first_block} record per tensor; block b finds its tensor by binary search over first_block and
// converts elements [(b - first_block) * 4096, +4096) of it.
struct CastSeg {
  const float* src;
  bf16* dst;
  long long n;
  long long blk0;
};
static_assert(sizeof(CastSeg) == 32, "table layout is part of the C ABI: 4 x int64 per tensor");
constexpr int kCastSegElems = 4096;
__global__ void __launch_bounds__(256) cast_multi_kernel(const CastSeg* __restrict__ segs, int nseg) {
  pdl_launch_dependents();
  pdl_wait();
  const long long b = blockIdx.x;
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&segs[mid].blk0) <= b) lo = mid; else hi = mid - 1;
  }
  const float* src = segs[lo].src;
  bf16* dst = segs[lo].dst;
  const long long n = segs[lo].n;
  const long long base = (b - segs[lo].blk0) * kCastSegElems;
#pragma unroll
  for (int it = 0; it < kCastSegElems / (256 * 8); ++it) {
    const long long i = base + (static_cast<long long>(it) * 256 + threadIdx.x) * 8;
    if (i + 8 <= n) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src + i)), c = __ldg(reinterpret_cast<const float4*>(src + i + 4));
      const float f[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
      *reinterpret_cast<uint4*>(dst + i) = pack8(f);
    } else {
      for (long long k = i; k < n; ++k) dst[k] = __float2bfloat16(src[k]);
    }
  }
}
__global__ void cast_bf16_f32_kernel(const bf16* __restrict__ src, float* __restrict__ dst, long long n) {
  pdl_launch_dependents();
  pdl_wait();
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 8;
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float f[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(src + i)), f);
      *reinterpret_cast<float4*>(dst + i) = make_float4(f[0], f[1], f[2], f[3]);
      *reinterpret_cast<float4*>(dst + i + 4) = make_float4(f[4], f[5], f[6], f[7]);
    } else {
      for (long long k = i; k < n; ++k) dst[k] = __bfloat162float(src[k]);
    }
  }
}
// dst = float(src) * scale : the up-cast after a reduced-precision all-reduce(SUM), with the 1/world_size folded in
__global__ void cast_bf16_f32_scale_kernel(const bf16* __restrict__ src, float* __restrict__ dst, long long n, float scale) {
  pdl_launch_dependents();
  pdl_wait();
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 8;
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8; i < n; i += stride) {
    if (i + 8 <= n) {
      float f[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(src + i)), f);
      *reinterpret_cast<float4*>(dst + i) = make_float4(f[0] * scale, f[1] * scale, f[2] * scale, f[3] * scale);
      *reinterpret_cast<float4*>(dst + i + 4) = make_float4(f[4] * scale, f[5] * scale, f[6] * scale, f[7] * scale);
    } else {
      for (long long k = i; k < n; ++k) dst[k] = __bfloat162float(src[k]) * scale;
    }
  }
}
__global__ void bcast_rows_kernel(const float* __restrict__ src, int div, int mod, bf16* __restrict__ out, int rows,
                                  int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = D >> 3;
  const long long total = static_cast<long long>(rows) * nvec;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / nvec), v = static_cast<int>(i % nvec);
    const float* s = src + static_cast<long long>((r / div) % mod) * D + v * 8;
    const float4 a = __ldg(reinterpret_cast<const float4*>(s)), b = __ldg(reinterpret_cast<const float4*>(s + 4));
    const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    reinterpret_cast<uint4*>(out + static_cast<long long>(r) * D)[v] = pack8(f);
  }
}

// out[r,:] = x[r,:] + bias[(r/div)%mod,:]   (frame_embs broadcast add, modeling_otter.py:224-226)
__global__ void add_rowbias_kernel(const bf16* __restrict__ x, const float* __restrict__ bias, int div, int mod,
                                   bf16* __restrict__ out, int rows, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = D >> 3;
  const long long total = static_cast<long long>(rows) * nvec;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / nvec), v = static_cast<int>(i % nvec);
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + static_cast<long long>(r) * D) + v), f);
    const float* s = bias + static_cast<long long>((r / div) % mod) * D + v * 8;
    const float4 a = __ldg(reinterpret_cast<const float4*>(s)), b = __ldg(reinterpret_cast<const float4*>(s + 4));
    f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w; f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
    reinterpret_cast<uint4*>(out + static_cast<long long>(r) * D)[v] = pack8(f);
  }
}
// out[g, c] (+)= sum over rows r with (r/div)%mod == g.  block (32,8): 64 columns x 8 row lanes; grid (D/64, mod)
__global__ void __launch_bounds__(256)
grouped_colsum_kernel(const bf16* __restrict__ x, long long ldx, int rows, int D, int div, int mod,
                      float* __restrict__ out, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s[8][64];
  const int col = blockIdx.x * 64 + threadIdx.x * 2;
  const int g = blockIdx.y;
  float a0 = 0.f, a1 = 0.f;
  if (col < D) {
    // rows of group g: r = (k*mod + g)*div + e, e in [0,div)
    const long long per = static_cast<long long>(div);
    for (long long blk = g; blk * per < rows; blk += mod) {
      for (long long e = threadIdx.y; e < per; e += 8) {
        const long long r = blk * per + e;
        if (r < rows) {
          const float2 v = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + r * ldx + col));
          a0 += v.x; a1 += v.y;
        }
      }
    }
  }
  s[threadIdx.y][threadIdx.x * 2] = a0; s[threadIdx.y][threadIdx.x * 2 + 1] = a1;
  __syncthreads();
  const int t = threadIdx.y * 32 + threadIdx.x;
  if (t < 64) {
    float acc = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) acc += s[y][t];
    const int gc = blockIdx.x * 64 + t;
    if (gc < D) {
      float* o = out + static_cast<long long>(g) * D + gc;
      *o = (accumulate ? *o : 0.f) + acc;
    }
  }
}

constexpr int kDotBlocks = 592;  // 4 per SM
__global__ void __launch_bounds__(256)
dot_partial_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, long long n, float* __restrict__ ws) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8];
  float acc = 0.f;
  const long long nvec = n >> 3;
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec;
       v += static_cast<long long>(gridDim.x) * blockDim.x) {
    float fa[8], fb[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(a) + v), fa);
    unpack8(__ldg(reinterpret_cast<const uint4*>(b) + v), fb);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc += fa[i] * fb[i];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    for (long long k = nvec * 8; k < n; ++k) acc += __bfloat162float(a[k]) * __bfloat162float(b[k]);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    ws[blockIdx.x] = t;
  }
}
__global__ void gate_grad_finalize_kernel(const float* __restrict__ ws, int nblk, const float* __restrict__ gate,
                                          float* __restrict__ dgate, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  // one warp, fixed summation order (lane-strided partials, then a shuffle tree) -> deterministic
  double t = 0.0;
  for (int i = threadIdx.x; i < nblk; i += 32) t += ws[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (threadIdx.x == 0) {
    const float th = tanhf(*gate);
    const float g = (1.0f - th * th) * static_cast<float>(t);
    *dgate = (accumulate ? *dgate : 0.f) + g;
  }
}
__global__ void __launch_bounds__(256)
sqmean_partial_kernel(const bf16* __restrict__ x, long long n, float* __restrict__ ws, bf16* __restrict__ dx) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8];
  float acc = 0.f;
  const float gscale = 2.0f / static_cast<float>(n);
  const long long nvec = n >> 3;
  for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec;
       v += static_cast<long long>(gridDim.x) * blockDim.x) {
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x) + v), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { acc += f[i] * f[i]; f[i] *= gscale; }
    if (dx) reinterpret_cast<uint4*>(dx)[v] = pack8(f);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i];
    ws[blockIdx.x] = t;
  }
}
__global__ void sqmean_finalize_kernel(const float* __restrict__ ws, int nblk, long long n, float* __restrict__ loss) {
  pdl_launch_dependents();
  pdl_wait();
  double t = 0.0;
  for (int i = threadIdx.x; i < nblk; i += 32) t += ws[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if (threadIdx.x == 0) *loss = static_cast<float>(t / static_cast<double>(n));
}

// ------------------------------------------------------------------------------------------------
// CLIP embeddings / media assembly / Fuyu scatter
// ------------------------------------------------------------------------------------------------
template <bool kF32>
__global__ void im2col_kernel(const void* __restrict__ pixels, int N, int H, int W, int patch, bf16* __restrict__ out,
                              int Kpad) {
  pdl_launch_dependents();
  pdl_wait();
  const int gw = W / patch, gh = H / patch;
  const int K = 3 * patch * patch;
  const long long total = static_cast<long long>(N) * gh * gw * Kpad;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % Kpad);
    const long long prow = i / Kpad;
    float v = 0.f;
    if (k < K) {
      const int c = k / (patch * patch), ij = k % (patch * patch), pi = ij / patch, pj = ij % patch;
      const int pw = static_cast<int>(prow % gw), ph = static_cast<int>((prow / gw) % gh);
      const long long n = prow / (static_cast<long long>(gw) * gh);
      const long long src = ((n * 3 + c) * H + (ph * patch + pi)) * W + (pw * patch + pj);
      v = kF32 ? static_cast<const float*>(pixels)[src] : __bfloat162float(static_cast<const bf16*>(pixels)[src]);
    }
    out[i] = __float2bfloat16(v);
  }
}
__global__ void clip_assemble_kernel(const bf16* __restrict__ patch_emb, const float* __restrict__ cls,
                                     const float* __restrict__ pos, bf16* __restrict__ out, int N, int np, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = D >> 3;
  const long long total = static_cast<long long>(N) * (np + 1) * nvec;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % nvec);
    const long long tok = i / nvec;
    const int t = static_cast<int>(tok % (np + 1));
    const long long n = tok / (np + 1);
    float f[8];
    if (t == 0) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(cls) + 2 * v), b = __ldg(reinterpret_cast<const float4*>(cls) + 2 * v + 1);
      f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    } else {
      unpack8(__ldg(reinterpret_cast<const uint4*>(patch_emb + (n * np + (t - 1)) * D) + v), f);
    }
    const float* pp = pos + static_cast<long long>(t) * D + v * 8;
    const float4 a = __ldg(reinterpret_cast<const float4*>(pp)), b = __ldg(reinterpret_cast<const float4*>(pp + 4));
    f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w; f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
    reinterpret_cast<uint4*>(out + tok * D)[v] = pack8(f);
  }
}
__global__ void media_from_clip_kernel(const bf16* __restrict__ hidden, const float* __restrict__ frame_embs, int F,
                                       bf16* __restrict__ out, int n_img, int v_tok, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = D >> 3;
  const long long total = static_cast<long long>(n_img) * v_tok * nvec;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % nvec);
    const long long tok = i / nvec;
    const int t = static_cast<int>(tok % v_tok);
    const long long img = tok / v_tok;
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(hidden + (img * (v_tok + 1) + 1 + t) * D) + v), f);
    if (frame_embs != nullptr) {
      const float* fe = frame_embs + static_cast<long long>(img % F) * D + v * 8;
      const float4 a = __ldg(reinterpret_cast<const float4*>(fe)), b = __ldg(reinterpret_cast<const float4*>(fe + 4));
      f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w; f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
    }
    reinterpret_cast<uint4*>(out + tok * D)[v] = pack8(f);
  }
}
__global__ void fuyu_scatter_kernel(const bf16* __restrict__ word, const bf16* __restrict__ cont,
                                    const long long* __restrict__ idx, const long long* __restrict__ b_off,
                                    bf16* __restrict__ out, int B, int S, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = D >> 3;
  const long long total = static_cast<long long>(B) * S * nvec;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % nvec);
    const long long tok = i / nvec;
    const int b = static_cast<int>(tok / S);
    const long long id = idx[tok];
    // b_off holds B+1 prefix offsets: ids outside sample b's [0, n_b) keep the word row instead of reading out of bounds
    const bool take = id >= 0 && id < b_off[b + 1] - b_off[b];
    const uint4* src = take ? reinterpret_cast<const uint4*>(cont + (b_off[b] + id) * D)
                            : reinterpret_cast<const uint4*>(word + tok * D);
    reinterpret_cast<uint4*>(out + tok * D)[v] = __ldg(src + v);
  }
}

static inline int grid_for(long long work_items, int block) {
  long long g = (work_items + block - 1) / block;
  const long long cap = static_cast<long long>(sm_count()) * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

}  // namespace otb

using namespace otb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int otb_layernorm_fwd(const void* x, int64_t ldx, const float* gamma, const float* beta, void* y,
                                 int64_t ldy, float* mean, float* rstd, int rows, int D, float eps, void* stream) {
  OTB_CHECK_ARG(x && gamma && beta && y && rows > 0 && D > 0, "otb_layernorm_fwd: bad argument");
  OTB_CHECK_ARG(D % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "otb_layernorm_fwd: D/ld must be multiples of 8");
  OTB_CHECK_CUDA(launch_k(ln_fwd_kernel, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), static_cast<const bf16*>(x), ldx, gamma, beta,
                                                          static_cast<bf16*>(y), ldy, mean, rstd, rows, D, eps));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

static int ln_fused_grid(int rows) {
  const int nbatch = (rows + otb::kLnR - 1) / otb::kLnR;
  return nbatch < otb::sm_count() ? nbatch : otb::sm_count();
}

extern "C" int otb_ln_chunks(int rows, int D) {
  if (D <= 4096) {        // workspace must hold one partial row per CTA of the one-pass kernel
    const int g = ln_fused_grid(rows);
    int colblocks0 = (D + 63) / 64, chunks0 = (4 * 132 + colblocks0 - 1) / colblocks0;   // 4 x the H100's SMs
    return g > chunks0 ? g : chunks0;
  }
  int colblocks = (D + 63) / 64;
  int chunks = (4 * 132 + colblocks - 1) / colblocks;
  if (chunks > (rows + 7) / 8) chunks = (rows + 7) / 8;
  if (chunks < 1) chunks = 1;
  return chunks;
}

extern "C" int otb_layernorm_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                                 const float* rstd, const float* gamma, const void* add, int64_t ldadd, void* dx,
                                 int64_t lddx, float* dgamma, float* dbeta, int accumulate, float* ws, int rows,
                                 int D, void* stream) {
  OTB_CHECK_ARG(dy && x && mean && rstd && gamma && rows > 0 && D > 0, "otb_layernorm_bwd: bad argument");
  OTB_CHECK_ARG(D % 8 == 0 && lddy % 8 == 0 && ldx % 8 == 0, "otb_layernorm_bwd: D/ld must be multiples of 8");
  // Parameter gradients take the one-pass kernel, which holds at most two 16 B vectors of a row per thread (D <= 4096);
  // wider rows take ln_bwd_dx_kernel + the param / finalize kernels below.  dx == nullptr (perceiver norm_media: the
  // frozen CLIP features need no input gradient) takes the one-pass kernel too: it then only produces the gamma / beta
  // partials.  Only dx wanted (the frozen MPT / Persimmon layers): ln_bwd_dx_kernel alone.
  if (D <= 4096 && (dgamma != nullptr || dbeta != nullptr)) {
    OTB_CHECK_ARG((dx == nullptr || lddx % 8 == 0) && (add == nullptr || ldadd % 8 == 0), "otb_layernorm_bwd: bad ld");
    OTB_CHECK_ARG(ws != nullptr, "otb_layernorm_bwd: workspace required for parameter gradients");
    const int grid = ln_fused_grid(rows);
    auto kern = (D <= 2048) ? ln_bwd_fused_kernel<1> : ln_bwd_fused_kernel<2>;
    OTB_CHECK_CUDA(launch_k(kern, dim3(grid), dim3(256), 0, ST(stream), static_cast<const bf16*>(dy), lddy,
                            static_cast<const bf16*>(x), ldx, mean, rstd, gamma, static_cast<const bf16*>(add), ldadd,
                            static_cast<bf16*>(dx), lddx, ws, rows, D));
    OTB_CHECK_CUDA(launch_k(ln_bwd_finalize_wide_kernel, dim3((D + 31) / 32), dim3(32, 8), 0, ST(stream), ws, dgamma,
                            dbeta, D, grid, accumulate));
    count_launch(2);
    OTB_CHECK_CUDA(cudaGetLastError());
    return OTB_OK;
  }
  if (dx != nullptr) {
    OTB_CHECK_ARG(lddx % 8 == 0 && (add == nullptr || ldadd % 8 == 0), "otb_layernorm_bwd: bad ld");
    OTB_CHECK_CUDA(launch_k(ln_bwd_dx_kernel, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), 
        static_cast<const bf16*>(dy), lddy, static_cast<const bf16*>(x), ldx, mean, rstd, gamma,
        static_cast<const bf16*>(add), ldadd, static_cast<bf16*>(dx), lddx, rows, D));
    count_launch();
  }
  if (dgamma != nullptr || dbeta != nullptr) {
    OTB_CHECK_ARG(ws != nullptr, "otb_layernorm_bwd: workspace required for parameter gradients");
    const int chunks = otb_ln_chunks(rows, D);
    dim3 grid((D + 63) / 64, chunks), block(32, 8);
    OTB_CHECK_CUDA(launch_k(ln_bwd_param_kernel, dim3(grid), dim3(block), 0, ST(stream), static_cast<const bf16*>(dy), lddy,
                                                          static_cast<const bf16*>(x), ldx, mean, rstd, ws, rows, D,
                                                          chunks));
    OTB_CHECK_CUDA(launch_k(ln_bwd_finalize_kernel, dim3((D + 255) / 256), dim3(256), 0, ST(stream), ws, dgamma, dbeta, D, chunks, accumulate));
    count_launch(2);
  }
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_text_time(const uint8_t* media_locations, int B, int L, int attend_previous, int32_t* text_time,
                             void* stream) {
  OTB_CHECK_ARG(media_locations && text_time && B > 0 && L > 0, "otb_text_time: bad argument");
  OTB_CHECK_CUDA(launch_k(text_time_kernel, dim3((B + 63) / 64), dim3(64), 0, ST(stream), media_locations, B, L, attend_previous, text_time));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_cast_f32_bf16_multi(const void* table, int n_tensors, int64_t total_blocks, void* stream) {
  OTB_CHECK_ARG(table && n_tensors > 0 && total_blocks > 0 && total_blocks < (1ll << 31),
                "otb_cast_f32_bf16_multi: bad argument");
  OTB_CHECK_CUDA(launch_k(cast_multi_kernel, dim3(static_cast<unsigned>(total_blocks)), dim3(256), 0, ST(stream),
                          static_cast<const CastSeg*>(table), n_tensors));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_cast_f32_bf16(const float* src, void* dst, int64_t n, void* stream) {
  OTB_CHECK_ARG(src && dst && n > 0, "otb_cast_f32_bf16: bad argument");
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
                "otb_cast_f32_bf16: pointers must be 16-byte aligned");
  OTB_CHECK_CUDA(launch_k(cast_f32_bf16_kernel, dim3(grid_for((n + 7) / 8, 256)), dim3(256), 0, ST(stream), src, static_cast<bf16*>(dst), n));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_cast_bf16_f32(const void* src, float* dst, int64_t n, void* stream) {
  OTB_CHECK_ARG(src && dst && n > 0, "otb_cast_bf16_f32: bad argument");
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
                "otb_cast_bf16_f32: pointers must be 16-byte aligned");
  OTB_CHECK_CUDA(launch_k(cast_bf16_f32_kernel, dim3(grid_for((n + 7) / 8, 256)), dim3(256), 0, ST(stream), static_cast<const bf16*>(src), dst, n));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_cast_bf16_f32_scale(const void* src, float* dst, int64_t n, float scale, void* stream) {
  OTB_CHECK_ARG(src && dst && n > 0, "otb_cast_bf16_f32_scale: bad argument");
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
                "otb_cast_bf16_f32_scale: pointers must be 16-byte aligned");
  OTB_CHECK_CUDA(launch_k(cast_bf16_f32_scale_kernel, dim3(grid_for((n + 7) / 8, 256)), dim3(256), 0, ST(stream),
                          static_cast<const bf16*>(src), dst, (long long)n, scale));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_bcast_rows(const float* src, int div, int mod, void* out, int rows, int D, void* stream) {
  OTB_CHECK_ARG(src && out && div > 0 && mod > 0 && rows > 0 && D % 8 == 0, "otb_bcast_rows: bad argument");
  OTB_CHECK_CUDA(launch_k(bcast_rows_kernel, dim3(grid_for(static_cast<long long>(rows) * (D / 8), 256)), dim3(256), 0, ST(stream), 
      src, div, mod, static_cast<bf16*>(out), rows, D));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_add_rowbias(const void* x, const float* bias, int div, int mod, void* out, int rows, int D,
                               void* stream) {
  OTB_CHECK_ARG(x && bias && out && div > 0 && mod > 0 && rows > 0 && D % 8 == 0, "otb_add_rowbias: bad argument");
  OTB_CHECK_CUDA(launch_k(add_rowbias_kernel, dim3(grid_for(static_cast<long long>(rows) * (D / 8), 256)), dim3(256), 0, ST(stream), 
      static_cast<const bf16*>(x), bias, div, mod, static_cast<bf16*>(out), rows, D));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_grouped_colsum(const void* x, int64_t ldx, int rows, int D, int div, int mod, float* out,
                                  int accumulate, void* stream) {
  OTB_CHECK_ARG(x && out && div > 0 && mod > 0 && rows > 0 && D % 2 == 0 && ldx % 2 == 0,
                "otb_grouped_colsum: bad argument");
  dim3 grid((D + 63) / 64, mod), block(32, 8);
  OTB_CHECK_CUDA(launch_k(grouped_colsum_kernel, dim3(grid), dim3(block), 0, ST(stream), static_cast<const bf16*>(x), ldx, rows, D, div, mod, out,
                                                          accumulate));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_dot_blocks(void) { return kDotBlocks; }
extern "C" int otb_gate_grad(const void* dy, const void* a, int64_t n, const float* gate, float* dgate,
                             int accumulate, float* ws, void* stream) {
  OTB_CHECK_ARG(dy && a && gate && dgate && ws && n > 0, "otb_gate_grad: bad argument");
  OTB_CHECK_CUDA(launch_k(dot_partial_kernel, dim3(kDotBlocks), dim3(256), 0, ST(stream), static_cast<const bf16*>(dy), static_cast<const bf16*>(a), n,
                                                           ws));
  OTB_CHECK_CUDA(launch_k(gate_grad_finalize_kernel, dim3(1), dim3(32), 0, ST(stream), ws, kDotBlocks, gate, dgate, accumulate));
  count_launch(2);
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_sqmean_loss(const void* x, int64_t n, float* loss, void* dx, float* ws, void* stream) {
  OTB_CHECK_ARG(x && loss && ws && n > 0 && n % 8 == 0, "otb_sqmean_loss: bad argument (n %% 8 == 0 required)");
  OTB_CHECK_CUDA(launch_k(sqmean_partial_kernel, dim3(kDotBlocks), dim3(256), 0, ST(stream), static_cast<const bf16*>(x), n, ws,
                                                              static_cast<bf16*>(dx)));
  OTB_CHECK_CUDA(launch_k(sqmean_finalize_kernel, dim3(1), dim3(32), 0, ST(stream), ws, kDotBlocks, n, loss));
  count_launch(2);
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_im2col_patches(const void* pixels, int pix_fp32, int N, int H, int W, int patch, void* out,
                                  int Kpad, void* stream) {
  OTB_CHECK_ARG(pixels && out && N > 0 && patch > 0 && H % patch == 0 && W % patch == 0 && Kpad >= 3 * patch * patch,
                "otb_im2col_patches: bad argument");
  const long long total = static_cast<long long>(N) * (H / patch) * (W / patch) * Kpad;
  if (pix_fp32)
    OTB_CHECK_CUDA(launch_k(im2col_kernel<true>, dim3(grid_for(total, 256)), dim3(256), 0, ST(stream), pixels, N, H, W, patch, static_cast<bf16*>(out), Kpad));
  else
    OTB_CHECK_CUDA(launch_k(im2col_kernel<false>, dim3(grid_for(total, 256)), dim3(256), 0, ST(stream), pixels, N, H, W, patch, static_cast<bf16*>(out), Kpad));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_clip_assemble(const void* patch_emb, const float* cls, const float* pos, void* out, int N, int np,
                                 int D, void* stream) {
  OTB_CHECK_ARG(patch_emb && cls && pos && out && N > 0 && np > 0 && D % 8 == 0, "otb_clip_assemble: bad argument");
  OTB_CHECK_CUDA(launch_k(clip_assemble_kernel, dim3(grid_for(static_cast<long long>(N) * (np + 1) * (D / 8), 256)), dim3(256), 0, ST(stream), 
      static_cast<const bf16*>(patch_emb), cls, pos, static_cast<bf16*>(out), N, np, D));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_media_from_clip(const void* hidden, const float* frame_embs, int F, void* out, int n_img, int v,
                                   int D, void* stream) {
  OTB_CHECK_ARG(hidden && out && n_img > 0 && v > 0 && D % 8 == 0 && F > 0, "otb_media_from_clip: bad argument");
  OTB_CHECK_CUDA(launch_k(media_from_clip_kernel, dim3(grid_for(static_cast<long long>(n_img) * v * (D / 8), 256)), dim3(256), 0, ST(stream), 
      static_cast<const bf16*>(hidden), frame_embs, F, static_cast<bf16*>(out), n_img, v, D));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_fuyu_scatter(const void* word, const void* cont, const int64_t* idx, const int64_t* b_off,
                                void* out, int B, int S, int D, void* stream) {
  OTB_CHECK_ARG(word && cont && idx && b_off && out && B > 0 && S > 0 && D % 8 == 0, "otb_fuyu_scatter: bad argument");
  OTB_CHECK_CUDA(launch_k(fuyu_scatter_kernel, dim3(grid_for(static_cast<long long>(B) * S * (D / 8), 256)), dim3(256), 0, ST(stream), 
      static_cast<const bf16*>(word), static_cast<const bf16*>(cont), reinterpret_cast<const long long*>(idx),
      reinterpret_cast<const long long*>(b_off), static_cast<bf16*>(out), B, S, D));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
