// otter_b200 — the two hot paths of a KV-cache decode step (one new token per sequence): attention of one query row per
// (sequence, head) over the T cached keys, and the linear layers at M = batch x beams <= 8 rows.
//
// Both are HBM streams (the cache rows, the weight matrix) with a handful of FMAs per byte, and both run on the CUDA
// cores: one query row, or eight activation rows, gives the tensor cores nothing to do — a wgmma tile is 64 rows, so
// 56 to 63 of them would be padding, and the kernels are bound by the bytes they read, not by arithmetic.  What matters
// is that every SM streams (enough CTAs) with enough 16-byte loads in flight to cover the HBM latency.
// Deterministic: partial results are combined in a fixed order, no atomics.
#include <algorithm>

#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

// 16-byte read of data no thread of the grid writes, not kept in L1 (each byte is used once)
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// ================================================================================================
// Decode attention
// ================================================================================================
// grid (split, head, batch), 256 threads = 16 half-warps.  A half-warp owns a key at a time: lane l of it holds dims
// [8 l, 8 l + 8) of q, reads the same dims of the key row (one 16 B load; the half-warp reads the 256 B row) and of
// the value row, and keeps 8 of the 128 output dims.  Half-warp g walks keys t0 + g, t0 + g + 16, ... of the split,
// four at a time (8 loads in flight per lane), with its own running (max, sum, out); the 16 are combined through shared
// memory in half-warp order and the split's (max, sum, 128 unnormalised outputs) go to the workspace.  A second kernel
// combines the splits of a (batch, head) in split order.  Scores are kept in the log2 domain (exp2f).
constexpr int kDecThreads = 256;
constexpr int kDecGroups = kDecThreads / 16;
constexpr int kDecUnroll = 4;
constexpr int kDecWsStride = 132;          // floats per (batch, head, split): max, sum, 2 pad, 128 outputs (16 B aligned)
constexpr int kDecMinKeys = 64;            // a split is not worth less than 4 keys per half-warp
constexpr int kDecMaxSplits = 64;
constexpr float kLog2eDec = 1.4426950408889634f;

struct DecodeParams {
  const bf16* q; const bf16* k; const bf16* v; bf16* out; float* ws; const float* slopes;
  long long ld_q, ld_out, kv_batch, ld_kv;
  int H, T, keys_per_split, nsplit;
  float scale_log2;
};

// keys per split (a multiple of 16) and the number of splits: aim at two CTAs per SM, never less than kDecMinKeys keys
static int decode_splits(int B, int H, int T, int* keys_per_split) {
  const long long bh = static_cast<long long>(B) * H;
  long long want = (2LL * sm_count() + bh - 1) / bh;
  want = std::min<long long>(want, kDecMaxSplits);
  want = std::min<long long>(want, (T + kDecMinKeys - 1) / kDecMinKeys);
  want = std::max<long long>(want, 1);
  int kps = static_cast<int>((T + want - 1) / want);
  kps = (kps + 15) / 16 * 16;
  *keys_per_split = kps;
  return (T + kps - 1) / kps;              // every split holds at least one key
}

__global__ void __launch_bounds__(kDecThreads) lm_attn_decode_kernel(DecodeParams p) {
  __shared__ float s_m[kDecGroups], s_l[kDecGroups];
  __shared__ __align__(16) float s_o[kDecGroups][128];
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int g = threadIdx.x >> 4, l = threadIdx.x & 15;
  pdl_launch_dependents();
  pdl_wait();
  const int t0 = split * p.keys_per_split;
  const int t1 = min(p.T, t0 + p.keys_per_split);
  float q[8];
  unpack8(*reinterpret_cast<const uint4*>(p.q + b * p.ld_q + h * 128 + l * 8), q);
#pragma unroll
  for (int i = 0; i < 8; ++i) q[i] *= p.scale_log2;
  const float slope = p.slopes ? p.slopes[h] * kLog2eDec : 0.f;
  const bf16* kbase = p.k + b * p.kv_batch + h * 128 + l * 8;
  const bf16* vbase = p.v + b * p.kv_batch + h * 128 + l * 8;

  float m = -INFINITY, lsum = 0.f, o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;
  // the two half-warps of a warp can leave the key loop at different trips: the shuffles name their own 16 lanes only
  const unsigned hw_mask = (threadIdx.x & 16) ? 0xffff0000u : 0x0000ffffu;
  for (int j0 = t0 + g; j0 < t1; j0 += kDecGroups * kDecUnroll) {      // half-warp uniform
    uint4 kr[kDecUnroll], vr[kDecUnroll];
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const int j = j0 + u * kDecGroups;
      kr[u] = vr[u] = make_uint4(0, 0, 0, 0);
      if (j < t1) {                                                     // rows >= T are never read
        kr[u] = ld_stream16(kbase + j * p.ld_kv);
        vr[u] = ld_stream16(vbase + j * p.ld_kv);
      }
    }
    float s[kDecUnroll], m_new = m;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const int j = j0 + u * kDecGroups;
      float kf[8], d = 0.f;
      unpack8(kr[u], kf);
#pragma unroll
      for (int i = 0; i < 8; ++i) d = fmaf(q[i], kf[i], d);
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) d += __shfl_xor_sync(hw_mask, d, off);
      s[u] = j < t1 ? d + slope * static_cast<float>(j - (p.T - 1)) : -INFINITY;
      m_new = fmaxf(m_new, s[u]);
    }
    const float c = exp2f(m - m_new);                                   // m_new is finite: key j0 is valid; exp2f(-inf) = 0
    lsum *= c;
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] *= c;
#pragma unroll
    for (int u = 0; u < kDecUnroll; ++u) {
      const float pj = exp2f(s[u] - m_new);
      float vf[8];
      unpack8(vr[u], vf);
      lsum += pj;
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmaf(pj, vf[i], o[i]);
    }
    m = m_new;
  }
  if (l == 0) { s_m[g] = m; s_l[g] = lsum; }
  *reinterpret_cast<float4*>(&s_o[g][l * 8]) = make_float4(o[0], o[1], o[2], o[3]);
  *reinterpret_cast<float4*>(&s_o[g][l * 8 + 4]) = make_float4(o[4], o[5], o[6], o[7]);
  __syncthreads();
  if (threadIdx.x < 128) {                                              // half-warps in order 0 .. 15
    const int d = threadIdx.x;
    float mm = -INFINITY;
#pragma unroll
    for (int i = 0; i < kDecGroups; ++i) mm = fmaxf(mm, s_m[i]);
    float ll = 0.f, acc = 0.f;
#pragma unroll
    for (int i = 0; i < kDecGroups; ++i) {
      const float c = exp2f(s_m[i] - mm);                               // 0 for a half-warp that had no key
      ll = fmaf(s_l[i], c, ll);
      acc = fmaf(s_o[i][d], c, acc);
    }
    float* w = p.ws + (static_cast<long long>(b * p.H + h) * p.nsplit + split) * kDecWsStride;
    if (d == 0) { w[0] = mm; w[1] = ll; }
    w[4 + d] = acc;
  }
}

// grid (head, batch), 128 threads: thread d combines output dim d over the splits in split order
__global__ void __launch_bounds__(128) lm_attn_decode_combine_kernel(DecodeParams p) {
  const int h = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
  pdl_launch_dependents();
  pdl_wait();
  const float* w = p.ws + static_cast<long long>(b * p.H + h) * p.nsplit * kDecWsStride;
  float mm = -INFINITY;
  for (int s = 0; s < p.nsplit; ++s) mm = fmaxf(mm, w[s * kDecWsStride]);
  float ll = 0.f, acc = 0.f;
  for (int s = 0; s < p.nsplit; ++s) {
    const float c = exp2f(w[s * kDecWsStride] - mm);
    ll = fmaf(w[s * kDecWsStride + 1], c, ll);
    acc = fmaf(w[s * kDecWsStride + 4 + d], c, acc);
  }
  p.out[b * p.ld_out + h * 128 + d] = __float2bfloat16(acc / ll);
}

// ================================================================================================
// y[M][N] = epilogue(x[M][K] . W[N][K]^T),  1 <= M <= 8
// ================================================================================================
// 256 threads = 8 warps.  A warp owns 4 consecutive rows of W (4 output columns) over one of `ksplit` interleaved
// shares of K: lane l reads 16 B vectors l, l + 32, ... of its share from each of the 4 rows (a warp reads 512
// contiguous bytes of a row per step, the next step's 4 loads are issued before this step's FMAs) and multiplies them
// with the MT activation rows held in shared memory, so one weight byte is read once and one shared-memory read of x
// feeds 4 weight rows.  x is staged per CTA in K-chunks of 4096 elements (MT x 8 KB; rows M .. MT-1 are zero).  The
// 32 lanes are summed by butterfly, the ksplit warps of a column group in warp order through shared memory, then the
// epilogue (the GEMM's order: + bias, GELU, x alpha, + residual) writes bf16.  ksplit in {1, 2, 4} is chosen from N so
// that a narrow matrix (out_proj: N = 4096) still gives every SM a CTA or two: 32 / ksplit columns per CTA.
constexpr int kLinThreads = 256;
constexpr int kLinWarps = kLinThreads / 32;
constexpr int kLinRows = 4;                 // weight rows per warp
constexpr int kLinChunk = 4096;             // K elements of x staged at a time

struct LinearSmallParams {
  const bf16* x; const bf16* w; const float* bias; const bf16* residual; bf16* out;
  long long ldx, ldw, ld_res, ld_out;
  int M, N, K, act, ksplit;
  float alpha;
};

template <int MT>
__global__ void __launch_bounds__(kLinThreads, 2) linear_small_m_kernel(LinearSmallParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint4* xs = reinterpret_cast<uint4*>(smem_raw);                      // [MT][kLinChunk / 8] vectors of 8 bf16
  __shared__ float red[kLinWarps][kLinRows * MT];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = kLinWarps / p.ksplit;                             // column groups of 4 per CTA
  const int grp = warp % groups, ks = warp / groups;
  const int n0 = (blockIdx.x * groups + grp) * kLinRows;
  const bool active = n0 < p.N;                                        // N % 8 == 0: a group is whole or absent
  pdl_launch_dependents();
  pdl_wait();

  float acc[kLinRows][MT];
#pragma unroll
  for (int r = 0; r < kLinRows; ++r)
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[r][m] = 0.f;

  const int step = 32 * p.ksplit;
  for (int k0 = 0; k0 < p.K; k0 += kLinChunk) {
    const int nvec = min(kLinChunk, p.K - k0) >> 3;
    if (k0) __syncthreads();                                           // the previous chunk has been read
    for (int i = threadIdx.x; i < MT * nvec; i += kLinThreads) {
      const int m = i / nvec, v = i - m * nvec;
      xs[m * (kLinChunk / 8) + v] = m < p.M ? *reinterpret_cast<const uint4*>(p.x + m * p.ldx + k0 + v * 8)
                                            : make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    if (active) {
      const bf16* wp = p.w + static_cast<long long>(n0) * p.ldw + k0;
      int v = ks * 32 + lane;
      uint4 wn[kLinRows];
      if (v < nvec) {
#pragma unroll
        for (int r = 0; r < kLinRows; ++r) wn[r] = ld_stream16(wp + r * p.ldw + v * 8);
      }
      while (v < nvec) {
        float wf[kLinRows][8];
#pragma unroll
        for (int r = 0; r < kLinRows; ++r) unpack8(wn[r], wf[r]);
        const int vn = v + step;
        if (vn < nvec) {
#pragma unroll
          for (int r = 0; r < kLinRows; ++r) wn[r] = ld_stream16(wp + r * p.ldw + vn * 8);
        }
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          float xf[8];
          unpack8(xs[m * (kLinChunk / 8) + v], xf);
#pragma unroll
          for (int r = 0; r < kLinRows; ++r)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[r][m] = fmaf(xf[i], wf[r][i], acc[r][m]);
        }
        v = vn;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kLinRows; ++r)
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const float s = warp_sum(acc[r][m]);
      if (lane == 0) red[warp][r * MT + m] = s;
    }
  __syncthreads();
  // one thread per output element of the CTA: (row m, column group, column of the group)
  const int t = threadIdx.x;
  if (t < p.M * groups * kLinRows) {
    const int m = t / (groups * kLinRows), c = t - m * (groups * kLinRows);
    const int g2 = c / kLinRows, r = c - g2 * kLinRows;
    const int n = (blockIdx.x * groups + g2) * kLinRows + r;
    if (n < p.N) {
      float v = 0.f;
      for (int s = 0; s < p.ksplit; ++s) v += red[s * groups + g2][r * MT + m];     // warp order
      if (p.bias) v += p.bias[n];
      if (p.act == 1) v = gelu_fast(v);
      v *= p.alpha;
      if (p.residual) v += __bfloat162float(p.residual[m * p.ld_res + n]);
      p.out[m * p.ld_out + n] = __float2bfloat16(v);
    }
  }
}

template <int MT>
static cudaError_t launch_linear_small(const LinearSmallParams& p, int ctas, cudaStream_t stream) {
  const int smem = MT * kLinChunk * 2;
  cudaError_t e = ensure_dyn_smem(linear_small_m_kernel<MT>, smem);
  if (e != cudaSuccess) return e;
  return launch_k(linear_small_m_kernel<MT>, dim3(ctas), dim3(kLinThreads), smem, stream, p);
}

}  // namespace otb

using namespace otb;

static int decode_check(const otb_lm_attn_decode_desc* d) {
  OTB_CHECK_ARG(d != nullptr && d->q && d->k && d->v && d->out && d->ws, "otb_lm_attn_decode: null pointer");
  OTB_CHECK_ARG(d->B > 0 && d->H > 0 && d->T > 0, "otb_lm_attn_decode: bad sizes");
  OTB_CHECK_ARG(d->B <= 65535 && d->H <= 65535, "otb_lm_attn_decode: B and H must be at most 65535");
  OTB_CHECK_ARG(d->head_dim == 128, "otb_lm_attn_decode: head_dim must be 128 (MPT-7B)");
  OTB_CHECK_ARG(d->ld_q % 8 == 0 && d->ld_kv % 8 == 0 && d->kv_batch_stride % 8 == 0,
                "otb_lm_attn_decode: row pitches and the batch stride must be multiples of 8");
  OTB_CHECK_ARG(d->ld_q >= d->H * 128 && d->ld_kv >= d->H * 128 && d->ld_out >= d->H * 128,
                "otb_lm_attn_decode: a row pitch is smaller than H * 128");
  OTB_CHECK_ARG(((reinterpret_cast<uintptr_t>(d->q) | reinterpret_cast<uintptr_t>(d->k) |
                  reinterpret_cast<uintptr_t>(d->v) | reinterpret_cast<uintptr_t>(d->ws)) & 15) == 0,
                "otb_lm_attn_decode: q, k, v and ws must be 16-byte aligned");
  return OTB_OK;
}

extern "C" long long otb_lm_attn_decode_ws_floats(int B, int H, int T) {
  if (B <= 0 || H <= 0 || T <= 0) return 0;
  int kps;
  return static_cast<long long>(B) * H * decode_splits(B, H, T, &kps) * kDecWsStride;
}

extern "C" int otb_lm_attn_decode(const otb_lm_attn_decode_desc* d, void* stream) {
  int rc = decode_check(d);
  if (rc) return rc;
  DecodeParams p;
  p.q = static_cast<const bf16*>(d->q); p.k = static_cast<const bf16*>(d->k); p.v = static_cast<const bf16*>(d->v);
  p.out = static_cast<bf16*>(d->out); p.ws = d->ws; p.slopes = d->alibi_slopes;
  p.ld_q = d->ld_q; p.ld_out = d->ld_out; p.kv_batch = d->kv_batch_stride; p.ld_kv = d->ld_kv;
  p.H = d->H; p.T = d->T;
  p.nsplit = decode_splits(d->B, d->H, d->T, &p.keys_per_split);
  p.scale_log2 = d->scale * kLog2eDec;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  OTB_CHECK_CUDA(launch_k(lm_attn_decode_kernel, dim3(p.nsplit, d->H, d->B), dim3(kDecThreads), 0, st, p));
  OTB_CHECK_CUDA(launch_k(lm_attn_decode_combine_kernel, dim3(d->H, d->B), dim3(128), 0, st, p));
  count_launch(2);
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_linear_small_m(const void* x, int64_t ldx, const void* w, int64_t ldw, int M, int N, int K, float alpha,
                                  const float* bias, int act, const void* residual, int64_t ld_res, void* out,
                                  int64_t ld_out, void* stream) {
  OTB_CHECK_ARG(x && w && out, "otb_linear_small_m: null pointer");
  OTB_CHECK_ARG(M >= 1 && M <= 8, "otb_linear_small_m: M = %d must be in 1..8 (otb_gemm_bf16 serves larger M)", M);
  OTB_CHECK_ARG(N > 0 && K > 0 && N % 8 == 0 && K % 8 == 0, "otb_linear_small_m: N and K must be positive multiples of 8");
  OTB_CHECK_ARG(act == 0 || act == 1, "otb_linear_small_m: act must be 0 (none) or 1 (GELU)");
  OTB_CHECK_ARG(ldx >= K && ldw >= K && ld_out >= N && ldx % 8 == 0 && ldw % 8 == 0 && (!residual || ld_res >= N),
                "otb_linear_small_m: bad row pitch (ldx, ldw >= K and multiples of 8; ld_out, ld_res >= N)");
  OTB_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15) == 0,
                "otb_linear_small_m: x and w must be 16-byte aligned");
  LinearSmallParams p;
  p.x = static_cast<const bf16*>(x); p.w = static_cast<const bf16*>(w); p.bias = bias;
  p.residual = static_cast<const bf16*>(residual); p.out = static_cast<bf16*>(out);
  p.ldx = ldx; p.ldw = ldw; p.ld_res = ld_res; p.ld_out = ld_out;
  p.M = M; p.N = N; p.K = K; p.act = act; p.alpha = alpha;
  // the smallest in-CTA K split that gives two CTAs per SM (4 if none does)
  const int groups_total = N / kLinRows;
  p.ksplit = 4;
  for (int ks = 1; ks < 4; ks *= 2)
    if ((groups_total + kLinWarps / ks - 1) / (kLinWarps / ks) >= 2 * sm_count()) { p.ksplit = ks; break; }
  const int per_cta = kLinWarps / p.ksplit;
  const int ctas = (groups_total + per_cta - 1) / per_cta;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int mt = M == 1 ? 1 : M == 2 ? 2 : M <= 4 ? 4 : 8;
  OTB_CHECK_CUDA(mt == 1 ? launch_linear_small<1>(p, ctas, st) : mt == 2 ? launch_linear_small<2>(p, ctas, st)
                 : mt == 4 ? launch_linear_small<4>(p, ctas, st) : launch_linear_small<8>(p, ctas, st));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
