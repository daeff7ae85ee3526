// otter_b200 — LLaMA decoder-layer specific kernels (SURVEY.md §8f rank 1: the LLaMA-7B text model of OTTER-Video / c3,
// and the grouped-query / scaled-RoPE LLaMA layers of Llama-2-70B and Llama-3).
//   reference: xformers_model/llama.py:74-89 (LlamaRMSNorm), :150-166 (rotate_half / apply_rotary_pos_emb),
//              :169-185 (LlamaMLP: down(silu(gate(x)) * up(x))), :186-259 (attention), :262-320 (decoder layer)
// HBM-bound element-wise passes around the wgmma GEMMs and the head-dim-128 causal attention kernel:
//   rmsnorm fwd / bwd         y = x * rsqrt(mean(x^2) + eps) * w;  backward: dx, and optionally the weight gradient
//                             (trainable decoder layers) through a deterministic two-stage column reduction
//   rope (in place)           q, k columns of the fused projection buffer, rotate_half convention, head dim 128;
//                             frequencies from theta, or from a table (linear / llama3 / yarn scaling) with a cos/sin factor
//   swiglu fwd / bwd          h = silu(g) * u ;  dg = dh * u * silu'(g), du = dh * silu(g)
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

// one warp per row; D % 8 == 0
__global__ void __launch_bounds__(256)
rmsnorm_fwd_kernel(const bf16* __restrict__ x, long long ldx, const float* __restrict__ w, bf16* __restrict__ y,
                   long long ldy, float* __restrict__ rstd_out, int rows, int D, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint4* px = reinterpret_cast<const uint4*>(x + static_cast<long long>(row) * ldx);
  const int nvec = D >> 3;
  float ss = 0.f;
  for (int v = lane; v < nvec; v += 32) {
    float f[8];
    unpack8(__ldg(px + v), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
  }
  const float rstd = rsqrtf(warp_sum(ss) / D + eps);
  if (lane == 0 && rstd_out != nullptr) rstd_out[row] = rstd;
  uint4* py = reinterpret_cast<uint4*>(y + static_cast<long long>(row) * ldy);
  for (int v = lane; v < nvec; v += 32) {
    float f[8];
    unpack8(__ldg(px + v), f);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
    const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = f[i] * rstd * ww[i];
    py[v] = pack8(f);
  }
}

// dx = rstd * (g - xhat * mean(g * xhat)) [+ add],  g = dy * w,  xhat = x * rstd
__global__ void __launch_bounds__(256)
rmsnorm_bwd_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x, long long ldx,
                   const float* __restrict__ rstd_in, const float* __restrict__ w, const bf16* __restrict__ add,
                   long long ldadd, bf16* __restrict__ dx, long long lddx, int rows, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint4* px = reinterpret_cast<const uint4*>(x + static_cast<long long>(row) * ldx);
  const uint4* pd = reinterpret_cast<const uint4*>(dy + static_cast<long long>(row) * lddy);
  const int nvec = D >> 3;
  const float rstd = rstd_in[row];
  float s = 0.f;
  for (int v = lane; v < nvec; v += 32) {
    float fx[8], fd[8];
    unpack8(__ldg(px + v), fx);
    unpack8(__ldg(pd + v), fd);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
    const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) s += fd[i] * ww[i] * fx[i] * rstd;
  }
  const float m = warp_sum(s) / D;
  uint4* po = reinterpret_cast<uint4*>(dx + static_cast<long long>(row) * lddx);
  const uint4* pa = add ? reinterpret_cast<const uint4*>(add + static_cast<long long>(row) * ldadd) : nullptr;
  for (int v = lane; v < nvec; v += 32) {
    float fx[8], fd[8], fa[8], o[8];
    unpack8(__ldg(px + v), fx);
    unpack8(__ldg(pd + v), fd);
    if (pa) unpack8(__ldg(pa + v), fa);
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
    const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[i] = rstd * (fd[i] * ww[i] - fx[i] * rstd * m);
      if (pa) o[i] += fa[i];
    }
    po[v] = pack8(o);
  }
}

// Weight-gradient variant: dx as rmsnorm_bwd_kernel (the row code below is the same, so dx has the same bits) and
// dw[j] = sum_r dy[r,j] * x[r,j] * rstd[r].  CTAs stride over groups of 8 rows, one warp per row; after the warps' dx of
// a group, thread t adds the group's rows, in row order, into its columns of the CTA's partial sums (vectors t, t + 256,
// ... of smem `colacc` [D]; the rows were just read, so they come from cache).  Each CTA writes its partials to
// ws[blockIdx.x][D]; rmsnorm_wgrad_finalize_kernel sums them in chunk order: deterministic, no atomics.
__global__ void __launch_bounds__(256)
rmsnorm_bwd_wgrad_kernel(const bf16* __restrict__ dy, long long lddy, const bf16* __restrict__ x, long long ldx,
                         const float* __restrict__ rstd_in, const float* __restrict__ w, const bf16* __restrict__ add,
                         long long ldadd, bf16* __restrict__ dx, long long lddx, float* __restrict__ ws, int rows, int D) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float4 colacc4[];
  float* colacc = reinterpret_cast<float*>(colacc4);
  const int lane = threadIdx.x & 31;
  const int nvec = D >> 3;
  for (int v = threadIdx.x; v < nvec; v += 256) {
#pragma unroll
    for (int i = 0; i < 8; ++i) colacc[v * 8 + i] = 0.f;
  }
  for (int grp = blockIdx.x; grp * 8 < rows; grp += gridDim.x) {
    const int row = grp * 8 + (threadIdx.x >> 5);
    if (row < rows) {
      const uint4* px = reinterpret_cast<const uint4*>(x + static_cast<long long>(row) * ldx);
      const uint4* pd = reinterpret_cast<const uint4*>(dy + static_cast<long long>(row) * lddy);
      const float rstd = rstd_in[row];
      float s = 0.f;
      for (int v = lane; v < nvec; v += 32) {
        float fx[8], fd[8];
        unpack8(__ldg(px + v), fx);
        unpack8(__ldg(pd + v), fd);
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
        const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) s += fd[i] * ww[i] * fx[i] * rstd;
      }
      const float m = warp_sum(s) / D;
      uint4* po = reinterpret_cast<uint4*>(dx + static_cast<long long>(row) * lddx);
      const uint4* pa = add ? reinterpret_cast<const uint4*>(add + static_cast<long long>(row) * ldadd) : nullptr;
      for (int v = lane; v < nvec; v += 32) {
        float fx[8], fd[8], fa[8], o[8];
        unpack8(__ldg(px + v), fx);
        unpack8(__ldg(pd + v), fd);
        if (pa) unpack8(__ldg(pa + v), fa);
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
        const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o[i] = rstd * (fd[i] * ww[i] - fx[i] * rstd * m);
          if (pa) o[i] += fa[i];
        }
        po[v] = pack8(o);
      }
    }
    const int r0 = grp * 8, nr = min(8, rows - r0);
    for (int v = threadIdx.x; v < nvec; v += 256) {
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = colacc[v * 8 + i];
      for (int r = 0; r < nr; ++r) {
        const long long rr = r0 + r;
        const float rs = __ldg(rstd_in + rr);
        float fx[8], fd[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(x + rr * ldx) + v), fx);
        unpack8(__ldg(reinterpret_cast<const uint4*>(dy + rr * lddy) + v), fd);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += fd[i] * (fx[i] * rs);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) colacc[v * 8 + i] = acc[i];
    }
  }
  float* wr = ws + static_cast<long long>(blockIdx.x) * D;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    reinterpret_cast<float4*>(wr)[2 * v] = colacc4[2 * v];
    reinterpret_cast<float4*>(wr)[2 * v + 1] = colacc4[2 * v + 1];
  }
}

// dw[c] (+)= sum over the chunks of ws[chunk][c]: a CTA owns 32 columns, its 8 thread rows stride over the chunks, then a
// fixed-order smem reduction (deterministic).
__global__ void __launch_bounds__(256)
rmsnorm_wgrad_finalize_kernel(const float* __restrict__ ws, float* __restrict__ dw, int D, int chunks, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sw[8][32];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float a = 0.f;
  if (c < D) {
    for (int k = threadIdx.y; k < chunks; k += 8) a += ws[static_cast<long long>(k) * D + c];
  }
  sw[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < D) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < 8; ++y) t += sw[y][threadIdx.x];
    dw[c] = (accumulate ? dw[c] : 0.f) + t;
  }
}

// In-place rotary embedding of `nblk` column blocks of H heads x 128 dims (q and k of the fused projection buffer).
// Thread = one (row, block, head, pair index i < 64): x_i' = x_i c - x_{i+64} s ; x_{i+64}' = x_{i+64} c + x_i s
// (rotate_half), angle = pos * inv_freq_i with inv_freq_i = theta^(-2i/128), or inv_tab[i] when a table is given (scaled
// RoPE); c, s are multiplied by attn_scale (yarn's attention factor, 1 otherwise); sign = -1 applies the transpose
// (backward).
__global__ void __launch_bounds__(256)
rope128_kernel(bf16* __restrict__ buf, long long ld, long long rows, int H, int S, int nblk, float log2_theta,
               const float* __restrict__ inv_tab, float attn_scale, float sign) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = rows * nblk * H * 64;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int i = static_cast<int>(idx & 63);
    const long long t = idx >> 6;
    const int h = static_cast<int>(t % H);
    const long long t2 = t / H;
    const int blk = static_cast<int>(t2 % nblk);
    const long long row = t2 / nblk;
    const int pos = static_cast<int>(row % S);
    const float inv_freq = inv_tab != nullptr ? __ldg(inv_tab + i) : exp2f(-log2_theta * static_cast<float>(2 * i) / 128.0f);
    float s, c;
    sincosf(static_cast<float>(pos) * inv_freq, &s, &c);
    c *= attn_scale;
    s *= sign * attn_scale;
    bf16* p = buf + row * ld + (static_cast<long long>(blk) * H + h) * 128 + i;
    const float a = __bfloat162float(p[0]), b = __bfloat162float(p[64]);
    p[0] = __float2bfloat16_rn(a * c - b * s);
    p[64] = __float2bfloat16_rn(b * c + a * s);
  }
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

// h = silu(g) * u      gu: [rows][2*I] with g at columns [0, I), u at [I, 2I)  (or separate pointers via ld)
__global__ void __launch_bounds__(256)
swiglu_fwd_kernel(const bf16* __restrict__ g, long long ldg, const bf16* __restrict__ u, long long ldu, bf16* __restrict__ h,
                  long long ldh, long long rows, int I) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = I >> 3;
  const long long total = rows * nvec;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = idx / nvec;
    const int v = static_cast<int>(idx % nvec);
    float fg[8], fu[8], o[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(g + row * ldg) + v), fg);
    unpack8(__ldg(reinterpret_cast<const uint4*>(u + row * ldu) + v), fu);
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = fg[i] * sigmoidf_(fg[i]) * fu[i];
    reinterpret_cast<uint4*>(h + row * ldh)[v] = pack8(o);
  }
}

// dg = dh * u * (sig + g * sig * (1 - sig)),  du = dh * g * sig
__global__ void __launch_bounds__(256)
swiglu_bwd_kernel(const bf16* __restrict__ dh, long long lddh, const bf16* __restrict__ g, long long ldg,
                  const bf16* __restrict__ u, long long ldu, bf16* __restrict__ dg, long long lddg, bf16* __restrict__ du,
                  long long lddu, long long rows, int I) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = I >> 3;
  const long long total = rows * nvec;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = idx / nvec;
    const int v = static_cast<int>(idx % nvec);
    float fd[8], fg[8], fu[8], og[8], ou[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(dh + row * lddh) + v), fd);
    unpack8(__ldg(reinterpret_cast<const uint4*>(g + row * ldg) + v), fg);
    unpack8(__ldg(reinterpret_cast<const uint4*>(u + row * ldu) + v), fu);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float sg = sigmoidf_(fg[i]);
      og[i] = fd[i] * fu[i] * (sg + fg[i] * sg * (1.0f - sg));
      ou[i] = fd[i] * fg[i] * sg;
    }
    reinterpret_cast<uint4*>(dg + row * lddg)[v] = pack8(og);
    reinterpret_cast<uint4*>(du + row * lddu)[v] = pack8(ou);
  }
}

constexpr int kRmsWGradMaxD = 16384;     // the weight-gradient kernel's column partials live in smem: D fp32

static inline int ew_grid(long long items) {
  long long g = (items + 255) / 256;
  const long long cap = static_cast<long long>(sm_count()) * 8;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace otb

using namespace otb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int otb_rmsnorm_fwd(const void* x, int64_t ldx, const float* weight, void* y, int64_t ldy, float* rstd, int rows,
                               int D, float eps, void* stream) {
  OTB_CHECK_ARG(x && weight && y && rows > 0 && D > 0 && D % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0, "otb_rmsnorm_fwd: bad argument");
  OTB_CHECK_CUDA(launch_k(rmsnorm_fwd_kernel, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), static_cast<const bf16*>(x),
                          (long long)ldx, weight, static_cast<bf16*>(y), (long long)ldy, rstd, rows, D, eps));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_rmsnorm_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* rstd, const float* weight,
                               const void* add, int64_t ldadd, void* dx, int64_t lddx, int rows, int D, void* stream) {
  OTB_CHECK_ARG(dy && x && rstd && weight && dx && rows > 0 && D > 0 && D % 8 == 0, "otb_rmsnorm_bwd: bad argument");
  OTB_CHECK_ARG(lddy % 8 == 0 && ldx % 8 == 0 && lddx % 8 == 0 && (add == nullptr || ldadd % 8 == 0), "otb_rmsnorm_bwd: bad ld");
  OTB_CHECK_CUDA(launch_k(rmsnorm_bwd_kernel, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), static_cast<const bf16*>(dy),
                          (long long)lddy, static_cast<const bf16*>(x), (long long)ldx, rstd, weight,
                          static_cast<const bf16*>(add), (long long)ldadd, static_cast<bf16*>(dx), (long long)lddx, rows, D));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_rmsnorm_bwd_chunks(int rows, int D) {
  if (rows <= 0 || D <= 0) return 1;
  const int groups = (rows + 7) / 8, cap = 4 * sm_count();     // 4 CTAs of 8 warps per SM
  return groups < cap ? groups : cap;
}

extern "C" int otb_rmsnorm_bwd_params(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* rstd,
                                      const float* weight, const void* add, int64_t ldadd, void* dx, int64_t lddx,
                                      float* dweight, int accumulate, float* ws, int rows, int D, void* stream) {
  OTB_CHECK_ARG(dy && x && rstd && weight && dx && dweight && ws && rows > 0 && D > 0 && D % 8 == 0,
                "otb_rmsnorm_bwd_params: bad argument");
  OTB_CHECK_ARG(D <= kRmsWGradMaxD, "otb_rmsnorm_bwd_params: D = %d exceeds %d", D, kRmsWGradMaxD);
  OTB_CHECK_ARG(lddy % 8 == 0 && ldx % 8 == 0 && lddx % 8 == 0 && (add == nullptr || ldadd % 8 == 0),
                "otb_rmsnorm_bwd_params: bad ld");
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "otb_rmsnorm_bwd_params: ws must be 16-byte aligned");
  const int chunks = otb_rmsnorm_bwd_chunks(rows, D);
  const int smem = D * static_cast<int>(sizeof(float));
  OTB_CHECK_CUDA(ensure_dyn_smem(rmsnorm_bwd_wgrad_kernel, kRmsWGradMaxD * static_cast<int>(sizeof(float))));   // once
  OTB_CHECK_CUDA(launch_k(rmsnorm_bwd_wgrad_kernel, dim3(chunks), dim3(256), smem, ST(stream), static_cast<const bf16*>(dy),
                          (long long)lddy, static_cast<const bf16*>(x), (long long)ldx, rstd, weight,
                          static_cast<const bf16*>(add), (long long)ldadd, static_cast<bf16*>(dx), (long long)lddx, ws, rows,
                          D));
  OTB_CHECK_CUDA(launch_k(rmsnorm_wgrad_finalize_kernel, dim3((D + 31) / 32), dim3(32, 8), 0, ST(stream),
                          static_cast<const float*>(ws), dweight, D, chunks, accumulate));
  count_launch(2);
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_rope128(void* buf, int64_t ld, int64_t rows, int H, int S, int nblk, float rope_theta, int backward,
                           void* stream) {
  OTB_CHECK_ARG(buf && rows > 0 && H > 0 && S > 0 && nblk > 0 && ld >= (int64_t)nblk * H * 128 && rope_theta > 1.f,
                "otb_rope128: bad argument");
  OTB_CHECK_CUDA(launch_k(rope128_kernel, dim3(ew_grid(rows * nblk * H * 64)), dim3(256), 0, ST(stream), static_cast<bf16*>(buf),
                          (long long)ld, (long long)rows, H, S, nblk, log2f(rope_theta), static_cast<const float*>(nullptr),
                          1.0f, backward ? -1.0f : 1.0f));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_rope128_freqs(void* buf, int64_t ld, int64_t rows, int H, int S, int nblk, const float* inv_freq,
                                 float attn_scale, int backward, void* stream) {
  OTB_CHECK_ARG(buf && inv_freq && rows > 0 && H > 0 && S > 0 && nblk > 0 && ld >= (int64_t)nblk * H * 128 &&
                    attn_scale > 0.f && attn_scale < INFINITY,
                "otb_rope128_freqs: bad argument");
  OTB_CHECK_CUDA(launch_k(rope128_kernel, dim3(ew_grid(rows * nblk * H * 64)), dim3(256), 0, ST(stream), static_cast<bf16*>(buf),
                          (long long)ld, (long long)rows, H, S, nblk, 0.0f, inv_freq, attn_scale, backward ? -1.0f : 1.0f));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_swiglu_fwd(const void* g, int64_t ldg, const void* u, int64_t ldu, void* h, int64_t ldh, int64_t rows, int I,
                              void* stream) {
  OTB_CHECK_ARG(g && u && h && rows > 0 && I > 0 && I % 8 == 0 && ldg % 8 == 0 && ldu % 8 == 0 && ldh % 8 == 0,
                "otb_swiglu_fwd: bad argument");
  OTB_CHECK_CUDA(launch_k(swiglu_fwd_kernel, dim3(ew_grid(rows * (I / 8))), dim3(256), 0, ST(stream), static_cast<const bf16*>(g),
                          (long long)ldg, static_cast<const bf16*>(u), (long long)ldu, static_cast<bf16*>(h), (long long)ldh,
                          (long long)rows, I));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_swiglu_bwd(const void* dh, int64_t lddh, const void* g, int64_t ldg, const void* u, int64_t ldu, void* dg,
                              int64_t lddg, void* du, int64_t lddu, int64_t rows, int I, void* stream) {
  OTB_CHECK_ARG(dh && g && u && dg && du && rows > 0 && I > 0 && I % 8 == 0, "otb_swiglu_bwd: bad argument");
  OTB_CHECK_ARG(lddh % 8 == 0 && ldg % 8 == 0 && ldu % 8 == 0 && lddg % 8 == 0 && lddu % 8 == 0, "otb_swiglu_bwd: bad ld");
  OTB_CHECK_CUDA(launch_k(swiglu_bwd_kernel, dim3(ew_grid(rows * (I / 8))), dim3(256), 0, ST(stream), static_cast<const bf16*>(dh),
                          (long long)lddh, static_cast<const bf16*>(g), (long long)ldg, static_cast<const bf16*>(u),
                          (long long)ldu, static_cast<bf16*>(dg), (long long)lddg, static_cast<bf16*>(du), (long long)lddu,
                          (long long)rows, I));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
