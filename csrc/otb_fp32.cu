// otter_b200 — fp32-grade forward path (parity mode): meets the north star's 1e-3 rel / 1e-5 abs against the
// reference's fp32 forward.  The dense contractions still run on the wgmma GEMM: each fp32 operand is split into
// three bf16 terms x = x0 + x1 + x2 (24 mantissa bits) and the six significant cross products
//   x0y0 + x0y1 + x1y0 + x1y1 + x0y2 + x2y0
// are evaluated as ONE bf16 GEMM over a 6x longer reduction dimension (operands concatenated along K by
// otb_split3_concat), accumulated in fp32 registers.  LayerNorm / softmax / attention run in fp32 on CUDA cores
// (they are < 0.1 % of the FLOPs).  Forward only; used by tests and by `otter_b200.precision("fp32")`.
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

__device__ __forceinline__ float warp_sum32(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// pattern 0 (A side): [x0 x0 x1 x1 x0 x2]   pattern 1 (B side): [y0 y1 y0 y1 y2 y0]
__global__ void split3_concat_kernel(const float* __restrict__ src, long long ld, int rows, int K, int pattern,
                                     bf16* __restrict__ dst) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(rows) * K;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / K), k = static_cast<int>(i % K);
    const float x = src[static_cast<long long>(r) * ld + k];
    const bf16 x0 = __float2bfloat16(x);
    const float r1 = x - __bfloat162float(x0);
    const bf16 x1 = __float2bfloat16(r1);
    const float r2 = r1 - __bfloat162float(x1);
    const bf16 x2 = __float2bfloat16(r2);
    bf16* d = dst + static_cast<long long>(r) * (6LL * K) + k;
    if (pattern == 0) {
      d[0] = x0; d[K] = x0; d[2LL * K] = x1; d[3LL * K] = x1; d[4LL * K] = x0; d[5LL * K] = x2;
    } else {
      d[0] = x0; d[K] = x1; d[2LL * K] = x0; d[3LL * K] = x1; d[4LL * K] = x2; d[5LL * K] = x0;
    }
  }
}

__global__ void __launch_bounds__(256)
ln_fwd_f32_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ gamma,
                  const float* __restrict__ beta, float* __restrict__ y, long long ldy, int rows, int D, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= rows) return;
  const float* xr = x + static_cast<long long>(row) * ldx;
  float s = 0.f;
  for (int c = lane; c < D; c += 32) s += xr[c];
  const float mean = warp_sum32(s) / D;
  float ss = 0.f;
  for (int c = lane; c < D; c += 32) { const float d = xr[c] - mean; ss += d * d; }
  const float rstd = 1.0f / sqrtf(warp_sum32(ss) / D + eps);
  float* yr = y + static_cast<long long>(row) * ldy;
  for (int c = lane; c < D; c += 32) yr[c] = (xr[c] - mean) * rstd * gamma[c] + beta[c];
}

__global__ void add_rowbias_f32_kernel(const float* __restrict__ x, const float* __restrict__ bias, int div, int mod,
                                       float* __restrict__ out, int rows, int D) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(rows) * D;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / D), c = static_cast<int>(i % D);
    out[i] = x[i] + bias[static_cast<long long>((r / div) % mod) * D + c];
  }
}

// epilogue of the chunked fp32-grade GEMM (same order as the fused one): act(acc + bias) * gate + residual
__global__ void epilogue_f32_kernel(const float* __restrict__ acc, const float* __restrict__ bias, int act,
                                    const float* __restrict__ scale_ptr, int scale_tanh,
                                    const float* __restrict__ residual, float* __restrict__ out, int M, int N) {
  pdl_launch_dependents();
  pdl_wait();
  float scale = 1.0f;
  if (scale_ptr != nullptr) scale = scale_tanh ? tanhf(*scale_ptr) : *scale_ptr;
  const long long total = static_cast<long long>(M) * N;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v = acc[i];
    if (bias != nullptr) v += bias[i % N];
    if (act == 1) v = 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    else if (act == 2) v = v / (1.0f + expf(-1.702f * v));
    v *= scale;
    if (residual != nullptr) v += residual[i];
    out[i] = v;
  }
}

// fp32 attention forward, one thread per query row (d = 64 in registers), exact two-pass softmax semantics of the
// reference incl. the media mask classes.  q/kv/out are fp32 matrices addressed like the bf16 kernels.
struct AttnF32 {
  const float* q; const float* kv1; const float* kv2; float* out; const int* text_time;
  long long ldq, ldkv1, ldkv2, ldo;
  int q_col0, k1_col0, v1_col0, k2_col0, v2_col0, o_col0, n_per_media, T_img, P, H, Sq, Sk1, Sk2, mask_ge, causal;
  float scale;
};
__global__ void __launch_bounds__(64) attn_fwd_f32_kernel(AttnF32 p) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * 64 + threadIdx.x, h = blockIdx.y, prob = blockIdx.z;
  if (row >= p.Sq) return;
  const long long grow = static_cast<long long>(prob) * p.Sq + row;
  float q[64], acc[64];
  const float* qp = p.q + grow * p.ldq + p.q_col0 + h * 64;
#pragma unroll
  for (int d = 0; d < 64; ++d) { q[d] = qp[d] * p.scale; acc[d] = 0.f; }
  int cls = 1, tt = 0;
  if (p.text_time != nullptr) {
    tt = p.text_time[grow];
    cls = p.mask_ge ? (tt == 0 ? 2 : 1) : ((tt == 0) ? 0 : (tt <= p.T_img ? 1 : 2));
  }
  // key j participates (class 1): eq -> slot of j equals tt; ge -> slot of j <= tt; causal -> j <= row
  auto allowed = [&](int j) {
    if (p.causal && j > row) return false;
    if (p.text_time == nullptr) return true;
    const int slot = j / p.n_per_media + 1;
    return p.mask_ge ? (slot <= tt) : (slot == tt);
  };
  float* op = p.out + grow * p.ldo + p.o_col0 + h * 64;
  if (cls == 0) {
#pragma unroll
    for (int d = 0; d < 64; ++d) op[d] = 0.f;
    return;
  }
  const int nk = p.Sk1 + p.Sk2;
  // pass 1: max
  float m = -INFINITY;
  if (cls == 1) {
    for (int j = 0; j < nk; ++j) {
      if (!allowed(j)) continue;
      const float* kp = (j < p.Sk1) ? p.kv1 + (static_cast<long long>(prob) * p.Sk1 + j) * p.ldkv1 + p.k1_col0 + h * 64
                                    : p.kv2 + (static_cast<long long>(prob) * p.Sk2 + (j - p.Sk1)) * p.ldkv2 + p.k2_col0 + h * 64;
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) s = fmaf(q[d], kp[d], s);
      m = fmaxf(m, s);
    }
  }
  float l = 0.f;
  for (int j = 0; j < nk; ++j) {
    float w;
    const bool src1 = j < p.Sk1;
    const long long krow = src1 ? (static_cast<long long>(prob) * p.Sk1 + j) : (static_cast<long long>(prob) * p.Sk2 + (j - p.Sk1));
    if (cls == 2) {
      w = 1.0f;
    } else {
      if (!allowed(j)) continue;
      const float* kp = src1 ? p.kv1 + krow * p.ldkv1 + p.k1_col0 + h * 64 : p.kv2 + krow * p.ldkv2 + p.k2_col0 + h * 64;
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) s = fmaf(q[d], kp[d], s);
      w = expf(s - m);
    }
    l += w;
    const float* vp = src1 ? p.kv1 + krow * p.ldkv1 + p.v1_col0 + h * 64 : p.kv2 + krow * p.ldkv2 + p.v2_col0 + h * 64;
#pragma unroll
    for (int d = 0; d < 64; ++d) acc[d] = fmaf(w, vp[d], acc[d]);
  }
  const float inv = 1.0f / l;
#pragma unroll
  for (int d = 0; d < 64; ++d) op[d] = acc[d] * inv;
}

static inline int grid1d(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  return static_cast<int>(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace otb

using namespace otb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int otb_split3_concat(const float* src, int64_t ld, int rows, int K, int pattern, void* dst, void* stream) {
  OTB_CHECK_ARG(src && dst && rows > 0 && K > 0 && ld >= K && (pattern == 0 || pattern == 1),
                "otb_split3_concat: bad argument");
  OTB_CHECK_CUDA(launch_k(split3_concat_kernel, dim3(grid1d(static_cast<long long>(rows) * K, 256)), dim3(256), 0, ST(stream), 
      src, ld, rows, K, pattern, static_cast<bf16*>(dst)));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_layernorm_fwd_f32(const float* x, int64_t ldx, const float* gamma, const float* beta, float* y,
                                     int64_t ldy, int rows, int D, float eps, void* stream) {
  OTB_CHECK_ARG(x && gamma && beta && y && rows > 0 && D > 0, "otb_layernorm_fwd_f32: bad argument");
  OTB_CHECK_CUDA(launch_k(ln_fwd_f32_kernel, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), x, ldx, gamma, beta, y, ldy, rows, D, eps));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_add_rowbias_f32(const float* x, const float* bias, int div, int mod, float* out, int rows, int D,
                                   void* stream) {
  OTB_CHECK_ARG(x && bias && out && div > 0 && mod > 0 && rows > 0 && D > 0, "otb_add_rowbias_f32: bad argument");
  OTB_CHECK_CUDA(launch_k(add_rowbias_f32_kernel, dim3(grid1d(static_cast<long long>(rows) * D, 256)), dim3(256), 0, ST(stream), x, bias, div, mod, out,
                                                                                              rows, D));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_epilogue_f32(const float* acc, const float* bias, int act, const float* scale_ptr, int scale_tanh,
                                const float* residual, float* out, int M, int N, void* stream) {
  OTB_CHECK_ARG(acc && out && M > 0 && N > 0 && act >= 0 && act <= 2, "otb_epilogue_f32: bad argument");
  OTB_CHECK_CUDA(launch_k(epilogue_f32_kernel, dim3(grid1d(static_cast<long long>(M) * N, 256)), dim3(256), 0, ST(stream), acc, bias, act, scale_ptr,
                                                                                        scale_tanh, residual, out, M, N));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
extern "C" int otb_attn_fwd_f32(const otb_attn_desc* d, void* stream) {
  OTB_CHECK_ARG(d && d->q && d->kv1 && d->out && d->head_dim == 64 && d->P > 0 && d->H > 0 && d->Sq > 0 && d->Sk1 > 0,
                "otb_attn_fwd_f32: bad argument");
  OTB_CHECK_ARG(d->Sk2 == 0 || d->kv2, "otb_attn_fwd_f32: kv2 missing");
  OTB_CHECK_ARG(d->text_time == nullptr || (d->Sk2 == 0 && d->n_per_media > 0 && d->T_img * d->n_per_media == d->Sk1),
                "otb_attn_fwd_f32: media mask needs a single key source with Sk1 == T_img * n_per_media");
  AttnF32 p;
  p.q = static_cast<const float*>(d->q); p.kv1 = static_cast<const float*>(d->kv1);
  p.kv2 = static_cast<const float*>(d->kv2); p.out = static_cast<float*>(d->out); p.text_time = d->text_time;
  p.ldq = d->ldq; p.ldkv1 = d->ldkv1; p.ldkv2 = d->ldkv2; p.ldo = d->ld_out;
  p.q_col0 = d->q_col0; p.k1_col0 = d->k1_col0; p.v1_col0 = d->v1_col0; p.k2_col0 = d->k2_col0; p.v2_col0 = d->v2_col0;
  p.o_col0 = d->out_col0; p.n_per_media = d->n_per_media; p.T_img = d->T_img; p.mask_ge = d->mask_ge; p.causal = d->causal;
  p.P = d->P; p.H = d->H; p.Sq = d->Sq; p.Sk1 = d->Sk1; p.Sk2 = d->Sk2; p.scale = d->scale;
  dim3 grid((d->Sq + 63) / 64, d->H, d->P);
  OTB_CHECK_CUDA(launch_k(attn_fwd_f32_kernel, dim3(grid), dim3(64), 0, ST(stream), p));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
