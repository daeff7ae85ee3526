// otter_b200 — fp32-grade BACKWARD path (parity mode): gradients of the perceiver / gated cross-attention blocks held to
// the north star's 1e-3 rel tolerance against the reference's fp32 autograd (modeling_otter.py:129-184, :238-340, :343-395).
// The dense contractions (dgrad / wgrad) reuse the three-term bf16 split GEMM of the forward path (otb_split3_concat +
// otb_gemm_bf16); this file holds the fp32 CUDA-core passes around them: LayerNorm backward, attention backward (exact
// two-pass softmax semantics incl. the media-mask classes), activation derivative, tanh-gate gradient, row-bias gradient.
// Deterministic (no atomics).  Used by tests and by `otter_b200.precision("fp32")`; never timed.
#include "otb_common.cuh"
#include "otb_host.h"
#include "../include/otter_b200.h"

namespace otb {

// ---- LayerNorm backward: dx (one warp per row) + the row statistics for the parameter pass ----
__global__ void __launch_bounds__(256)
ln_bwd_dx_f32_kernel(const float* __restrict__ dy, long long lddy, const float* __restrict__ x, long long ldx,
                     const float* __restrict__ gamma, float* __restrict__ dx, long long lddx, float* __restrict__ stats,
                     int rows, int D, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= rows) return;
  const float* xr = x + static_cast<long long>(row) * ldx;
  const float* gr = dy + static_cast<long long>(row) * lddy;
  float s = 0.f;
  for (int c = lane; c < D; c += 32) s += xr[c];
  const float mean = warp_sum(s) / D;
  float ss = 0.f;
  for (int c = lane; c < D; c += 32) { const float d = xr[c] - mean; ss += d * d; }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) / D + eps);
  float s1 = 0.f, s2 = 0.f;
  for (int c = lane; c < D; c += 32) {
    const float g = gr[c] * gamma[c];
    s1 += g;
    s2 += g * (xr[c] - mean) * rstd;
  }
  s1 = warp_sum(s1) / D;
  s2 = warp_sum(s2) / D;
  if (lane == 0) { stats[2 * row] = mean; stats[2 * row + 1] = rstd; }
  if (dx != nullptr) {
    float* o = dx + static_cast<long long>(row) * lddx;
    for (int c = lane; c < D; c += 32) {
      const float xh = (xr[c] - mean) * rstd;
      o[c] = rstd * (gr[c] * gamma[c] - s1 - xh * s2);
    }
  }
}

// dgamma[c] = sum_r dy[r][c] * xhat[r][c],  dbeta[c] = sum_r dy[r][c]    (one thread per column, rows in order)
__global__ void __launch_bounds__(128)
ln_bwd_param_f32_kernel(const float* __restrict__ dy, long long lddy, const float* __restrict__ x, long long ldx,
                        const float* __restrict__ stats, float* __restrict__ dgamma, float* __restrict__ dbeta, int rows,
                        int D) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= D) return;
  float g = 0.f, b = 0.f, gc = 0.f, bc = 0.f;       // Kahan-compensated: 1e-3 must hold for thousands of rows
  for (int r = 0; r < rows; ++r) {
    const float d = dy[static_cast<long long>(r) * lddy + c];
    const float xh = (x[static_cast<long long>(r) * ldx + c] - stats[2 * r]) * stats[2 * r + 1];
    float y = d * xh - gc, t = g + y;
    gc = (t - g) - y; g = t;
    y = d - bc; t = b + y;
    bc = (t - b) - y; b = t;
  }
  dgamma[c] = g;
  dbeta[c] = b;
}

// ---- activation derivative: out = dy * act'(pre)   act 1 = exact GELU (erf), 2 = quick-GELU ----
__global__ void act_bwd_f32_kernel(const float* __restrict__ dy, const float* __restrict__ pre, int act,
                                   float* __restrict__ out, long long n) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = pre[i];
    float d;
    if (act == 1) {
      d = 0.5f * (1.0f + erff(v * 0.70710678118654752f)) + v * 0.39894228040143268f * expf(-0.5f * v * v);
    } else {
      const float sg = 1.0f / (1.0f + expf(-1.702f * v));
      d = sg + 1.702f * v * sg * (1.0f - sg);
    }
    out[i] = dy[i] * d;
  }
}

// ---- tanh-gate gradient: out[0] = (1 - tanh(g)^2) * sum_i dy[i] * f[i]   (one CTA, double accumulation) ----
__global__ void __launch_bounds__(1024)
gate_grad_f32_kernel(const float* __restrict__ dy, const float* __restrict__ f, long long n,
                     const float* __restrict__ gate, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[32];
  double acc = 0.0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) acc += static_cast<double>(dy[i]) * static_cast<double>(f[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 32; ++w) t += red[w];
    const float th = tanhf(*gate);
    out[0] = static_cast<float>(t * (1.0 - static_cast<double>(th) * th));
  }
}

// ---- gradient of otb_add_rowbias_f32's bias: out[m][c] = sum over rows r with (r / div) % mod == m of dy[r][c] ----
__global__ void __launch_bounds__(128)
rowbias_grad_f32_kernel(const float* __restrict__ dy, int div, int mod, int rows, int D, int out_rows,
                        float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
  if (c >= D) return;
  float s = 0.f, comp = 0.f;
  if (m < mod) {
    for (long long base = static_cast<long long>(m) * div; base < rows; base += static_cast<long long>(mod) * div)
      for (int t = 0; t < div && base + t < rows; ++t) {
        const float y = dy[(base + t) * D + c] - comp, u = s + y;
        comp = (u - s) - y; s = u;
      }
  }
  if (m < out_rows) out[static_cast<long long>(m) * D + c] = s;     // rows >= mod of the table receive zero
}

// ---- attention backward ----
struct AttnBwdF32 {
  const float* q; const float* kv1; const float* kv2; const float* o; const float* dout; const int* text_time;
  float* dq; float* dkv1; float* dkv2; float* stats;                 // stats [P][H][Sq][3] = m, l, delta
  long long ldq, ldkv1, ldkv2, ldo, lddo, lddq, lddkv1, lddkv2;
  int q_col0, k1_col0, v1_col0, k2_col0, v2_col0, o_col0, do_col0, dq_col0, dk1_col0, dv1_col0, dk2_col0, dv2_col0;
  int n_per_media, T_img, P, H, Sq, Sk1, Sk2, mask_ge, causal;
  float scale;
};

__device__ __forceinline__ int row_cls(const AttnBwdF32& p, int tt) {
  if (p.text_time == nullptr) return 1;
  return p.mask_ge ? (tt == 0 ? 2 : 1) : ((tt == 0) ? 0 : (tt <= p.T_img ? 1 : 2));
}
__device__ __forceinline__ bool key_allowed(const AttnBwdF32& p, int tt, int row, int j) {
  if (p.causal && j > row) return false;
  if (p.text_time == nullptr) return true;
  const int slot = j / p.n_per_media + 1;
  return p.mask_ge ? (slot <= tt) : (slot == tt);
}
__device__ __forceinline__ const float* key_ptr(const AttnBwdF32& p, int prob, int h, int j, bool value) {
  if (j < p.Sk1)
    return p.kv1 + (static_cast<long long>(prob) * p.Sk1 + j) * p.ldkv1 + (value ? p.v1_col0 : p.k1_col0) + h * 64;
  return p.kv2 + (static_cast<long long>(prob) * p.Sk2 + (j - p.Sk1)) * p.ldkv2 + (value ? p.v2_col0 : p.k2_col0) + h * 64;
}

// one thread per query row: softmax statistics, delta = dO . O, and dq
__global__ void __launch_bounds__(64) attn_bwd_q_f32_kernel(AttnBwdF32 p) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x * 64 + threadIdx.x, h = blockIdx.y, prob = blockIdx.z;
  if (row >= p.Sq) return;
  const long long grow = static_cast<long long>(prob) * p.Sq + row;
  float q[64], go[64], acc[64];
  const float* qp = p.q + grow * p.ldq + p.q_col0 + h * 64;
  const float* gp = p.dout + grow * p.lddo + p.do_col0 + h * 64;
  const float* op = p.o + grow * p.ldo + p.o_col0 + h * 64;
  float delta = 0.f;
#pragma unroll
  for (int d = 0; d < 64; ++d) { q[d] = qp[d] * p.scale; go[d] = gp[d]; delta = fmaf(go[d], op[d], delta); acc[d] = 0.f; }
  const int tt = p.text_time ? p.text_time[grow] : 0;
  const int cls = row_cls(p, tt);
  const int nk = p.Sk1 + p.Sk2;
  float* st = p.stats + ((static_cast<long long>(prob) * p.H + h) * p.Sq + row) * 3;
  float* dqp = p.dq + grow * p.lddq + p.dq_col0 + h * 64;
  if (cls != 1) {                       // 0: output is the constant 0;  2: uniform weights, independent of q and k
    st[0] = 0.f; st[1] = (cls == 0) ? 0.f : static_cast<float>(nk); st[2] = delta;
#pragma unroll
    for (int d = 0; d < 64; ++d) dqp[d] = 0.f;
    return;
  }
  float m = -INFINITY;
  for (int j = 0; j < nk; ++j) {
    if (!key_allowed(p, tt, row, j)) continue;
    const float* kp = key_ptr(p, prob, h, j, false);
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < 64; ++d) s = fmaf(q[d], kp[d], s);
    m = fmaxf(m, s);
  }
  float l = 0.f;
  for (int j = 0; j < nk; ++j) {
    if (!key_allowed(p, tt, row, j)) continue;
    const float* kp = key_ptr(p, prob, h, j, false);
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < 64; ++d) s = fmaf(q[d], kp[d], s);
    l += expf(s - m);
  }
  st[0] = m; st[1] = l; st[2] = delta;
  const float inv = 1.0f / l;
  for (int j = 0; j < nk; ++j) {
    if (!key_allowed(p, tt, row, j)) continue;
    const float* kp = key_ptr(p, prob, h, j, false);
    const float* vp = key_ptr(p, prob, h, j, true);
    float s = 0.f, dp = 0.f;
#pragma unroll
    for (int d = 0; d < 64; ++d) { s = fmaf(q[d], kp[d], s); dp = fmaf(go[d], vp[d], dp); }
    const float ds = expf(s - m) * inv * (dp - delta);
#pragma unroll
    for (int d = 0; d < 64; ++d) acc[d] = fmaf(ds, kp[d], acc[d]);
  }
#pragma unroll
  for (int d = 0; d < 64; ++d) dqp[d] = acc[d] * p.scale;
}

// one thread per key row, query rows visited in order: dK (kValue = false) or dV (kValue = true)
template <bool kValue>
__global__ void __launch_bounds__(64) attn_bwd_kv_f32_kernel(AttnBwdF32 p) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = blockIdx.x * 64 + threadIdx.x, h = blockIdx.y, prob = blockIdx.z;
  const int nk = p.Sk1 + p.Sk2;
  if (j >= nk) return;
  float k[64], v[64], acc[64];
  const float* kp = key_ptr(p, prob, h, j, false);
  const float* vp = key_ptr(p, prob, h, j, true);
#pragma unroll
  for (int d = 0; d < 64; ++d) { k[d] = kp[d]; v[d] = kValue ? 0.f : vp[d]; acc[d] = 0.f; }
  for (int row = 0; row < p.Sq; ++row) {
    const long long grow = static_cast<long long>(prob) * p.Sq + row;
    const float* st = p.stats + ((static_cast<long long>(prob) * p.H + h) * p.Sq + row) * 3;
    const float m = st[0], l = st[1], delta = st[2];
    if (l == 0.f) continue;                                            // class 0 row
    const int tt = p.text_time ? p.text_time[grow] : 0;
    const int cls = row_cls(p, tt);
    const float* gp = p.dout + grow * p.lddo + p.do_col0 + h * 64;
    if (cls == 2) {
      if (kValue) {
        const float w = 1.0f / l;
#pragma unroll
        for (int d = 0; d < 64; ++d) acc[d] = fmaf(w, gp[d], acc[d]);
      }
      continue;
    }
    if (!key_allowed(p, tt, row, j)) continue;
    const float* qp = p.q + grow * p.ldq + p.q_col0 + h * 64;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < 64; ++d) s = fmaf(qp[d] * p.scale, k[d], s);
    const float w = expf(s - m) / l;
    if (kValue) {
#pragma unroll
      for (int d = 0; d < 64; ++d) acc[d] = fmaf(w, gp[d], acc[d]);
    } else {
      float dp = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) dp = fmaf(gp[d], v[d], dp);
      const float ds = w * (dp - delta) * p.scale;
#pragma unroll
      for (int d = 0; d < 64; ++d) acc[d] = fmaf(ds, qp[d], acc[d]);
    }
  }
  float* out;
  if (j < p.Sk1) out = p.dkv1 + (static_cast<long long>(prob) * p.Sk1 + j) * p.lddkv1 + (kValue ? p.dv1_col0 : p.dk1_col0) + h * 64;
  else out = p.dkv2 + (static_cast<long long>(prob) * p.Sk2 + (j - p.Sk1)) * p.lddkv2 + (kValue ? p.dv2_col0 : p.dk2_col0) + h * 64;
#pragma unroll
  for (int d = 0; d < 64; ++d) out[d] = acc[d];
}

static inline int grid1d_b(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = static_cast<long long>(sm_count()) * 16;
  return static_cast<int>(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace otb

using namespace otb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int otb_layernorm_bwd_f32(const float* dy, int64_t lddy, const float* x, int64_t ldx, const float* gamma,
                                     float* dx, int64_t lddx, float* dgamma, float* dbeta, float* ws, int rows, int D,
                                     float eps, void* stream) {
  OTB_CHECK_ARG(dy && x && gamma && ws && rows > 0 && D > 0 && lddy >= D && ldx >= D && (dx == nullptr || lddx >= D),
                "otb_layernorm_bwd_f32: bad argument");
  OTB_CHECK_ARG((dgamma == nullptr) == (dbeta == nullptr), "otb_layernorm_bwd_f32: dgamma and dbeta go together");
  OTB_CHECK_CUDA(launch_k(ln_bwd_dx_f32_kernel, dim3((rows + 7) / 8), dim3(256), 0, ST(stream), dy, (long long)lddy, x,
                          (long long)ldx, gamma, dx, (long long)lddx, ws, rows, D, eps));
  count_launch();
  if (dgamma != nullptr) {
    OTB_CHECK_CUDA(launch_k(ln_bwd_param_f32_kernel, dim3((D + 127) / 128), dim3(128), 0, ST(stream), dy, (long long)lddy, x,
                            (long long)ldx, (const float*)ws, dgamma, dbeta, rows, D));
    count_launch();
  }
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_act_bwd_f32(const float* dy, const float* pre, int act, float* out, int64_t n, void* stream) {
  OTB_CHECK_ARG(dy && pre && out && n > 0 && (act == 1 || act == 2), "otb_act_bwd_f32: bad argument");
  OTB_CHECK_CUDA(launch_k(act_bwd_f32_kernel, dim3(grid1d_b(n, 256)), dim3(256), 0, ST(stream), dy, pre, act, out, (long long)n));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_gate_grad_f32(const float* dy, const float* f, int64_t n, const float* gate, float* out, void* stream) {
  OTB_CHECK_ARG(dy && f && gate && out && n > 0, "otb_gate_grad_f32: bad argument");
  OTB_CHECK_CUDA(launch_k(gate_grad_f32_kernel, dim3(1), dim3(1024), 0, ST(stream), dy, f, (long long)n, gate, out));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_rowbias_grad_f32(const float* dy, int div, int mod, int rows, int D, int out_rows, float* out,
                                    void* stream) {
  OTB_CHECK_ARG(dy && out && div > 0 && mod > 0 && rows > 0 && D > 0 && out_rows >= mod && out_rows <= 65535,
                "otb_rowbias_grad_f32: bad argument");
  OTB_CHECK_CUDA(launch_k(rowbias_grad_f32_kernel, dim3((D + 127) / 128, out_rows), dim3(128), 0, ST(stream), dy, div, mod,
                          rows, D, out_rows, out));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

// d: the forward problem with fp32 pointers, d->out = the forward output O.  g: fp32 gradients (dout in, dq / dkv1 / dkv2
// out, every element of the addressed head columns is written); g->dq_ws: fp32 [P*H*Sq*3] statistics scratch.
extern "C" int otb_attn_bwd_f32(const otb_attn_desc* d, const otb_attn_grads* g, void* stream) {
  OTB_CHECK_ARG(d && g && d->q && d->kv1 && d->out && g->dout && g->dq && g->dkv1 && g->dq_ws && d->head_dim == 64 &&
                    d->P > 0 && d->H > 0 && d->Sq > 0 && d->Sk1 > 0,
                "otb_attn_bwd_f32: bad argument");
  OTB_CHECK_ARG(d->Sk2 == 0 || (d->kv2 && g->dkv2), "otb_attn_bwd_f32: kv2 / dkv2 missing");
  OTB_CHECK_ARG(d->text_time == nullptr || (d->Sk2 == 0 && d->n_per_media > 0 && d->T_img * d->n_per_media == d->Sk1),
                "otb_attn_bwd_f32: media mask needs a single key source with Sk1 == T_img * n_per_media");
  AttnBwdF32 p;
  p.q = static_cast<const float*>(d->q); p.kv1 = static_cast<const float*>(d->kv1); p.kv2 = static_cast<const float*>(d->kv2);
  p.o = static_cast<const float*>(d->out); p.dout = static_cast<const float*>(g->dout); p.text_time = d->text_time;
  p.dq = static_cast<float*>(g->dq); p.dkv1 = static_cast<float*>(g->dkv1); p.dkv2 = static_cast<float*>(g->dkv2);
  p.stats = g->dq_ws;
  p.ldq = d->ldq; p.ldkv1 = d->ldkv1; p.ldkv2 = d->ldkv2; p.ldo = d->ld_out; p.lddo = g->ld_dout; p.lddq = g->ld_dq;
  p.lddkv1 = g->ld_dkv1; p.lddkv2 = g->ld_dkv2;
  p.q_col0 = d->q_col0; p.k1_col0 = d->k1_col0; p.v1_col0 = d->v1_col0; p.k2_col0 = d->k2_col0; p.v2_col0 = d->v2_col0;
  p.o_col0 = d->out_col0; p.do_col0 = g->dout_col0; p.dq_col0 = g->dq_col0; p.dk1_col0 = g->dk1_col0; p.dv1_col0 = g->dv1_col0;
  p.dk2_col0 = g->dk2_col0; p.dv2_col0 = g->dv2_col0;
  p.n_per_media = d->n_per_media; p.T_img = d->T_img; p.P = d->P; p.H = d->H; p.Sq = d->Sq; p.Sk1 = d->Sk1; p.Sk2 = d->Sk2;
  p.mask_ge = d->mask_ge; p.causal = d->causal; p.scale = d->scale;
  OTB_CHECK_CUDA(launch_k(attn_bwd_q_f32_kernel, dim3((d->Sq + 63) / 64, d->H, d->P), dim3(64), 0, ST(stream), p));
  const dim3 gk((d->Sk1 + d->Sk2 + 63) / 64, d->H, d->P);
  OTB_CHECK_CUDA(launch_k(attn_bwd_kv_f32_kernel<false>, gk, dim3(64), 0, ST(stream), p));
  OTB_CHECK_CUDA(launch_k(attn_bwd_kv_f32_kernel<true>, gk, dim3(64), 0, ST(stream), p));
  count_launch(3);
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
