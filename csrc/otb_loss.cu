// otter_b200 — §8f "next" row 2: the two steps either side of the hot path in the reference's training step.
//   (1) label masking  pipeline/train/instruction_following.py:163-190 — python double loop with torch.where syncs;
//       here one thread per sequence, bit-exact integer semantics (both interval passes of the reference).
//   (2) LM-head loss   src/otter_ai/models/mpt/modeling_mpt.py:430-436 — labels rolled by -1, last position ignored,
//       F.cross_entropy(mean over non-ignored targets); here fused forward + gradient, HBM-bound:
//       2 reads + 1 write of the [rows][vocab] logits, deterministic two-stage loss reduction.
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

// One CTA per sequence: the row is staged in shared memory (coalesced), one thread runs the two sequential
// pairing passes of the reference on it, and the labels go back out coalesced.
__global__ void __launch_bounds__(128)
label_mask_kernel(const long long* __restrict__ ids, int B, int L, long long eos_id, long long answer_id,
                  long long eoc_id, long long mask_val, long long* __restrict__ labels) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ long long lm_smem[];
  long long* x = lm_smem;        // [L]
  long long* y = lm_smem + L;    // [L]
  const int b = blockIdx.x;
  const long long* gx = ids + static_cast<long long>(b) * L;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const long long v = gx[i];
    x[i] = v;
    y[i] = (v == eos_id) ? eos_id : mask_val;                                                 // :166
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // pass 1 (:170-183): each <answer> pairs with the first not-yet-consumed <|endofchunk|> after it
    int e = 0;
    for (int a = 0; a < L; ++a) {
      if (x[a] != answer_id) continue;
      while (e < L && !(x[e] == eoc_id && e >= a)) ++e;      // while E[j] < a: j += 1
      if (e < L) {
        for (int p = a + 1; p <= e; ++p) y[p] = x[p];        // labels[a+1 : e+1] = ids[a+1 : e+1]
        ++e;                                                 // j += 1
      }
    }
    // pass 2 (:185-186): zip(answers, endofchunks) — k-th <answer> with k-th <|endofchunk|>
    int pa = 0, pe = 0;
    while (true) {
      while (pa < L && x[pa] != answer_id) ++pa;
      while (pe < L && x[pe] != eoc_id) ++pe;
      if (pa >= L || pe >= L) break;
      for (int p = pa + 1; p <= pe; ++p) y[p] = x[p];
      ++pa; ++pe;
    }
    y[0] = mask_val;                                                                          // :188
  }
  __syncthreads();
  long long* gy = labels + static_cast<long long>(b) * L;
  for (int i = threadIdx.x; i < L; i += blockDim.x) gy[i] = y[i];
}

__device__ __forceinline__ float ld_logit(const float* p, long long i) { return p[i]; }
__device__ __forceinline__ float ld_logit(const bf16* p, long long i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ void st_logit(float* p, long long i, float v) { p[i] = v; }
__device__ __forceinline__ void st_logit(bf16* p, long long i, float v) { p[i] = __float2bfloat16(v); }

// target of row (b, t): labels[b, t+1], last position ignored  (torch.roll(labels, -1); _labels[:, -1] = -100)
__device__ __forceinline__ long long shifted_target(const long long* labels, int L, long long row) {
  const int t = static_cast<int>(row % L);
  return (t == L - 1) ? -100 : labels[row + 1];
}

__global__ void ce_count_kernel(const long long* __restrict__ labels, long long rows, int L, float* __restrict__ count) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ int red[32];
  int c = 0;
  for (long long r = threadIdx.x; r < rows; r += blockDim.x) c += (shifted_target(labels, L, r) != -100) ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
    *count = static_cast<float>(t);
  }
}

// One CTA per (b, t) row.  When the row fits in shared memory (V * sizeof(T) <= 200 KB: 100 KB for MPT's 50 432
// bf16 logits) it is read from HBM exactly once with 16-byte loads, reduced from smem, and the gradient is written
// once: 1 read + 1 write = the algorithmic minimum.  Larger rows fall back to re-reading global memory.
template <typename T, bool kSmem>
__global__ void __launch_bounds__(512)
ce_row_kernel(const T* __restrict__ logits, long long ld, const long long* __restrict__ labels, int L, int V,
              const float* __restrict__ count, float* __restrict__ row_loss, T* __restrict__ dlogits, long long ldd) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(16) uint8_t ce_smem[];
  __shared__ float red[16];
  __shared__ float tgt_logit;
  const long long row = blockIdx.x;
  const long long tgt = shifted_target(labels, L, row);
  const T* x = logits + row * ld;
  T* dx = dlogits ? dlogits + row * ldd : nullptr;
  constexpr int VEC = 16 / sizeof(T);
  const int nvec = ((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (dx == nullptr || (reinterpret_cast<uintptr_t>(dx) & 15) == 0))
                       ? V / VEC : 0;                          // vector body; the scalar tail covers the rest
  if (tgt == -100) {                                           // ignored position: zero loss, zero gradient
    if (threadIdx.x == 0) row_loss[row] = 0.f;
    if (dx) {
      const uint4 z = make_uint4(0, 0, 0, 0);
      for (int v = threadIdx.x; v < nvec; v += blockDim.x) reinterpret_cast<uint4*>(dx)[v] = z;
      for (int v = nvec * VEC + threadIdx.x; v < V; v += blockDim.x) st_logit(dx, v, 0.f);
    }
    return;
  }
  T* sx = reinterpret_cast<T*>(ce_smem);
  const T* src = x;
  float m = -INFINITY;
  if constexpr (kSmem) {
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(x) + v);
      reinterpret_cast<uint4*>(sx)[v] = u;
      const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
      for (int i = 0; i < VEC; ++i) m = fmaxf(m, ld_logit(e, i));
    }
    for (int v = nvec * VEC + threadIdx.x; v < V; v += blockDim.x) {
      const T t = x[v];
      sx[v] = t;
      m = fmaxf(m, ld_logit(&t, 0));
    }
    src = sx;
  } else {
    for (int v = threadIdx.x; v < V; v += blockDim.x) m = fmaxf(m, ld_logit(x, v));
  }
  // block max
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  float M = red[0];
  for (int i = 1; i < (blockDim.x >> 5); ++i) M = fmaxf(M, red[i]);
  __syncthreads();
  // block sum of exp(x - M); with the row in smem the exponentials are kept in place (as T) for the gradient
  float s = 0.f;
  if constexpr (kSmem) {
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
      const float e = __expf(ld_logit(sx, v) - M);
      s += e;
      if (v == tgt) tgt_logit = ld_logit(sx, v);    // the target logit, needed for the loss
      st_logit(sx, v, e);
    }
  } else {
    for (int v = threadIdx.x; v < V; v += blockDim.x) s += __expf(ld_logit(src, v) - M);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float S = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) S += red[i];
  const float lse = M + logf(S);
  if (threadIdx.x == 0) row_loss[row] = lse - (kSmem ? tgt_logit : ld_logit(src, tgt));
  if (dx) {
    const float inv = 1.0f / fmaxf(*count, 1.0f);
    const float invS = 1.0f / S;
    auto prob = [&](int c) { return kSmem ? ld_logit(sx, c) * invS : __expf(ld_logit(src, c) - lse); };
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
      __align__(16) T o[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const int c = v * VEC + i;
        st_logit(o, i, (prob(c) - ((c == tgt) ? 1.f : 0.f)) * inv);
      }
      reinterpret_cast<uint4*>(dx)[v] = *reinterpret_cast<const uint4*>(o);
    }
    for (int v = nvec * VEC + threadIdx.x; v < V; v += blockDim.x)
      st_logit(dx, v, (prob(v) - ((v == tgt) ? 1.f : 0.f)) * inv);
  }
}

__global__ void ce_finalize_kernel(const float* __restrict__ row_loss, long long rows, const float* __restrict__ count,
                                   float* __restrict__ loss) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[8];
  double t = 0.0;
  for (long long r = threadIdx.x; r < rows; r += blockDim.x) t += row_loss[r];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int i = 0; i < 8; ++i) a += red[i];
    *loss = static_cast<float>(a / fmax(static_cast<double>(*count), 1.0));      // nan-free when nothing is supervised
  }
}

template <typename T>
__global__ void scale_by_scalar_kernel(T* __restrict__ x, long long n, const float* __restrict__ g) {
  pdl_launch_dependents();
  pdl_wait();
  const float s = *g;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    st_logit(x, i, ld_logit(x, i) * s);
}

}  // namespace otb

using namespace otb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int otb_label_mask(const int64_t* input_ids, int B, int L, int64_t eos_id, int64_t answer_id, int64_t eoc_id,
                              int64_t mask_val, int64_t* labels, void* stream) {
  OTB_CHECK_ARG(input_ids && labels && B > 0 && L > 0, "otb_label_mask: bad argument");
  const size_t lm_smem = static_cast<size_t>(L) * 16;
  OTB_CHECK_ARG(lm_smem <= 200 * 1024, "otb_label_mask: L too long for the shared-memory staging (max 12800)");
  OTB_CHECK_CUDA(ensure_dyn_smem(label_mask_kernel, 200 * 1024));
  OTB_CHECK_CUDA(launch_k(label_mask_kernel, dim3(B), dim3(128), lm_smem, ST(stream),
                          reinterpret_cast<const long long*>(input_ids), B, L, (long long)eos_id, (long long)answer_id,
                          (long long)eoc_id, (long long)mask_val, reinterpret_cast<long long*>(labels)));
  count_launch();
  return OTB_OK;
}

extern "C" int otb_shifted_cross_entropy(const void* logits, int logits_fp32, int64_t ld, const int64_t* labels, int B,
                                         int L, int V, float* loss, void* dlogits, int64_t ldd, float* ws,
                                         void* stream) {
  OTB_CHECK_ARG(logits && labels && loss && ws && B > 0 && L > 0 && V > 0 && ld >= V, "otb_shifted_cross_entropy: bad argument");
  OTB_CHECK_ARG(dlogits == nullptr || ldd >= V, "otb_shifted_cross_entropy: bad ldd");
  const long long rows = static_cast<long long>(B) * L;
  float* count = ws;            // ws: [1 + rows] floats
  float* row_loss = ws + 1;
  const long long* lab = reinterpret_cast<const long long*>(labels);
  OTB_CHECK_CUDA(launch_k(ce_count_kernel, dim3(1), dim3(1024), 0, ST(stream), lab, rows, L, count));
  const size_t row_bytes = static_cast<size_t>(V) * (logits_fp32 ? 4 : 2);
  const bool in_smem = row_bytes <= 200 * 1024;
  const size_t ce_smem = in_smem ? ((row_bytes + 15) & ~size_t(15)) : 0;
  OTB_CHECK_CUDA(ensure_dyn_smem(ce_row_kernel<float, true>, 200 * 1024 + 16));
  OTB_CHECK_CUDA(ensure_dyn_smem(ce_row_kernel<bf16, true>, 200 * 1024 + 16));
#define OTB_CE_LAUNCH(T_, S_)                                                                                       \
  OTB_CHECK_CUDA(launch_k(ce_row_kernel<T_, S_>, dim3((unsigned)rows), dim3(512), ce_smem, ST(stream),              \
                          static_cast<const T_*>(logits), (long long)ld, lab, L, V, (const float*)count, row_loss,  \
                          static_cast<T_*>(dlogits), (long long)ldd))
  if (logits_fp32) { if (in_smem) OTB_CE_LAUNCH(float, true); else OTB_CE_LAUNCH(float, false); }
  else             { if (in_smem) OTB_CE_LAUNCH(bf16, true);  else OTB_CE_LAUNCH(bf16, false); }
#undef OTB_CE_LAUNCH
  OTB_CHECK_CUDA(launch_k(ce_finalize_kernel, dim3(1), dim3(256), 0, ST(stream), (const float*)row_loss, rows,
                          (const float*)count, loss));
  count_launch(3);
  return OTB_OK;
}

extern "C" int otb_scale_by_scalar(void* x, int x_fp32, int64_t n, const float* scalar, void* stream) {
  OTB_CHECK_ARG(x && scalar && n > 0, "otb_scale_by_scalar: bad argument");
  long long g = (n + 255) / 256;
  if (g > 132 * 16) g = 132 * 16;
  if (x_fp32)
    OTB_CHECK_CUDA(launch_k(scale_by_scalar_kernel<float>, dim3((unsigned)g), dim3(256), 0, ST(stream),
                            static_cast<float*>(x), (long long)n, scalar));
  else
    OTB_CHECK_CUDA(launch_k(scale_by_scalar_kernel<bf16>, dim3((unsigned)g), dim3(256), 0, ST(stream),
                            static_cast<bf16*>(x), (long long)n, scalar));
  count_launch();
  return OTB_OK;
}
