// otter_b200 — dropout on the input of the LoRA adapters of the MPT / LLaMA decoder layers (otter_b200/lora.py).
//   peft's LoRA forward: base(x) + lora_B(lora_A(dropout(x))) * scaling; the dropout is the only element-wise pass the
//   adapters need (the projections and `scaling` run on the GEMM and its epilogue alpha).
// The keep mask is a pure function of (seed, stream_id, element index e = row * cols + col): Philox4x32-10 keyed by the
// 64-bit seed, counter {e / 4 (low word), e / 4 (high word), stream_id, 0}; output word e % 4 decides element e:
//   keep  iff  u32 >= threshold,  threshold = (uint32_t)floor(p * 2^32)   (computed on the host in double)
// so the backward regenerates the forward's mask instead of storing it, whatever the launch geometry.
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

constexpr uint32_t kPhiloxM0 = 0xD2511F53u, kPhiloxM1 = 0xCD9E8D57u;
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u, kPhiloxW1 = 0xBB67AE85u;

// Philox4x32-10 (Salmon et al., SC'11; the Random123 reference rounds)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(kPhiloxM0, c.x), lo0 = kPhiloxM0 * c.x;
    const uint32_t hi1 = __umulhi(kPhiloxM1, c.z), lo1 = kPhiloxM1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += kPhiloxW0;
    k1 += kPhiloxW1;
  }
  return c;
}

// keep flags of elements 8v .. 8v+7 (e = 8v is a multiple of 8: two Philox blocks)
__device__ __forceinline__ void keep8(unsigned long long e0, unsigned long long seed, uint32_t stream_id, uint32_t thr,
                                      bool keep[8]) {
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const unsigned long long q = (e0 >> 2) + b;
    const uint4 u = philox4x32_10(make_uint4(static_cast<uint32_t>(q), static_cast<uint32_t>(q >> 32), stream_id, 0u),
                                  static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
    keep[4 * b + 0] = u.x >= thr;
    keep[4 * b + 1] = u.y >= thr;
    keep[4 * b + 2] = u.z >= thr;
    keep[4 * b + 3] = u.w >= thr;
  }
}

// out = x * keep * scale (bwd == 0)  or  dx += g * keep * scale (bwd != 0, `out` is dx); one thread per 16-byte vector
__global__ void __launch_bounds__(256)
lora_dropout_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, long long ld, long long rows, int cols,
                    uint32_t thr, float scale, unsigned long long seed, uint32_t stream_id, int bwd) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = cols >> 3;
  const long long total = rows * nvec;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = idx / nvec;
    const int v = static_cast<int>(idx % nvec);
    bool keep[8];
    keep8(static_cast<unsigned long long>(row) * cols + 8ull * v, seed, stream_id, thr, keep);
    float f[8], o[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + row * ld) + v), f);
    uint4* po = reinterpret_cast<uint4*>(out + row * ld) + v;
    if (bwd) {
      unpack8(*po, o);
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = __fmaf_rn(f[i], keep[i] ? scale : 0.0f, o[i]);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = keep[i] ? __fmul_rn(f[i], scale) : 0.0f;
    }
    *po = pack8(o);
  }
}

static int lora_dropout_launch(const char* name, const void* x, void* out, int64_t rows, int cols, int64_t ld, float p,
                               uint64_t seed, uint32_t stream_id, int bwd, void* stream) {
  OTB_CHECK_ARG(x && out && rows > 0 && cols > 0 && cols % 8 == 0 && ld >= cols && ld % 8 == 0, "%s: bad argument", name);
  OTB_CHECK_ARG(p >= 0.0f && p < 1.0f, "%s: p = %g must be in [0, 1)", name, static_cast<double>(p));
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                "%s: x and out must be 16-byte aligned", name);
  const uint32_t thr = static_cast<uint32_t>(static_cast<double>(p) * 4294967296.0);
  const float scale = 1.0f / (1.0f - p);
  const long long items = static_cast<long long>(rows) * (cols / 8);
  long long grid = (items + 255) / 256;
  const long long cap = static_cast<long long>(sm_count()) * 8;
  grid = grid > cap ? cap : grid;
  OTB_CHECK_CUDA(launch_k(lora_dropout_kernel, dim3(static_cast<unsigned>(grid)), dim3(256), 0,
                          static_cast<cudaStream_t>(stream), static_cast<const bf16*>(x), static_cast<bf16*>(out),
                          (long long)ld, (long long)rows, cols, thr, scale, (unsigned long long)seed, stream_id, bwd));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

}  // namespace otb

extern "C" int otb_lora_dropout_fwd(const void* x, void* out, int64_t rows, int cols, int64_t ld, float p, uint64_t seed,
                                    uint32_t stream_id, void* stream) {
  return otb::lora_dropout_launch("otb_lora_dropout_fwd", x, out, rows, cols, ld, p, seed, stream_id, 0, stream);
}

extern "C" int otb_lora_dropout_bwd_add(const void* g, void* dx, int64_t rows, int cols, int64_t ld, float p, uint64_t seed,
                                        uint32_t stream_id, void* stream) {
  return otb::lora_dropout_launch("otb_lora_dropout_bwd_add", g, dx, rows, cols, ld, p, seed, stream_id, 1, stream);
}
