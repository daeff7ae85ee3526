// otter_b200 — common device-side building blocks for the sm_90a (Hopper) kernels.
//
// Everything here is a thin inline-PTX wrapper: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma) with
// its shared-memory descriptors, and the fp32 shared-memory accumulator tiles the attention kernels read row by row.
// No CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace otb {

typedef __nv_bfloat16 bf16;

// ----------------------------------------------------------------------------------------------
// small utilities
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// named barrier among `nthreads` threads (a multiple of 32) — the warps that share id `id` (1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// Programmatic dependent launch: every kernel lets its successor's CTAs start early (launch_dependents) and
// itself waits for the complete predecessor grid (and its memory) right before the first global access, so
// prologues (barrier init, descriptor prefetch, launch latency) overlap the predecessor's tail.
// Both are no-ops when the kernel was not launched with the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  // make generic-proxy smem writes visible to the async proxy (TMA store, wgmma operand reads)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug turns into a trap (CUDA error) after ~2 s instead of a hung GPU.  No printf here: a
// function call between wgmma issue and wait makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 0x3ff) == 0 && (clock64() - t0) > 4000000000LL) __trap();
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 2D tiled load global -> shared, completion signalled on an mbarrier (complete_tx bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
// smem box += into global (fp32 add performed at L2): the accumulate epilogue without reading the old values
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma: warpgroup MMA (4 warps, 128 threads), bf16 x bf16 -> fp32, accumulator in registers
// ----------------------------------------------------------------------------------------------
// D[64 x N] (+)= A[64 x 16] . B[16 x N] with both operands read from shared memory through descriptors.  TA / TB = 1:
// the operand is MN-major (A stored [k][m], B stored [k][n]) — the transposed reads dgrad / wgrad / P V need, with no
// transpose copy.  scale_d = 0 ignores the old accumulator (first k-step).  Every thread of the warpgroup executes it.
template <int N, int TA, int TB>
struct Wgmma;

template <int TA, int TB>
struct Wgmma<64, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %36;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
};

template <int TA, int TB>
struct Wgmma<128, TA, TB> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, %67, %68;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
  }
};

// the accumulator registers are about to be read or written by wgmma (orders earlier register / smem accesses)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N committed groups of this warpgroup still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void wgmma_keep(float (&d)[R]) {   // registers stay live across the asynchronous MMA
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ----------------------------------------------------------------------------------------------
// fp32 accumulator tiles in shared memory
// ----------------------------------------------------------------------------------------------
// The attention kernels keep the softmax and epilogue code "thread t owns row t": a warpgroup's m64 fragments are
// stored to a [rows][N] fp32 tile and each thread reads its row back.  16 B units are XOR-swizzled with (row & 7), so
// both the fragment stores (8 rows x 2 units per warp) and the row reads (a quarter-warp = 8 consecutive rows) are free
// of bank conflicts.  N >= 32.
template <int N>
__device__ __forceinline__ float* acc_at(uint8_t* tile, int row, int col) {
  return reinterpret_cast<float*>(tile + row * (N * 4) + ((((col >> 2) ^ (row & 7))) << 4) + (col & 3) * 4);
}
// wgmma fragment of m64nN (rows row0 .. row0+63 of the tile) <-> tile.  Thread t of the warpgroup holds rows
// row0 + 16 (t/32) + (t%32)/4 (+8), columns 8 j + 2 (t%4) (+1).
template <int N>
__device__ __forceinline__ void acc_store(uint8_t* tile, int row0, const float (&d)[N / 2]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int col = 8 * j + 2 * (t & 3);
    *reinterpret_cast<float2*>(acc_at<N>(tile, r, col)) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(acc_at<N>(tile, r + 8, col)) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// 32 consecutive columns [col0, col0 + 32) of one row (col0 a multiple of 4); 16-column variant below
template <int N>
__device__ __forceinline__ void acc_ld32(uint8_t* tile, int row, int col0, uint32_t (&r)[32]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float4 v = *reinterpret_cast<const float4*>(acc_at<N>(tile, row, col0 + 4 * k));
    r[4 * k] = __float_as_uint(v.x); r[4 * k + 1] = __float_as_uint(v.y);
    r[4 * k + 2] = __float_as_uint(v.z); r[4 * k + 3] = __float_as_uint(v.w);
  }
}
template <int N>
__device__ __forceinline__ void acc_ld16(uint8_t* tile, int row, int col0, uint32_t (&r)[16]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float4 v = *reinterpret_cast<const float4*>(acc_at<N>(tile, row, col0 + 4 * k));
    r[4 * k] = __float_as_uint(v.x); r[4 * k + 1] = __float_as_uint(v.y);
    r[4 * k + 2] = __float_as_uint(v.z); r[4 * k + 3] = __float_as_uint(v.w);
  }
}

// A 128-row product by one warpgroup: tile[128 x N] = sum_k A_k . B_k over `ksteps` k16 steps, as two m64 halves.
// a(h, k) is the descriptor of rows [64 h, 64 h + 64) of A at k-step k, b(k) the one of B.  Operands must be resident
// (and, if written by threads, fenced to the async proxy); the caller synchronises before reading the tile.
template <int N, int TA, int TB, typename ADesc, typename BDesc>
__device__ __forceinline__ void wg_mma_tile(uint8_t* tile, int ksteps, ADesc a, BDesc b) {
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    wgmma_keep(d);
    wgmma_fence();
#pragma unroll 1
    for (int k = 0; k < ksteps; ++k) Wgmma<N, TA, TB>::mma(d, a(h, k), b(k), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_keep(d);
    acc_store<N>(tile, 64 * h, d);
  }
}
// Same product accumulated into registers: d[h] holds rows [64 h, 64 h + 64) of an H x 64-row tile (accumulate = false
// starts from zero).
template <int N, int TA, int TB, int H, typename ADesc, typename BDesc>
__device__ __forceinline__ void wg_mma_regs(float (&d)[H][N / 2], bool accumulate, int ksteps, ADesc a, BDesc b) {
#pragma unroll
  for (int h = 0; h < H; ++h) wgmma_keep(d[h]);
  wgmma_fence();
#pragma unroll
  for (int h = 0; h < H; ++h)
#pragma unroll 1
    for (int k = 0; k < ksteps; ++k) Wgmma<N, TA, TB>::mma(d[h], a(h, k), b(k), (accumulate || k != 0) ? 1 : 0);
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < H; ++h) wgmma_keep(d[h]);
}

// ----------------------------------------------------------------------------------------------
// Descriptors
// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, SWIZZLE_128B:
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type (1 = SW128); base offset 0 (1024 B-aligned atoms)
// K-major operand tile  [rows][64 bf16 = 128 B], 8-row swizzle atoms of 1024 B:
//     SBO = 1024 (next 8-row group), LBO unused (1).  K-step of 16 elements = +32 B on the start address; rows 64..127
//     of a 128-row tile start 8 KB further.
// MN-major operand tile [chunk of 64 MN][k rows][128 B]:
//     SBO = 1024 (next 8 k-rows), LBO = bytes between 64-element MN chunks. K-step of 16 = +16 rows = +2048 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ----------------------------------------------------------------------------------------------
// math helpers shared by epilogues / elementwise kernels
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}
// x * sigmoid(1.702 x).  The reciprocal is MUFU.RCP (1 ulp): an IEEE division costs ~20 instructions and a branch to a
// slow path per element, and the bf16 result cannot tell the difference.
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float quick_gelu(float x) { return x * rcp_approx(1.0f + __expf(-1.702f * x)); }

// Branch-free erf for the bf16-output GEMM epilogues (Abramowitz-Stegun 7.1.26, |error| <= 1.5e-7 — five orders of
// magnitude below bf16 resolution; the fp32-grade path keeps erff).  Returns erf(x/sqrt2) and exp(-x^2/2), which is
// exactly what GELU and its derivative need: ~14 instructions instead of erff's two divergent branches.
__device__ __forceinline__ void erf_exp_half(float x, float& erf_v, float& exp_v) {
  const float a = fabsf(x) * 0.70710678118654752f;
  const float t = rcp_approx(fmaf(0.3275911f, a, 1.0f));   // 1-ulp reciprocal: 5 orders below bf16 resolution
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  exp_v = exp2f(-0.72134752044448170f * x * x);           // exp(-x^2 / 2)
  erf_v = copysignf(fmaf(-p * t, exp_v, 1.0f), x);
}
__device__ __forceinline__ float gelu_fast(float x) {
  float e, g;
  erf_exp_half(x, e, g);
  return 0.5f * x * (1.0f + e);
}
__device__ __forceinline__ float gelu_grad_fast(float x) {
  float e, g;
  erf_exp_half(x, e, g);
  return fmaf(x * 0.3989422804014327f, g, 0.5f * (1.0f + e));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

}  // namespace otb
