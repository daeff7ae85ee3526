// otter_b200 — wgmma / TMA GEMM with fused epilogues (the >99.9 %-of-FLOPs kernel of the hot path).
//
//   D[M,N] = epilogue( A[M,K] . B[N,K]^T ),  bf16 operands, fp32 accumulation in registers.
//
// Serves every nn.Linear on the path and its autograd dgrad / wgrad:
//   forward  y  = x W^T      : A = x  [M][K]  K-major,  B = W  [N][K]  K-major
//   dgrad    dx = dy W       : A = dy [M][N'] K-major,  B = W  [N'][K'] read as MN-major (no transpose copy)
//   wgrad    dW = dy^T x     : A = dy read MN-major,    B = x  read MN-major (reduction over tokens)
// (reference: modeling_otter.py:139-148,164-184,253-256,284-288,340,363-370; clip.py:106-149)
//
// Structure (one CTA per SM, persistent over 128 x 128 output tiles, 384 threads = 3 warpgroups):
//   warpgroup 2 : TMA producer  — one thread streams 128B-swizzled A / B tiles into a 4-deep smem ring
//   warpgroups 0, 1 : MMA + epilogue — each issues wgmma.m64n128k16 for its 64 rows (accumulator: 64 fp32 registers
//                 per thread), then parks the fragments in a swizzled fp32 smem tile and runs the fused
//                 bias/GELU/gate/residual epilogue with one thread per (row, column half): 16 B stores or a TMA store
// Shared memory: 4 x 32 KB ring + 2 x 32 KB fp32 tiles + 32 KB TMA-store stage = 224 KB of the 227 KB an H100 CTA may
// use; deeper rings or 256-wide tiles do not fit beside the fp32 tiles.
#include <cstdlib>

#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

constexpr int kBM = 128;
constexpr int kBN = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 384;   // 2 MMA/epilogue warpgroups + 1 producer warpgroup
constexpr int kStages = 4;
constexpr int kABytes = kBM * kBK * 2;              // 16 KB
constexpr int kBBytes = kBN * kBK * 2;              // 16 KB
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kAccBytes = 64 * kBN * 4;             // one warpgroup's 64 x 128 fp32 tile
constexpr int kEpiWarpStage = 32 * 128;             // one epilogue warp's store stage: 32 rows x 128 B (64 bf16 columns)
constexpr int kEpiStageBytes = 8 * kEpiWarpStage;   // 32 KB, sits between the fp32 tiles and the barriers
constexpr int kGemmSmemBytes = kStages * kStageBytes + 2 * kAccBytes + 1024 /*align slack*/ + 256 /*barriers*/;

struct GemmEpi {
  const float* bias;
  const bf16* aux_in;
  bf16* aux_out;
  const float* scale_ptr;
  const bf16* residual;
  void* out;
  long long ld_out, ld_aux_in, ld_aux_out, ld_res;
  int act, scale_tanh, out_fp32, accumulate;
  float alpha;
  int res_fp32;   // residual is fp32 [M][N] (fp32-grade parity path)
  int tma_out;    // bf16 output leaves through a swizzled smem stage + TMA store (full 128 B lines, bounds clipped by TMA)
  int cls;        // index into kEpiCls when the options match one of the compiled classes, else -1 (run-time options)
};


// One epilogue warp's share of a warpgroup's 64 x BN accumulator tile `acc`: 32-row quarter q, column half `half`.
template <int BN>
__device__ __forceinline__ void epilogue_tile(const GemmEpi& ep, float scale, uint8_t* acc, int m0, int n0, int M,
                                              int N, int q, int half, int lane) {
  const int row = m0 + q * 32 + lane;
  const bool row_ok = row < M;
  const long long lrow = row;
#pragma unroll 1
  for (int c = half * (BN / 64); c < (half + 1) * (BN / 64); ++c) {
    const int colbase = n0 + c * 32;
    const bool act_chunk = row_ok && colbase < N;
    // Issue every global read of this 32-column chunk up front (they do not depend on the accumulator):
    // each thread reads 64 B of its own row, so the loads of a warp are uncoalesced — what matters is
    // having all of them in flight together instead of one dependent load per 8 columns.
    uint4 res[4], aux[4];
    float4 old[8];
    if (act_chunk) {
      if (ep.residual != nullptr && !ep.res_fp32) {
        const uint4* pr = reinterpret_cast<const uint4*>(ep.residual + lrow * ep.ld_res + colbase);
#pragma unroll
        for (int g = 0; g < 4; ++g) if (colbase + g * 8 < N) res[g] = __ldg(pr + g);
      }
      if (ep.aux_in != nullptr) {
        const uint4* pa = reinterpret_cast<const uint4*>(ep.aux_in + lrow * ep.ld_aux_in + colbase);
#pragma unroll
        for (int g = 0; g < 4; ++g) if (colbase + g * 8 < N) aux[g] = __ldg(pa + g);
      }
      if (ep.out_fp32 && ep.accumulate) {
        const float4* po = reinterpret_cast<const float4*>(reinterpret_cast<float*>(ep.out) + lrow * ep.ld_out + colbase);
#pragma unroll
        for (int g = 0; g < 8; ++g) if (colbase + g * 4 < N) old[g] = po[g];
      }
    }
    uint32_t r[32];
    acc_ld32<BN>(acc, q * 32 + lane, c * 32, r);
    if (act_chunk) {
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int col = colbase + g * 8;
        if (col >= N) break;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[g * 8 + i]);
        if (ep.bias != nullptr) {
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(ep.bias + col));
          const float4 b1 = __ldg(reinterpret_cast<const float4*>(ep.bias + col + 4));
          v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w;
          v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
        }
        if (ep.aux_out != nullptr) {
          uint4 o;
          o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
          o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
          *reinterpret_cast<uint4*>(ep.aux_out + lrow * ep.ld_aux_out + col) = o;
        }
        if (ep.aux_in == nullptr) {
          if (ep.act == 1) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = gelu_fast(v[i]);
          } else if (ep.act == 2) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = quick_gelu(v[i]);
          } else if (ep.act == 3) {                     // relu^2 (Persimmon "relu2")
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float r_ = fmaxf(v[i], 0.f); v[i] = r_ * r_; }
          }
        } else {   // backward of the activation whose pre-activation is aux_in: act 3 -> 2 relu(z), otherwise gelu'(z)
          const float2 a0 = unpack_bf16x2(aux[g].x), a1 = unpack_bf16x2(aux[g].y), a2 = unpack_bf16x2(aux[g].z),
                       a3 = unpack_bf16x2(aux[g].w);
          if (ep.act == 3) {
            v[0] *= 2.f * fmaxf(a0.x, 0.f); v[1] *= 2.f * fmaxf(a0.y, 0.f);
            v[2] *= 2.f * fmaxf(a1.x, 0.f); v[3] *= 2.f * fmaxf(a1.y, 0.f);
            v[4] *= 2.f * fmaxf(a2.x, 0.f); v[5] *= 2.f * fmaxf(a2.y, 0.f);
            v[6] *= 2.f * fmaxf(a3.x, 0.f); v[7] *= 2.f * fmaxf(a3.y, 0.f);
          } else {
            v[0] *= gelu_grad_fast(a0.x); v[1] *= gelu_grad_fast(a0.y);
            v[2] *= gelu_grad_fast(a1.x); v[3] *= gelu_grad_fast(a1.y);
            v[4] *= gelu_grad_fast(a2.x); v[5] *= gelu_grad_fast(a2.y);
            v[6] *= gelu_grad_fast(a3.x); v[7] *= gelu_grad_fast(a3.y);
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] *= scale;
        if (ep.residual != nullptr && ep.res_fp32) {
          const float* pr = reinterpret_cast<const float*>(ep.residual) + lrow * ep.ld_res + col;
          const float4 r0 = __ldg(reinterpret_cast<const float4*>(pr)), r1 = __ldg(reinterpret_cast<const float4*>(pr + 4));
          v[0] += r0.x; v[1] += r0.y; v[2] += r0.z; v[3] += r0.w;
          v[4] += r1.x; v[5] += r1.y; v[6] += r1.z; v[7] += r1.w;
        } else if (ep.residual != nullptr) {
          const float2 a0 = unpack_bf16x2(res[g].x), a1 = unpack_bf16x2(res[g].y), a2 = unpack_bf16x2(res[g].z),
                       a3 = unpack_bf16x2(res[g].w);
          v[0] += a0.x; v[1] += a0.y; v[2] += a1.x; v[3] += a1.y;
          v[4] += a2.x; v[5] += a2.y; v[6] += a3.x; v[7] += a3.y;
        }
        if (ep.out_fp32) {
          float* o = reinterpret_cast<float*>(ep.out) + lrow * ep.ld_out + col;
          float4 o0 = make_float4(0.f, 0.f, 0.f, 0.f), o1 = o0;
          if (ep.accumulate) { o0 = old[2 * g]; o1 = old[2 * g + 1]; }
          o0.x += v[0]; o0.y += v[1]; o0.z += v[2]; o0.w += v[3];
          o1.x += v[4]; o1.y += v[5]; o1.z += v[6]; o1.w += v[7];
          *reinterpret_cast<float4*>(o) = o0;
          *reinterpret_cast<float4*>(o + 4) = o1;
        } else {
          uint4 o;
          o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
          o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
          *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(ep.out) + lrow * ep.ld_out + col) = o;
        }
      }
    }
  }
}

// TMA-store variant of the epilogue.  The direct epilogue above has every thread write 16 B pieces of its own row:
// 32 different 128 B lines per warp store instruction, partially written sectors on the way to L2, and the
// accumulate class first READS its old fp32 values the same way.  Here a warp assembles 32 rows x 128 B (64 bf16 or
// 32 fp32 columns) in a SWIZZLE_128B smem stage — thread = row, the 16 B unit j of row r lands at unit j ^ (r & 7),
// which is bank-conflict free and exactly the layout the output tensor map expects — and one lane hands the 4 KB box
// to the TMA engine, which writes whole lines, clips rows >= M / columns >= N, and for `accumulate` performs the
// fp32 add at L2 (cp.reduce.async.bulk ... add) so the old values never travel to the SM.
// The stage is reused once the previous bulk operation has finished READING it (wait_group.read), which overlaps
// with the accumulator read and the math of the next chunk.  The pre-activation side output (aux_out) keeps direct stores.
// CLS >= 0: the epilogue options of launch class kEpiCls[CLS] are compile-time constants — the per-group option tests
// (uniform branches that cut the 32 independent element streams of a chunk into tiny basic blocks) disappear and the
// chunk becomes one block the scheduler can interleave.  CLS = -1: options read from `ep` at run time (any combination).
struct EpiCls { bool bias, aux_out; int act; bool aux_in, scale, res, out_f32, acc; };
constexpr int kNumEpiCls = 14;
constexpr EpiCls kEpiCls[kNumEpiCls] = {
    /* 0 plain                      */ {false, false, 0, false, false, false, false, false},
    /* 1 * gate                     */ {false, false, 0, false, true, false, false, false},
    /* 2 bias                       */ {true, false, 0, false, false, false, false, false},
    /* 3 bias + quick-GELU          */ {true, false, 2, false, false, false, false, false},
    /* 4 bias + residual            */ {true, false, 0, false, false, true, false, false},
    /* 5 residual                   */ {false, false, 0, false, false, true, false, false},
    /* 6 GELU + pre-activation      */ {false, true, 1, false, false, false, false, false},
    /* 7 branch out, * gate, + res  */ {false, true, 0, false, true, true, false, false},
    /* 8 * gelu'(aux) * gate        */ {false, false, 0, true, true, false, false, false},
    /* 9 * gelu'(aux)               */ {false, false, 0, true, false, false, false, false},
    /* 10 fp32 store                */ {false, false, 0, false, false, false, true, false},
    /* 11 fp32 store * gate         */ {false, false, 0, false, true, false, true, false},
    /* 12 fp32 accumulate           */ {false, false, 0, false, false, false, true, true},
    /* 13 fp32 accumulate * gate    */ {false, false, 0, false, true, false, true, true},
};

template <int BN, int CLS>
__device__ __forceinline__ void epilogue_tile_tma(const GemmEpi& ep, float scale, uint8_t* acc, int m0, int n0, int M,
                                                  int N, int q, int half, int lane, uint8_t* stage,
                                                  const CUtensorMap* map_d) {
  constexpr bool kS = CLS >= 0;
  constexpr EpiCls kC = kEpiCls[kS ? CLS : 0];
  const bool f_bias = kS ? kC.bias : (ep.bias != nullptr);
  const bool f_auxo = kS ? kC.aux_out : (ep.aux_out != nullptr);
  const int f_act = kS ? kC.act : ep.act;
  const bool f_auxi = kS ? kC.aux_in : (ep.aux_in != nullptr);
  const bool f_scale = kS ? kC.scale : true;
  const bool f_res = kS ? kC.res : (ep.residual != nullptr);
  const bool f_f32 = kS ? kC.out_f32 : (ep.out_fp32 != 0);
  const bool f_acc = kS ? kC.acc : (ep.accumulate != 0);
  const int row0 = m0 + q * 32;
  if (row0 >= M) return;                                      // warp-uniform: no row of this quarter is inside
  const int row = row0 + lane;
  const bool row_ok = row < M;
  const long long lrow = row;
  uint8_t* my_row = stage + lane * 128;
  const int xr = lane & 7;
#pragma unroll 1
  for (int c = half * (BN / 64); c < (half + 1) * (BN / 64); ++c) {     // 32-column chunks of this warp's half
    const int colbase = n0 + c * 32;
    if (colbase >= N) break;                                  // warp-uniform
    const bool act_chunk = row_ok;
    uint4 res[4], aux[4];
    if (act_chunk) {
      if (f_res) {
        const uint4* pr = reinterpret_cast<const uint4*>(ep.residual + lrow * ep.ld_res + colbase);
#pragma unroll
        for (int g = 0; g < 4; ++g) if (colbase + g * 8 < N) res[g] = __ldg(pr + g);
      }
      if (f_auxi) {
        const uint4* pa = reinterpret_cast<const uint4*>(ep.aux_in + lrow * ep.ld_aux_in + colbase);
#pragma unroll
        for (int g = 0; g < 4; ++g) if (colbase + g * 8 < N) aux[g] = __ldg(pa + g);
      }
    }
    uint32_t r[32];
    acc_ld32<BN>(acc, q * 32 + lane, c * 32, r);
    // bf16: two chunks share one 128 B-wide box (units 0-3 / 4-7); fp32: one chunk is one box (units 0-7).
    const bool first_of_box = f_f32 || (c & 1) == 0;
    const bool last_of_box = f_f32 || (c & 1) == 1 || colbase + 32 >= N;
    if (first_of_box) {                                       // the previous box must have left the stage
      if (lane == 0) tma_store_wait_read<0>();
      __syncwarp();
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int col = colbase + g * 8;
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = __uint_as_float(r[g * 8 + i]);
      if (act_chunk && col < N) {
        if (f_bias) {
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(ep.bias + col));
          const float4 b1 = __ldg(reinterpret_cast<const float4*>(ep.bias + col + 4));
          v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w;
          v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
        }
        if (f_auxo) {
          uint4 x;
          x.x = pack_bf16x2(v[0], v[1]); x.y = pack_bf16x2(v[2], v[3]);
          x.z = pack_bf16x2(v[4], v[5]); x.w = pack_bf16x2(v[6], v[7]);
          *reinterpret_cast<uint4*>(ep.aux_out + lrow * ep.ld_aux_out + col) = x;
        }
        if (!f_auxi) {
          if (f_act == 1) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = gelu_fast(v[i]);
          } else if (f_act == 2) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = quick_gelu(v[i]);
          } else if (f_act == 3) {                     // relu^2 (Persimmon "relu2")
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float r_ = fmaxf(v[i], 0.f); v[i] = r_ * r_; }
          }
        } else {   // backward of the activation whose pre-activation is aux_in: act 3 -> 2 relu(z), otherwise gelu'(z)
          const float2 a0 = unpack_bf16x2(aux[g].x), a1 = unpack_bf16x2(aux[g].y), a2 = unpack_bf16x2(aux[g].z),
                       a3 = unpack_bf16x2(aux[g].w);
          if (f_act == 3) {
            v[0] *= 2.f * fmaxf(a0.x, 0.f); v[1] *= 2.f * fmaxf(a0.y, 0.f);
            v[2] *= 2.f * fmaxf(a1.x, 0.f); v[3] *= 2.f * fmaxf(a1.y, 0.f);
            v[4] *= 2.f * fmaxf(a2.x, 0.f); v[5] *= 2.f * fmaxf(a2.y, 0.f);
            v[6] *= 2.f * fmaxf(a3.x, 0.f); v[7] *= 2.f * fmaxf(a3.y, 0.f);
          } else {
            v[0] *= gelu_grad_fast(a0.x); v[1] *= gelu_grad_fast(a0.y);
            v[2] *= gelu_grad_fast(a1.x); v[3] *= gelu_grad_fast(a1.y);
            v[4] *= gelu_grad_fast(a2.x); v[5] *= gelu_grad_fast(a2.y);
            v[6] *= gelu_grad_fast(a3.x); v[7] *= gelu_grad_fast(a3.y);
          }
        }
        if (f_scale) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] *= scale;
        }
        if (f_res) {
          const float2 a0 = unpack_bf16x2(res[g].x), a1 = unpack_bf16x2(res[g].y), a2 = unpack_bf16x2(res[g].z),
                       a3 = unpack_bf16x2(res[g].w);
          v[0] += a0.x; v[1] += a0.y; v[2] += a1.x; v[3] += a1.y;
          v[4] += a2.x; v[5] += a2.y; v[6] += a3.x; v[7] += a3.y;
        }
      }
      // rows >= M and columns >= N hold don't-care values: the TMA engine clips them
      if (f_f32) {
        *reinterpret_cast<float4*>(my_row + (((2 * g) ^ xr) << 4)) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(my_row + (((2 * g + 1) ^ xr) << 4)) = make_float4(v[4], v[5], v[6], v[7]);
      } else {
        uint4 o;
        o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
        o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
        *reinterpret_cast<uint4*>(my_row + ((((c & 1) * 4 + g) ^ xr) << 4)) = o;
      }
    }
    if (last_of_box) {
      fence_proxy_async_smem();                               // generic-proxy writes -> visible to the TMA engine
      __syncwarp();
      if (lane == 0) {
        const int box_col = f_f32 ? colbase : (colbase & ~63);
        if (f_acc) tma_reduce_add_2d(map_d, stage, box_col, row0);
        else tma_store_2d(map_d, stage, box_col, row0);
        tma_store_commit();
      }
    }
  }
}

// per-tile dispatch on the launch's epilogue class (host: epi_class_of)
template <int BN>
__device__ __forceinline__ void epilogue_dispatch_tma(const GemmEpi& ep, float scale, uint8_t* acc, int m0, int n0,
                                                      int M, int N, int q, int half, int lane, uint8_t* stage,
                                                      const CUtensorMap* map_d) {
#define OTB_EPI_CASE(C_) case C_: epilogue_tile_tma<BN, C_>(ep, scale, acc, m0, n0, M, N, q, half, lane, stage, map_d); break;
  switch (ep.cls) {
    OTB_EPI_CASE(0) OTB_EPI_CASE(1) OTB_EPI_CASE(2) OTB_EPI_CASE(3) OTB_EPI_CASE(4) OTB_EPI_CASE(5) OTB_EPI_CASE(6)
    OTB_EPI_CASE(7) OTB_EPI_CASE(8) OTB_EPI_CASE(9) OTB_EPI_CASE(10) OTB_EPI_CASE(11) OTB_EPI_CASE(12) OTB_EPI_CASE(13)
    default: epilogue_tile_tma<BN, -1>(ep, scale, acc, m0, n0, M, N, q, half, lane, stage, map_d); break;
  }
#undef OTB_EPI_CASE
}

// Persistent warp-specialised kernel, one CTA per SM.  Warpgroup 2 (one thread) is the TMA producer; warpgroups 0 and 1
// each own 64 rows of the 128 x 128 tile: 4 wgmma.m64n128k16 per 64-deep k-block, one k-block kept in flight while the
// next one issues (wait_group 1), its ring slot released as soon as the previous k-block's MMAs retire.  At the end of
// a tile the warpgroup parks its fragments in its 32 KB fp32 tile and runs the epilogue row by row from there, while
// the producer already streams the next tile's operands into the ring.
template <bool A_MN, bool B_MN, bool TS>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_d, int M, int N, int K, GemmEpi ep) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* acc_tiles = smem + kStages * kStageBytes;                 // 2 x 32 KB (one per MMA warpgroup)
  uint8_t* epi_stage = acc_tiles + 2 * kAccBytes;                    // 8 x 4 KB (1024-aligned), TMA-store epilogue only
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_stage + (TS ? kEpiStageBytes : 0));
  uint64_t* full_bar = bars;                        // [kStages]
  uint64_t* empty_bar = bars + kStages;             // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  const int tiles_m = (M + kBM - 1) / kBM;
  const int tiles_n = (N + kBN - 1) / kBN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = (K + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrive per MMA warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // predecessor grid complete before any global / TMA access

  if (wg == 2) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 256) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int m0 = (t % tiles_m) * kBM;
        const int n0 = (t / tiles_m) * kBN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * kStageBytes;
          uint8_t* sb = sa + kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          const int k0 = kb * kBK;
          if constexpr (!A_MN) {
            tma_load_2d(sa, &map_a, &full_bar[stage], k0, m0);  // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int c = 0; c < kBM / 64; ++c)                  // box {64 m, 64 k rows} per 64-wide chunk
              tma_load_2d(sa + c * (kBK * 128), &map_a, &full_bar[stage], m0 + c * 64, k0);
          }
          if constexpr (!B_MN) {
            tma_load_2d(sb, &map_b, &full_bar[stage], k0, n0);  // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int c = 0; c < kBN / 64; ++c)
              tma_load_2d(sb + c * (kBK * 128), &map_b, &full_bar[stage], n0 + c * 64, k0);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue warpgroups: rows [64 wg, 64 wg + 64) of each tile =====================
    constexpr uint32_t a_lbo = A_MN ? kBK * 128 : 16, a_kstep = A_MN ? 2048 : 32;
    constexpr uint32_t b_lbo = B_MN ? kBK * 128 : 16, b_kstep = B_MN ? 2048 : 32;
    // this warpgroup's 64 rows of A: 8 KB into a K-major tile, the second 64-wide chunk of an MN-major one
    constexpr uint32_t a_rows = 64 * 128;
    uint8_t* acc = acc_tiles + wg * kAccBytes;
    const int q = warp & 1, half = (warp >> 1) & 1;      // epilogue: 32-row quarter of the 64 rows, column half
    float scale = ep.alpha;
    if (ep.scale_ptr != nullptr) {
      const float s = __ldg(ep.scale_ptr);
      scale *= ep.scale_tanh ? tanhf(s) : s;
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int m0 = (t % tiles_m) * kBM;
      const int n0 = (t / tiles_m) * kBN;
      float d[kBN / 2];
#pragma unroll
      for (int i = 0; i < kBN / 2; ++i) d[i] = 0.f;
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * kStageBytes);
        const uint32_t sb = sa + kABytes;
        const uint64_t da = make_smem_desc(sa + wg * a_rows, a_lbo, 1024);
        const uint64_t db = make_smem_desc(sb, b_lbo, 1024);
        wgmma_keep(d);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
          Wgmma<kBN, A_MN, B_MN>::mma(d, da + ((k * a_kstep) >> 4), db + ((k * b_kstep) >> 4), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();                                 // the previous k-block's MMAs retired: its slot is free
        wgmma_keep(d);
        if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_keep(d);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
      acc_store<kBN>(acc, 0, d);
      named_bar_sync(1 + wg, 128);
      if constexpr (TS)
        epilogue_dispatch_tma<kBN>(ep, scale, acc, m0 + 64 * wg, n0, M, N, q, half, lane, epi_stage + warp * kEpiWarpStage,
                                   &map_d);
      else
        epilogue_tile<kBN>(ep, scale, acc, m0 + 64 * wg, n0, M, N, q, half, lane);
      named_bar_sync(1 + wg, 128);                      // the fp32 tile is read before the next tile overwrites it
    }
    if (TS && lane == 0) tma_store_wait_read<0>();     // the stage must outlive the last bulk store's reads
  }
}

template <bool A_MN, bool B_MN, bool TS>
static int launch_gemm(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                       const GemmEpi& ep, cudaStream_t stream) {
  CUtensorMap ma, mb;
  int rc;
  if (!A_MN) rc = make_tmap_bf16_2d(&ma, A, M, K, lda, kBM, 64);   // [M][K], box 128 rows x 64 k
  else       rc = make_tmap_bf16_2d(&ma, A, K, M, lda, kBK, 64);   // [K][M], box 64 k-rows x 64 m
  if (rc) return rc;
  if (!B_MN) rc = make_tmap_bf16_2d(&mb, B, N, K, ldb, kBN, 64);
  else       rc = make_tmap_bf16_2d(&mb, B, K, N, ldb, kBK, 64);
  if (rc) return rc;
  CUtensorMap md = ma;                                               // placeholder when the direct epilogue is used
  if (TS) {                                                          // [M][N] output, box 32 rows x 128 B
    rc = ep.out_fp32 ? make_tmap_f32_2d(&md, ep.out, M, N, ep.ld_out, 32, 32)
                     : make_tmap_bf16_2d(&md, ep.out, M, N, ep.ld_out, 32, 64);
    if (rc) return rc;
  }
  auto kern = gemm_bf16_kernel<A_MN, B_MN, TS>;
  constexpr int smem_bytes = kGemmSmemBytes + (TS ? kEpiStageBytes : 0);
  OTB_CHECK_CUDA(ensure_dyn_smem(kern, smem_bytes));   // per (instantiation, device)
  const int tiles = ((M + kBM - 1) / kBM) * ((N + kBN - 1) / kBN);
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  int nattr = 0;
  if (pdl_enabled()) {
    attr[nattr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[nattr].val.programmaticStreamSerializationAllowed = 1;
    ++nattr;
  }
  cfg.gridDim = dim3(tiles < sm_count() ? tiles : sm_count());
  cfg.attrs = attr;
  cfg.numAttrs = nattr;
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  OTB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, ma, mb, md, M, N, K, ep));
  count_launch();
  return OTB_OK;
}

}  // namespace otb

extern "C" int otb_gemm_bf16(const void* A, int a_mn_major, int64_t lda, const void* B, int b_mn_major, int64_t ldb,
                             int M, int N, int K, const otb_gemm_epilogue* e, void* stream) {
  using namespace otb;
  OTB_CHECK_ARG(A && B && e && e->out, "otb_gemm_bf16: null pointer");
  OTB_CHECK_ARG(M > 0 && N > 0 && K > 0, "otb_gemm_bf16: bad shape %d %d %d", M, N, K);
  OTB_CHECK_ARG(N % 8 == 0, "otb_gemm_bf16: N=%d must be a multiple of 8", N);
  OTB_CHECK_ARG(e->ld_out % 8 == 0 && e->ld_out >= N, "otb_gemm_bf16: bad ld_out");
  OTB_CHECK_ARG(!e->accumulate || e->out_fp32, "otb_gemm_bf16: accumulate requires fp32 output");
  OTB_CHECK_ARG(e->aux_in == nullptr || (e->ld_aux_in % 8 == 0 && e->ld_aux_in >= N), "otb_gemm_bf16: bad ld_aux_in");
  OTB_CHECK_ARG(e->aux_out == nullptr || (e->ld_aux_out % 8 == 0 && e->ld_aux_out >= N),
                "otb_gemm_bf16: bad ld_aux_out");
  OTB_CHECK_ARG(e->residual == nullptr || (e->ld_res % 8 == 0 && e->ld_res >= N), "otb_gemm_bf16: bad ld_res");
  OTB_CHECK_ARG(e->act >= 0 && e->act <= 3, "otb_gemm_bf16: bad act");
  if (a_mn_major) OTB_CHECK_ARG(M % 8 == 0 && lda >= M, "otb_gemm_bf16: MN-major A needs M%%8==0, lda>=M");
  else OTB_CHECK_ARG(lda >= K, "otb_gemm_bf16: lda < K");
  if (b_mn_major) OTB_CHECK_ARG(ldb >= N, "otb_gemm_bf16: ldb < N");
  else OTB_CHECK_ARG(ldb >= K, "otb_gemm_bf16: ldb < K");

  GemmEpi ep;
  ep.bias = e->bias;
  ep.aux_in = static_cast<const bf16*>(e->aux_in);
  ep.aux_out = static_cast<bf16*>(e->aux_out);
  ep.scale_ptr = e->scale_ptr;
  ep.residual = static_cast<const bf16*>(e->residual);
  ep.out = e->out;
  ep.ld_out = e->ld_out; ep.ld_aux_in = e->ld_aux_in; ep.ld_aux_out = e->ld_aux_out; ep.ld_res = e->ld_res;
  ep.act = e->act; ep.scale_tanh = e->scale_tanh; ep.out_fp32 = e->out_fp32; ep.accumulate = e->accumulate;
  ep.alpha = e->alpha;
  ep.res_fp32 = e->res_fp32;
  OTB_CHECK_ARG(!e->res_fp32 || e->out_fp32, "otb_gemm_bf16: fp32 residual requires fp32 output");
  // Outputs leave through the smem-staged TMA-store / reduce-add epilogue (full 128 B lines, fp32 accumulate performed
  // at L2).  OTB_GEMM_EPI_TMA=0 selects direct stores.
  static const bool epi_tma = [] { const char* v = getenv("OTB_GEMM_EPI_TMA"); return !(v && v[0] == '0'); }();
  ep.tma_out = (epi_tma && !e->res_fp32 && (reinterpret_cast<uintptr_t>(e->out) & 15) == 0 &&
                (!e->out_fp32 || e->ld_out % 4 == 0)) ? 1 : 0;
  ep.cls = -1;
  if (ep.tma_out && e->res_fp32 == 0) {
    const bool scaled = (e->scale_ptr != nullptr) || e->alpha != 1.0f;
    for (int c = 0; c < kNumEpiCls; ++c) {
      const EpiCls& k = kEpiCls[c];
      if (k.bias == (e->bias != nullptr) && k.aux_out == (e->aux_out != nullptr) && k.aux_in == (e->aux_in != nullptr) &&
          k.act == (e->aux_in ? 0 : e->act) && (e->aux_in == nullptr || e->act != 3) && k.scale == scaled &&
          k.res == (e->residual != nullptr) && k.out_f32 == (e->out_fp32 != 0) && k.acc == (e->accumulate != 0)) {
        ep.cls = c;
        break;
      }
    }
  }
  static const bool cls_off = [] { const char* v = getenv("OTB_GEMM_EPI_CLS"); return v && v[0] == '0'; }();
  if (cls_off) ep.cls = -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  const int sel = (a_mn_major ? 2 : 0) | (b_mn_major ? 1 : 0);
#define OTB_GEMM_CASE(A_, B_)                                                    \
  return ep.tma_out ? launch_gemm<A_, B_, true>(A, lda, B, ldb, M, N, K, ep, st) \
                    : launch_gemm<A_, B_, false>(A, lda, B, ldb, M, N, K, ep, st)
  switch (sel) {
    case 0: OTB_GEMM_CASE(false, false);
    case 1: OTB_GEMM_CASE(false, true);
    case 3: OTB_GEMM_CASE(true, true);
    default: break;
  }
#undef OTB_GEMM_CASE
  return set_error(OTB_ERR_UNSUPPORTED, "otb_gemm_bf16: layout (A MN-major, B K-major) not instantiated");
}
