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
// Structure (one CTA per SM, persistent over 128 x 128 output tiles, 384 threads = 3 warpgroups), ping-pong:
//   warpgroup 2 : TMA producer  — one thread streams 128B-swizzled A / B tiles of the CTA's tiles, in order, into a
//                 4-deep smem ring (register budget lowered to 40 with setmaxnreg)
//   warpgroups 0, 1 : MMA + epilogue — they take alternate tiles of the CTA's sequence.  Each owns a whole 128 x 128
//                 tile: two wgmma.m64n128k16 per k16 step, 128 fp32 accumulator registers per thread (budget raised to
//                 232).  While one warpgroup runs its mainloop, the other runs the epilogue of its previous tile, so
//                 the tensor cores do not wait for epilogues.  The epilogue parks the whole accumulator in a swizzled
//                 fp32 smem tile shared by both warpgroups (their epilogues take turns) and runs the fused
//                 bias/GELU/gate/residual epilogue with one thread per (row, column half), leaving through TMA stores.
// Tiles are walked in groups of 32 M-tiles (tile_origin) so one wave's operands stay in L2.
// Shared memory: 4 x 32 KB ring + 64 KB fp32 park tile + 32 KB TMA-store stage = 224 KB of the 227 KB an H100 CTA may
// use.  Two 64 KB park tiles do not fit; one shared tile lets a warpgroup park its whole accumulator before the
// epilogue, so no accumulator register stays live through it and the existing epilogue code runs unchanged.
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

constexpr int kBM = 128;
constexpr int kBN = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 384;   // 2 MMA/epilogue warpgroups + 1 producer warpgroup
constexpr int kStages = 4;
constexpr int kGroupM = 32;                         // M-tiles per group of the tile walk
constexpr int kProducerRegs = 40;                   // setmaxnreg budgets: 40 x 128 + 232 x 256 <= 64 K registers
constexpr int kMmaRegs = 232;
constexpr int kABytes = kBM * kBK * 2;              // 16 KB
constexpr int kBBytes = kBN * kBK * 2;              // 16 KB
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kAccBytes = 64 * kBN * 4;             // 64 x 128 fp32: one half of the park tile
constexpr int kParkBytes = 2 * kAccBytes;           // the 128 x 128 fp32 park tile, 64 KB
constexpr int kEpiWarpStage = 32 * 128;             // one epilogue warp's store stage: 32 rows x 128 B (64 bf16 columns)
constexpr int kEpiStageBytes = 8 * kEpiWarpStage;   // 32 KB, sits between the park tile and the barriers
constexpr int kGemmSmemBytes =
    kStages * kStageBytes + kParkBytes + kEpiStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
// named barriers: 1 + wg = the 128 threads of MMA warpgroup wg; kOrderBar + wg = "wg may issue its mainloop";
// kEpiOrderBar + wg = "wg may fill the park tile"
constexpr int kOrderBar = 3;
constexpr int kEpiOrderBar = 5;

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
  int res_fp32;   // residual is fp32 [M][N] (fp32-grade parity path; run-time options only)
  int cls;        // index into kEpiCls when the options match one of the compiled classes, else -1 (run-time options)
};

// One epilogue warp's share of a warpgroup's 64 x BN accumulator tile `acc`: 32-row quarter q, column half `half`.
// Stores of 16 B pieces of each thread's own row would touch 32 different 128 B lines per warp store instruction and
// leave partially written sectors on the way to L2, and an accumulate would first have to READ its old fp32 values
// the same way.  Instead a warp assembles 32 rows x 128 B (64 bf16 or 32 fp32 columns) in a SWIZZLE_128B smem stage —
// thread = row, the 16 B unit j of row r lands at unit j ^ (r & 7), which is bank-conflict free and exactly the layout
// the output tensor map expects — and one lane hands the 4 KB box to the TMA engine, which writes whole lines, clips
// rows >= M / columns >= N, and for `accumulate` performs the fp32 add at L2 (cp.reduce.async.bulk ... add) so the old
// values never travel to the SM.
// The stage is reused once the previous bulk operation has finished READING it (wait_group.read), which overlaps
// with the accumulator read and the math of the next chunk.  The pre-activation side output (aux_out) keeps direct stores.
// CLS >= 0: the epilogue options of launch class kEpiCls[CLS] are compile-time constants — the per-group option tests
// (uniform branches that cut the 32 independent element streams of a chunk into tiny basic blocks) disappear and the
// chunk becomes one block the scheduler can interleave.  CLS = -1: options read from `ep` at run time (any combination,
// including the fp32 residual).
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
__device__ __forceinline__ void epilogue_tile(const GemmEpi& ep, float scale, uint8_t* acc, int m0, int n0, int M,
                                              int N, int q, int half, int lane, uint8_t* stage,
                                              const CUtensorMap* map_d) {
  constexpr bool kS = CLS >= 0;
  constexpr EpiCls kC = kEpiCls[kS ? CLS : 0];
  const bool f_bias = kS ? kC.bias : (ep.bias != nullptr);
  const bool f_auxo = kS ? kC.aux_out : (ep.aux_out != nullptr);
  const int f_act = kS ? kC.act : ep.act;
  const bool f_auxi = kS ? kC.aux_in : (ep.aux_in != nullptr);
  const bool f_scale = kS ? kC.scale : true;
  const bool f_res = kS ? kC.res : (ep.residual != nullptr && !ep.res_fp32);   // bf16 residual, loaded up front
  const bool f_res32 = !kS && ep.residual != nullptr && ep.res_fp32;         // fp32 residual, loaded at its use
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
        if (f_auxo) *reinterpret_cast<uint4*>(ep.aux_out + lrow * ep.ld_aux_out + col) = pack8(v);
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
          float a[8];
          unpack8(aux[g], a);
          if (f_act == 3) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] *= 2.f * fmaxf(a[i], 0.f);
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] *= gelu_grad_fast(a[i]);
          }
        }
        if (f_scale) {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] *= scale;
        }
        if (f_res) {
          float a[8];
          unpack8(res[g], a);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] += a[i];
        }
        if (f_res32) {
          const float* pr = reinterpret_cast<const float*>(ep.residual) + lrow * ep.ld_res + col;
          const float4 r0 = __ldg(reinterpret_cast<const float4*>(pr)), r1 = __ldg(reinterpret_cast<const float4*>(pr + 4));
          v[0] += r0.x; v[1] += r0.y; v[2] += r0.z; v[3] += r0.w;
          v[4] += r1.x; v[5] += r1.y; v[6] += r1.z; v[7] += r1.w;
        }
      }
      // rows >= M and columns >= N hold don't-care values: the TMA engine clips them
      if (f_f32) {
        *reinterpret_cast<float4*>(my_row + (((2 * g) ^ xr) << 4)) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(my_row + (((2 * g + 1) ^ xr) << 4)) = make_float4(v[4], v[5], v[6], v[7]);
      } else {
        *reinterpret_cast<uint4*>(my_row + ((((c & 1) * 4 + g) ^ xr) << 4)) = pack8(v);
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
__device__ __forceinline__ void epilogue_dispatch(const GemmEpi& ep, float scale, uint8_t* acc, int m0, int n0, int M,
                                                  int N, int q, int half, int lane, uint8_t* stage,
                                                  const CUtensorMap* map_d) {
#define OTB_EPI_CASE(C_) case C_: epilogue_tile<BN, C_>(ep, scale, acc, m0, n0, M, N, q, half, lane, stage, map_d); break;
  switch (ep.cls) {
    OTB_EPI_CASE(0) OTB_EPI_CASE(1) OTB_EPI_CASE(2) OTB_EPI_CASE(3) OTB_EPI_CASE(4) OTB_EPI_CASE(5) OTB_EPI_CASE(6)
    OTB_EPI_CASE(7) OTB_EPI_CASE(8) OTB_EPI_CASE(9) OTB_EPI_CASE(10) OTB_EPI_CASE(11) OTB_EPI_CASE(12) OTB_EPI_CASE(13)
    default: epilogue_tile<BN, -1>(ep, scale, acc, m0, n0, M, N, q, half, lane, stage, map_d); break;
  }
#undef OTB_EPI_CASE
}

// Tile t of the launch -> (m0, n0).  Tiles are walked in groups of kGroupM M-tiles, M fastest inside a group, so the
// operands one wave of CTAs reads stay in L2: at M = 16384, N = 4096, K = 2048 one wave touches ~32 M-tiles x ~4
// N-tiles, ~18 MB, where an M-fastest walk reads all 64 MB of A per wave.  Launches with tiles_m <= kGroupM keep the
// plain M-fastest order.  The last group may be narrower (ragged M).
__device__ __forceinline__ void tile_origin(int t, int tiles_m, int tiles_n, int& m0, int& n0) {
  const int per_group = kGroupM * tiles_n;
  const int first_m = (t / per_group) * kGroupM;
  const int gm = min(kGroupM, tiles_m - first_m);
  const int r = t % per_group;
  m0 = (first_m + r % gm) * kBM;
  n0 = (r / gm) * kBN;
}

// Persistent warp-specialised ping-pong kernel, one CTA per SM.  Warpgroup 2 (one thread) is the TMA producer and loads
// the CTA's tiles in order into the ring.  MMA warpgroup wg takes tiles wg, wg + 2, ... of the CTA's sequence and skips
// the ring slots of the other's tiles.  Per 64-deep k-block it issues 4 k16 steps x 2 wgmma.m64n128k16 (rows 0-63 and
// 64-127), keeps one k-block in flight while the next one issues (wait_group 1), and releases a ring slot as soon as
// its MMAs retire.  A named-barrier hand-off orders the mainloops: a warpgroup starts issuing a tile once the other has
// issued the previous one, so the two alternate on the tensor cores and each one's epilogue runs under the other's
// mainloop.  Each output element is summed by the same instructions in the same k order as with one warpgroup per
// 64 rows.
template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_d, int M, int N, int K, GemmEpi ep) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* park = smem + kStages * kStageBytes;                      // 64 KB, shared by the MMA warpgroups in turn
  uint8_t* epi_stage = park + kParkBytes;                            // 8 x 4 KB (1024-aligned), one per epilogue warp
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_stage + kEpiStageBytes);
  uint64_t* full_bar = bars;                        // [kStages]
  uint64_t* empty_bar = bars + kStages;             // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  const int tiles_m = (M + kBM - 1) / kBM;
  const int tiles_n = (N + kBN - 1) / kBN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = (K + kBK - 1) / kBK;
  const int cta_tiles = (num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;   // >= 1: the grid is <= num_tiles

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);   // released by the warpgroup that owns the slot's tile
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // predecessor grid complete before any global / TMA access

  if (wg == 2) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == 256) {
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < cta_tiles; ++i) {
        int m0, n0;
        tile_origin(blockIdx.x + i * gridDim.x, tiles_m, tiles_n, m0, n0);
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
    // ===================== MMA + epilogue warpgroups: whole tiles, alternating =====================
    setmaxnreg_inc<kMmaRegs>();
    constexpr uint32_t a_lbo = A_MN ? kBK * 128 : 16, a_kstep = A_MN ? 2048 : 32;
    constexpr uint32_t b_lbo = B_MN ? kBK * 128 : 16, b_kstep = B_MN ? 2048 : 32;
    // rows 64-127 of A: 8 KB into a K-major tile, the second 64-wide chunk of an MN-major one
    constexpr uint32_t a_rows = 64 * 128;
    const int q = warp & 1, half = (warp >> 1) & 1;      // epilogue: 32-row quarter of the 64 rows, column half
    float scale = ep.alpha;
    if (ep.scale_ptr != nullptr) {
      const float s = __ldg(ep.scale_ptr);
      scale *= ep.scale_tanh ? tanhf(s) : s;
    }
    // it = ring position (k-blocks loaded so far by the producer) of this warpgroup's current tile
    for (uint32_t i = wg, it = wg * num_kb; i < (uint32_t)cta_tiles; i += 2, it += 2 * num_kb) {
      int m0, n0;
      tile_origin(blockIdx.x + i * gridDim.x, tiles_m, tiles_n, m0, n0);
      float d[2][kBN / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < kBN / 2; ++j) d[h][j] = 0.f;
      if (i > 0) named_bar_sync(kOrderBar + wg, 256);   // the other warpgroup has issued tile i - 1
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        const int stage = (it + kb) % kStages;
        mbar_wait(&full_bar[stage], ((it + kb) / kStages) & 1);
        const uint32_t sa = smem_u32(smem + stage * kStageBytes);
        const uint32_t sb = sa + kABytes;
        const uint64_t da = make_smem_desc(sa, a_lbo, 1024);
        const uint64_t db = make_smem_desc(sb, b_lbo, 1024);
        wgmma_keep(d[0]);
        wgmma_keep(d[1]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            Wgmma<kBN, A_MN, B_MN>::mma(d[h], da + ((h * a_rows + k * a_kstep) >> 4), db + ((k * b_kstep) >> 4),
                                        (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();                                 // the previous k-block's MMAs retired: its slot is free
        wgmma_keep(d[0]);
        wgmma_keep(d[1]);
        if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
      }
      if (i + 1 < (uint32_t)cta_tiles) named_bar_arrive(kOrderBar + (wg ^ 1), 256);   // hand the tensor cores over
      wgmma_wait<0>();
      wgmma_keep(d[0]);
      wgmma_keep(d[1]);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
      // Epilogue: the whole 128 x 128 fp32 tile is parked in the shared park tile (so no accumulator register stays
      // live through the epilogue), then the fused epilogue runs on each 64-row half with one thread per (row, column
      // half).  The two warpgroups' epilogues take turns on the park tile in tile order, like their mainloops.
      if (i > 0) named_bar_sync(kEpiOrderBar + wg, 256);    // the other warpgroup has finished tile i - 1's epilogue
      acc_store<kBN>(park, 0, d[0]);
      acc_store<kBN>(park, 64, d[1]);
      named_bar_sync(1 + wg, 128);
#pragma unroll 1
      for (int h = 0; h < 2; ++h)
        epilogue_dispatch<kBN>(ep, scale, park + h * kAccBytes, m0 + 64 * h, n0, M, N, q, half, lane,
                               epi_stage + warp * kEpiWarpStage, &map_d);
      named_bar_sync(1 + wg, 128);                        // the park tile is read before the other warpgroup refills it
      if (i + 1 < (uint32_t)cta_tiles) named_bar_arrive(kEpiOrderBar + (wg ^ 1), 256);
      // the stage must outlive the last bulk store's reads.  Waited for here, inside the loop: the same wait after the
      // loop makes ptxas allocate the MMA warpgroups' code within the 168-register launch budget instead of the
      // setmaxnreg one, and the epilogue spills.
      if (i + 2 >= (uint32_t)cta_tiles && lane == 0) tma_store_wait_read<0>();
    }
  }
}

template <bool A_MN, bool B_MN>
static int launch_gemm(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                       const GemmEpi& ep, cudaStream_t stream) {
  CUtensorMap ma, mb, md;
  int rc;
  if (!A_MN) rc = make_tmap_bf16_2d(&ma, A, M, K, lda, kBM, 64);   // [M][K], box 128 rows x 64 k
  else       rc = make_tmap_bf16_2d(&ma, A, K, M, lda, kBK, 64);   // [K][M], box 64 k-rows x 64 m
  if (rc) return rc;
  if (!B_MN) rc = make_tmap_bf16_2d(&mb, B, N, K, ldb, kBN, 64);
  else       rc = make_tmap_bf16_2d(&mb, B, K, N, ldb, kBK, 64);
  if (rc) return rc;
  rc = ep.out_fp32 ? make_tmap_f32_2d(&md, ep.out, M, N, ep.ld_out, 32, 32)    // [M][N] output, box 32 rows x 128 B
                   : make_tmap_bf16_2d(&md, ep.out, M, N, ep.ld_out, 32, 64);
  if (rc) return rc;
  auto kern = gemm_bf16_kernel<A_MN, B_MN>;
  OTB_CHECK_CUDA(ensure_dyn_smem(kern, kGemmSmemBytes));   // per (instantiation, device)
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
  cfg.dynamicSmemBytes = kGemmSmemBytes;
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
  // the output tensor map of the TMA-store epilogue needs a 16-byte aligned base
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(e->out) & 15) == 0, "otb_gemm_bf16: out must be 16-byte aligned");
  // the epilogue reads bias / residual / aux_in and writes aux_out in 16 B vectors
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(e->bias) & 15) == 0, "otb_gemm_bf16: bias must be 16-byte aligned");
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(e->residual) & 15) == 0,
                "otb_gemm_bf16: residual must be 16-byte aligned");
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(e->aux_in) & 15) == 0, "otb_gemm_bf16: aux_in must be 16-byte aligned");
  OTB_CHECK_ARG((reinterpret_cast<uintptr_t>(e->aux_out) & 15) == 0,
                "otb_gemm_bf16: aux_out must be 16-byte aligned");
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
  ep.cls = -1;
  if (e->res_fp32 == 0) {                                   // the fp32 residual takes the run-time options
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
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  const int sel = (a_mn_major ? 2 : 0) | (b_mn_major ? 1 : 0);
  switch (sel) {
    case 0: return launch_gemm<false, false>(A, lda, B, ldb, M, N, K, ep, st);
    case 1: return launch_gemm<false, true>(A, lda, B, ldb, M, N, K, ep, st);
    case 3: return launch_gemm<true, true>(A, lda, B, ldb, M, N, K, ep, st);
    default: break;
  }
  return set_error(OTB_ERR_UNSUPPORTED, "otb_gemm_bf16: layout (A MN-major, B K-major) not instantiated");
}
