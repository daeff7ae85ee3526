// otter_b200 — causal self-attention of the frozen LM decoder layers (SURVEY.md §8f rank 1), head dim 128.
//
//   MPT-7B / LLaMA shapes: H query heads x 128, S = L (256 ... 2048), Q/K/V read in place from the fused Wqkv GEMM
//   output (bf16, head h at columns col0 + h*128), optional ALiBi key bias slope_h * (j - (S-1)) added to the scaled
//   scores (mpt/attention.py:51-56,457-464), causal mask (mpt/attention.py:68-75).  Grouped-query attention
//   (Llama-2-70B, Llama-3): kv_heads K/V heads, query head h reads K/V head h / (H / kv_heads) (HF's repeat_kv).
//
// Same machinery as otb_attn.cu (wgmma from 128B-swizzled TMA tiles, one warpgroup, softmax rows owned by threads and
// read from swizzled fp32 smem tiles), with every 128-wide operand held as two 64-column SW128 panels:
//   forward  (q tile, head, batch): S = Q K^T (8 k-steps over d) in two 64-key halves, two sweeps over the key tiles at
//            or below the diagonal (row max, then exp + O += P V with V consumed MN-major across both panels; O lives in
//            registers), O / l and LSE out.
//   backward (head, batch): 64-key tiles, so that dV_j and dK_j (64 x 128 each) stay in registers across the query
//            tiles: for key tile j, for query tile i that sees it: S, dP = dO V^T, P / dS staged in smem, dV_j += P^T dO,
//            dK_j += dS^T Q, dQ_i = dS K_j through a 64 KB fp32 tile and accumulated across key tiles in an fp32
//            workspace.  The weights of the LM are frozen: there is no wgrad, only these activation gradients.
//            With a group of g = H / kv_heads > 1 query heads per K/V head, each CTA still owns one query head: it writes
//            its fp32 dK/dV partials to the workspace and lm_attn_kv_reduce_kernel sums the g partials of a K/V head in
//            a fixed order (deterministic, no atomics; H*B CTAs instead of kv_heads*B).
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

constexpr int kLmThreads = 128;
constexpr int kPanel = 128 * 128;        // [128 rows][64 bf16] = 16 KB
constexpr int kTile2 = 2 * kPanel;       // [128 rows][128 bf16] as two panels
constexpr int kBwdKeys = 64;             // backward key tile
constexpr int kKPanel = kBwdKeys * 128;  // [64 keys][64 bf16] = 8 KB
constexpr float kLog2e = 1.4426950408889634f;

struct LmAttnParams {
  int B, H, S, causal;
  int q_col0, k_col0, v_col0;
  int kv_group;                          // H / kv_heads: query head h reads K/V head h / kv_group
  float scale, scale_log2;
  const float* slopes;                   // [H] ALiBi slopes or nullptr
  bf16* out; long long ldo; int o_col0;
  float* lse;                            // [B][H][S] natural log
  const bf16* dout; long long ld_do; int do_col0;
  bf16* dqkv; long long ld_dqkv; int dq_col0, dk_col0, dv_col0;
  float* dq_ws;                          // [B*S][H*128] fp32
  float* dk_ws; float* dv_ws;            // kv_group > 1: per-query-head dK / dV partials, [B*S][H*128] fp32 each
};

__device__ __forceinline__ float lm_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 16 B unit of row r, columns [c, c+8) of a [rows][64] SW128 panel
__device__ __forceinline__ void lm_st_sw128(uint8_t* panel, int r, int c_in_panel, uint4 v) {
  const int unit = (c_in_panel >> 3) ^ (r & 7);
  *reinterpret_cast<uint4*>(panel + r * 128 + unit * 16) = v;
}
// number of keys of the key tile starting at key k0 (at most `tk` keys) a query row may see: [0, hi)
__device__ __forceinline__ int lm_row_hi(const LmAttnParams& p, bool row_ok, int row, int k0, int tk) {
  if (!row_ok) return 0;
  const int valid = min(tk, p.S - k0);
  return p.causal ? max(0, min(valid, row - k0 + 1)) : valid;
}

// ================================================================================================
// forward
// ================================================================================================
__global__ void __launch_bounds__(kLmThreads)
lm_attn_fwd_kernel(const __grid_constant__ CUtensorMap map_qkv, LmAttnParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_q = smem;                     // 32 KB
  uint8_t* s_k = s_q + kTile2;             // 2 stages x 32 KB
  uint8_t* s_v = s_k + 2 * kTile2;         // 2 stages x 32 KB
  uint8_t* s_p = s_v + 2 * kTile2;         // 32 KB: P as two 64-key panels of [128 rows][128 B]
  uint8_t* acc_s = s_p + kTile2;           // 32 KB: S of one 64-key half [128][64] fp32
  uint64_t* bars = reinterpret_cast<uint64_t*>(acc_s + kTile2);
  uint64_t* full = bars;                   // [2]
  uint64_t* bar_q = bars + 2;

  const int tid = threadIdx.x;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int kvh = h / p.kv_group;

  if (tid == 0) {
    mbar_init(&full[0], 1); mbar_init(&full[1], 1); mbar_init(bar_q, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  const int nt_all = (p.S + 127) / 128;
  const int nt = p.causal ? min(nt_all, qt + 1) : nt_all;       // key tiles at or below the diagonal
  const int nsteps = (nt == 1) ? 1 : 2 * nt;

  const int row = qt * 128 + tid;
  const bool row_ok = row < p.S;
  const float slope2 = (p.slopes != nullptr) ? __ldg(p.slopes + h) * kLog2e : 0.f;

  auto issue_load = [&](int s) {  // thread 0 only
    const int j = (nt == 1) ? 0 : (s % nt);
    const bool need_v = (nt == 1) || (s >= nt);
    const int st = s & 1;
    const int krow = b * p.S + j * 128;
    mbar_arrive_expect_tx(&full[st], need_v ? 2 * kTile2 : kTile2);
#pragma unroll
    for (int pp = 0; pp < 2; ++pp) {
      tma_load_2d(s_k + st * kTile2 + pp * kPanel, &map_qkv, &full[st], p.k_col0 + kvh * 128 + pp * 64, krow);
      if (need_v) tma_load_2d(s_v + st * kTile2 + pp * kPanel, &map_qkv, &full[st], p.v_col0 + kvh * 128 + pp * 64, krow);
    }
  };
  const uint32_t q_addr = smem_u32(s_q), p_addr = smem_u32(s_p);
  auto compute_s_half = [&](int st, int kh) {  // S[:, 64 kh : 64 kh + 64] = Q K^T over d = 128: panel k>>2, step k&3
    const uint32_t k_addr = smem_u32(s_k + st * kTile2) + kh * 8192;
    wg_mma_tile<64, 0, 0>(
        acc_s, 8, [&](int hh, int k) { return make_smem_desc(q_addr + (k >> 2) * kPanel + hh * 8192 + (k & 3) * 32, 16, 1024); },
        [&](int k) { return make_smem_desc(k_addr + (k >> 2) * kPanel + (k & 3) * 32, 16, 1024); });
    __syncthreads();
  };
  float o[2][64];                // O rows [64 hh, 64 hh + 64) as wgmma fragments
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
#pragma unroll
    for (int i = 0; i < 64; ++i) o[hh][i] = 0.f;
  bool o_started = false;

  if (tid == 0) {
    tma_prefetch_desc(&map_qkv);
    mbar_arrive_expect_tx(bar_q, kTile2);
#pragma unroll
    for (int pp = 0; pp < 2; ++pp)
      tma_load_2d(s_q + pp * kPanel, &map_qkv, bar_q, p.q_col0 + h * 128 + pp * 64, b * p.S + qt * 128);
    issue_load(0);
  }
  mbar_wait(bar_q, 0);

  float m_run = -INFINITY, l_run = 0.f;      // m_run in the log2 domain: max of s*scale*log2e + bias*log2e
  for (int s = 0; s < nsteps; ++s) {
    if (tid == 0 && s + 1 < nsteps) issue_load(s + 1);   // its buffer was last read by the MMAs of step s - 1
    const int st = s & 1;
    mbar_wait(&full[st], (s >> 1) & 1);
    const int j = (nt == 1) ? 0 : (s % nt);
    const bool is_p2 = (nt == 1) || (s >= nt);
    const bool do_max = (nt == 1) || (s < nt);
    const int hi = lm_row_hi(p, row_ok, row, j * 128, 128);
    const float kf0 = static_cast<float>(j * 128 - (p.S - 1));    // ALiBi distance of the tile's first key
    if (do_max) {
#pragma unroll 1
      for (int kh = 0; kh < 2; ++kh) {
        compute_s_half(st, kh);
#pragma unroll 1
        for (int c2 = 0; c2 < 2; ++c2) {
          const int c = kh * 2 + c2;
          uint32_t r[32];
          acc_ld32<64>(acc_s, tid, c2 * 32, r);
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int cc = c * 32 + i;
            const float t = fmaf(__uint_as_float(r[i]), p.scale_log2, slope2 * (kf0 + static_cast<float>(cc)));
            if (cc < hi) m_run = fmaxf(m_run, t);
          }
        }
        __syncthreads();
      }
    }
    if (is_p2) {
      const float mb2 = (m_run == -INFINITY) ? 0.f : m_run;        // final here
#pragma unroll 1
      for (int kh = 0; kh < 2; ++kh) {
        compute_s_half(st, kh);
#pragma unroll 1
        for (int c2 = 0; c2 < 2; ++c2) {
          const int c = kh * 2 + c2;
          uint32_t r[32];
          acc_ld32<64>(acc_s, tid, c2 * 32, r);
          float pv[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int cc = c * 32 + i;
            const float t = fmaf(__uint_as_float(r[i]), p.scale_log2, slope2 * (kf0 + static_cast<float>(cc)));
            const float v = (cc < hi) ? lm_ex2(t - mb2) : 0.f;
            pv[i] = v;
            l_run += v;
          }
          uint8_t* panel = s_p + kh * kPanel;
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            uint4 ov;
            ov.x = pack_bf16x2(pv[g * 8 + 0], pv[g * 8 + 1]); ov.y = pack_bf16x2(pv[g * 8 + 2], pv[g * 8 + 3]);
            ov.z = pack_bf16x2(pv[g * 8 + 4], pv[g * 8 + 5]); ov.w = pack_bf16x2(pv[g * 8 + 6], pv[g * 8 + 7]);
            lm_st_sw128(panel, tid, c2 * 32 + g * 8, ov);
          }
        }
        __syncthreads();
      }
      fence_proxy_async_smem();
      __syncthreads();
      // O += P V: A = P K-major over keys, B = V MN-major, N = 128 over 2 panels
      const uint32_t v_addr = smem_u32(s_v + st * kTile2);
      wg_mma_regs<128, 0, 1>(
          o, o_started, 8,
          [&](int hh, int k) { return make_smem_desc(p_addr + (k >> 2) * kPanel + hh * 8192 + (k & 3) * 32, 16, 1024); },
          [&](int k) { return make_smem_desc(v_addr + k * 2048, kPanel, 1024); });
      o_started = true;
    }
  }

  // ---- epilogue: O / l -> bf16, LSE (O parked in the S and P buffers: [128][128] fp32 = 64 KB) ----
  __syncthreads();
  uint8_t* acc_o = s_p;
  acc_store<128>(acc_o, 0, o[0]);
  acc_store<128>(acc_o, 64, o[1]);
  __syncthreads();
  const float inv_l = (l_run > 0.f) ? 1.0f / l_run : 0.f;
#pragma unroll 1
  for (int c = 0; c < 4; ++c) {
    uint32_t r[32];
    acc_ld32<128>(acc_o, tid, c * 32, r);
    if (row_ok) {
      bf16* dst = p.out + static_cast<long long>(b * p.S + row) * p.ldo + p.o_col0 + h * 128 + c * 32;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        uint4 ov;
        ov.x = pack_bf16x2(__uint_as_float(r[g * 8 + 0]) * inv_l, __uint_as_float(r[g * 8 + 1]) * inv_l);
        ov.y = pack_bf16x2(__uint_as_float(r[g * 8 + 2]) * inv_l, __uint_as_float(r[g * 8 + 3]) * inv_l);
        ov.z = pack_bf16x2(__uint_as_float(r[g * 8 + 4]) * inv_l, __uint_as_float(r[g * 8 + 5]) * inv_l);
        ov.w = pack_bf16x2(__uint_as_float(r[g * 8 + 6]) * inv_l, __uint_as_float(r[g * 8 + 7]) * inv_l);
        *reinterpret_cast<uint4*>(dst + g * 8) = ov;
      }
    }
  }
  if (row_ok && p.lse != nullptr) {
    p.lse[(static_cast<long long>(b) * p.H + h) * p.S + row] =
        (l_run > 0.f) ? (m_run + log2f(l_run)) * 0.6931471805599453f : 0.f;
  }
}

// ================================================================================================
// backward (activation gradients only)
// ================================================================================================
// kGrouped: dK / dV partials of this query head go to p.dk_ws / p.dv_ws in fp32 (summed by lm_attn_kv_reduce_kernel);
// otherwise they are final and written to dqkv in bf16.
template <bool kGrouped>
__global__ void __launch_bounds__(kLmThreads)
lm_attn_bwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                   const __grid_constant__ CUtensorMap map_do, LmAttnParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_k = smem;                     // 16 KB  K_j  [64 keys][128 d] (2 panels of 8 KB)
  uint8_t* s_v = s_k + 2 * kKPanel;        // 16 KB  V_j
  uint8_t* s_q = s_v + 2 * kKPanel;        // 32 KB  Q_i  [128 rows][128 d] (2 panels)
  uint8_t* s_do = s_q + kTile2;            // 32 KB  dO_i
  uint8_t* s_p = s_do + kTile2;            // 16 KB  P   [128 rows][64 keys] (1 panel)
  uint8_t* s_ds = s_p + kPanel;            // 16 KB  dS * scale
  uint8_t* acc_s = s_ds + kPanel;          // 32 KB  S  [128][64] fp32  } dQ [128][128] fp32 over both;
  uint8_t* acc_dp = acc_s + kTile2;        // 32 KB  dP [128][64] fp32  } dV, dK [64][128] at the end of a key tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(acc_dp + kTile2);
  uint64_t* bar_kv = bars;
  uint64_t* bar_qdo = bars + 1;

  const int tid = threadIdx.x;
  const int h = blockIdx.x, b = blockIdx.y;
  const int kvh = h / p.kv_group;

  if (tid == 0) {
    mbar_init(bar_kv, 1); mbar_init(bar_qdo, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  const int nkt = (p.S + kBwdKeys - 1) / kBwdKeys, nqt = (p.S + 127) / 128;
  const float slope2 = (p.slopes != nullptr) ? __ldg(p.slopes + h) * kLog2e : 0.f;
  const uint32_t a_k = smem_u32(s_k), a_v = smem_u32(s_v), a_q = smem_u32(s_q), a_do = smem_u32(s_do);
  const uint32_t a_p = smem_u32(s_p), a_ds = smem_u32(s_ds);

  uint32_t ph_kv = 0, ph_qdo = 0;
  if (tid == 0) { tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_kv); tma_prefetch_desc(&map_do); }

  for (int j = 0; j < nkt; ++j) {
    const int k0 = j * kBwdKeys;
    const int kvalid = min(kBwdKeys, p.S - k0);
    const int krow = b * p.S + k0;
    if (tid == 0) {
      mbar_arrive_expect_tx(bar_kv, 4 * kKPanel);
#pragma unroll
      for (int pp = 0; pp < 2; ++pp) {
        tma_load_2d(s_k + pp * kKPanel, &map_kv, bar_kv, p.k_col0 + kvh * 128 + pp * 64, krow);
        tma_load_2d(s_v + pp * kKPanel, &map_kv, bar_kv, p.v_col0 + kvh * 128 + pp * 64, krow);
      }
    }
    float dv[1][64], dk[1][64];      // dV_j, dK_j: the 64 keys of this tile x 128 d
#pragma unroll
    for (int i = 0; i < 64; ++i) { dv[0][i] = 0.f; dk[0][i] = 0.f; }
    const int i_first = p.causal ? k0 / 128 : 0;
    for (int i = i_first; i < nqt; ++i) {
      const int row = i * 128 + tid;
      const bool row_ok = row < p.S;
      const long long grow = static_cast<long long>(b) * p.S + row;
      if (tid == 0) {
        mbar_arrive_expect_tx(bar_qdo, 2 * kTile2);
#pragma unroll
        for (int pp = 0; pp < 2; ++pp) {
          tma_load_2d(s_q + pp * kPanel, &map_q, bar_qdo, p.q_col0 + h * 128 + pp * 64, b * p.S + i * 128);
          tma_load_2d(s_do + pp * kPanel, &map_do, bar_qdo, p.do_col0 + h * 128 + pp * 64, b * p.S + i * 128);
        }
      }
      // per-row scalars (overlap the TMA): delta = rowsum(dO . O), lse
      float delta = 0.f, lse = 0.f;
      if (row_ok) {
        const uint4* po = reinterpret_cast<const uint4*>(p.out + grow * p.ldo + p.o_col0 + h * 128);
        const uint4* pd = reinterpret_cast<const uint4*>(p.dout + grow * p.ld_do + p.do_col0 + h * 128);
#pragma unroll 4
        for (int g = 0; g < 16; ++g) {
          const uint4 a = __ldg(po + g), d = __ldg(pd + g);
          const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y), a2 = unpack_bf16x2(a.z), a3 = unpack_bf16x2(a.w);
          const float2 d0 = unpack_bf16x2(d.x), d1 = unpack_bf16x2(d.y), d2 = unpack_bf16x2(d.z), d3 = unpack_bf16x2(d.w);
          delta += a0.x * d0.x + a0.y * d0.y + a1.x * d1.x + a1.y * d1.y + a2.x * d2.x + a2.y * d2.y + a3.x * d3.x +
                   a3.y * d3.y;
        }
        lse = p.lse[(static_cast<long long>(b) * p.H + h) * p.S + row];
      }
      const int hi = lm_row_hi(p, row_ok, row, k0, kBwdKeys);
      const float lse_l2 = lse * kLog2e;
      const float kf0 = static_cast<float>(k0 - (p.S - 1));

      if (i == i_first) mbar_wait(bar_kv, ph_kv);
      mbar_wait(bar_qdo, ph_qdo);
      ph_qdo ^= 1;
      // S = Q K^T, dP = dO V^T: [128 rows][64 keys], 8 k-steps over d (panel k>>2, step k&3)
      wg_mma_tile<64, 0, 0>(
          acc_s, 8, [&](int hh, int k) { return make_smem_desc(a_q + (k >> 2) * kPanel + hh * 8192 + (k & 3) * 32, 16, 1024); },
          [&](int k) { return make_smem_desc(a_k + (k >> 2) * kKPanel + (k & 3) * 32, 16, 1024); });
      wg_mma_tile<64, 0, 0>(
          acc_dp, 8,
          [&](int hh, int k) { return make_smem_desc(a_do + (k >> 2) * kPanel + hh * 8192 + (k & 3) * 32, 16, 1024); },
          [&](int k) { return make_smem_desc(a_v + (k >> 2) * kKPanel + (k & 3) * 32, 16, 1024); });
      __syncthreads();

#pragma unroll 1
      for (int c = 0; c < 2; ++c) {
        uint32_t rs[32], rp[32];
        acc_ld32<64>(acc_s, tid, c * 32, rs);
        acc_ld32<64>(acc_dp, tid, c * 32, rp);
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float pv[8], dv8[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int cc = c * 32 + g * 8 + e;
            float pr = 0.f, ds = 0.f;
            if (cc < hi) {
              const float t = fmaf(__uint_as_float(rs[g * 8 + e]), p.scale_log2, slope2 * (kf0 + static_cast<float>(cc)));
              pr = lm_ex2(t - lse_l2);
              ds = pr * (__uint_as_float(rp[g * 8 + e]) - delta) * p.scale;
            }
            pv[e] = pr; dv8[e] = ds;
          }
          uint4 o;
          o.x = pack_bf16x2(pv[0], pv[1]); o.y = pack_bf16x2(pv[2], pv[3]);
          o.z = pack_bf16x2(pv[4], pv[5]); o.w = pack_bf16x2(pv[6], pv[7]);
          lm_st_sw128(s_p, tid, c * 32 + g * 8, o);
          o.x = pack_bf16x2(dv8[0], dv8[1]); o.y = pack_bf16x2(dv8[2], dv8[3]);
          o.z = pack_bf16x2(dv8[4], dv8[5]); o.w = pack_bf16x2(dv8[6], dv8[7]);
          lm_st_sw128(s_ds, tid, c * 32 + g * 8, o);
        }
      }
      fence_proxy_async_smem();
      __syncthreads();

      // dV += P^T dO ; dK += dS^T Q   A MN-major (M = the 64 keys: one panel), K-step = 16 query rows = +2048 B;
      // B MN-major (N = d: 2 panels of 64, LBO = panel stride), same K-step.
      const bool acc = i > i_first;
      wg_mma_regs<128, 1, 1>(
          dv, acc, 8, [&](int, int k) { return make_smem_desc(a_p + k * 2048, kPanel, 1024); },
          [&](int k) { return make_smem_desc(a_do + k * 2048, kPanel, 1024); });
      wg_mma_regs<128, 1, 1>(
          dk, acc, 8, [&](int, int k) { return make_smem_desc(a_ds + k * 2048, kPanel, 1024); },
          [&](int k) { return make_smem_desc(a_q + k * 2048, kPanel, 1024); });
      // dQ = dS K   A K-major over the 64 keys, B = K_j MN-major (N = d over 2 panels of [64 keys][128 B])
      uint8_t* acc_dq = acc_s;             // [128][128] fp32 over acc_s and acc_dp
      wg_mma_tile<128, 0, 1>(
          acc_dq, 4, [&](int hh, int k) { return make_smem_desc(a_ds + hh * 8192 + k * 32, 16, 1024); },
          [&](int k) { return make_smem_desc(a_k + k * 2048, kKPanel, 1024); });
      __syncthreads();

      // dQ tile: accumulate across the key tiles this query tile sees through the fp32 workspace
      const int j_last = p.causal ? min((i * 128 + 127) / kBwdKeys, nkt - 1) : nkt - 1;
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        uint32_t r[32];
        acc_ld32<128>(acc_dq, tid, c * 32, r);
        if (row_ok) {
          float v[32];
#pragma unroll
          for (int e = 0; e < 32; ++e) v[e] = __uint_as_float(r[e]);
          float* ws = (j_last > 0) ? p.dq_ws + grow * (p.H * 128) + h * 128 + c * 32 : nullptr;
          if (j > 0) {
#pragma unroll
            for (int e = 0; e < 32; e += 4) {
              const float4 w = *reinterpret_cast<const float4*>(ws + e);
              v[e] += w.x; v[e + 1] += w.y; v[e + 2] += w.z; v[e + 3] += w.w;
            }
          }
          if (j == j_last) {
            bf16* dst = p.dqkv + grow * p.ld_dqkv + p.dq_col0 + h * 128 + c * 32;
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              uint4 o;
              o.x = pack_bf16x2(v[g * 8 + 0], v[g * 8 + 1]); o.y = pack_bf16x2(v[g * 8 + 2], v[g * 8 + 3]);
              o.z = pack_bf16x2(v[g * 8 + 4], v[g * 8 + 5]); o.w = pack_bf16x2(v[g * 8 + 6], v[g * 8 + 7]);
              *reinterpret_cast<uint4*>(dst + g * 8) = o;
            }
          } else {
#pragma unroll
            for (int e = 0; e < 32; e += 4)
              *reinterpret_cast<float4*>(ws + e) = make_float4(v[e], v[e + 1], v[e + 2], v[e + 3]);
          }
        }
      }
      __syncthreads();
    }
    ph_kv ^= 1;

    // dV_j, dK_j complete: row t of the [64][128] tiles = key t of this tile
    acc_store<128>(acc_s, 0, dv[0]);
    acc_store<128>(acc_dp, 0, dk[0]);
    __syncthreads();
    {
      const bool key_ok = tid < kvalid;
#pragma unroll 1
      for (int w = 0; w < 2; ++w) {      // 0: dV, 1: dK
        uint8_t* src = w ? acc_dp : acc_s;
#pragma unroll 1
        for (int c = 0; c < 4; ++c) {
          if (key_ok) {
            uint32_t r[32];
            acc_ld32<128>(src, tid, c * 32, r);
            if constexpr (kGrouped) {
              float* dst = (w ? p.dk_ws : p.dv_ws) + static_cast<long long>(krow + tid) * (p.H * 128) + h * 128 + c * 32;
#pragma unroll
              for (int e = 0; e < 32; e += 4)
                *reinterpret_cast<float4*>(dst + e) = make_float4(__uint_as_float(r[e]), __uint_as_float(r[e + 1]),
                                                                  __uint_as_float(r[e + 2]), __uint_as_float(r[e + 3]));
              continue;
            }
            bf16* dst = p.dqkv + static_cast<long long>(krow + tid) * p.ld_dqkv + (w ? p.dk_col0 : p.dv_col0) + h * 128 +
                        c * 32;
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              uint4 o;
              o.x = pack_bf16x2(__uint_as_float(r[g * 8 + 0]), __uint_as_float(r[g * 8 + 1]));
              o.y = pack_bf16x2(__uint_as_float(r[g * 8 + 2]), __uint_as_float(r[g * 8 + 3]));
              o.z = pack_bf16x2(__uint_as_float(r[g * 8 + 4]), __uint_as_float(r[g * 8 + 5]));
              o.w = pack_bf16x2(__uint_as_float(r[g * 8 + 6]), __uint_as_float(r[g * 8 + 7]));
              *reinterpret_cast<uint4*>(dst + g * 8) = o;
            }
          }
        }
      }
    }
    __syncthreads();
  }
}

// dK / dV of K/V head kvh = sum over r = 0 .. kv_group-1 (in this order) of the partials of query head kvh*kv_group + r.
// Thread = 8 columns of one (row, dK or dV, K/V head).
__global__ void __launch_bounds__(256) lm_attn_kv_reduce_kernel(LmAttnParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int nkv = p.H / p.kv_group;
  const long long total = static_cast<long long>(p.B) * p.S * 2 * nkv * 16;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int u = static_cast<int>(idx & 15);
    const long long t = idx >> 4;
    const int kvh = static_cast<int>(t % nkv);
    const long long t2 = t / nkv;
    const int w = static_cast<int>(t2 & 1);               // 0: dV, 1: dK
    const long long row = t2 >> 1;
    const float* src = (w ? p.dk_ws : p.dv_ws) + row * (p.H * 128) + kvh * p.kv_group * 128 + u * 8;
    float a[8];
    {
      const float4 x0 = reinterpret_cast<const float4*>(src)[0], x1 = reinterpret_cast<const float4*>(src)[1];
      a[0] = x0.x; a[1] = x0.y; a[2] = x0.z; a[3] = x0.w; a[4] = x1.x; a[5] = x1.y; a[6] = x1.z; a[7] = x1.w;
    }
    for (int r = 1; r < p.kv_group; ++r) {
      const float4 x0 = reinterpret_cast<const float4*>(src + r * 128)[0], x1 = reinterpret_cast<const float4*>(src + r * 128)[1];
      a[0] += x0.x; a[1] += x0.y; a[2] += x0.z; a[3] += x0.w; a[4] += x1.x; a[5] += x1.y; a[6] += x1.z; a[7] += x1.w;
    }
    *reinterpret_cast<uint4*>(p.dqkv + row * p.ld_dqkv + (w ? p.dk_col0 : p.dv_col0) + kvh * 128 + u * 8) = pack8(a);
  }
}

constexpr int kLmFwdSmem = 6 * kTile2 + kTile2 + 1024 + 128;
constexpr int kLmBwdSmem = 4 * kKPanel + 2 * kTile2 + 2 * kPanel + 2 * kTile2 + 1024 + 128;

}  // namespace otb

using namespace otb;

static int lm_check(const otb_lm_attn_desc* d) {
  OTB_CHECK_ARG(d != nullptr && d->qkv != nullptr && d->out != nullptr, "otb_lm_attn: null pointer");
  OTB_CHECK_ARG(d->B > 0 && d->H > 0 && d->S > 0, "otb_lm_attn: bad sizes");
  OTB_CHECK_ARG(d->head_dim == 128, "otb_lm_attn: head_dim must be 128 (MPT-7B / LLaMA)");
  OTB_CHECK_ARG(d->kv_heads >= 0 && (d->kv_heads == 0 || d->H % d->kv_heads == 0),
                "otb_lm_attn: kv_heads must divide H (0 means H)");
  OTB_CHECK_ARG(d->ld_qkv % 8 == 0 && d->ld_out % 8 == 0, "otb_lm_attn: row pitches must be multiples of 8");
  OTB_CHECK_ARG(d->q_col0 % 8 == 0 && d->k_col0 % 8 == 0 && d->v_col0 % 8 == 0 && d->out_col0 % 8 == 0,
                "otb_lm_attn: column offsets must be multiples of 8");
  return OTB_OK;
}

static void lm_fill(const otb_lm_attn_desc* d, LmAttnParams& p) {
  p.B = d->B; p.H = d->H; p.S = d->S; p.causal = d->causal;
  p.q_col0 = d->q_col0; p.k_col0 = d->k_col0; p.v_col0 = d->v_col0;
  p.kv_group = d->kv_heads ? d->H / d->kv_heads : 1;
  p.scale = d->scale; p.scale_log2 = d->scale * kLog2e;
  p.slopes = d->alibi_slopes;
  p.out = static_cast<bf16*>(d->out); p.ldo = d->ld_out; p.o_col0 = d->out_col0;
  p.lse = d->lse;
  p.dout = nullptr; p.ld_do = 0; p.do_col0 = 0;
  p.dqkv = nullptr; p.ld_dqkv = 0; p.dq_col0 = p.dk_col0 = p.dv_col0 = 0;
  p.dq_ws = p.dk_ws = p.dv_ws = nullptr;
}

extern "C" int otb_lm_attn_fwd(const otb_lm_attn_desc* d, void* stream) {
  int rc = lm_check(d);
  if (rc) return rc;
  LmAttnParams p;
  lm_fill(d, p);
  CUtensorMap mqkv;
  rc = make_tmap_bf16_2d(&mqkv, d->qkv, (uint64_t)d->B * d->S, d->qkv_cols, d->ld_qkv, 128, 64);
  if (rc) return rc;
  OTB_CHECK_CUDA(ensure_dyn_smem(lm_attn_fwd_kernel, kLmFwdSmem));
  dim3 grid((d->S + 127) / 128, d->H, d->B);
  OTB_CHECK_CUDA(launch_k(lm_attn_fwd_kernel, grid, dim3(kLmThreads), kLmFwdSmem, static_cast<cudaStream_t>(stream), mqkv, p));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_lm_attn_bwd(const otb_lm_attn_desc* d, const otb_lm_attn_grads* g, void* stream) {
  int rc = lm_check(d);
  if (rc) return rc;
  OTB_CHECK_ARG(g && d->lse && g->dout && g->dqkv, "otb_lm_attn_bwd: null tensor");
  OTB_CHECK_ARG(d->S <= kBwdKeys || g->dq_ws != nullptr, "otb_lm_attn_bwd: dq workspace required for S > 64");
  OTB_CHECK_ARG(d->kv_heads == 0 || d->kv_heads == d->H || g->dq_ws != nullptr,
                "otb_lm_attn_bwd: workspace required when kv_heads < H");
  OTB_CHECK_ARG(g->ld_dout % 8 == 0 && g->ld_dqkv % 8 == 0, "otb_lm_attn_bwd: row pitches must be multiples of 8");
  LmAttnParams p;
  lm_fill(d, p);
  p.dout = static_cast<const bf16*>(g->dout); p.ld_do = g->ld_dout; p.do_col0 = g->dout_col0;
  p.dqkv = static_cast<bf16*>(g->dqkv); p.ld_dqkv = g->ld_dqkv;
  p.dq_col0 = g->dq_col0; p.dk_col0 = g->dk_col0; p.dv_col0 = g->dv_col0;
  p.dq_ws = g->dq_ws;
  const bool grouped = p.kv_group > 1;
  if (grouped) {                         // [3][B*S][H*128]: dQ, dK partials, dV partials
    const long long plane = static_cast<long long>(d->B) * d->S * d->H * 128;
    p.dk_ws = g->dq_ws + plane;
    p.dv_ws = g->dq_ws + 2 * plane;
  }
  CUtensorMap mq, mkv, mdo;
  rc = make_tmap_bf16_2d(&mq, d->qkv, (uint64_t)d->B * d->S, d->qkv_cols, d->ld_qkv, 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&mkv, d->qkv, (uint64_t)d->B * d->S, d->qkv_cols, d->ld_qkv, kBwdKeys, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&mdo, g->dout, (uint64_t)d->B * d->S, g->dout_cols, g->ld_dout, 128, 64);
  if (rc) return rc;
  const auto kernel = grouped ? lm_attn_bwd_kernel<true> : lm_attn_bwd_kernel<false>;
  OTB_CHECK_CUDA(ensure_dyn_smem(kernel, kLmBwdSmem));
  dim3 grid(d->H, d->B);
  OTB_CHECK_CUDA(launch_k(kernel, grid, dim3(kLmThreads), kLmBwdSmem, static_cast<cudaStream_t>(stream), mq, mkv, mdo, p));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  if (grouped) {
    const long long units = static_cast<long long>(d->B) * d->S * 2 * (d->H / p.kv_group) * 16;
    const long long cap = static_cast<long long>(sm_count()) * 8;
    const int blocks = static_cast<int>(std::min((units + 255) / 256, cap));
    OTB_CHECK_CUDA(launch_k(lm_attn_kv_reduce_kernel, dim3(blocks), dim3(256), 0, static_cast<cudaStream_t>(stream), p));
    count_launch();
    OTB_CHECK_CUDA(cudaGetLastError());
  }
  return OTB_OK;
}
