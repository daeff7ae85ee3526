// otter_b200 — fused attention cores on wgmma / TMA (forward + backward).
//
// One kernel family serves the three attention cores of the hot path:
//   (A) perceiver latent x (vision ++ latent) attention      modeling_otter.py:168-179   (two key sources)
//   (B) gated cross-attention text x latent with media mask   modeling_otter.py:290-333   (text_time mask)
//   (C) CLIP ViT self-attention (no mask)                     xformers_model/clip.py:112-128
//
// Layout: no head permutes — Q/K/V/O are read/written in place inside the projection GEMM outputs
// ([rows][cols] bf16, head h at columns col0 + h*64), addressed through TMA tensor maps.
//
// Forward, per CTA = (128-row query tile, head, problem), one warpgroup (thread t owns query row t):
//   S = Q K^T on wgmma (two m64n128k16 halves) parked in a swizzled fp32 smem tile and read back row by row; softmax in
//   fp32 registers (two sweeps over the key tiles: row max, then exp/accumulate — no rescaling of O); P (bf16) staged
//   in 128B-swizzled smem; O += P V on wgmma with V consumed MN-major straight from its TMA tile, O accumulated in
//   registers across key tiles; O/l written once.  K/V tiles are double-buffered TMA loads.
// Backward, per CTA = (head, problem): loops key tiles (outer) x query tiles (inner) with S, dP = dO V^T (in two
//   64-key halves through 32 KB fp32 tiles), dV += P^T dO, dK += dS^T Q (accumulated in registers across query tiles)
//   and dQ = dS K, all on wgmma; P / dS are staged in smem and consumed K-major and MN-major from the same bytes.
//
// Mask semantics of (B) (bit-exact w.r.t. the reference, SURVEY.md §8a-5): with tt = text_time[b,row]
//   tt == 0        -> attention row zeroed after softmax (output row exactly 0, no gradients)
//   1 <= tt <= T   -> only keys of media slot tt-1 participate
//   tt > T         -> every key masked with -FLT_MAX => uniform attention 1/(T*n); dS = 0, dV gets dO/(T*n)
#include <cstdlib>

#include "otb_attn_common.cuh"
#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

// ================================================================================================
// forward
// ================================================================================================
__global__ void __launch_bounds__(kAttnThreads)
attn_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv1,
                const __grid_constant__ CUtensorMap map_kv2, AttnParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_q = smem;                        // 16 KB
  uint8_t* s_k = s_q + kTileBytes;            // 2 x 16 KB
  uint8_t* s_v = s_k + 2 * kTileBytes;        // 2 x 16 KB
  uint8_t* s_p = s_v + 2 * kTileBytes;        // 32 KB: P as two 64-key chunks of [128 rows][128 B]
  uint8_t* acc_s = s_p + 2 * kTileBytes;      // 64 KB: S [128][128] fp32 (O [128][64] at the end)
  uint64_t* bars = reinterpret_cast<uint64_t*>(acc_s + 4 * kTileBytes);
  uint64_t* full = bars;        // [2]
  uint64_t* bar_q = bars + 2;

  const int tid = threadIdx.x;
  const int qt = blockIdx.x, h = blockIdx.y, prob = blockIdx.z;

  if (tid == 0) {
    mbar_init(&full[0], 1); mbar_init(&full[1], 1); mbar_init(bar_q, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // predecessor grid complete before any global / TMA access

  const int nt1 = (p.Sk1 + 127) / 128, nt2 = (p.Sk2 + 127) / 128, nt = nt1 + nt2;
  const int nsteps = (nt == 1) ? 1 : 2 * nt;

  const int row = qt * 128 + tid;
  const bool row_ok = row < p.Sq;
  int tt = 0;
  if (p.text_time != nullptr && row_ok) tt = p.text_time[prob * p.Sq + row];
  const int cls = row_ok ? row_class(p, tt) : 0;

  auto issue_load = [&](int s) {  // thread 0 only
    const int j = (nt == 1) ? 0 : (s % nt);
    const bool need_v = (nt == 1) || (s >= nt);
    const KeyTile kt = key_tile(p, prob, j, nt1);
    const int st = s & 1;
    mbar_arrive_expect_tx(&full[st], need_v ? 2 * kTileBytes : kTileBytes);
    const CUtensorMap* m = kt.src ? &map_kv2 : &map_kv1;
    tma_load_2d(s_k + st * kTileBytes, m, &full[st], (kt.src ? p.k2_col0 : p.k1_col0) + h * 64, kt.row0);
    if (need_v) tma_load_2d(s_v + st * kTileBytes, m, &full[st], (kt.src ? p.v2_col0 : p.v1_col0) + h * 64, kt.row0);
  };
  const uint32_t q_addr = smem_u32(s_q);
  auto compute_s = [&](int st) {  // S = Q K^T into acc_s
    const uint32_t k_addr = smem_u32(s_k + st * kTileBytes);
    wg_mma_tile<128, 0, 0>(
        acc_s, 4, [&](int hh, int k) { return make_smem_desc(q_addr + hh * 8192 + k * 32, 16, 1024); },
        [&](int k) { return make_smem_desc(k_addr + k * 32, 16, 1024); });
  };
  float o[2][32];               // O rows [64 h, 64 h + 64) as wgmma fragments
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[hh][i] = 0.f;
  bool o_started = false;
  auto issue_pv = [&](int st) {  // O += P V   (A = P K-major over keys, B = V MN-major)
    const uint32_t v_addr = smem_u32(s_v + st * kTileBytes), p_addr = smem_u32(s_p);
    wg_mma_regs<64, 0, 1>(
        o, o_started, 8,
        [&](int hh, int k) { return make_smem_desc(p_addr + (k >> 2) * kTileBytes + hh * 8192 + (k & 3) * 32, 16, 1024); },
        [&](int k) { return make_smem_desc(v_addr + k * 2048, 16, 1024); });
    o_started = true;
  };

  if (tid == 0) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_kv1); tma_prefetch_desc(&map_kv2);
    mbar_arrive_expect_tx(bar_q, kTileBytes);
    tma_load_2d(s_q, &map_q, bar_q, p.q_col0 + h * 64, prob * p.Sq + qt * 128);
    issue_load(0);
  }
  mbar_wait(bar_q, 0);
  mbar_wait(&full[0], 0);
  compute_s(0);
  __syncthreads();

  float m_run = -INFINITY, l_run = 0.f;
  for (int s = 0; s < nsteps; ++s) {
    if (tid == 0 && s + 1 < nsteps) issue_load(s + 1);   // its buffer was last read by the MMAs of step s - 1
    const int j = (nt == 1) ? 0 : (s % nt);
    const bool is_p2 = (nt == 1) || (s >= nt);
    const bool do_max = (nt == 1) || (s < nt);
    const KeyTile kt = key_tile(p, prob, j, nt1);
    const RowRange rr = row_range(p, cls, tt, kt, row);
    if (do_max) {
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        uint32_t r[32];
        acc_ld32<128>(acc_s, tid, c * 32, r);
        if (cls == 1) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int cc = c * 32 + i;
            if (cc >= rr.lo && cc < rr.hi) m_run = fmaxf(m_run, __uint_as_float(r[i]));
          }
        }
      }
    }
    if (is_p2) {
      const float mb2 = (m_run == -INFINITY) ? 0.f : m_run * p.scale_log2;   // m_run is final here
#pragma unroll 1
      for (int c = 0; c < 4; ++c) {
        uint32_t r[32];
        acc_ld32<128>(acc_s, tid, c * 32, r);
        float pv[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int cc = c * 32 + i;
          float v = 0.f;
          if (cc >= rr.lo && cc < rr.hi)
            v = (cls == 1) ? ex2_approx(fmaf(__uint_as_float(r[i]), p.scale_log2, -mb2)) : 1.0f;
          pv[i] = v;
          l_run += v;
        }
        uint8_t* chunk = s_p + (c >> 1) * kTileBytes;
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          uint4 ov;
          ov.x = pack_bf16x2(pv[g * 8 + 0], pv[g * 8 + 1]); ov.y = pack_bf16x2(pv[g * 8 + 2], pv[g * 8 + 3]);
          ov.z = pack_bf16x2(pv[g * 8 + 4], pv[g * 8 + 5]); ov.w = pack_bf16x2(pv[g * 8 + 6], pv[g * 8 + 7]);
          st_sw128(chunk, tid, (c & 1) * 32 + g * 8, ov);
        }
      }
      fence_proxy_async_smem();
    }
    __syncthreads();                                     // P published, S read
    if (is_p2) issue_pv(s & 1);
    if (s + 1 < nsteps) {
      mbar_wait(&full[(s + 1) & 1], ((s + 1) >> 1) & 1);
      compute_s((s + 1) & 1);
    }
    __syncthreads();
  }

  // ---- epilogue: O / l -> bf16, LSE ----
  acc_store<64>(acc_s, 0, o[0]);
  acc_store<64>(acc_s, 64, o[1]);
  __syncthreads();
  const float inv_l = (l_run > 0.f) ? 1.0f / l_run : 0.f;
#pragma unroll 1
  for (int c = 0; c < 2; ++c) {
    uint32_t r[32];
    acc_ld32<64>(acc_s, tid, c * 32, r);
    if (row_ok) {
      bf16* dst = p.out + static_cast<long long>(prob * p.Sq + row) * p.ldo + p.o_col0 + h * 64 + c * 32;
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
    p.lse[(static_cast<long long>(prob) * p.H + h) * p.Sq + row] =
        (cls == 1 && l_run > 0.f) ? (m_run * p.scale + logf(l_run)) : 0.f;
  }
}

// ================================================================================================
// backward
// ================================================================================================
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_do,
                const __grid_constant__ CUtensorMap map_kv1, const __grid_constant__ CUtensorMap map_kv2,
                AttnParams p) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_k = smem;                      // 16 KB  K_j  [128 keys][64 d]
  uint8_t* s_v = s_k + kTileBytes;          // 16 KB  V_j
  uint8_t* s_q = s_v + kTileBytes;          // 16 KB  Q_i  [128 rows][64 d]
  uint8_t* s_do = s_q + kTileBytes;         // 16 KB  dO_i
  uint8_t* s_p = s_do + kTileBytes;         // 32 KB  P   [128 rows][128 keys] (2 chunks)
  uint8_t* s_ds = s_p + 2 * kTileBytes;     // 32 KB  dS * scale
  uint8_t* acc_s = s_ds + 2 * kTileBytes;   // 32 KB  S of one 64-key half [128][64] fp32; dQ, dV afterwards
  uint8_t* acc_dp = acc_s + 2 * kTileBytes; // 32 KB  dP of the same half; dK afterwards
  uint64_t* bars = reinterpret_cast<uint64_t*>(acc_dp + 2 * kTileBytes);
  uint64_t* bar_kv = bars;
  uint64_t* bar_qdo = bars + 1;

  const int tid = threadIdx.x;
  const int h = blockIdx.x, prob = blockIdx.y;

  if (tid == 0) {
    mbar_init(bar_kv, 1); mbar_init(bar_qdo, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();   // predecessor grid complete before any global / TMA access

  const int nt1 = (p.Sk1 + 127) / 128, nt2 = (p.Sk2 + 127) / 128, nkt = nt1 + nt2;
  const int nqt = (p.Sq + 127) / 128;
  const uint32_t a_q = smem_u32(s_q), a_k = smem_u32(s_k), a_v = smem_u32(s_v), a_do = smem_u32(s_do);
  const uint32_t a_p = smem_u32(s_p), a_ds = smem_u32(s_ds);

  uint32_t ph_kv = 0, ph_qdo = 0;
  if (tid == 0) {
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_do); tma_prefetch_desc(&map_kv1); tma_prefetch_desc(&map_kv2);
  }

  for (int j = 0; j < nkt; ++j) {
    const KeyTile kt = key_tile(p, prob, j, nt1);
    if (tid == 0) {
      const CUtensorMap* m = kt.src ? &map_kv2 : &map_kv1;
      mbar_arrive_expect_tx(bar_kv, 2 * kTileBytes);
      tma_load_2d(s_k, m, bar_kv, (kt.src ? p.k2_col0 : p.k1_col0) + h * 64, kt.row0);
      tma_load_2d(s_v, m, bar_kv, (kt.src ? p.v2_col0 : p.v1_col0) + h * 64, kt.row0);
    }
    float dv[2][32], dk[2][32];   // dV_j, dK_j: key rows [64 h, 64 h + 64)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int i = 0; i < 32; ++i) { dv[hh][i] = 0.f; dk[hh][i] = 0.f; }
    for (int i = 0; i < nqt; ++i) {
      const int row = i * 128 + tid;
      const bool row_ok = row < p.Sq;
      const long long grow = static_cast<long long>(prob) * p.Sq + row;
      if (tid == 0) {
        mbar_arrive_expect_tx(bar_qdo, 2 * kTileBytes);
        tma_load_2d(s_q, &map_q, bar_qdo, p.q_col0 + h * 64, prob * p.Sq + i * 128);
        tma_load_2d(s_do, &map_do, bar_qdo, p.do_col0 + h * 64, prob * p.Sq + i * 128);
      }
      // per-row scalars (overlaps the TMA): delta = rowsum(dO . O), lse, class
      int tt = 0;
      float delta = 0.f, lse = 0.f;
      if (row_ok) {
        if (p.text_time != nullptr) tt = p.text_time[grow];
        const uint4* po = reinterpret_cast<const uint4*>(p.o + grow * p.ldo + p.o_col0 + h * 64);
        const uint4* pd = reinterpret_cast<const uint4*>(p.dout + grow * p.ld_do + p.do_col0 + h * 64);
#pragma unroll
        for (int g = 0; g < 8; ++g) {
          const uint4 a = __ldg(po + g), b = __ldg(pd + g);
          const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y), a2 = unpack_bf16x2(a.z), a3 = unpack_bf16x2(a.w);
          const float2 b0 = unpack_bf16x2(b.x), b1 = unpack_bf16x2(b.y), b2 = unpack_bf16x2(b.z), b3 = unpack_bf16x2(b.w);
          delta += a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y + a2.x * b2.x + a2.y * b2.y + a3.x * b3.x +
                   a3.y * b3.y;
        }
        lse = p.lse[(static_cast<long long>(prob) * p.H + h) * p.Sq + row];
      }
      const int cls = row_ok ? row_class(p, tt) : 0;
      const float inv_cnt = 1.0f / static_cast<float>(p.Sk1 + p.Sk2);
      const RowRange rr = row_range(p, cls, tt, kt, row);
      const float lse_l2 = lse * 1.4426950408889634f;

      if (i == 0) mbar_wait(bar_kv, ph_kv);
      mbar_wait(bar_qdo, ph_qdo);
      ph_qdo ^= 1;

#pragma unroll 1
      for (int kh = 0; kh < 2; ++kh) {           // keys [64 kh, 64 kh + 64): S = Q K^T, dP = dO V^T
        wg_mma_tile<64, 0, 0>(
            acc_s, 4, [&](int hh, int k) { return make_smem_desc(a_q + hh * 8192 + k * 32, 16, 1024); },
            [&](int k) { return make_smem_desc(a_k + kh * 8192 + k * 32, 16, 1024); });
        wg_mma_tile<64, 0, 0>(
            acc_dp, 4, [&](int hh, int k) { return make_smem_desc(a_do + hh * 8192 + k * 32, 16, 1024); },
            [&](int k) { return make_smem_desc(a_v + kh * 8192 + k * 32, 16, 1024); });
        __syncthreads();
#pragma unroll 1
        for (int c2 = 0; c2 < 2; ++c2) {
          const int c = kh * 2 + c2;
          uint32_t rs[32], rp[32];
          acc_ld32<64>(acc_s, tid, c2 * 32, rs);
          acc_ld32<64>(acc_dp, tid, c2 * 32, rp);
          uint8_t* pchunk = s_p + kh * kTileBytes;
          uint8_t* dchunk = s_ds + kh * kTileBytes;
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            float pv[8], dsv[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int cc = c * 32 + g * 8 + e;
              float pr = 0.f, ds = 0.f;
              if (cc >= rr.lo && cc < rr.hi) {
                if (cls == 1) {
                  pr = ex2_approx(fmaf(__uint_as_float(rs[g * 8 + e]), p.scale_log2, -lse_l2));
                  ds = pr * (__uint_as_float(rp[g * 8 + e]) - delta) * p.scale;
                } else {
                  pr = inv_cnt;
                }
              }
              pv[e] = pr; dsv[e] = ds;
            }
            uint4 o;
            o.x = pack_bf16x2(pv[0], pv[1]); o.y = pack_bf16x2(pv[2], pv[3]);
            o.z = pack_bf16x2(pv[4], pv[5]); o.w = pack_bf16x2(pv[6], pv[7]);
            st_sw128(pchunk, tid, c2 * 32 + g * 8, o);
            o.x = pack_bf16x2(dsv[0], dsv[1]); o.y = pack_bf16x2(dsv[2], dsv[3]);
            o.z = pack_bf16x2(dsv[4], dsv[5]); o.w = pack_bf16x2(dsv[6], dsv[7]);
            st_sw128(dchunk, tid, c2 * 32 + g * 8, o);
          }
        }
        __syncthreads();                          // acc_s / acc_dp read before the next half overwrites them
      }
      fence_proxy_async_smem();
      __syncthreads();

      // dV += P^T dO ; dK += dS^T Q      A MN-major: key half hh = chunk hh, k-step = 16 q rows; B MN-major
      wg_mma_regs<64, 1, 1>(
          dv, i > 0, 8, [&](int hh, int k) { return make_smem_desc(a_p + hh * kTileBytes + k * 2048, kTileBytes, 1024); },
          [&](int k) { return make_smem_desc(a_do + k * 2048, 16, 1024); });
      wg_mma_regs<64, 1, 1>(
          dk, i > 0, 8, [&](int hh, int k) { return make_smem_desc(a_ds + hh * kTileBytes + k * 2048, kTileBytes, 1024); },
          [&](int k) { return make_smem_desc(a_q + k * 2048, 16, 1024); });
      // dQ = dS K   A K-major over keys (2 chunks), B = K_j MN-major
      wg_mma_tile<64, 0, 1>(
          acc_s, 8,
          [&](int hh, int k) { return make_smem_desc(a_ds + (k >> 2) * kTileBytes + hh * 8192 + (k & 3) * 32, 16, 1024); },
          [&](int k) { return make_smem_desc(a_k + k * 2048, 16, 1024); });
      __syncthreads();

      // dQ tile: accumulate across key tiles through the fp32 workspace (same thread owns the same row)
#pragma unroll 1
      for (int c = 0; c < 2; ++c) {
        uint32_t r[32];
        acc_ld32<64>(acc_s, tid, c * 32, r);
        if (row_ok) {
          float v[32];
#pragma unroll
          for (int e = 0; e < 32; ++e) v[e] = __uint_as_float(r[e]);
          float* ws = (nkt > 1) ? p.dq_ws + grow * (p.H * 64) + h * 64 + c * 32 : nullptr;
          if (j > 0) {
#pragma unroll
            for (int e = 0; e < 32; e += 4) {
              const float4 w = *reinterpret_cast<const float4*>(ws + e);
              v[e] += w.x; v[e + 1] += w.y; v[e + 2] += w.z; v[e + 3] += w.w;
            }
          }
          if (j == nkt - 1) {
            bf16* dst = p.dq + grow * p.ld_dq + p.dq_col0 + h * 64 + c * 32;
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

    // dV_j, dK_j complete: row t of the tiles = key t of this tile
    acc_store<64>(acc_s, 0, dv[0]); acc_store<64>(acc_s, 64, dv[1]);
    acc_store<64>(acc_dp, 0, dk[0]); acc_store<64>(acc_dp, 64, dk[1]);
    __syncthreads();
    {
      const bool key_ok = tid < kt.valid;
      bf16* base = kt.src ? p.dkv2 : p.dkv1;
      const long long ld = kt.src ? p.ld_dkv2 : p.ld_dkv1;
      const int dkc = kt.src ? p.dk2_col0 : p.dk1_col0, dvc = kt.src ? p.dv2_col0 : p.dv1_col0;
#pragma unroll 1
      for (int w = 0; w < 2; ++w) {      // 0: dV, 1: dK
        uint8_t* src = w ? acc_dp : acc_s;
#pragma unroll 1
        for (int c = 0; c < 2; ++c) {
          uint32_t r[32];
          acc_ld32<64>(src, tid, c * 32, r);
          if (key_ok) {
            bf16* dst = base + static_cast<long long>(kt.row0 + tid) * ld + (w ? dkc : dvc) + h * 64 + c * 32;
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

constexpr int kAttnFwdSmem = 11 * kTileBytes + 1024 + 128;
constexpr int kAttnBwdSmem = 12 * kTileBytes + 1024 + 128;

}  // namespace otb

using namespace otb;

static int check_common(const otb_attn_desc* d) {
  OTB_CHECK_ARG(d != nullptr, "otb_attn: null descriptor");
  OTB_CHECK_ARG(d->P > 0 && d->H > 0 && d->Sq > 0 && d->Sk1 > 0 && d->Sk2 >= 0, "otb_attn: bad sizes");
  OTB_CHECK_ARG(d->head_dim == 64, "otb_attn: head_dim must be 64 (Otter/CLIP-L: 64)");
  OTB_CHECK_ARG(d->q && d->kv1 && (d->Sk2 == 0 || d->kv2), "otb_attn: null tensor");
  OTB_CHECK_ARG(d->text_time == nullptr || (d->Sk2 == 0 && d->n_per_media > 0 && d->T_img * d->n_per_media == d->Sk1),
                "otb_attn: media mask needs a single key source with Sk1 == T_img * n_per_media");
  OTB_CHECK_ARG(!d->causal || (d->Sk2 == 0 && d->Sq == d->Sk1 && d->text_time == nullptr),
                "otb_attn: causal needs self-attention (Sq == Sk1, one key source, no media mask)");
  return OTB_OK;
}

static void fill_params(const otb_attn_desc* d, AttnParams& p) {
  p.P = d->P; p.H = d->H; p.Sq = d->Sq; p.Sk1 = d->Sk1; p.Sk2 = d->Sk2;
  p.q_col0 = d->q_col0; p.k1_col0 = d->k1_col0; p.v1_col0 = d->v1_col0; p.k2_col0 = d->k2_col0; p.v2_col0 = d->v2_col0;
  p.scale = d->scale; p.scale_log2 = d->scale * 1.4426950408889634f;
  p.out = static_cast<bf16*>(d->out); p.ldo = d->ld_out; p.o_col0 = d->out_col0;
  p.lse = d->lse;
  p.text_time = d->text_time; p.n_per_media = d->n_per_media; p.T_img = d->T_img;
  p.mask_ge = d->mask_ge; p.causal = d->causal;
  p.o = static_cast<const bf16*>(d->out);
  p.dout = nullptr; p.dq = nullptr; p.dkv1 = nullptr; p.dkv2 = nullptr; p.dq_ws = nullptr;
  p.ld_do = p.ld_dq = p.ld_dkv1 = p.ld_dkv2 = 0;
  p.do_col0 = p.dq_col0 = p.dk1_col0 = p.dv1_col0 = p.dk2_col0 = p.dv2_col0 = 0;
}

extern "C" int otb_attn_fwd(const otb_attn_desc* d, void* stream) {
  int rc = check_common(d);
  if (rc) return rc;
  OTB_CHECK_ARG(d->out != nullptr, "otb_attn_fwd: null out");
  AttnParams p;
  fill_params(d, p);
  CUtensorMap mq, mk1, mk2;
  rc = make_tmap_bf16_2d(&mq, d->q, (uint64_t)d->P * d->Sq, d->q_cols, d->ldq, 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&mk1, d->kv1, (uint64_t)d->P * d->Sk1, d->kv1_cols, d->ldkv1, 128, 64);
  if (rc) return rc;
  if (d->Sk2 > 0) rc = make_tmap_bf16_2d(&mk2, d->kv2, (uint64_t)d->P * d->Sk2, d->kv2_cols, d->ldkv2, 128, 64);
  else mk2 = mk1;
  if (rc) return rc;
  dim3 grid((d->Sq + 127) / 128, d->H, d->P);
  OTB_CHECK_CUDA(ensure_dyn_smem(attn_fwd_kernel, kAttnFwdSmem));
  OTB_CHECK_CUDA(launch_k(attn_fwd_kernel, grid, dim3(kAttnThreads), kAttnFwdSmem, static_cast<cudaStream_t>(stream), mq,
                          mk1, mk2, p));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_attn_bwd(const otb_attn_desc* d, const otb_attn_grads* g, void* stream) {
  int rc = check_common(d);
  if (rc) return rc;
  OTB_CHECK_ARG(g && d->out && d->lse && g->dout && g->dq && g->dkv1 && (d->Sk2 == 0 || g->dkv2),
                "otb_attn_bwd: null tensor");
  const int nkt = (d->Sk1 + 127) / 128 + (d->Sk2 + 127) / 128;
  OTB_CHECK_ARG(nkt == 1 || g->dq_ws != nullptr, "otb_attn_bwd: dq workspace required for >1 key tile");
  AttnParams p;
  fill_params(d, p);
  p.dout = static_cast<const bf16*>(g->dout); p.ld_do = g->ld_dout; p.do_col0 = g->dout_col0;
  p.dq = static_cast<bf16*>(g->dq); p.ld_dq = g->ld_dq; p.dq_col0 = g->dq_col0;
  p.dkv1 = static_cast<bf16*>(g->dkv1); p.ld_dkv1 = g->ld_dkv1; p.dk1_col0 = g->dk1_col0; p.dv1_col0 = g->dv1_col0;
  p.dkv2 = static_cast<bf16*>(g->dkv2); p.ld_dkv2 = g->ld_dkv2; p.dk2_col0 = g->dk2_col0; p.dv2_col0 = g->dv2_col0;
  p.dq_ws = g->dq_ws;
  CUtensorMap mq, mdo, mk1, mk2;
  rc = make_tmap_bf16_2d(&mq, d->q, (uint64_t)d->P * d->Sq, d->q_cols, d->ldq, 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&mdo, g->dout, (uint64_t)d->P * d->Sq, g->dout_cols, g->ld_dout, 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&mk1, d->kv1, (uint64_t)d->P * d->Sk1, d->kv1_cols, d->ldkv1, 128, 64);
  if (rc) return rc;
  if (d->Sk2 > 0) rc = make_tmap_bf16_2d(&mk2, d->kv2, (uint64_t)d->P * d->Sk2, d->kv2_cols, d->ldkv2, 128, 64);
  else mk2 = mk1;
  if (rc) return rc;
  OTB_CHECK_CUDA(ensure_dyn_smem(attn_bwd_kernel, kAttnBwdSmem));
  dim3 grid(d->H, d->P);
  OTB_CHECK_CUDA(launch_k(attn_bwd_kernel, dim3(grid), dim3(kAttnThreads), kAttnBwdSmem, static_cast<cudaStream_t>(stream), mq, mdo, mk1, mk2, p));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
