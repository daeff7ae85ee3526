// otter_b200 — the north star's literal kernel: gated cross-attention core + output projection + tanh gate + residual
// in ONE kernel (SURVEY.md §7 option (a); reference modeling_otter.py:290-340 and :380-389):
//
//     x1 = ( softmax(mask(Q K^T / 8)) V  Wo^T ) * tanh(attn_gate) + x
//
// The unfused path writes the attention output O [B*L, 512] to HBM, and a second launch (the to_out GEMM with the
// gate + residual epilogue) reads it back.  Here a CTA (one warpgroup) owns 128 text rows x 512 output columns:
//   phase 1  for each of the 8 heads: S = Q_h K_h^T (wgmma, keys = one 64-row tile: T_img * n <= 64, the training
//            layout T = 1) through a fp32 smem tile, media-masked softmax with thread t owning row t, P -> smem,
//            O_h = P V_h in registers, O_h / l -> bf16 into a 128B-swizzled smem tile that is directly the K-major A
//            operand of phase 2 (O never travels to HBM on the way to the projection; the CTAs of output-column block 0
//            also store O and the LSE for the backward pass).  Q_h+1 / K_h+1 / V_h+1 load while O_h is written out.
//   phase 2  Y[128 x 512] = O[128 x 512] Wo[n0 : n0+512, :]^T — four 128-column chunks of 8 k-blocks each through a
//            2-stage TMA ring that reuses the phase-1 buffers; accumulators in registers, parked in a fp32 tile for
//            the row-wise epilogue: the pre-gate branch output a1 (kept for the gate gradient), then
//            y = a1 * tanh(g) + x, both written once.
// The attention is recomputed by the D/512 CTAs that share a row tile (16 MFLOP against the 67 MFLOP of the
// projection slice; Q/K/V come from L2).
#include "otb_attn_common.cuh"
#include "otb_host.h"

namespace otb {

constexpr int kXfThreads = 128;
constexpr int kXfCols = 512;                 // output columns per CTA
constexpr int kXfChunk = 128;                // output columns per phase-2 accumulator
constexpr int kXfStageBytes = kXfChunk * 128;  // one Wo tile: 128 output rows x 64 k (bf16) = 16 KB

struct XFusedParams {
  AttnParams a;                              // attention problem (one key source, Sk1 <= 64); a.out = O, a.lse
  const float* gate;                         // attn_gate, device scalar
  const bf16* residual; long long ld_res;    // x   [B*L][D]
  bf16* aux; long long ld_aux;               // a1  [B*L][D]   pre-gate branch output (may be null)
  bf16* y; long long ld_y;                   // x1  [B*L][D]
  int D;
};

__global__ void __launch_bounds__(kXfThreads, 1)
xattn_out_fused_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_kv,
                       const __grid_constant__ CUtensorMap map_w, XFusedParams fp) {
  const AttnParams& p = fp.a;
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // phase 1 (80 KB of the 96 KB work area)
  uint8_t* s_q = smem;                              // 16 KB   Q_h  [128 rows][64]
  uint8_t* s_k = s_q + kTileBytes;                  //  8 KB   K_h  [64 keys][64]
  uint8_t* s_v = s_k + kTileBytes / 2;              //  8 KB   V_h
  uint8_t* s_p = s_v + kTileBytes / 2;              // 16 KB   P    [128 rows][64 keys]
  uint8_t* acc_s = s_p + kTileBytes;                // 32 KB   S / O_h [128][64] fp32
  // phase 2 (the same 96 KB)
  uint8_t* s_w = smem;                              // 2 x 16 KB Wo stages
  uint8_t* acc_y = smem + 2 * kTileBytes;           // 64 KB   Y chunk [128][128] fp32
  uint8_t* s_o = smem + 6 * kTileBytes;             // 8 x 16 KB   O_h tiles = A operand of the projection
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_o + 8 * kTileBytes);
  uint64_t* in_full = bars;           // Q_h, K_h, V_h landed
  uint64_t* w_full = bars + 1;        // [2]

  const int tid = threadIdx.x;
  const int n0 = blockIdx.x * kXfCols, qt = blockIdx.y, prob = blockIdx.z;
  const int H = p.H;

  if (tid == 0) {
    mbar_init(in_full, 1); mbar_init(&w_full[0], 1); mbar_init(&w_full[1], 1);
    fence_mbar_init();
    tma_prefetch_desc(&map_q); tma_prefetch_desc(&map_kv); tma_prefetch_desc(&map_w);
  }
  __syncthreads();
  pdl_wait();

  auto load_head = [&](int h) {   // thread 0
    mbar_arrive_expect_tx(in_full, 2 * kTileBytes);
    tma_load_2d(s_q, &map_q, in_full, p.q_col0 + h * 64, prob * p.Sq + qt * 128);
    tma_load_2d(s_k, &map_kv, in_full, p.k1_col0 + h * 64, prob * p.Sk1);
    tma_load_2d(s_v, &map_kv, in_full, p.v1_col0 + h * 64, prob * p.Sk1);
  };
  if (tid == 0) load_head(0);

  const int row = qt * 128 + tid;
  const bool row_ok = row < p.Sq;
  const long long grow = static_cast<long long>(prob) * p.Sq + row;
  int tt = 0;
  if (p.text_time != nullptr && row_ok) tt = p.text_time[grow];
  const int cls = row_ok ? row_class(p, tt) : 0;
  KeyTile kt;
  kt.src = 0; kt.row0 = prob * p.Sk1; kt.valid = p.Sk1; kt.key_base = 0;
  const RowRange rr = row_range(p, cls, tt, kt, row);
  const bool store_o = (blockIdx.x == 0);
  const int nch = ((p.Sk1 + 15) & ~15) >> 4;       // 16-key chunks holding a valid key
  const uint32_t a_q = smem_u32(s_q), a_k = smem_u32(s_k), a_v = smem_u32(s_v), a_p = smem_u32(s_p);

  for (int h = 0; h < H; ++h) {
    mbar_wait(in_full, h & 1);
    // S = Q_h K_h^T: [128 rows][64 keys] (keys >= Sk1 belong to the next problem or are zero-filled: masked below)
    wg_mma_tile<64, 0, 0>(
        acc_s, 4, [&](int hh, int k) { return make_smem_desc(a_q + hh * 8192 + k * 32, 16, 1024); },
        [&](int k) { return make_smem_desc(a_k + k * 32, 16, 1024); });
    __syncthreads();
    // ---- sweep 1: row max ----
    float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    if (cls == 1) {
      for (int c = 0; c < nch; ++c) {
        uint32_t r[16];
        acc_ld16<64>(acc_s, tid, c * 16, r);
#pragma unroll
        for (int i = 0; i < 16; ++i)
          if (c * 16 + i >= rr.lo && c * 16 + i < rr.hi) mx[i & 3] = fmaxf(mx[i & 3], __uint_as_float(r[i]));
      }
    }
    const float m_run = fmaxf(fmaxf(mx[0], mx[1]), fmaxf(mx[2], mx[3]));
    // ---- sweep 2: P (every 16-key chunk is written: chunks past the valid keys hold zeros) ----
    float ls[4] = {0.f, 0.f, 0.f, 0.f};
    const float mb = (m_run == -INFINITY) ? 0.f : m_run * p.scale_log2;
#pragma unroll 1
    for (int c = 0; c < 4; ++c) {
      uint32_t r[16];
      acc_ld16<64>(acc_s, tid, c * 16, r);
      float pv[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        float v = 0.f;
        if (c * 16 + i >= rr.lo && c * 16 + i < rr.hi)
          v = (cls == 1) ? ex2_approx(fmaf(__uint_as_float(r[i]), p.scale_log2, -mb)) : 1.0f;
        pv[i] = v;
        ls[i & 3] += v;
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        uint4 o;
        o.x = pack_bf16x2(pv[u * 8 + 0], pv[u * 8 + 1]); o.y = pack_bf16x2(pv[u * 8 + 2], pv[u * 8 + 3]);
        o.z = pack_bf16x2(pv[u * 8 + 4], pv[u * 8 + 5]); o.w = pack_bf16x2(pv[u * 8 + 6], pv[u * 8 + 7]);
        st_sw128(s_p, tid, c * 16 + u * 8, o);
      }
    }
    const float l_run = (ls[0] + ls[1]) + (ls[2] + ls[3]);
    fence_proxy_async_smem();
    __syncthreads();
    // O_h = P V_h   (A = P K-major over the 64 keys, B = V MN-major)
    float o[2][32];
    wg_mma_regs<64, 0, 1>(
        o, false, 4, [&](int hh, int k) { return make_smem_desc(a_p + hh * 8192 + k * 32, 16, 1024); },
        [&](int k) { return make_smem_desc(a_v + k * 2048, 16, 1024); });
    acc_store<64>(acc_s, 0, o[0]);
    acc_store<64>(acc_s, 64, o[1]);
    __syncthreads();                                  // Q_h / K_h / V_h are dead, O_h is in acc_s
    if (tid == 0 && h + 1 < H) load_head(h + 1);
    // O_h / l -> bf16: into the smem tile that phase 2 consumes, and (column block 0) to HBM for the backward pass
    {
      const float inv_l = (l_run > 0.f) ? 1.0f / l_run : 0.f;
      uint8_t* tile = s_o + h * kTileBytes;
      bf16* dst = p.out + grow * p.ldo + p.o_col0 + h * 64;
#pragma unroll 1
      for (int c = 0; c < 2; ++c) {
        uint32_t r[32];
        acc_ld32<64>(acc_s, tid, c * 32, r);
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
          uint4 o4;
          o4.x = pack_bf16x2(__uint_as_float(r[g4 * 8 + 0]) * inv_l, __uint_as_float(r[g4 * 8 + 1]) * inv_l);
          o4.y = pack_bf16x2(__uint_as_float(r[g4 * 8 + 2]) * inv_l, __uint_as_float(r[g4 * 8 + 3]) * inv_l);
          o4.z = pack_bf16x2(__uint_as_float(r[g4 * 8 + 4]) * inv_l, __uint_as_float(r[g4 * 8 + 5]) * inv_l);
          o4.w = pack_bf16x2(__uint_as_float(r[g4 * 8 + 6]) * inv_l, __uint_as_float(r[g4 * 8 + 7]) * inv_l);
          if (!row_ok) o4 = make_uint4(0u, 0u, 0u, 0u);
          st_sw128(tile, tid, c * 32 + g4 * 8, o4);
          if (store_o && row_ok) *reinterpret_cast<uint4*>(dst + c * 32 + g4 * 8) = o4;
        }
      }
      if (store_o && row_ok && p.lse != nullptr)
        p.lse[(static_cast<long long>(prob) * p.H + h) * p.Sq + row] =
            (cls == 1 && l_run > 0.f) ? (m_run * p.scale + logf(l_run)) : 0.f;
    }
    __syncthreads();                                  // acc_s is read before S_h+1 overwrites it
  }
  fence_proxy_async_smem();                           // the O tiles (generic-proxy stores) feed wgmma next
  __syncthreads();

  // ---- phase 2: Y = O Wo^T, 128 columns at a time; a1 = acc, y = a1 * tanh(g) + x ----
  const int nkb = H;                                  // 64-wide k-blocks of O (one per head)
  const int nw = (kXfCols / kXfChunk) * nkb;
  auto load_w = [&](int i) {                          // thread 0
    const int c = i / nkb, kb = i % nkb, st = i & 1;
    mbar_arrive_expect_tx(&w_full[st], kXfStageBytes);
    tma_load_2d(s_w + st * kXfStageBytes, &map_w, &w_full[st], kb * 64, n0 + c * kXfChunk);
  };
  if (tid == 0) { load_w(0); if (nw > 1) load_w(1); }
  const float gt = tanhf(__ldg(fp.gate));
  const uint32_t a_o = smem_u32(s_o), a_w = smem_u32(s_w);
  float y[2][64];
  for (int i = 0; i < nw; ++i) {
    const int c = i / nkb, kb = i % nkb, st = i & 1;
    mbar_wait(&w_full[st], (i >> 1) & 1);
    wg_mma_regs<128, 0, 0>(
        y, kb > 0, 4, [&](int hh, int k) { return make_smem_desc(a_o + kb * kTileBytes + hh * 8192 + k * 32, 16, 1024); },
        [&](int k) { return make_smem_desc(a_w + st * kXfStageBytes + k * 32, 16, 1024); });
    if (tid == 0 && i + 2 < nw) load_w(i + 2);       // the MMAs that read this stage have retired
    if (kb != nkb - 1) continue;
    acc_store<128>(acc_y, 0, y[0]);
    acc_store<128>(acc_y, 64, y[1]);
    __syncthreads();
#pragma unroll 1
    for (int ch = 0; ch < kXfChunk / 32; ++ch) {
      const int col = n0 + c * kXfChunk + ch * 32;
      uint4 res[4];
      if (row_ok) {
        const uint4* pr = reinterpret_cast<const uint4*>(fp.residual + grow * fp.ld_res + col);
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) res[g4] = __ldg(pr + g4);
      }
      uint32_t r[32];
      acc_ld32<128>(acc_y, tid, ch * 32, r);
      if (row_ok) {
#pragma unroll
        for (int g4 = 0; g4 < 4; ++g4) {
          float v[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = __uint_as_float(r[g4 * 8 + e]);
          if (fp.aux != nullptr) {
            uint4 a;
            a.x = pack_bf16x2(v[0], v[1]); a.y = pack_bf16x2(v[2], v[3]);
            a.z = pack_bf16x2(v[4], v[5]); a.w = pack_bf16x2(v[6], v[7]);
            *reinterpret_cast<uint4*>(fp.aux + grow * fp.ld_aux + col + g4 * 8) = a;
          }
          const float2 x0 = unpack_bf16x2(res[g4].x), x1 = unpack_bf16x2(res[g4].y), x2 = unpack_bf16x2(res[g4].z),
                       x3 = unpack_bf16x2(res[g4].w);
          uint4 o;
          o.x = pack_bf16x2(v[0] * gt + x0.x, v[1] * gt + x0.y); o.y = pack_bf16x2(v[2] * gt + x1.x, v[3] * gt + x1.y);
          o.z = pack_bf16x2(v[4] * gt + x2.x, v[5] * gt + x2.y); o.w = pack_bf16x2(v[6] * gt + x3.x, v[7] * gt + x3.y);
          *reinterpret_cast<uint4*>(fp.y + grow * fp.ld_y + col + g4 * 8) = o;
        }
      }
    }
    __syncthreads();                                  // acc_y is read before the next chunk overwrites it
  }
}

constexpr int kXfSmem = 14 * kTileBytes + 1024 + 128;

}  // namespace otb

using namespace otb;

extern "C" int otb_xattn_out_fused(const otb_attn_desc* d, const void* wo, int64_t ld_wo, const float* gate,
                                   const void* residual, int64_t ld_res, void* aux, int64_t ld_aux, void* y, int64_t ld_y,
                                   int D, void* stream) {
  OTB_CHECK_ARG(d && wo && gate && residual && y, "otb_xattn_out_fused: null pointer");
  OTB_CHECK_ARG(d->P > 0 && d->H > 0 && d->H <= 8 && d->Sq > 0 && d->head_dim == 64, "otb_xattn_out_fused: bad sizes");
  OTB_CHECK_ARG(d->Sk2 == 0 && d->Sk1 > 0 && d->Sk1 <= 64,
                "otb_xattn_out_fused: one key source with at most 64 keys (T_img * n <= 64); use otb_attn_fwd + otb_gemm_bf16");
  OTB_CHECK_ARG(!d->causal && d->q && d->kv1 && d->out, "otb_xattn_out_fused: bad attention descriptor");
  OTB_CHECK_ARG(d->text_time == nullptr || (d->n_per_media > 0 && d->T_img * d->n_per_media == d->Sk1),
                "otb_xattn_out_fused: media mask needs Sk1 == T_img * n_per_media");
  OTB_CHECK_ARG(D > 0 && D % kXfCols == 0, "otb_xattn_out_fused: D must be a multiple of 512");
  OTB_CHECK_ARG(ld_res >= D && ld_y >= D && (aux == nullptr || ld_aux >= D) && ld_res % 8 == 0 && ld_y % 8 == 0 &&
                    ld_aux % 8 == 0 && ld_wo >= d->H * 64, "otb_xattn_out_fused: bad row pitch");
  XFusedParams fp;
  AttnParams& p = fp.a;
  p.P = d->P; p.H = d->H; p.Sq = d->Sq; p.Sk1 = d->Sk1; p.Sk2 = 0;
  p.q_col0 = d->q_col0; p.k1_col0 = d->k1_col0; p.v1_col0 = d->v1_col0; p.k2_col0 = 0; p.v2_col0 = 0;
  p.scale = d->scale; p.scale_log2 = d->scale * 1.4426950408889634f;
  p.out = static_cast<bf16*>(d->out); p.ldo = d->ld_out; p.o_col0 = d->out_col0; p.lse = d->lse;
  p.text_time = d->text_time; p.n_per_media = d->n_per_media; p.T_img = d->T_img; p.mask_ge = d->mask_ge; p.causal = 0;
  p.o = nullptr; p.dout = nullptr; p.dq = nullptr; p.dkv1 = nullptr; p.dkv2 = nullptr; p.dq_ws = nullptr;
  p.ld_do = p.ld_dq = p.ld_dkv1 = p.ld_dkv2 = 0;
  p.do_col0 = p.dq_col0 = p.dk1_col0 = p.dv1_col0 = p.dk2_col0 = p.dv2_col0 = 0;
  fp.gate = gate;
  fp.residual = static_cast<const bf16*>(residual); fp.ld_res = ld_res;
  fp.aux = static_cast<bf16*>(aux); fp.ld_aux = ld_aux;
  fp.y = static_cast<bf16*>(y); fp.ld_y = ld_y;
  fp.D = D;
  CUtensorMap mq, mkv, mw;
  int rc = make_tmap_bf16_2d(&mq, d->q, (uint64_t)d->P * d->Sq, d->q_cols, d->ldq, 128, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&mkv, d->kv1, (uint64_t)d->P * d->Sk1, d->kv1_cols, d->ldkv1, 64, 64);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&mw, wo, (uint64_t)D, (uint64_t)d->H * 64, ld_wo, kXfChunk, 64);
  if (rc) return rc;
  OTB_CHECK_CUDA(ensure_dyn_smem(xattn_out_fused_kernel, kXfSmem));
  dim3 grid(D / kXfCols, (d->Sq + 127) / 128, d->P);
  OTB_CHECK_CUDA(launch_k(xattn_out_fused_kernel, grid, dim3(kXfThreads), kXfSmem, static_cast<cudaStream_t>(stream), mq,
                          mkv, mw, fp));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
