// otter_b200 — Persimmon / Fuyu decoder-layer specific kernels (SURVEY.md §8f rank 3).
//
// The reference's PersimmonAttention (src/otter_ai/models/fuyu/modeling_persimmon.py:266-319) takes the fused
// query_key_value output [rows][heads][3][64], applies a LayerNorm over the 64 head dims to q and to k
// (q_layernorm / k_layernorm, :283-285, flash-attn's fused_layer_norm), rotates the first `rot` dims of q and k
// (partial rotary, non-interleaved / rotate_half convention, :287-303, fused_apply_rotary_emb) and hands q, k, v to
// flash_attn_func(causal=True).  Here one kernel does split + qk-LayerNorm + partial RoPE and writes q | k | v as
// three head-major column blocks [rows][3 * heads * 64] — the layout the fused attention kernel reads in place —
// and one kernel is its backward (un-rotate, LayerNorm backward, re-interleave) with a deterministic two-stage
// reduction for the four [64] affine-parameter gradients.  One warp per (row, head); lane l owns dims 2l, 2l+1.
#include <algorithm>

#include "otb_common.cuh"
#include "otb_host.h"

namespace otb {

constexpr int kQkBlock = 256;            // 8 warps
constexpr int kQkMaxBlocks = 592;        // 4 per SM: partial [blocks][4][64] rows of the parameter-gradient reduction

// cos / sin of the rotary angle for rotary dim index i (0 <= i < rot): angle = pos * theta^(-2 (i mod rot/2) / rot)
__device__ __forceinline__ void rope_cs(int pos, int i, int rot, float log2_theta, float& c, float& s) {
  const int half = rot >> 1;
  const float inv_freq = exp2f(-log2_theta * static_cast<float>(2 * (i % half)) / static_cast<float>(rot));
  sincosf(static_cast<float>(pos) * inv_freq, &s, &c);
}

// forward: fused [rows][H][3][64] -> qkv [rows][3*H*64] (q | k | v blocks), stats [rows][H][4] = mean_q, rstd_q, mean_k, rstd_k
__global__ void __launch_bounds__(kQkBlock)
qkln_rope_fwd_kernel(const bf16* __restrict__ fused, long long ld_fused, const float* __restrict__ qg,
                     const float* __restrict__ qb, const float* __restrict__ kg, const float* __restrict__ kb,
                     bf16* __restrict__ qkv, long long ld_qkv, float* __restrict__ stats, long long rows, int H, int S,
                     int rot, float log2_theta, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * kQkBlock + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * kQkBlock) >> 5;
  const int d0 = 2 * lane;
  const float2 gq = make_float2(qg[d0], qg[d0 + 1]), bq = make_float2(qb[d0], qb[d0 + 1]);
  const float2 gk = make_float2(kg[d0], kg[d0 + 1]), bk = make_float2(kb[d0], kb[d0 + 1]);
  const int hr = rot >> 1;                         // rotate_half pairs dim i with i + rot/2
  for (long long item = warp0; item < rows * H; item += nwarps) {
    const long long row = item / H;
    const int h = static_cast<int>(item % H);
    const int pos = static_cast<int>(row % S);
    const bf16* src = fused + row * ld_fused + static_cast<long long>(h) * 192;
    const float2 q = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(src + d0));
    const float2 k = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(src + 64 + d0));
    const uint32_t v = *reinterpret_cast<const uint32_t*>(src + 128 + d0);
    float y[2][2];
    float st[4];
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      const float2 x = w ? k : q;
      const float mean = warp_sum(x.x + x.y) * (1.0f / 64.0f);
      const float dx = x.x - mean, dy = x.y - mean;
      const float var = warp_sum(dx * dx + dy * dy) * (1.0f / 64.0f);
      const float rstd = rsqrtf(var + eps);
      const float2 g = w ? gk : gq, b = w ? bk : bq;
      y[w][0] = dx * rstd * g.x + b.x;
      y[w][1] = dy * rstd * g.y + b.y;
      st[2 * w] = mean; st[2 * w + 1] = rstd;
    }
    // partial rotary on dims [0, rot): lanes owning dims < rot/2 pair with the lane hr/2 further on
    const int pl = hr >> 1;                                       // lanes per half (rot = 32: 8)
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      const float o0 = __shfl_xor_sync(0xffffffffu, y[w][0], pl);
      const float o1 = __shfl_xor_sync(0xffffffffu, y[w][1], pl);
      if (d0 < rot) {
        float c0, s0, c1, s1;
        rope_cs(pos, d0, rot, log2_theta, c0, s0);
        rope_cs(pos, d0 + 1, rot, log2_theta, c1, s1);
        const float sign = (d0 < hr) ? -1.0f : 1.0f;              // rotate_half: first half gets -x2, second half +x1
        y[w][0] = y[w][0] * c0 + sign * o0 * s0;
        y[w][1] = y[w][1] * c1 + sign * o1 * s1;
      }
    }
    bf16* dst = qkv + row * ld_qkv + static_cast<long long>(h) * 64 + d0;
    const long long blk = static_cast<long long>(H) * 64;
    *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(y[0][0], y[0][1]);
    *reinterpret_cast<uint32_t*>(dst + blk) = pack_bf16x2(y[1][0], y[1][1]);
    *reinterpret_cast<uint32_t*>(dst + 2 * blk) = v;
    if (lane < 4 && stats != nullptr)
      stats[item * 4 + lane] = (lane == 0) ? st[0] : (lane == 1) ? st[1] : (lane == 2) ? st[2] : st[3];
  }
}

// backward: dqkv [rows][3*H*64] -> dfused [rows][H][3][64]; partial parameter gradients ws [gridDim.x][4][64]
// (dgamma_q, dbeta_q, dgamma_k, dbeta_k)
__global__ void __launch_bounds__(kQkBlock)
qkln_rope_bwd_kernel(const bf16* __restrict__ dqkv, long long ld_dqkv, const bf16* __restrict__ fused,
                     long long ld_fused, const float* __restrict__ stats, const float* __restrict__ qg,
                     const float* __restrict__ kg, bf16* __restrict__ dfused, long long ld_dfused,
                     float* __restrict__ ws, long long rows, int H, int S, int rot, float log2_theta) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[kQkBlock / 32][4][64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long warp0 = (static_cast<long long>(blockIdx.x) * kQkBlock + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * kQkBlock) >> 5;
  const int d0 = 2 * lane, hr = rot >> 1, pl = hr >> 1;
  const float2 g2[2] = {make_float2(qg[d0], qg[d0 + 1]), make_float2(kg[d0], kg[d0 + 1])};
  float acc[2][2][2] = {};                         // [q/k][gamma/beta][elem]
  const long long blk = static_cast<long long>(H) * 64;
  for (long long item = warp0; item < rows * H; item += nwarps) {
    const long long row = item / H;
    const int h = static_cast<int>(item % H);
    const int pos = static_cast<int>(row % S);
    const bf16* gsrc = dqkv + row * ld_dqkv + static_cast<long long>(h) * 64 + d0;
    const bf16* xsrc = fused + row * ld_fused + static_cast<long long>(h) * 192;
    bf16* dst = dfused + row * ld_dfused + static_cast<long long>(h) * 192;
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      float2 dy = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(gsrc + w * blk));
      // transpose of the rotation: dx_i = dy_i cos_i + dy_{i+hr} sin_i ; dx_{i+hr} = dy_{i+hr} cos_i - dy_i sin_i
      const float o0 = __shfl_xor_sync(0xffffffffu, dy.x, pl);
      const float o1 = __shfl_xor_sync(0xffffffffu, dy.y, pl);
      if (d0 < rot) {
        float c0, s0, c1, s1;
        rope_cs(pos, d0, rot, log2_theta, c0, s0);
        rope_cs(pos, d0 + 1, rot, log2_theta, c1, s1);
        const float sign = (d0 < hr) ? 1.0f : -1.0f;
        dy.x = dy.x * c0 + sign * o0 * s0;
        dy.y = dy.y * c1 + sign * o1 * s1;
      }
      const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(xsrc + w * 64 + d0));
      const float mean = stats[item * 4 + 2 * w], rstd = stats[item * 4 + 2 * w + 1];
      const float xh0 = (x.x - mean) * rstd, xh1 = (x.y - mean) * rstd;
      acc[w][0][0] += dy.x * xh0; acc[w][0][1] += dy.y * xh1;
      acc[w][1][0] += dy.x;       acc[w][1][1] += dy.y;
      const float a0 = dy.x * g2[w].x, a1 = dy.y * g2[w].y;        // d x-hat
      const float m1 = warp_sum(a0 + a1) * (1.0f / 64.0f);
      const float m2 = warp_sum(a0 * xh0 + a1 * xh1) * (1.0f / 64.0f);
      *reinterpret_cast<uint32_t*>(dst + w * 64 + d0) = pack_bf16x2(rstd * (a0 - m1 - xh0 * m2), rstd * (a1 - m1 - xh1 * m2));
    }
    *reinterpret_cast<uint32_t*>(dst + 128 + d0) = *reinterpret_cast<const uint32_t*>(gsrc + 2 * blk);      // dv
  }
  // deterministic block reduction of the parameter-gradient partials (fixed order over warps)
#pragma unroll
  for (int w = 0; w < 2; ++w)
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      red[warp][2 * w + t][d0] = acc[w][t][0];
      red[warp][2 * w + t][d0 + 1] = acc[w][t][1];
    }
  __syncthreads();
  if (threadIdx.x < 256) {
    const int j = threadIdx.x;                      // 4 x 64 outputs
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kQkBlock / 32; ++w) s += red[w][j >> 6][j & 63];
    ws[static_cast<long long>(blockIdx.x) * 256 + j] = s;
  }
}

// out[j] (+)= sum_b ws[b][j], j < 256 = dgamma_q | dbeta_q | dgamma_k | dbeta_k
__global__ void qkln_param_finalize_kernel(const float* __restrict__ ws, int nblocks, float* __restrict__ dqg,
                                           float* __restrict__ dqb, float* __restrict__ dkg, float* __restrict__ dkb,
                                           int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = threadIdx.x;
  float s = 0.f;
  for (int b = 0; b < nblocks; ++b) s += ws[static_cast<long long>(b) * 256 + j];
  float* out = (j < 64) ? dqg : (j < 128) ? dqb : (j < 192) ? dkg : dkb;
  const int i = j & 63;
  out[i] = accumulate ? out[i] + s : s;
}

static int qk_grid(long long items) {
  long long g = (items * 32 + kQkBlock - 1) / kQkBlock;
  const long long cap = std::min<long long>(kQkMaxBlocks, static_cast<long long>(sm_count()) * 4);
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace otb

using namespace otb;
#define ST(s) static_cast<cudaStream_t>(s)

extern "C" int otb_qkln_rope_ws_floats(void) { return kQkMaxBlocks * 256; }

extern "C" int otb_qkln_rope_fwd(const void* fused, int64_t ld_fused, const float* q_gamma, const float* q_beta,
                                 const float* k_gamma, const float* k_beta, void* qkv, int64_t ld_qkv, float* stats,
                                 int64_t rows, int H, int S, int rotary_dims, float rope_theta, float eps, void* stream) {
  OTB_CHECK_ARG(fused && q_gamma && q_beta && k_gamma && k_beta && qkv && rows > 0 && H > 0 && S > 0,
                "otb_qkln_rope_fwd: bad argument");
  OTB_CHECK_ARG(ld_fused >= 192LL * H && ld_qkv >= 192LL * H && ld_fused % 2 == 0 && ld_qkv % 2 == 0,
                "otb_qkln_rope_fwd: bad row pitch");
  OTB_CHECK_ARG((rotary_dims == 0 || (rotary_dims >= 4 && rotary_dims <= 64 && (rotary_dims & (rotary_dims - 1)) == 0)) &&
                    rope_theta > 1.f, "otb_qkln_rope_fwd: rotary_dims must be 0 or a power of two in [4, 64]");
  OTB_CHECK_CUDA(launch_k(qkln_rope_fwd_kernel, dim3(qk_grid(rows * H)), dim3(kQkBlock), 0, ST(stream),
                          static_cast<const bf16*>(fused), (long long)ld_fused, q_gamma, q_beta, k_gamma, k_beta,
                          static_cast<bf16*>(qkv), (long long)ld_qkv, stats, (long long)rows, H, S, rotary_dims,
                          log2f(rope_theta), eps));
  count_launch();
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}

extern "C" int otb_qkln_rope_bwd(const void* dqkv, int64_t ld_dqkv, const void* fused, int64_t ld_fused,
                                 const float* stats, const float* q_gamma, const float* k_gamma, void* dfused,
                                 int64_t ld_dfused, float* dq_gamma, float* dq_beta, float* dk_gamma, float* dk_beta,
                                 int accumulate, float* ws, int64_t rows, int H, int S, int rotary_dims,
                                 float rope_theta, void* stream) {
  OTB_CHECK_ARG(dqkv && fused && stats && q_gamma && k_gamma && dfused && ws && rows > 0 && H > 0 && S > 0,
                "otb_qkln_rope_bwd: bad argument");
  OTB_CHECK_ARG(dq_gamma && dq_beta && dk_gamma && dk_beta, "otb_qkln_rope_bwd: null parameter gradient");
  OTB_CHECK_ARG((rotary_dims == 0 || (rotary_dims >= 4 && rotary_dims <= 64 && (rotary_dims & (rotary_dims - 1)) == 0)) &&
                    rope_theta > 1.f, "otb_qkln_rope_bwd: rotary_dims must be 0 or a power of two in [4, 64]");
  const int grid = qk_grid(rows * H);
  OTB_CHECK_CUDA(launch_k(qkln_rope_bwd_kernel, dim3(grid), dim3(kQkBlock), 0, ST(stream),
                          static_cast<const bf16*>(dqkv), (long long)ld_dqkv, static_cast<const bf16*>(fused),
                          (long long)ld_fused, stats, q_gamma, k_gamma, static_cast<bf16*>(dfused),
                          (long long)ld_dfused, ws, (long long)rows, H, S, rotary_dims, log2f(rope_theta)));
  OTB_CHECK_CUDA(launch_k(qkln_param_finalize_kernel, dim3(1), dim3(256), 0, ST(stream), (const float*)ws, grid, dq_gamma,
                          dq_beta, dk_gamma, dk_beta, accumulate));
  count_launch(2);
  OTB_CHECK_CUDA(cudaGetLastError());
  return OTB_OK;
}
