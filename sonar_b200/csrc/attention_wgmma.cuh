// The consumer-warpgroup tail shared by the two wgmma flash-attention kernels (attention_tc.cu: text self-attention,
// attention_relpos_tc.cu: Conformer relative-position attention).  Once a warpgroup holds S[64 x 128] of one 128-key tile in
// the m64n128 accumulator layout (a row = the 4 lanes of a quad, see common.cuh), both kernels mask, soft-max, multiply P
// with the MN-major V tile and store their rows the same way.
//
// Every function is force-inlined and calls nothing: a function call anywhere in a kernel that issues wgmma makes ptxas
// serialize every wgmma (DESIGN.md §4).  Callers keep each of them under a warpgroup-uniform branch.
#pragma once

#include "common.cuh"

#include <math_constants.h>

namespace sb {
namespace attn {

constexpr float kScaleLog2 = 0.125f * 1.4426950408889634f;  // 1/sqrt(64) * log2(e)

// keys >= kv_valid lie beyond the sequence: -inf -> probability exactly 0.  cq = 2 (lane % 4), the fragment's first column.
__device__ __forceinline__ void mask_keys(float (&s)[64], int kv_valid, int cq) {
  if (kv_valid < 128) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (8 * j + cq >= kv_valid) s[4 * j] = s[4 * j + 2] = -CUDART_INF_F;
      if (8 * j + cq + 1 >= kv_valid) s[4 * j + 1] = s[4 * j + 3] = -CUDART_INF_F;
    }
  }
}

// Online softmax of one key tile: updates the running row maxima m_run and this lane's share of the row sums l_run, returns
// the rescale factors of the previous tiles in alpha and the numerators, packed to bf16, as the A fragments of P.V in pa.
__device__ __forceinline__ void online_softmax(const float (&s)[64], float (&m_run)[2], float (&l_run)[2], float (&alpha)[2],
                                               uint32_t (&pa)[8][4]) {
  float mx[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    mx[0] = fmaxf(mx[0], fmaxf(s[4 * j], s[4 * j + 1]));
    mx[1] = fmaxf(mx[1], fmaxf(s[4 * j + 2], s[4 * j + 3]));
  }
  float mxs[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float m_new = fmaxf(m_run[r], mx[r]);              // finite: key 0 of every tile is valid
    alpha[r] = ex2_approx((m_run[r] - m_new) * kScaleLog2);  // 0 on the first key tile (m_run = -inf)
    m_run[r] = m_new;
    mxs[r] = m_new * kScaleLog2;
  }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float p0 = ex2_approx(fmaf(s[4 * j], kScaleLog2, -mxs[0])), p1 = ex2_approx(fmaf(s[4 * j + 1], kScaleLog2, -mxs[0]));
    const float p2 = ex2_approx(fmaf(s[4 * j + 2], kScaleLog2, -mxs[1])), p3 = ex2_approx(fmaf(s[4 * j + 3], kScaleLog2, -mxs[1]));
    sum[0] += p0 + p1;
    sum[1] += p2 + p3;
    pa[j >> 1][(j & 1) * 2] = pack_bf16x2(p0, p1);  // A fragment of k-step j / 2: (row, keys) then (row + 8, keys)
    pa[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
  }
  l_run[0] = l_run[0] * alpha[0] + sum[0];
  l_run[1] = l_run[1] * alpha[1] + sum[1];
}

// O[64 x 64] = alpha O + P . V for the V tile behind v_desc (MN-major, SWIZZLE_128B); the first key tile overwrites O.
// All 8 k-steps run (a branch around a wgmma would serialize them): masked keys have P = 0 exactly, and the V rows behind
// them are other sequences' finite values or TMA zero fill.
__device__ __forceinline__ void pv_accumulate(float (&o)[32], const uint32_t (&pa)[8][4], const float (&alpha)[2],
                                              uint64_t v_desc, bool first_key_tile) {
  if (!first_key_tile) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
      o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
    }
  }
  wgmma_fence_regs(o);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 8; ++k)
    wgmma_m64n64k16_rs_bt(o, pa[k], v_desc + uint64_t(k * (2048 >> 4)), (!first_key_tile || k > 0) ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(o);
}

// out[tok0 + qrow, col + c] = bf16(O / l) for this lane's rows qrow = qrow0 and qrow0 + 8 that lie below len; D = row
// stride of out in elements, col = the head's first column + cq.
__device__ __forceinline__ void store_rows(const float (&o)[32], const float (&l_run)[2], __nv_bfloat16* __restrict__ out,
                                           int tok0, int qrow0, int len, int D, int col) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int qrow = qrow0 + 8 * r;
    if (qrow < len) {
      const float inv = 1.0f / l;
      uint32_t* dst = reinterpret_cast<uint32_t*>(out + (long long)(tok0 + qrow) * D + col);
#pragma unroll
      for (int j = 0; j < 8; ++j) dst[4 * j] = pack_bf16x2(o[4 * j + 2 * r] * inv, o[4 * j + 2 * r + 1] * inv);
    }
  }
}

}  // namespace attn
}  // namespace sb
