// SONAR speech encoder on sm_90a (BASELINE.json config 3; SURVEY §8 rows a11/a12, App. B.2/B.3):
//   w2v-BERT frontend (stack 2 fbank frames -> LN(160) -> Linear 160->1024)
//   -> 24 Conformer blocks -> model.layer_norm -> attention pooler (1 BOS query, POST-LN decoder layers;
//   AttentionPooler of latent_attention.cu, shared with the text encoder) -> [B,1024]
// following SonarSpeechEncoderModel.forward (sonar/models/sonar_speech/model.py:59-77), factory.py:53-152,
// nn/encoder_pooler.py:70-83; parameter names per sonar_speech/handler.py:63-100.
//
// Every Linear / pointwise conv is the wgmma GEMM of gemm_wgmma.cu (SiLU / ReLU / bias / x += epilogues; the
// macaron 0.5 is folded into the FFN output weights on the host, BatchNorm is folded to scale+shift).  Tokens are
// PACKED (row = cu[b] + t), so padded positions never exist: the reference zeroes them before the depthwise conv and
// masks them in the softmax; here they are simply out of range.
//
// Relative-position attention (Transformer-XL):  score(i,j) = ((q_i+u).k_j + (q_i+v).p_{i-j}) / 8
//   = (q_i.k_j + u.k_j + q_i.p_{i-j} + v.p_{i-j}) / 8.  p = r_proj(R) is one small GEMM per layer and v.p one tiny
//   kernel; the flash kernel computes q.p for the band of relative offsets each 16-query x 64-key tile can reach with
//   the same mma path as q.k^T and applies the Transformer-XL shift as an anti-diagonal read from shared memory.

#include "../../include/sonar_b200.h"
#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>
#include <algorithm>
#include <memory>
#include <new>
#include <vector>

namespace sb {
namespace {

constexpr int kFeat = 160, kFeatPad = 192;

// ---------------------------------------------------------------------------------------------
// frontend: row (b,t) = LN(fbank[b, 2t:2t+2, :]) -> bf16 [T, 192] (cols 160..191 zero)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
frontend_ln_kernel(const float* __restrict__ fbank, int Tpad, const int32_t* __restrict__ cu,
                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                   __nv_bfloat16* __restrict__ out) {
  const int b = blockIdx.x;
  const int t = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int start = cu[b], len = cu[b + 1] - start;
  if (t >= len) return;
  const float* src = fbank + ((long long)b * Tpad + 2 * t) * 80;
  float v[5];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 5; ++i) { v[i] = src[i * 32 + lane]; s += v[i]; }
  const float mean = warp_sum(s) / float(kFeat);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 5; ++i) { const float d = v[i] - mean; q += d * d; }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / float(kFeat) + eps);
  __nv_bfloat16* o = out + (long long)(start + t) * kFeatPad;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const int n = i * 32 + lane;
    o[n] = __float2bfloat16_rn((v[i] - mean) * rstd * gamma[n] + beta[n]);
  }
  o[kFeat + lane] = __float2bfloat16_rn(0.f);
}

// vp[h, n] = sum_d v_bias[h, d] * p[n, h*64 + d]      (one warp per (n, h))
__global__ void __launch_bounds__(256)
relpos_bias_kernel(const __nv_bfloat16* __restrict__ p, const float* __restrict__ v_bias, int Npad, int H,
                   float* __restrict__ vp) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int h = blockIdx.y, lane = threadIdx.x & 31;
  if (n >= Npad) return;
  const __nv_bfloat162 pv = *reinterpret_cast<const __nv_bfloat162*>(p + (long long)n * H * 64 + h * 64 + lane * 2);
  const float s = warp_sum(v_bias[h * 64 + lane * 2] * __low2float(pv) + v_bias[h * 64 + lane * 2 + 1] * __high2float(pv));
  if (lane == 0) vp[(long long)h * Npad + n] = s;
}

// ---------------------------------------------------------------------------------------------
// relative-position flash attention over packed sequences (mma.sync m16n8k16, online softmax)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp16(uint32_t dst, const void* src, bool ok) {
  const int sz = ok ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void ldsm4(uint32_t a, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void ldsm4t(uint32_t a, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ uint32_t toff(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

// Dynamic shared memory layout of attention_relpos_kernel (bytes).  G (per warp two [16 x 88] fp32 band products, one per
// 16-row m-tile) also serves as the Q staging area before the key loop and as the output staging area after it.
constexpr int kRpThreads = 128;                                   // 4 warps x 32 query rows
constexpr int kRpGStride = 88;                                    // floats per G row: 8-byte stores of 4 rows hit 32 distinct banks
constexpr int kRpG = 0, kRpGBytes = 4 * 2 * 16 * kRpGStride * 4;  // 45056
constexpr int kRpKV = kRpG + kRpGBytes;                           // 2 stages x (K 8 KB | V 8 KB)
constexpr int kRpP = kRpKV + 2 * 16384;                           // ring of 256 rows of p (32 KB): 192 live + 64 in flight
constexpr int kRpVp = kRpP + 256 * 128, kRpU = kRpVp + 256 * 4, kRpKb = kRpU + 64 * 4;
constexpr int kRpBar = kRpKb + 64 * 4;                            // 2 mbarriers: TMA completion per K/V/p stage
constexpr int kRpSmem = kRpBar + 16 + 1024;                       // 113168 B incl. 1 KB alignment slack -> two CTAs per SM
constexpr uint32_t kRpBlockBytes = 3 * 8192;                      // K + V + 64 new rows of p per key block
static_assert(kRpGBytes >= 16384, "Q / output staging lives inside G");

__device__ __forceinline__ void cp4(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(ok ? 4 : 0) : "memory");
}

// score(i,j) = (q_i.k_j + u.k_j + q_i.p[c-1-i+j] + v.p[c-1-i+j]) / 8 with c = S_center.  Per 64-key block the CTA needs the
// 192 rows of p its 128 queries can reach; consecutive key blocks share 128 of them, so p lives in a 256-row ring and only
// 64 new rows arrive per block, prefetched with K and V one block ahead (cp.async double buffering).  The kernel is bound
// by shared-memory wavefronts (ldmatrix), so each warp owns 32 query rows = two m-tiles that share every K, V and p
// fragment it loads.  A warp multiplies its queries with its own 96-row window of p on the tensor cores (mma.sync), adds
// v.p, parks the two [16 x 80] results in shared memory and reads them back along the anti-diagonals -- the
// Transformer-XL "shift" -- while it masks and soft-maxes q.k^T.
__global__ void __launch_bounds__(kRpThreads, 2)
attention_relpos_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_p,
                        const int32_t* __restrict__ cu, int H, const float* __restrict__ u_bias,
                        const float* __restrict__ vp, int Npad, int S_center, __nv_bfloat16* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));  // SW128 tiles
  uint8_t* sQ = smem + kRpG;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kRpBar);
  float* s_vp = reinterpret_cast<float*>(smem + kRpVp);
  float* s_u = reinterpret_cast<float*>(smem + kRpU);
  float* s_kb = reinterpret_cast<float*>(smem + kRpKb);
  const int qblk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int start = cu[b], len = cu[b + 1] - start;
  const int q0 = qblk * 128;
  if (q0 >= len) return;
  const int D = H * 64;
  const float* vpbase = vp + (long long)h * Npad;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t sQa = smem_u32(sQ), sKVa = smem_u32(smem + kRpKV), sPa = smem_u32(smem + kRpP), sVpa = smem_u32(s_vp);
  float* sG = reinterpret_cast<float*>(smem + kRpG) + warp * 2 * 16 * kRpGStride;  // [m-tile][16][stride]
  const int band_first = S_center - 1 - (q0 + 127);  // p row of ring position 0
  const int nkb = (len + 63) / 64;

  // One elected thread feeds the CTA by TMA (128-byte swizzle = toff()): K/V of key block kb -> stage kb&1 and the 64
  // rows of p at ring positions [r_lo, r_lo+64).  Rows past the utterance belong to the next one (or are zero-filled
  // past the buffer): their keys are masked below and their probabilities are exactly 0.  Rows of p outside the table
  // (negative or >= Npad) are zero-filled by the TMA unit.  v.p (64 floats) rides on cp.async from 64 threads.
  auto issue_loads = [&](int kb, int r_lo) {
    if (tid == 0) {
      uint64_t* bar = &full_bar[kb & 1];
      uint8_t* stage = smem + kRpKV + (kb & 1) * 16384;
      mbar_arrive_expect_tx(bar, kRpBlockBytes);
      tma_load_2d(stage, &tm_qkv, bar, D + h * 64, start + kb * 64);
      tma_load_2d(stage + 8192, &tm_qkv, bar, 2 * D + h * 64, start + kb * 64);
      tma_load_2d(smem + kRpP + (r_lo & 255) * 128, &tm_p, bar, h * 64, band_first + r_lo);
    }
    if (tid < 64) {
      const int rr = r_lo + tid, idx = band_first + rr;
      const bool ok = idx >= 0 && idx < Npad;
      cp4(sVpa + (rr & 255) * 4, vpbase + (ok ? idx : 0), ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  if (tid == 0) {
    mbar_init(&full_bar[0], 1);
    mbar_init(&full_bar[1], 1);
    fence_mbar_init();
  }
  if (tid < 64) s_u[tid] = u_bias[h * 64 + tid];
  __syncthreads();
  if (tid == 0) {  // Q (two 64-row boxes), K/V of block 0 and its 192 rows of p: one transaction on barrier 0
    uint64_t* bar = &full_bar[0];
    mbar_arrive_expect_tx(bar, 7 * 8192);
    tma_load_2d(sQ, &tm_qkv, bar, h * 64, start + q0);
    tma_load_2d(sQ + 8192, &tm_qkv, bar, h * 64, start + q0 + 64);
    tma_load_2d(smem + kRpKV, &tm_qkv, bar, D + h * 64, start);
    tma_load_2d(smem + kRpKV + 8192, &tm_qkv, bar, 2 * D + h * 64, start);
#pragma unroll
    for (int i = 0; i < 3; ++i) tma_load_2d(smem + kRpP + i * 8192, &tm_p, bar, h * 64, band_first + i * 64);
  }
  for (int rr = tid; rr < 192; rr += kRpThreads) {
    const int idx = band_first + rr;
    const bool ok = idx >= 0 && idx < Npad;
    cp4(sVpa + rr * 4, vpbase + (ok ? idx : 0), ok);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  mbar_wait(&full_bar[0], 0);
  uint32_t qf[2][4][4];
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const int r = warp * 32 + m * 16 + (lane & 15);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      ldsm4(sQa + toff(r, kk * 2 + (lane >> 4)), qf[m][kk][0], qf[m][kk][1], qf[m][kk][2], qf[m][kk][3]);
  }
  float o[2][8][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int j = 0; j < 8; ++j) o[m][j][0] = o[m][j][1] = o[m][j][2] = o[m][j][3] = 0.f;
  float m_run[2][2], l_run[2][2];
#pragma unroll
  for (int m = 0; m < 2; ++m) m_run[m][0] = m_run[m][1] = -CUDART_INF_F, l_run[m][0] = l_run[m][1] = 0.f;
  const float sl2 = 0.125f * 1.4426950408889634f;
  const int rl_lo = lane >> 2, rl_hi = rl_lo + 8;  // this thread's two rows inside each 16-row m-tile
  // band row (ring-relative to the block) of (query i, key j) is 127 - i + j.  The warp's 32 rows reach the 96-row window
  // starting at wrow0; m-tile 0 (rows 32w..32w+15) uses window columns [16, 96), m-tile 1 uses [0, 80).
  const int wrow0 = 96 - 32 * warp;
  const int kc = (lane & 3) * 2;
  const int mtx = lane >> 3;

  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * 64;
    const int ring0 = kb * 64;  // ring position of band row 0 of this block
    // block kb has landed (waited below / before the loop); everyone is past block kb-1 (and past the Q fragments)
    __syncthreads();
    if (kb + 1 < nkb) issue_loads(kb + 1, 192 + ring0);
    if (kb > 0) mbar_wait(&full_bar[kb & 1], (kb >> 1) & 1);  // block 0 was awaited before the Q fragments were read
    const uint32_t sKa = sKVa + (kb & 1) * 16384, sVa = sKa + 8192;
    if (tid < 64) {  // u . k_j for the 64 keys of this block
      const uint8_t* sK = smem + kRpKV + (kb & 1) * 16384;
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 u4 = *reinterpret_cast<const uint4*>(sK + toff(tid, c));
        const uint32_t w[4] = {u4.x, u4.y, u4.z, u4.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const __nv_bfloat162 k2 = *reinterpret_cast<const __nv_bfloat162*>(&w[e]);
          acc = fmaf(s_u[c * 8 + 2 * e], __low2float(k2), acc);
          acc = fmaf(s_u[c * 8 + 2 * e + 1], __high2float(k2), acc);
        }
      }
      s_kb[tid] = acc;
    }
    // ---- G_m[16 x 80] = Q_m . Pwindow_m^T (+ v.p), parked in shared memory; window n-tile pair np feeds both m-tiles ----
#pragma unroll
    for (int nq = 0; nq < 3; ++nq) {  // two n-tile pairs per pass: up to 8 independent accumulator chains in flight
      float ga[2][2][2][4];  // [pair][m-tile][n-tile of the pair][c]
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int t = 0; t < 2; ++t) ga[a][m][t][0] = ga[a][m][t][1] = ga[a][m][t][2] = ga[a][m][t][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int a = 0; a < 2; ++a) {
          const int np = nq * 2 + a;
          const bool use0 = np >= 1, use1 = np <= 4;  // m-tile 0: window n-tiles 2..11; m-tile 1: 0..9
          const int prow = (ring0 + wrow0 + (np * 2 + (mtx >> 1)) * 8 + (lane & 7)) & 255;
          uint32_t b0, b1, b2, b3;
          ldsm4(sPa + toff(prow, kk * 2 + (mtx & 1)), b0, b1, b2, b3);
          if (use0) {
            mma_m16n8k16_bf16(ga[a][0][0], qf[0][kk], b0, b1);
            mma_m16n8k16_bf16(ga[a][0][1], qf[0][kk], b2, b3);
          }
          if (use1) {
            mma_m16n8k16_bf16(ga[a][1][0], qf[1][kk], b0, b1);
            mma_m16n8k16_bf16(ga[a][1][1], qf[1][kk], b2, b3);
          }
        }
      }
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const int np = nq * 2 + a;
        const bool use0 = np >= 1, use1 = np <= 4;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int wc = (np * 2 + t) * 8 + kc;  // window column of this thread's pair
          const float2 v01 = *reinterpret_cast<const float2*>(s_vp + ((ring0 + wrow0 + wc) & 255));
          if (use0) {
            float* g0 = sG + wc - 16;  // m-tile 0 stores relative to its own 80-column window
            *reinterpret_cast<float2*>(g0 + rl_lo * kRpGStride) = make_float2(ga[a][0][t][0] + v01.x, ga[a][0][t][1] + v01.y);
            *reinterpret_cast<float2*>(g0 + rl_hi * kRpGStride) = make_float2(ga[a][0][t][2] + v01.x, ga[a][0][t][3] + v01.y);
          }
          if (use1) {
            float* g1 = sG + 16 * kRpGStride + wc;
            *reinterpret_cast<float2*>(g1 + rl_lo * kRpGStride) = make_float2(ga[a][1][t][0] + v01.x, ga[a][1][t][1] + v01.y);
            *reinterpret_cast<float2*>(g1 + rl_hi * kRpGStride) = make_float2(ga[a][1][t][2] + v01.x, ga[a][1][t][3] + v01.y);
          }
        }
      }
    }
    float s[2][8][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int j = 0; j < 8; ++j) s[m][j][0] = s[m][j][1] = s[m][j][2] = s[m][j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        const int key = (jp * 2 + (mtx >> 1)) * 8 + (lane & 7);
        uint32_t b0, b1, b2, b3;
        ldsm4(sKa + toff(key, kk * 2 + (mtx & 1)), b0, b1, b2, b3);
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          mma_m16n8k16_bf16(s[m][jp * 2], qf[m][kk], b0, b1);
          mma_m16n8k16_bf16(s[m][jp * 2 + 1], qf[m][kk], b2, b3);
        }
      }
    }
    __syncthreads();  // s_kb visible (each warp's own G only needed __syncwarp)
    uint32_t pf[2][4][4];
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      const float* g_lo = sG + (m * 16 + rl_lo) * kRpGStride + 15 - rl_lo + kc;  // band column of (i, j): 15 - r + key
      const float* g_hi = sG + (m * 16 + rl_hi) * kRpGStride + 15 - rl_hi + kc;
      float mx[2] = {-CUDART_INF_F, -CUDART_INF_F};
      if (k0 + 64 <= len) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 kb2 = *reinterpret_cast<const float2*>(s_kb + j * 8 + kc);
          s[m][j][0] += kb2.x + g_lo[j * 8];
          s[m][j][1] += kb2.y + g_lo[j * 8 + 1];
          s[m][j][2] += kb2.x + g_hi[j * 8];
          s[m][j][3] += kb2.y + g_hi[j * 8 + 1];
          mx[0] = fmaxf(mx[0], fmaxf(s[m][j][0], s[m][j][1]));
          mx[1] = fmaxf(mx[1], fmaxf(s[m][j][2], s[m][j][3]));
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int kl = j * 8 + kc + (e & 1);
            float val = -CUDART_INF_F;
            if (k0 + kl < len) val = s[m][j][e] + s_kb[kl] + ((e < 2) ? g_lo : g_hi)[j * 8 + (e & 1)];
            s[m][j][e] = val;
            mx[e >> 1] = fmaxf(mx[e >> 1], val);
          }
        }
      }
      float corr[2], msc[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mnew = fmaxf(m_run[m][r], mx[r]);  // finite: key 0 of every block is inside the utterance
        corr[r] = ex2_approx((m_run[m][r] - mnew) * sl2);
        m_run[m][r] = mnew;
        msc[r] = mnew * sl2;
        l_run[m][r] *= corr[r];
      }
      float ls[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float p0 = ex2_approx(fmaf(s[m][j][0], sl2, -msc[0])), p1 = ex2_approx(fmaf(s[m][j][1], sl2, -msc[0]));
        const float p2 = ex2_approx(fmaf(s[m][j][2], sl2, -msc[1])), p3 = ex2_approx(fmaf(s[m][j][3], sl2, -msc[1]));
        ls[0] += p0 + p1;
        ls[1] += p2 + p3;
        pf[m][j >> 1][(j & 1) * 2 + 0] = pack_bf16x2(p0, p1);
        pf[m][j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
        o[m][j][0] *= corr[0]; o[m][j][1] *= corr[0]; o[m][j][2] *= corr[1]; o[m][j][3] *= corr[1];
      }
      l_run[m][0] += ls[0];
      l_run[m][1] += ls[1];
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        const int key = kk * 16 + (mtx & 1) * 8 + (lane & 7);
        uint32_t b0, b1, b2, b3;
        ldsm4t(sVa + toff(key, jp * 2 + (mtx >> 1)), b0, b1, b2, b3);
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          mma_m16n8k16_bf16(o[m][jp * 2], pf[m][kk], b0, b1);
          mma_m16n8k16_bf16(o[m][jp * 2 + 1], pf[m][kk], b2, b3);
        }
      }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");  // this thread's share of block kb+1; the loop-top barrier publishes it
  }
  __syncthreads();  // every warp is done with its G before the region is reused for the output rows
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float l = l_run[m][r];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      inv[r] = 1.0f / l;
    }
    const int r0 = warp * 32 + m * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int bo = (lane & 3) * 4;
      *reinterpret_cast<uint32_t*>(sQ + toff(r0, j) + bo) = pack_bf16x2(o[m][j][0] * inv[0], o[m][j][1] * inv[0]);
      *reinterpret_cast<uint32_t*>(sQ + toff(r0 + 8, j) + bo) = pack_bf16x2(o[m][j][2] * inv[1], o[m][j][3] * inv[1]);
    }
  }
  __syncwarp();
  __nv_bfloat16* obase = out + (long long)start * D + h * 64;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = i * 32 + lane;
    const int r = warp * 32 + (idx >> 3), c = idx & 7;
    if (q0 + r < len)
      *reinterpret_cast<uint4*>(obase + (long long)(q0 + r) * D + c * 8) = *reinterpret_cast<const uint4*>(sQ + toff(r, c));
  }
}

// ---------------------------------------------------------------------------------------------
// conv module middle: GLU -> depthwise conv (k taps, "same", zero outside the utterance) -> BN(scale,shift) -> SiLU
//   g bf16 [T, 2D] (pointwise_conv1 output: value | gate), out bf16 [T, D]
// ---------------------------------------------------------------------------------------------
// Two adjacent channels per thread: value pairs come out of shared memory as 64-bit loads.  Per output the taps are applied
// in the order k = 0..KS-1 with IEEE fma, one fma per channel (Hopper has no packed fp32 FMA).
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

template <int KS>
__global__ void __launch_bounds__(128, 5)
glu_dwconv_kernel(const __nv_bfloat16* __restrict__ g, const int32_t* __restrict__ cu, int D,
                  const float* __restrict__ dw, const float* __restrict__ bn_scale, const float* __restrict__ bn_shift,
                  __nv_bfloat16* __restrict__ out) {
  constexpr int TP = 64, HALO = KS / 2, ROWS = TP + KS - 1, PP = 16, TAPLD = 66;
  __shared__ __align__(16) float tile[ROWS][64];
  __shared__ __align__(8) float taps[KS][TAPLD];  // this block's 64 channels, transposed to [tap][channel] (row pad: 2-way banks)
  const int b = blockIdx.z, c0 = blockIdx.y * 64, t0 = blockIdx.x * TP;
  const int start = cu[b], len = cu[b + 1] - start;
  if (t0 >= len) return;
  const int tid = threadIdx.x;
  for (int i = tid; i < 64 * KS; i += 128) taps[i % KS][i / KS] = __ldg(dw + (long long)c0 * KS + i);  // coalesced read of dw [D, KS]
  // 16-byte loads, 8 channels of value and gate per thread; every load of the block is in flight before the first use
  constexpr int kIt = (ROWS * 8 + 127) / 128;
  uint4 a4[kIt], g4[kIt];
#pragma unroll
  for (int it = 0; it < kIt; ++it) {
    const int i = tid + it * 128;
    const int pos = t0 - HALO + (i >> 3);
    a4[it] = g4[it] = make_uint4(0u, 0u, 0u, 0u);  // bf16 zeros: 0 * sigmoid(0) = 0 outside the utterance
    if (i < ROWS * 8 && pos >= 0 && pos < len) {
      const __nv_bfloat16* row = g + (long long)(start + pos) * 2 * D + c0 + (i & 7) * 8;
      a4[it] = __ldg(reinterpret_cast<const uint4*>(row));
      g4[it] = __ldg(reinterpret_cast<const uint4*>(row + D));
    }
  }
#pragma unroll
  for (int it = 0; it < kIt; ++it) {
    const int i = tid + it * 128;
    if (i < ROWS * 8) {
      const int p = i >> 3, c8 = (i & 7) * 8;
      const uint32_t aw[4] = {a4[it].x, a4[it].y, a4[it].z, a4[it].w}, gw[4] = {g4[it].x, g4[it].y, g4[it].z, g4[it].w};
      float v[8];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const __nv_bfloat162 a2 = *reinterpret_cast<const __nv_bfloat162*>(&aw[e]);
        const __nv_bfloat162 g2 = *reinterpret_cast<const __nv_bfloat162*>(&gw[e]);
        v[2 * e] = __low2float(a2) * sigmoid_fast(__low2float(g2));
        v[2 * e + 1] = __high2float(a2) * sigmoid_fast(__high2float(g2));
      }
      *reinterpret_cast<float4*>(&tile[p][c8]) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(&tile[p][c8 + 4]) = make_float4(v[4], v[5], v[6], v[7]);
    }
  }
  __syncthreads();
  const int cp = (tid & 31) * 2, pg = tid >> 5;  // channel pair; 4 groups of 16 positions, a register window slides down them
  float2 win[PP + KS - 1];
#pragma unroll
  for (int i = 0; i < PP + KS - 1; ++i) win[i] = *reinterpret_cast<const float2*>(&tile[pg * PP + i][cp]);
  float2 acc[PP];
#pragma unroll
  for (int pp = 0; pp < PP; ++pp) acc[pp] = make_float2(0.f, 0.f);
#pragma unroll
  for (int k = 0; k < KS; ++k) {  // tap-major: PP independent chains in flight
    const float2 w = *reinterpret_cast<const float2*>(&taps[k][cp]);
#pragma unroll
    for (int pp = 0; pp < PP; ++pp) acc[pp] = fma2(w, win[pp + k], acc[pp]);
  }
  const float2 sc = *reinterpret_cast<const float2*>(bn_scale + c0 + cp), sh = *reinterpret_cast<const float2*>(bn_shift + c0 + cp);
#pragma unroll
  for (int pp = 0; pp < PP; ++pp) {
    const int pos = t0 + pg * PP + pp;
    if (pos < len)
      *reinterpret_cast<uint32_t*>(out + (long long)(start + pos) * D + c0 + cp) =
          pack_bf16x2(silu_fast(acc[pp].x * sc.x + sh.x), silu_fast(acc[pp].y * sc.y + sh.y));
  }
}

// ---------------------------------------------------------------------------------------------
// launches: the speech encoder's forward and the kernel-level entry points below call the same functions
// ---------------------------------------------------------------------------------------------
// p rows of the relative-position table for a batch whose longest utterance has smax positions
int npad_of(int smax) { return ((2 * smax - 1) + 255) / 256 * 256; }

// fbank fp32 [B, padded_frames, 80] -> out bf16 [T, 192]
int speech_frontend(const float* fbank, int padded_frames, const int32_t* cu, int B, int max_len, const float* gamma,
                    const float* beta, float eps, __nv_bfloat16* out, cudaStream_t stream) {
  frontend_ln_kernel<<<dim3((unsigned)B, (unsigned)((max_len + 7) / 8)), 256, 0, stream>>>(fbank, padded_frames, cu, gamma,
                                                                                          beta, eps, out);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

// g bf16 [T, 2D] (value | gate) -> out bf16 [T, D]: GLU -> depthwise conv (31 taps) -> BatchNorm scale / shift -> SiLU
int conformer_conv(const __nv_bfloat16* g, const int32_t* cu, int B, int max_len, int D, const float* dw, const float* bn_scale,
                   const float* bn_shift, __nv_bfloat16* out, cudaStream_t stream) {
  static bool carve_set[64] = {};
  if (first_use_on_device(carve_set))  // 5 CTAs x 32 KB of static shared memory per SM: ask for the large carve-out
    SB_CUDA_CHECK(cudaFuncSetAttribute(glu_dwconv_kernel<31>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                       cudaSharedmemCarveoutMaxShared));
  glu_dwconv_kernel<31><<<dim3((unsigned)((max_len + 63) / 64), (unsigned)(D / 64), (unsigned)B), 128, 0, stream>>>(
      g, cu, D, dw, bn_scale, bn_shift, out);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

// Relative-position attention: impl 0 = the wgmma kernel (attention_relpos_tc.cu, B <= kRelposTcMaxBatch), impl 1 = v.p
// (relpos_bias_kernel into vp [H, Npad]) followed by the mma.sync kernel.  qkv [T, 3D], p [Npad, D], out [T, D] bf16;
// qu / qv [T, D] bf16 scratch of impl 0; S_center = the batch's longest utterance.
int attention_relpos(const __nv_bfloat16* qkv, const __nv_bfloat16* p, const float* u_bias, const float* v_bias,
                     const int32_t* cu, int B, int H, long long T, int Npad, int S_center, int impl, __nv_bfloat16* qu,
                     __nv_bfloat16* qv, float* vp, __nv_bfloat16* out, int num_sms, cudaStream_t stream) {
  if (impl == 0)
    return attention_relpos_tc(qkv, p, u_bias, v_bias, cu, B, H, T, Npad, S_center, qu, qv, out, num_sms, stream);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    SB_CUDA_CHECK(cudaFuncSetAttribute(attention_relpos_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kRpSmem));
  const int D = H * 64;
  // TMA views: 64 x 64 boxes of the packed qkv rows [T, 3D] and of the projected table [Npad, D]
  CUtensorMap tm_qkv, tm_p;
  int rc;
  if ((rc = make_tmap_2d(&tm_qkv, qkv, 2, T, 3ll * D, 3ll * D, 64, 64))) return rc;
  if ((rc = make_tmap_2d(&tm_p, p, 2, Npad, D, D, 64, 64))) return rc;
  relpos_bias_kernel<<<dim3((unsigned)((Npad + 7) / 8), (unsigned)H), 256, 0, stream>>>(p, v_bias, Npad, H, vp);
  SB_CUDA_CHECK(cudaGetLastError());
  attention_relpos_kernel<<<dim3((unsigned)((S_center + 127) / 128), (unsigned)H, (unsigned)B), kRpThreads, kRpSmem, stream>>>(
      tm_qkv, tm_p, cu, H, u_bias, vp, Npad, S_center, out);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

}  // namespace
}  // namespace sb

using namespace sb;

struct SbSpeechEncoder {
  SbSpeechConfig cfg;
  SbSpeechWeights w;
  std::vector<SbConformerLayerWeights> layers;
  AttentionPooler pooler;
  int num_sms;
  static constexpr int kMaxBatch = 65535;  // grid z of the attention and conv kernels
  StagingRing staging;  // cu_seqlens
};

namespace {

struct SpWs {
  int32_t* cu;          // [B+1]
  __nv_bfloat16* a192;  // [T,192]
  float* x;             // [T,D]
  __nv_bfloat16* h;     // [T,D]
  __nv_bfloat16* big;   // [T,max(F,3D,2D)]
  __nv_bfloat16* p;     // [Npad,D]
  float* vp;            // [H,Npad]
  __nv_bfloat16* qu;    // [T,D]
  __nv_bfloat16* qv;    // [T,D]
  AttentionPooler::Ws pool;
  size_t bytes;
};

SpWs carve_sp(const SbSpeechEncoder* e, int B, long long T, int smax, void* base) {
  const size_t D = e->cfg.model_dim, F = e->cfg.ffn_inner_dim, H = e->cfg.num_heads;
  const size_t np = npad_of(smax);
  size_t wide = F > 3 * D ? F : 3 * D;
  Carver c(base);
  SpWs w;
  const size_t t = (size_t)T;
  w.cu = c.take<int32_t>(sizeof(int32_t) * ((size_t)B + 1));
  w.a192 = c.take<__nv_bfloat16>(t * kFeatPad * 2);
  w.x = c.take<float>(t * D * 4);
  w.h = c.take<__nv_bfloat16>(t * D * 2);
  w.big = c.take<__nv_bfloat16>(t * wide * 2);
  w.p = c.take<__nv_bfloat16>(np * D * 2);
  w.vp = c.take<float>(H * np * 4);
  w.qu = c.take<__nv_bfloat16>(t * D * 2);  // bf16(q + u), bf16(q + v): A operands of the wgmma attention
  w.qv = c.take<__nv_bfloat16>(t * D * 2);
  w.pool = e->pooler.take(c, (size_t)B);
  w.bytes = c.off;
  return w;
}

}  // namespace

extern "C" {

int sb_speech_encoder_create(const SbSpeechConfig* cfg, const SbSpeechWeights* w, SbSpeechEncoder** out) {
  if (!cfg || !w || !out) { set_last_error("sb_speech_encoder_create: null argument"); return SB_ERR_INVALID; }
  *out = nullptr;
  const int D = cfg->model_dim, H = cfg->num_heads;
  if (D <= 0 || D % 256 != 0 || D > 1024 || H <= 0 || D != 64 * H || cfg->ffn_inner_dim % 256 != 0 ||
      cfg->pooler_ffn_inner_dim % 256 != 0 || cfg->conv_kernel != 31 || cfg->num_layers < 0 || cfg->pooler_layers < 0 ||
      cfg->attn_impl < 0 || cfg->attn_impl > 1) {
    set_last_error("sb_speech_encoder_create: unsupported configuration (need d%%256==0 <=1024, head_dim 64, conv kernel 31)");
    return SB_ERR_INVALID;
  }
  if (!w->front_ln_g || !w->front_ln_b || !w->front_w || !w->front_b || !w->final_ln_g || !w->final_ln_b ||
      !w->zeros || (cfg->num_layers && !w->layers)) {
    set_last_error("sb_speech_encoder_create: missing weight pointer");
    return SB_ERR_INVALID;
  }
  for (int i = 0; i < cfg->num_layers; ++i)
    if (has_null_pointer(w->layers[i])) {
      set_last_error("sb_speech_encoder_create: conformer layer %d has a null weight pointer", i);
      return SB_ERR_INVALID;
    }
  int num_sms = 0;
  if (int rc = require_hopper("sb_speech_encoder_create", &num_sms)) return rc;
  std::unique_ptr<SbSpeechEncoder> e(new (std::nothrow) SbSpeechEncoder());
  if (!e) { set_last_error("out of host memory"); return SB_ERR_INVALID; }
  e->cfg = *cfg;
  e->w = *w;
  e->layers.assign(w->layers, w->layers + cfg->num_layers);
  e->num_sms = num_sms;
  if (int rc = e->staging.create("sb_speech_encoder_create", SbSpeechEncoder::kMaxBatch + 1)) return rc;
  // the projection has no bias: zeros; every GEMM of this engine may take the weight-streaming path
  if (int rc = e->pooler.create("sb_speech_encoder_create", w->pooler, cfg->pooler_layers, w->pooler_q0, w->proj_w, w->zeros,
                                D, D, cfg->pooler_ffn_inner_dim, cfg->ln_eps, num_sms, 2, 1))
    return rc;
  *out = e.release();
  return SB_OK;
}

void sb_speech_encoder_destroy(SbSpeechEncoder* e) { delete e; }

int sb_speech_encoder_workspace_bytes(const SbSpeechEncoder* e, int32_t B, int64_t total_positions, int32_t max_positions,
                                      size_t* bytes) {
  if (!e || !bytes || B <= 0 || total_positions <= 0 || max_positions <= 0) {
    set_last_error("sb_speech_encoder_workspace_bytes: bad argument");
    return SB_ERR_INVALID;
  }
  *bytes = carve_sp(e, B, total_positions, max_positions, nullptr).bytes + kWorkspaceAlign;
  return SB_OK;
}

int sb_speech_encoder_forward(SbSpeechEncoder* e, const float* fbank, int32_t padded_frames, const int32_t* lens_host,
                              int32_t B, const void* relpos_table, int32_t relpos_rows, float* out, float* encoded_packed,
                              void* workspace, size_t workspace_bytes, void* stream_v) {
  if (!e || !fbank || !lens_host || !relpos_table || !out || !workspace) {
    set_last_error("sb_speech_encoder_forward: null argument");
    return SB_ERR_INVALID;
  }
  if (B <= 0 || B > SbSpeechEncoder::kMaxBatch) { set_last_error("sb_speech_encoder_forward: bad batch size %d", B); return SB_ERR_INVALID; }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  // ---- cu_seqlens on the host, staged through a pinned ring ----
  int32_t* cu_h;
  long long T;
  int rc = e->staging.acquire(&cu_h);
  if (!rc) rc = host_cu_seqlens("sb_speech_encoder_forward", lens_host, B, padded_frames / 2, 1, cu_h, &T);
  if (rc) return rc;
  int smax = 0;
  for (int b = 0; b < B; ++b) smax = std::max(smax, cu_h[b + 1] - cu_h[b]);
  const int Npad = npad_of(smax);
  if (relpos_rows != Npad) {
    set_last_error("sb_speech_encoder_forward: relative-position table must have %d rows for max length %d (got %d)", Npad,
                   smax, relpos_rows);
    return SB_ERR_INVALID;
  }
  SpWs w;
  rc = bind_workspace("sb_speech_encoder_forward", workspace, workspace_bytes, &w,
                      [&](void* p) { return carve_sp(e, B, T, smax, p); });
  if (rc) return rc;
  SB_CUDA_CHECK(cudaMemcpyAsync(w.cu, cu_h, sizeof(int32_t) * (B + 1), cudaMemcpyHostToDevice, stream));
  if ((rc = e->staging.record(stream))) return rc;
  const int D = e->cfg.model_dim, F = e->cfg.ffn_inner_dim, H = e->cfg.num_heads;
  const float eps = e->cfg.ln_eps;
  // the mma.sync kernel (A/B runs, second implementation in the tests) is the only one for more than 2047 utterances
  const int attn_impl = (e->cfg.attn_impl == 1 || B > kRelposTcMaxBatch) ? 1 : 0;
  // every GEMM may take the weight-streaming path (as the pooler's do)
  auto gemm = [&](const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int fp32,
                  const float* bias, int M, int N, int K, int epi) {
    GemmArgs g = gemm_args(A, lda, W, ldw, C, ldc, fp32, bias, M, N, K, epi, e->num_sms);
    g.allow_skinny = 1;
    return gemm_bf16(g, stream);
  };
  // ---- frontend ----
  if ((rc = speech_frontend(fbank, padded_frames, w.cu, B, smax, e->w.front_ln_g, e->w.front_ln_b, eps, w.a192, stream)))
    return rc;
  if ((rc = gemm(w.a192, kFeatPad, e->w.front_w, kFeatPad, w.x, D, 1, e->w.front_b, (int)T, D, kFeatPad, EPI_BIAS))) return rc;
  // ---- conformer blocks ----
  for (int li = 0; li < e->cfg.num_layers; ++li) {
    const SbConformerLayerWeights& L = e->layers[li];
    // (a) half-step FFN 1 (0.5 folded into w2/b2)
    if ((rc = layernorm_bf16(w.x, L.ffn1_ln_g, L.ffn1_ln_b, eps, w.h, T, D, stream))) return rc;
    if ((rc = gemm(w.h, D, L.ffn1_w1, D, w.big, F, 0, L.ffn1_b1, (int)T, F, D, EPI_BIAS_SILU))) return rc;
    if ((rc = gemm(w.big, F, L.ffn1_w2, F, w.x, D, 1, L.ffn1_b2, (int)T, D, F, EPI_BIAS_RESIDUAL))) return rc;
    // (b) relative-position self-attention
    if ((rc = layernorm_bf16(w.x, L.attn_ln_g, L.attn_ln_b, eps, w.h, T, D, stream))) return rc;
    if ((rc = gemm(w.h, D, L.wqkv, D, w.big, 3 * D, 0, L.bqkv, (int)T, 3 * D, D, EPI_BIAS))) return rc;
    if ((rc = gemm(relpos_table, D, L.wr, D, w.p, D, 0, e->w.zeros, Npad, D, D, EPI_BIAS))) return rc;
    if ((rc = attention_relpos(w.big, w.p, L.u_bias, L.v_bias, w.cu, B, H, T, Npad, smax, attn_impl, w.qu, w.qv, w.vp, w.h,
                               e->num_sms, stream)))
      return rc;
    if ((rc = gemm(w.h, D, L.wo, D, w.x, D, 1, L.bo, (int)T, D, D, EPI_BIAS_RESIDUAL))) return rc;
    // (c) convolution module
    if ((rc = layernorm_bf16(w.x, L.conv_ln_g, L.conv_ln_b, eps, w.h, T, D, stream))) return rc;
    if ((rc = gemm(w.h, D, L.pw1, D, w.big, 2 * D, 0, e->w.zeros, (int)T, 2 * D, D, EPI_BIAS))) return rc;
    if ((rc = conformer_conv(w.big, w.cu, B, smax, D, L.dw, L.bn_scale, L.bn_shift, w.h, stream))) return rc;
    if ((rc = gemm(w.h, D, L.pw2, D, w.x, D, 1, e->w.zeros, (int)T, D, D, EPI_BIAS_RESIDUAL))) return rc;
    // (d) half-step FFN 2
    if ((rc = layernorm_bf16(w.x, L.ffn2_ln_g, L.ffn2_ln_b, eps, w.h, T, D, stream))) return rc;
    if ((rc = gemm(w.h, D, L.ffn2_w1, D, w.big, F, 0, L.ffn2_b1, (int)T, F, D, EPI_BIAS_SILU))) return rc;
    if ((rc = gemm(w.big, F, L.ffn2_w2, F, w.x, D, 1, L.ffn2_b2, (int)T, D, F, EPI_BIAS_RESIDUAL))) return rc;
    // (e) block LayerNorm: the residual stream itself is normalised
    if ((rc = layernorm_dual(w.x, L.ln_g, L.ln_b, eps, w.x, nullptr, T, D, stream))) return rc;
  }
  // ---- model.layer_norm (fp32 in place, bf16 copy = pooler memory) ----
  if ((rc = layernorm_dual(w.x, e->w.final_ln_g, e->w.final_ln_b, eps, w.x, w.h, T, D, stream))) return rc;
  if (encoded_packed) SB_CUDA_CHECK(cudaMemcpyAsync(encoded_packed, w.x, sizeof(float) * (size_t)T * D, cudaMemcpyDeviceToDevice, stream));
  return e->pooler.forward(w.pool, w.h, w.cu, B, out, stream);
}

int sb_attention_relpos(const void* qkv, const void* p, const float* u_bias, const float* v_bias, const int32_t* cu_seqlens,
                        int32_t B, int32_t H, int64_t total_tokens, int32_t Npad, int32_t S_center, int32_t impl, void* qu,
                        void* qv, float* vp, void* out, void* stream) {
  if (!qkv || !p || !u_bias || !v_bias || !cu_seqlens || !out || (impl == 0 && (!qu || !qv)) || (impl == 1 && !vp)) {
    set_last_error("sb_attention_relpos: null argument");
    return SB_ERR_INVALID;
  }
  const int D = 64 * H;
  if (impl < 0 || impl > 1 || B <= 0 || B > 65535 || total_tokens <= 0 || S_center <= 0 || H <= 0 || D % 256 != 0 || D > 1024 ||
      Npad != npad_of(S_center)) {
    set_last_error("sb_attention_relpos: bad argument (impl %d, B %d, H %d, T %lld, Npad %d, S_center %d)", impl, B, H,
                   (long long)total_tokens, Npad, S_center);
    return SB_ERR_INVALID;
  }
  int sms = 0;
  if (int rc = require_hopper("sb_attention_relpos", &sms)) return rc;
  return attention_relpos(static_cast<const __nv_bfloat16*>(qkv), static_cast<const __nv_bfloat16*>(p), u_bias, v_bias,
                          cu_seqlens, B, H, total_tokens, Npad, S_center, impl, static_cast<__nv_bfloat16*>(qu),
                          static_cast<__nv_bfloat16*>(qv), vp, static_cast<__nv_bfloat16*>(out), sms,
                          reinterpret_cast<cudaStream_t>(stream));
}

int sb_conformer_conv(const void* g, const int32_t* cu_seqlens, int32_t B, int32_t max_len, int32_t D, const float* dw,
                      const float* bn_scale, const float* bn_shift, void* out, void* stream) {
  if (!g || !cu_seqlens || !dw || !bn_scale || !bn_shift || !out) {
    set_last_error("sb_conformer_conv: null argument");
    return SB_ERR_INVALID;
  }
  if (B <= 0 || B > 65535 || max_len <= 0 || D <= 0 || D % 64 != 0) {
    set_last_error("sb_conformer_conv: bad argument (B %d, max_len %d, D %d)", B, max_len, D);
    return SB_ERR_INVALID;
  }
  return conformer_conv(static_cast<const __nv_bfloat16*>(g), cu_seqlens, B, max_len, D, dw, bn_scale, bn_shift,
                        static_cast<__nv_bfloat16*>(out), reinterpret_cast<cudaStream_t>(stream));
}

int sb_speech_frontend(const float* fbank, int32_t padded_frames, const int32_t* cu_seqlens, int32_t B, int32_t max_len,
                       const float* gamma, const float* beta, float eps, void* out, void* stream) {
  if (!fbank || !cu_seqlens || !gamma || !beta || !out) {
    set_last_error("sb_speech_frontend: null argument");
    return SB_ERR_INVALID;
  }
  if (B <= 0 || B > 65535 || max_len <= 0 || 2ll * max_len > padded_frames) {
    set_last_error("sb_speech_frontend: bad argument (B %d, max_len %d, padded_frames %d)", B, max_len, padded_frames);
    return SB_ERR_INVALID;
  }
  return speech_frontend(fbank, padded_frames, cu_seqlens, B, max_len, gamma, beta, eps, static_cast<__nv_bfloat16*>(out),
                         reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
