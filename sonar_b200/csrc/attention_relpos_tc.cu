// Transformer-XL relative-position self-attention of the w2v-BERT Conformer blocks on wgmma (BASELINE.json config 3,
// SURVEY §8 row a11 / App. B.2; reference wiring sonar/models/sonar_speech/factory.py:64-71, parameter names
// sdpa.u_bias / sdpa.v_bias / sdpa.r_proj in sonar_speech/handler.py:81-83):
//
//     score(i, j) = ((q_i + u) . k_j + (q_i + v) . p[c - 1 - i + j]) / 8,      p = r_proj(R) [2S-1 -> Npad rows],  c = S_center
//
// over PACKED utterances (row = cu[b] + t), keys >= len get probability exactly 0.
//
// Work decomposition.  An ITEM is (utterance b, 128-query tile, head h); a UNIT is one 128-key tile of it; each of the two
// consumer warpgroups owns 64 query rows (w = 0, 1) of the unit:
//     S1[64 x 128] = Qu . K^T                       Qu = bf16(q + u), Qv = bf16(q + v): prepared once per layer by
//     Bw[64 x 192] = Qv . Pw^T                      relpos_qprep_kernel, so no bias vector is added inside this kernel
//       Pw = the 256 rows of p the tile can reach: row n0 + cB, n0 = c - 1 - (q0 + 127) + j0, and the score of (query il,
//       key jl) of the tile uses column cB = 127 - il + jl -- the Transformer-XL "shift": every query row reads B at its
//       own offset.  Warpgroup w needs cB in [64 - 64 w, 254 - 64 w], i.e. 192 rows of Pw from row 64 - 64 w, and its
//       query row rl then reads column 63 - rl + jl of Bw.  The accumulator layout of wgmma fixes which thread holds which
//       column, so Bw goes through a shared-memory buffer (fp32, row stride 197 floats: the skewed reads and the fragment
//       writes are at most 2-way bank conflicted) in two 96-column halves and every thread gathers the position terms of
//       its S1 fragment from there.
//     P = exp2((S1 + shift(B) - m) / 8 * log2 e)    online softmax on the accumulator fragments (a row = 4 lanes)
//     O[64 x 64] += P . V                           A = P from registers, V the MN-major B operand
// Warpgroup 0 = TMA producer (one thread); Qu | Qv stay for the item, K | Pw and V are single slots that are released as
// soon as the products reading them have retired, so the next unit's loads run under this unit's softmax.

#include "attention_wgmma.cuh"
#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>

namespace sb {
namespace {

constexpr int kTile = 128 * 64 * 2;              // one [128 x 64] bf16 operand tile = 16 KB
constexpr int kOperandBytes = 6 * kTile;          // Qu | Qv | K | P_lo | P_hi | V  (96 KB)
constexpr int kOffQu = 0, kOffQv = kTile, kOffK = 2 * kTile, kOffPlo = 3 * kTile, kOffV = 5 * kTile;
constexpr int kBLd = 197;                         // floats per row of a warpgroup's Bw buffer (192 + skew padding)
constexpr int kBBytes = 64 * kBLd * 4;            // per consumer warpgroup
constexpr int kBarBytes = 512;
constexpr int kMaxBatch = kRelposTcMaxBatch;
constexpr int kSmemBytes = kOperandBytes + 2 * kBBytes + kBarBytes + 2 * (kMaxBatch + 1) * 4 + 1024;
constexpr int kThreads = 384;
static_assert(kSmemBytes <= 232448, "shared memory budget of one sm_90 block");

enum { Q_FULL = 0, Q_EMPTY, KP_FULL, KP_EMPTY, V_FULL, V_EMPTY, kNumBars };

// The unit sequence of this CTA: items first + i * stride; an item = (query tile, head) of one utterance, expanded
// into its key tiles.  tile_cu[b] = number of query tiles before utterance b.
struct RelStream {
  const int32_t* cu;
  const int32_t* tile_cu;
  int B, H, num_items, item, stride;
  int h, tok0, len, q0, nt, kt;
  bool valid;
  __device__ __forceinline__ void load_item() {
    valid = item < num_items;
    if (!valid) return;
    const int tile = item / H;
    h = item - tile * H;
    int lo = 0, hi = B - 1;  // last b with tile_cu[b] <= tile
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (tile_cu[mid] <= tile) lo = mid; else hi = mid - 1;
    }
    tok0 = cu[lo];
    len = cu[lo + 1] - tok0;
    q0 = (tile - tile_cu[lo]) * 128;
    nt = (len + 127) >> 7;
    kt = 0;
  }
  __device__ __forceinline__ void init(const int32_t* cu_, const int32_t* tile_cu_, int B_, int H_, int first, int stride_) {
    cu = cu_; tile_cu = tile_cu_; B = B_; H = H_; num_items = tile_cu_[B_] * H_; item = first; stride = stride_;
    load_item();
  }
  __device__ __forceinline__ void advance() {
    if (++kt == nt) {
      item += stride;
      load_item();
    }
  }
};

__global__ void __launch_bounds__(kThreads, 1)
attention_relpos_tc_kernel(const __grid_constant__ CUtensorMap tm_qu, const __grid_constant__ CUtensorMap tm_qv,
                           const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_p,
                           const int32_t* cu_g, int B, int H, int S_center, __nv_bfloat16* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* smem_bw = reinterpret_cast<float*>(smem + kOperandBytes);  // [2][64][kBLd]
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kOperandBytes + 2 * kBBytes);  // [kNumBars]
  int32_t* cu = reinterpret_cast<int32_t*>(smem + kOperandBytes + 2 * kBBytes + kBarBytes);
  int32_t* tile_cu = cu + (kMaxBatch + 1);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg_idx = threadIdx.x >> 7;
  const int D = H * 64;
  for (int i = threadIdx.x; i <= B; i += kThreads) cu[i] = cu_g[i];
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_qu);
    tma_prefetch_desc(&tm_qv);
    tma_prefetch_desc(&tm_qkv);
    tma_prefetch_desc(&tm_p);
    mbar_init(&bar[Q_FULL], 1);
    mbar_init(&bar[Q_EMPTY], 8);   // one arrive per consumer warp
    mbar_init(&bar[KP_FULL], 1);
    mbar_init(&bar[KP_EMPTY], 8);
    mbar_init(&bar[V_FULL], 1);
    mbar_init(&bar[V_EMPTY], 8);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // query-tile prefix over the utterances (B <= kMaxBatch)
    int acc = 0;
    for (int b = 0; b < B; ++b) {
      tile_cu[b] = acc;
      acc += (cu[b + 1] - cu[b] + 127) >> 7;
    }
    tile_cu[B] = acc;
  }
  __syncthreads();

  RelStream u;
  u.init(cu, tile_cu, B, H, blockIdx.x, gridDim.x);
  uint32_t n = 0, ni = 0;  // units / items so far

  if (wg_idx == 0) {
    // ============================ TMA producer ============================
    if (warp == 0 && lane == 0) {
      while (u.valid) {
        const int col = u.h * 64;
        if (u.kt == 0) {  // the item's biased queries
          mbar_wait(&bar[Q_EMPTY], (ni & 1) ^ 1);
          mbar_arrive_expect_tx(&bar[Q_FULL], 2 * kTile);
          tma_load_2d(smem + kOffQu, &tm_qu, &bar[Q_FULL], col, u.tok0 + u.q0);
          tma_load_2d(smem + kOffQv, &tm_qv, &bar[Q_FULL], col, u.tok0 + u.q0);
          ++ni;
        }
        const int j0 = u.kt * 128;
        const int n0 = S_center - 1 - (u.q0 + 127) + j0;  // p row of window column 0 (may be negative: zero filled)
        mbar_wait(&bar[KP_EMPTY], (n & 1) ^ 1);
        mbar_arrive_expect_tx(&bar[KP_FULL], 3 * kTile);
        tma_load_2d(smem + kOffK, &tm_qkv, &bar[KP_FULL], D + col, u.tok0 + j0);
        tma_load_2d(smem + kOffPlo, &tm_p, &bar[KP_FULL], col, n0);
        tma_load_2d(smem + kOffPlo + kTile, &tm_p, &bar[KP_FULL], col, n0 + 128);
        mbar_wait(&bar[V_EMPTY], (n & 1) ^ 1);
        mbar_arrive_expect_tx(&bar[V_FULL], kTile);
        tma_load_2d(smem + kOffV, &tm_qkv, &bar[V_FULL], 2 * D + col, u.tok0 + j0);
        ++n;
        u.advance();
      }
    }
  } else {
    // ============================ scores, softmax, P.V: 64 query rows per warpgroup ============================
    const int cwg = wg_idx - 1;
    const int fr = (warp & 3) * 16 + (lane >> 2);  // fragment rows fr and fr + 8 of this warpgroup's 64
    const int cq = 2 * (lane & 3);                 // fragment columns 8 j + cq, + 1
    float* bw = smem_bw + cwg * 64 * kBLd;
    const uint32_t bar_id = 1 + cwg;
    const uint32_t sbase = smem_u32(smem);
    float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};  // l_run: this lane's share of the row sum
    float o[32];
    while (u.valid) {
      const int kv_valid = min(128, u.len - u.kt * 128);
      const bool active = u.q0 + cwg * 64 < u.len;  // (warpgroup-uniform) this half of the query tile holds queries
      const bool last = (u.kt == u.nt - 1);
      if (u.kt == 0) {
        m_run[0] = m_run[1] = -CUDART_INF_F;
        l_run[0] = l_run[1] = 0.f;
        mbar_wait(&bar[Q_FULL], ni & 1);
        ++ni;
      }
      mbar_wait(&bar[KP_FULL], n & 1);
      float s[64];
      if (active) {
        const uint64_t qu = wgmma_desc_kmajor_sw128(sbase + kOffQu + cwg * 64 * 128);
        const uint64_t qv = wgmma_desc_kmajor_sw128(sbase + kOffQv + cwg * 64 * 128);
        const uint64_t kd = wgmma_desc_kmajor_sw128(sbase + kOffK);
        // Pw rows [64 - 64 cwg + 96 hb, + 96) for half hb of this warpgroup's window
        const uint32_t pw = sbase + kOffPlo + (64 - 64 * cwg) * 128;
        float bb[48];
        // the two Bw halves first and S1 last: at most 64 + 32 accumulator registers are live next to each product
        wgmma_fence_regs(bb);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n96k16_ss(bb, qv + uint64_t(2 * k), wgmma_desc_kmajor_sw128(pw) + uint64_t(2 * k), k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(bb);
        named_bar_sync(bar_id, 128);  // the previous unit's gathers are done
#pragma unroll
        for (int j = 0; j < 12; ++j) {
          float* d = bw + fr * kBLd + 8 * j + cq;
          d[0] = bb[4 * j]; d[1] = bb[4 * j + 1];
          d[8 * kBLd] = bb[4 * j + 2]; d[8 * kBLd + 1] = bb[4 * j + 3];
        }
        wgmma_fence_regs(bb);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n96k16_ss(bb, qv + uint64_t(2 * k), wgmma_desc_kmajor_sw128(pw + 96 * 128) + uint64_t(2 * k), k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(bb);
#pragma unroll
        for (int j = 0; j < 12; ++j) {
          float* d = bw + fr * kBLd + 96 + 8 * j + cq;
          d[0] = bb[4 * j]; d[1] = bb[4 * j + 1];
          d[8 * kBLd] = bb[4 * j + 2]; d[8 * kBLd + 1] = bb[4 * j + 3];
        }
        wgmma_fence_regs(s);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(s, qu + uint64_t(2 * k), kd + uint64_t(2 * k), k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&bar[KP_EMPTY]);             // K and Pw are dead
        if (last) mbar_arrive(&bar[Q_EMPTY]);    // last key tile of the item: Qu, Qv are dead too
      }
      uint32_t pa[8][4];
      float alpha[2] = {1.f, 1.f};
      if (active) {
        named_bar_sync(bar_id, 128);  // Bw complete
        // the shift: query row rl, key jl reads Bw[rl][63 - rl + jl]
        const float* g0 = bw + fr * kBLd + 63 - fr + cq;
        const float* g1 = bw + (fr + 8) * kBLd + 63 - (fr + 8) + cq;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          s[4 * j] += g0[8 * j];
          s[4 * j + 1] += g0[8 * j + 1];
          s[4 * j + 2] += g1[8 * j];
          s[4 * j + 3] += g1[8 * j + 1];
        }
        attn::mask_keys(s, kv_valid, cq);
        attn::online_softmax(s, m_run, l_run, alpha, pa);
      }
      mbar_wait(&bar[V_FULL], n & 1);
      if (active) attn::pv_accumulate(o, pa, alpha, wgmma_desc_mnmajor_sw128(sbase + kOffV), u.kt == 0);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar[V_EMPTY]);
      if (active && last) attn::store_rows(o, l_run, out, u.tok0, u.q0 + cwg * 64 + fr, u.len, D, u.h * 64 + cq);
      ++n;
      u.advance();
    }
  }
}

// qu = bf16(q + u), qv = bf16(q + v): q = first D columns of the packed qkv rows; u, v fp32 [D]  (8 elements per thread)
__global__ void __launch_bounds__(256)
relpos_qprep_kernel(const __nv_bfloat16* __restrict__ qkv, const float* __restrict__ u_bias, const float* __restrict__ v_bias,
                    long long T, int D, __nv_bfloat16* __restrict__ qu, __nv_bfloat16* __restrict__ qv) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int per_row = D / 8;
  if (i >= T * per_row) return;
  const long long t = i / per_row;
  const int c = int(i - t * per_row) * 8;
  const uint4 q8 = *reinterpret_cast<const uint4*>(qkv + t * 3 * D + c);
  const uint32_t w[4] = {q8.x, q8.y, q8.z, q8.w};
  uint32_t a[4], b[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const __nv_bfloat162 p = *reinterpret_cast<const __nv_bfloat162*>(&w[e]);
    const float x0 = __low2float(p), x1 = __high2float(p);
    a[e] = pack_bf16x2(x0 + u_bias[c + 2 * e], x1 + u_bias[c + 2 * e + 1]);
    b[e] = pack_bf16x2(x0 + v_bias[c + 2 * e], x1 + v_bias[c + 2 * e + 1]);
  }
  *reinterpret_cast<uint4*>(qu + t * D + c) = make_uint4(a[0], a[1], a[2], a[3]);
  *reinterpret_cast<uint4*>(qv + t * D + c) = make_uint4(b[0], b[1], b[2], b[3]);
}

}  // namespace

// qkv [T, 3D] bf16 packed rows (q | k | v), p [Npad, D] bf16 = r_proj(relative-position table), u_bias / v_bias fp32 [D],
// qu / qv [T, D] bf16 scratch, out [T, D] bf16.  S_center = the batch's maximum length (row c-1-i+j of p <-> offset i-j).
int attention_relpos_tc(const __nv_bfloat16* qkv, const __nv_bfloat16* p, const float* u_bias, const float* v_bias,
                        const int32_t* cu_seqlens, int B, int H, long long total_tokens, int Npad, int S_center,
                        __nv_bfloat16* qu, __nv_bfloat16* qv, __nv_bfloat16* out, int num_sms, cudaStream_t stream) {
  if (B <= 0 || total_tokens <= 0) return 0;
  if (B > kMaxBatch) {
    set_last_error("attention_relpos_tc: at most %d utterances per batch (got %d)", kMaxBatch, B);
    return -1;
  }
  const int D = H * 64;
  const long long nthr = total_tokens * (D / 8);
  relpos_qprep_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, stream>>>(qkv, u_bias, v_bias, total_tokens, D, qu, qv);
  SB_CUDA_CHECK(cudaGetLastError());
  CUtensorMap tm_qu, tm_qv, tm_qkv, tm_p;
  int rc;
  if ((rc = make_tmap_2d(&tm_qu, qu, 2, total_tokens, D, D, 128, 64))) return rc;
  if ((rc = make_tmap_2d(&tm_qv, qv, 2, total_tokens, D, D, 128, 64))) return rc;
  if ((rc = make_tmap_2d(&tm_qkv, qkv, 2, total_tokens, 3ll * D, 3ll * D, 128, 64))) return rc;
  if ((rc = make_tmap_2d(&tm_p, p, 2, Npad, D, D, 128, 64))) return rc;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    SB_CUDA_CHECK(cudaFuncSetAttribute(attention_relpos_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  }
  const int grid = num_sms > 0 ? num_sms : device_sm_count();
  attention_relpos_tc_kernel<<<(unsigned)grid, kThreads, kSmemBytes, stream>>>(tm_qu, tm_qv, tm_qkv, tm_p, cu_seqlens, B, H,
                                                                               S_center, out);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace sb
