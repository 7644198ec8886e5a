// wgmma self-attention over PACKED variable-length sequences (any length the position table allows).
//
// Reference semantics: fairseq2 StandardMultiheadAttention + create_default_sdpa
// (sonar/models/sonar_text/factory.py:130-141) = F.scaled_dot_product_attention with a key-padding mask,
// scale 1/sqrt(64), no causal mask (SURVEY App. A.2 / F4).  Padded positions do not exist on the device, so the
// "mask" is simply: keys >= len get probability exactly 0.
//
// Work decomposition.  An ITEM is (sentence b, head h).  Its queries are cut into 128-row tiles, its keys into 128-key
// tiles, and a UNIT is one (query tile, key tile) pair; each of the two consumer warpgroups owns 64 query rows of it:
//     S[64 x 128] = Q[64 x 64] . K[128 x 64]^T       4 x wgmma.m64n128k16, operands K-major in shared memory
//     P           = exp2((S - m) * scale)            softmax numerators on the accumulator fragments (a row = 4 lanes)
//     O[64 x 64] += P[64 x 128] . V[128 x 64]        <= 8 x wgmma.m64n64k16, A = P from REGISTERS, V the MN-major B operand
// For sentences of at most 128 tokens an item is exactly one unit; longer sentences run nq x nkv units with the usual
// online-softmax rescaling of the register accumulator between key tiles.
//
// One persistent CTA per SM, warp-specialised:
//   warpgroup 0    TMA producer (one thread): [128 x 64] bf16 tiles (SWIZZLE_128B) of the next units into two rings -- Q|K
//                  pairs (3 stages, released as soon as S = Q K^T has retired) and V tiles (6 stages, released when P.V has
//                  retired): the op is HBM-bound (reads 6 B, writes 2 B per token and dim; 1.2 % of the encoder FLOPs) and
//                  what matters is bytes in flight per SM
//   warpgroups 1-2 S, softmax, P.V and the output rows of their 64 queries.  P never touches shared memory: the
//                  accumulator layout of S is the A-operand register layout of P.V.

#include "attention_wgmma.cuh"
#include "common.cuh"
#include "sonar_b200_internal.h"

#include <limits.h>
#include <math_constants.h>

namespace sb {
namespace {

constexpr int kTile = 128 * 64 * 2;  // one [128 x 64] bf16 operand tile = 16 KB
constexpr int kQkStages = 3;         // Q | K pairs (32 KB each)
constexpr int kVStages = 6;          // V tiles (16 KB each)
constexpr int kRingBytes = kQkStages * 2 * kTile + kVStages * kTile;  // 192 KB
constexpr int kBarBytes = 512;
constexpr int kCuSmemInts = 8192;  // cu_seqlens is staged in shared memory when the batch has < 8192 sentences
constexpr int kSmemBytes = kRingBytes + kBarBytes + kCuSmemInts * 4 + 1024;  // + alignment slack
static_assert(kSmemBytes <= 232448, "shared memory budget of one sm_90 block");
constexpr int kThreads = 384;

// The unit sequence of this CTA: items blockIdx.x + i * gridDim.x, i = 0, 1, ..., each expanded into its
// (query tile, key tile) units.  Every warp role walks identical copies.
struct UnitStream {
  const int32_t* cu;
  int H, num_items, item, stride;
  int b, h, tok0, len, nt, qt, kt;  // current item / unit
  bool valid;
  __device__ __forceinline__ void load_item() {
    for (;;) {
      valid = item < num_items;
      if (!valid) return;
      b = item / H;
      h = item - b * H;
      tok0 = cu[b];
      len = cu[b + 1] - tok0;
      nt = (len + 127) >> 7;
      qt = kt = 0;
      if (len > 0) return;
      item += stride;  // empty sentence: no units (the pooling kernel writes zeros for it)
    }
  }
  __device__ __forceinline__ void init(const int32_t* cu_, int H_, int num_items_, int first, int stride_) {
    cu = cu_; H = H_; num_items = num_items_; item = first; stride = stride_;
    load_item();
  }
  __device__ __forceinline__ void advance() {
    if (++kt == nt) {
      kt = 0;
      if (++qt == nt) {
        item += stride;
        load_item();
      }
    }
  }
};

__global__ void __launch_bounds__(kThreads, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tm_qkv, const int32_t* cu, int B, int H,
                    __nv_bfloat16* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_qk = smem;                              // [kQkStages][Q | K]
  uint8_t* smem_v = smem + kQkStages * 2 * kTile;       // [kVStages]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kRingBytes);
  uint64_t* full_qk = bars;                       // [kQkStages] TMA: Q and K landed
  uint64_t* empty_qk = full_qk + kQkStages;       // [kQkStages] S retired in every consumer warp -> the Q | K pair is free
  uint64_t* full_v = empty_qk + kQkStages;        // [kVStages] TMA: V landed
  uint64_t* empty_v = full_v + kVStages;          // [kVStages] P.V retired in every consumer warp -> the V tile is free
  int32_t* cu_smem = reinterpret_cast<int32_t*>(smem + kRingBytes + kBarBytes);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg_idx = threadIdx.x >> 7;
  const int D = H * 64;
  const int num_items = B * H;
  // every role looks sentence boundaries up once per item: keep them in shared memory (one LDS instead of an L2 round trip)
  const int32_t* cu_g = cu;
  if (B + 1 <= kCuSmemInts) {
    for (int i = threadIdx.x; i <= B; i += kThreads) cu_smem[i] = cu_g[i];
    cu = cu_smem;
  }
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_qkv);
    for (int i = 0; i < kQkStages; ++i) {
      mbar_init(&full_qk[i], 1);
      mbar_init(&empty_qk[i], 8);
    }
    for (int i = 0; i < kVStages; ++i) {
      mbar_init(&full_v[i], 1);
      mbar_init(&empty_v[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  UnitStream u;
  u.init(cu, H, num_items, blockIdx.x, gridDim.x);
  int sq = 0, sv = 0;
  uint32_t phq = 0, phv = 0;

  if (wg_idx == 0) {
    // ============================ TMA producer ============================
    if (warp == 0 && lane == 0) {
      while (u.valid) {
        const int col = u.h * 64;
        const int qrow = u.tok0 + u.qt * 128, krow = u.tok0 + u.kt * 128;
        uint8_t* qk = smem_qk + sq * 2 * kTile;
        mbar_wait(&empty_qk[sq], phq ^ 1);
        mbar_arrive_expect_tx(&full_qk[sq], 2 * kTile);
        tma_load_2d(qk, &tm_qkv, &full_qk[sq], col, qrow);
        tma_load_2d(qk + kTile, &tm_qkv, &full_qk[sq], D + col, krow);
        mbar_wait(&empty_v[sv], phv ^ 1);
        mbar_arrive_expect_tx(&full_v[sv], kTile);
        tma_load_2d(smem_v + sv * kTile, &tm_qkv, &full_v[sv], 2 * D + col, krow);
        u.advance();
        if (++sq == kQkStages) { sq = 0; phq ^= 1; }
        if (++sv == kVStages) { sv = 0; phv ^= 1; }
      }
    }
  } else {
    // ============================ S, softmax, P.V: 64 query rows per warpgroup, a row = the 4 lanes of a quad ============
    const int cwg = wg_idx - 1;
    const int r_lo = cwg * 64 + (warp & 3) * 16 + (lane >> 2);  // query rows r_lo and r_lo + 8 of the tile
    const int cq = 2 * (lane & 3);                              // fragment columns 8 j + cq, + 1
    float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};  // l_run: this lane's share of the row sum
    float o[32];
    while (u.valid) {
      const int kv_valid = min(128, u.len - u.kt * 128);
      const bool active = u.qt * 128 + cwg * 64 < u.len;  // (warpgroup-uniform) this half of the query tile holds queries
      const bool last = (u.kt == u.nt - 1);
      if (u.kt == 0) { m_run[0] = m_run[1] = -CUDART_INF_F; l_run[0] = l_run[1] = 0.f; }
      float s[64];
      mbar_wait(&full_qk[sq], phq);
      if (active) {
        const uint8_t* base = smem_qk + sq * 2 * kTile;
        const uint64_t qd = wgmma_desc_kmajor_sw128(smem_u32(base) + cwg * 64 * 128);
        const uint64_t kd = wgmma_desc_kmajor_sw128(smem_u32(base + kTile));
        wgmma_fence_regs(s);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(s, qd + uint64_t(2 * k), kd + uint64_t(2 * k), k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_qk[sq]);  // Q and K are dead once S has retired
      uint32_t pa[8][4];
      float alpha[2] = {1.f, 1.f};
      if (active) {
        attn::mask_keys(s, kv_valid, cq);
        attn::online_softmax(s, m_run, l_run, alpha, pa);
      }
      mbar_wait(&full_v[sv], phv);
      if (active) attn::pv_accumulate(o, pa, alpha, wgmma_desc_mnmajor_sw128(smem_u32(smem_v + sv * kTile)), u.kt == 0);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_v[sv]);
      if (active && last) attn::store_rows(o, l_run, out, u.tok0, u.qt * 128 + r_lo, u.len, D, u.h * 64 + cq);
      u.advance();
      if (++sq == kQkStages) { sq = 0; phq ^= 1; }
      if (++sv == kVStages) { sv = 0; phv ^= 1; }
    }
  }
}

}  // namespace

int attention_packed(const __nv_bfloat16* qkv, const int32_t* cu_seqlens, int B, int H, long long total_tokens, int num_sms,
                     __nv_bfloat16* out, cudaStream_t stream) {
  if (B <= 0 || total_tokens <= 0) return 0;
  if (H <= 0 || (long long)B * H > INT_MAX) {  // the kernel counts (sentence, head) items in an int
    set_last_error("attention_packed: unsupported B=%d H=%d", B, H);
    return -1;
  }
  CUtensorMap tm;
  int rc = make_tmap_2d(&tm, qkv, 2, total_tokens, 3ll * H * 64, 3ll * H * 64, 128, 64);
  if (rc) return rc;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    SB_CUDA_CHECK(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  }
  long long items = (long long)B * H;
  long long grid = (num_sms > 0 ? num_sms : device_sm_count());
  if (grid > items) grid = items;
  attention_tc_kernel<<<(unsigned)grid, kThreads, kSmemBytes, stream>>>(tm, cu_seqlens, B, H, out);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace sb
