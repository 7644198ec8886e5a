// bf16 x bf16 -> fp32-accumulate GEMM on the Hopper tensor cores (wgmma, accumulators in registers),
// fed by TMA, warp-specialised, persistent.  C = epi(A[M,K] · W[N,K]^T + bias[N]).
//
// This is the contraction behind every `F.linear` of the SONAR text encoder layer
// (reference wiring: sonar/models/sonar_text/factory.py:130-153 -- q/k/v/out
// projections and the 1024->8192->1024 ReLU FFN; nn.Linear weight layout [out,in]).
//
// Tile shape per CTA: 128(M) x 256(N) x 64(K) per pipeline stage.  Two consumer warpgroups each own 64 rows of the
//   tile: four wgmma.m64n256k16 per stage into 128 fp32 accumulator registers per thread.
//   cta_group = 2: two CTAs of a cluster take the two 128-row halves of a 256-row tile and the same 256 columns;
//   each loads half of the W tile and TMA-multicasts it into both CTAs' shared memory, so W crosses L2 -> SM once
//   per pair.  cta_group = 1: independent CTAs.
// Warp roles (384 threads): warpgroup 0 = producer (one thread issues TMA; the group gives its registers away with
//   setmaxnreg), warpgroups 1-2 = MMA + epilogue.
// Epilogue, column-wise modes (bias, ReLU, SiLU, residual, accumulate, LnFold consumer): every thread applies bias and
//   activation to its accumulator fragments in registers and writes them straight into the 128B-swizzled staging
//   layout of the TMA store (stmatrix for bf16, st.shared.v2 for fp32), one 64-row x 128-byte box at a time, double
//   buffered, so the store of one box reads while the next is written.
// Epilogue, row-wise modes (LayerNorm statistics, running top-k / log-sum-exp): the fragments of 2 x 32 columns at a
//   time go through a padded shared-memory buffer so that ONE THREAD OWNS ONE ROW of 32 consecutive columns (thread t
//   of the warpgroup: row t % 64, column half t / 64 of the tile), then swizzled smem -> TMA store.
// LayerNorm folding (LnFold, sonar_b200_internal.h): a consumer GEMM scales its accumulator rows by the LayerNorm
// statistics of its input; the residual-stream GEMMs emit those statistics and the bf16 copy of the stream.
// Operand smem layout: K-major, 128-byte rows, SWIZZLE_128B (TMA writes it, wgmma reads it).

#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>

namespace sb {

// The row-wise epilogues need one thread per row (the fragment -> row transposition buffer); the others are column-wise.
constexpr bool epi_row_wise(int epi) { return epi == EPI_BIAS_RESIDUAL_STATS || epi == EPI_TOPK; }

// Shared memory: the row-wise epilogues keep 3 ring stages next to their transposition buffers (2 x 17 KB); the
// column-wise ones have no such buffer and spend the space on a 4th stage, so the producer can run 4 k-blocks of the next
// tile ahead while the epilogue runs.  The other layout that fits, 3 stages and four staging boxes per warpgroup (a whole
// bf16 tile, one store wait per tile), measured slower in the same call on an H100 80GB HBM3 (700 W): median 4.43 k against
// 4.48 k sentences/s over three alternating bench.py runs each, with a spread of 0.013 k and 0.033 k within each layout.
template <int kCtaGroup, int kEpi>
struct GemmCfg {
  static constexpr bool ROW_WISE = epi_row_wise(kEpi);
  static constexpr int BLOCK_M = 128;                 // rows per CTA (64 per consumer warpgroup)
  static constexpr int BLOCK_N = 256;                 // wgmma N
  static constexpr int BLOCK_K = 64;                  // 128 bytes of bf16 = one swizzle atom
  static constexpr int LOAD_N = BLOCK_N / kCtaGroup;  // W rows each CTA loads (multicast to the pair)
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGES = ROW_WISE ? 3 : 4;     // 48 KB per mainloop stage
  static constexpr int EPI_GROUPS = 2;                // column halves of a tile row = row-wise result lists per tile
  static constexpr int CD_BYTES = 2 * 64 * 128;       // per consumer warpgroup: two 64-row x 128-byte TMA boxes
  static constexpr int TRANS_LD = 68;                 // floats per row of the fragment -> row-per-thread buffer (64 + pad)
  static constexpr int TRANS_BYTES = ROW_WISE ? 64 * TRANS_LD * 4 : 0;
  static constexpr int LN_BYTES = 64 * 8;             // per consumer warpgroup: (mean, rstd) of its rows (LnFold consumer)
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES =
      STAGES * (A_BYTES + B_BYTES) + 2 * (CD_BYTES + TRANS_BYTES + LN_BYTES) + BAR_BYTES + 1024 /*align slack*/;
  static constexpr int THREADS = 384;
  static_assert(SMEM_BYTES <= 232448, "shared memory budget of one sm_90 block");
  static_assert(2 * STAGES * 8 <= BAR_BYTES, "ring barriers");
};

// Tile scheduler shared by the three warp roles (each role walks an identical copy).
// Default: tiles are dealt round-robin with n fastest, so the clusters running concurrently share A rows
// through L2 and every weight tile stays L2-resident.
// Sweep (top-k epilogue): a work item is (m-block, n-chunk); the cluster walks all n tiles of the chunk so the
// running top-k / log-sum-exp of a row lives in the epilogue thread's registers for the whole item.  Items of one
// m-block sit next to each other, and the same chunk of different m-blocks runs concurrently on different
// clusters, so W streams through L2 once.
template <bool kSweep>
struct TileSched {
  int num_m_tiles, num_n_tiles, cluster_id, num_clusters, n_chunks, tiles_per_chunk;
  int k_splits = 1;  // split-K (accumulate epilogue, few tiles): item = split * tiles + tile, `chunk` returns the split
  int i = 0, j = 0;
  __device__ __forceinline__ bool next(int& m_blk, int& n_blk, int& chunk, bool& first, bool& last) {
    if constexpr (!kSweep) {
      const int item = cluster_id + i * num_clusters;
      ++i;
      const int tiles = num_m_tiles * num_n_tiles;
      if (item >= tiles * k_splits) return false;
      const int tile = (k_splits == 1) ? item : item % tiles;
      chunk = (k_splits == 1) ? 0 : item / tiles;
      m_blk = tile / num_n_tiles;
      n_blk = tile % num_n_tiles;
      first = last = true;
      return true;
    } else {
      for (;;) {
        const int item = cluster_id + i * num_clusters;
        if (item >= num_m_tiles * n_chunks) return false;
        m_blk = item / n_chunks;
        chunk = item % n_chunks;
        const int n_begin = chunk * tiles_per_chunk;
        const int cnt = min(tiles_per_chunk, num_n_tiles - n_begin);
        if (j < cnt) {
          n_blk = n_begin + j;
          first = (j == 0);
          last = (j == cnt - 1);
          ++j;
          return true;
        }
        j = 0;
        ++i;
      }
    }
  }
};

// insert (v, idx) into a descending list kept in registers; equal values keep the earlier entry first.  Past the
// insertion point every entry moves down one place: the displaced entry must not be compared again, or it would pass
// the entries of its own value behind it and a tie at the list's end would lose its earliest entry.
template <int KC>
__device__ __forceinline__ void topk_insert(float (&tv)[KC], int (&ti)[KC], float v, int idx) {
  float cv = v;
  int ci = idx;
  bool shifting = false;
#pragma unroll
  for (int p = 0; p < KC; ++p) {
    const bool gt = shifting || cv > tv[p];
    shifting = gt;
    const float ov = tv[p];
    const int oi = ti[p];
    tv[p] = gt ? cv : ov;
    ti[p] = gt ? ci : oi;
    cv = gt ? ov : cv;
    ci = gt ? oi : ci;
  }
}


template <int kCtaGroup, int kEpi, typename OutT>
__global__ void __launch_bounds__(GemmCfg<kCtaGroup, kEpi>::THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                       const __grid_constant__ CUtensorMap tm_c, const float* __restrict__ bias,
                       const OutT* residual, long long ldr, int M, int N, int K, float* __restrict__ cand_val,
                       int* __restrict__ cand_idx, float* __restrict__ lse_part, int n_chunks, const LnFold lf,
                       const ColFilter cf, int k_splits, int* __restrict__ splitk_flags) {
  constexpr bool kSweep = (kEpi == EPI_TOPK);
  using Cfg = GemmCfg<kCtaGroup, kEpi>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + Cfg::STAGES * Cfg::A_BYTES;
  uint8_t* smem_cd = smem_b + Cfg::STAGES * Cfg::B_BYTES;
  uint8_t* smem_tr = smem_cd + 2 * Cfg::CD_BYTES;
  uint8_t* smem_ln = smem_tr + 2 * Cfg::TRANS_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_ln + 2 * Cfg::LN_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg_idx = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // (warp-uniform by construction)
  const uint32_t cta_rank = (kCtaGroup == 2) ? cluster_ctarank() : 0u;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    tma_prefetch_desc(&tm_c);
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);               // the producer's arrive.expect_tx (+ TMA bytes, the peer's W half included)
      mbar_init(&empty_bar[i], 8 * kCtaGroup);  // one arrive per consumer warp of every CTA that reads or fills the slot
    }
    fence_mbar_init();
  }
  if (kCtaGroup == 2) cluster_sync_all(); else __syncthreads();  // barriers of both CTAs live before any remote arrive

  const int tile_m = Cfg::BLOCK_M * kCtaGroup;
  const int num_m_tiles = (M + tile_m - 1) / tile_m;
  const int num_n_tiles = (N + Cfg::BLOCK_N - 1) / Cfg::BLOCK_N;  // N tail only with the top-k epilogue
  const int num_kb = K / Cfg::BLOCK_K;
  const int cluster_id = blockIdx.x / kCtaGroup;
  const int num_clusters = gridDim.x / kCtaGroup;
  TileSched<kSweep> sched{num_m_tiles, num_n_tiles, cluster_id, num_clusters, n_chunks,
                          (num_n_tiles + n_chunks - 1) / n_chunks, (kEpi == EPI_BIAS_ACCUM) ? k_splits : 1};
  // split-K: split s of a tile runs k-blocks [s * num_kb / k_splits, (s + 1) * num_kb / k_splits)
  auto kb_begin = [&](int split) { return (kEpi == EPI_BIAS_ACCUM && k_splits > 1) ? split * num_kb / k_splits : 0; };
  auto kb_end = [&](int split) { return (kEpi == EPI_BIAS_ACCUM && k_splits > 1) ? (split + 1) * num_kb / k_splits : num_kb; };
  int m_blk, n_blk, chunk;
  bool first_in_item, last_in_item;

  if (wg_idx == 0) {
    // ===================== TMA producer (one thread) =====================
    setmaxnreg_dec<40>();
    if (warp_idx == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      while (sched.next(m_blk, n_blk, chunk, first_in_item, last_in_item)) {
        const int m0 = m_blk * tile_m + int(cta_rank) * Cfg::BLOCK_M;
        const int n0 = n_blk * Cfg::BLOCK_N + int(cta_rank) * Cfg::LOAD_N;
        const int kb1 = kb_end(chunk);
        for (int kb = kb_begin(chunk); kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);  // the consumers of BOTH CTAs have released the slot
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::A_BYTES + Cfg::B_BYTES);
          tma_load_2d(smem_a + stage * Cfg::A_BYTES, &tm_a, &full_bar[stage], kb * Cfg::BLOCK_K, m0);
          uint8_t* b_dst = smem_b + stage * Cfg::B_BYTES + int(cta_rank) * (Cfg::LOAD_N * Cfg::BLOCK_K * 2);
          if (kCtaGroup == 2) tma_load_2d_multicast(b_dst, &tm_b, &full_bar[stage], kb * Cfg::BLOCK_K, n0, 0x3);
          else tma_load_2d(b_dst, &tm_b, &full_bar[stage], kb * Cfg::BLOCK_K, n0);
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers: 2 warpgroups x 64 rows, MMA then epilogue =====================
    setmaxnreg_inc<232>();
    const int cwg = wg_idx - 1;           // rows [64 cwg, 64 cwg + 64) of the CTA's tile
    const int t = threadIdx.x & 127;
    const int half = t >> 6;              // epilogue: columns [128 half, 128 half + 128) of the tile ...
    const int erow = t & 63;              // ... of row erow of this warpgroup
    const int row_in_tile = cwg * 64 + erow;
    const int frow = (warp_idx & 3) * 16 + (lane >> 2);  // accumulator fragment: rows frow and frow + 8
    uint8_t* smem_cd_wg = smem_cd + cwg * Cfg::CD_BYTES;
    float* trans = reinterpret_cast<float*>(smem_tr + cwg * Cfg::TRANS_BYTES);
    float2* ln_sm = reinterpret_cast<float2*>(smem_ln + cwg * Cfg::LN_BYTES);
    const uint32_t bar_id = 1 + cwg;  // named barrier of this warpgroup
    const uint64_t a_desc0 = wgmma_desc_kmajor_sw128(smem_u32(smem_a) + cwg * 64 * 128);
    const uint64_t b_desc0 = wgmma_desc_kmajor_sw128(smem_u32(smem_b));
    auto release = [&](int stage) {  // this warp's wgmma reads of the slot have retired
      if (kCtaGroup == 2) { if (lane < 2) mbar_arrive_cluster(&empty_bar[stage], lane); }
      else if (lane == 0) mbar_arrive(&empty_bar[stage]);
    };
    int stage = 0;
    uint32_t phase = 0;
    float acc[128];
    constexpr int KC = kTopkCandidates;
    [[maybe_unused]] float tv[KC];
    [[maybe_unused]] int ti[KC];
    [[maybe_unused]] float run_max = -CUDART_INF_F, run_sum = 0.f;  // online log-sum-exp of the row (optional)
    [[maybe_unused]] int q_n = 0;  // top-k sweep: candidates pending in this thread's shared-memory queue
    // ---- LayerNorm folding, consumer side: the (mean, M2) partials of this thread's input row are fetched ONE TILE AHEAD
    // (a lookahead copy of the scheduler names the next tile) so their latency hides under the current tile's mainloop ----
    [[maybe_unused]] bool fold_in = false;
    [[maybe_unused]] float2 part_next[8];
    [[maybe_unused]] TileSched<kSweep> sched_ahead = sched;
    [[maybe_unused]] auto fetch_parts = [&]() {
      int mb, nb, ch;
      bool f0, f1;
      if (!sched_ahead.next(mb, nb, ch, f0, f1)) return;
      const int r = mb * tile_m + int(cta_rank) * Cfg::BLOCK_M + row_in_tile;
      if (r < M) {
        const float2* sp = reinterpret_cast<const float2*>(lf.stats_in) + (long long)r * lf.chunks;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (i < lf.chunks) part_next[i] = sp[i];
      }
    };
    if constexpr (kEpi == EPI_BIAS || kEpi == EPI_BIAS_RELU) {
      fold_in = lf.stats_in != nullptr;
      if (fold_in) fetch_parts();
    }
    while (sched.next(m_blk, n_blk, chunk, first_in_item, last_in_item)) {
      const int m0 = m_blk * tile_m + int(cta_rank) * Cfg::BLOCK_M;
      const int n0 = n_blk * Cfg::BLOCK_N;
      const int grow = m0 + row_in_tile;
      [[maybe_unused]] float ln_mean = 0.f, ln_rstd = 1.f;
      if constexpr (kEpi == EPI_BIAS || kEpi == EPI_BIAS_RELU) {
        if (fold_in) {
          if (grow < M) {  // Chan merge of `chunks` partials of kLnPartCols columns each
            float msum = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (i < lf.chunks) msum += part_next[i].x;
            ln_mean = msum / float(lf.chunks);
            float m2 = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i)
              if (i < lf.chunks) { const float dm = part_next[i].x - ln_mean; m2 += part_next[i].y + float(kLnPartCols) * dm * dm; }
            ln_rstd = 1.0f / sqrtf(m2 / float(kLnPartCols * lf.chunks) + lf.eps);
          }
          // to the fragment layout (read after the mainloop; the previous tile read its values before its last store)
          if (half == 0) ln_sm[erow] = make_float2(ln_mean, ln_rstd);
          fetch_parts();  // for the next tile
        }
      }
      // ---- producer side: the first residual chunk of this thread's row is fetched while the MMAs run ----
      [[maybe_unused]] float4 rnext[8];
      [[maybe_unused]] float st_n = 0.f, st_mean = 0.f, st_m2 = 0.f;
      if constexpr (kEpi == EPI_BIAS_RESIDUAL_STATS) {
#pragma unroll
        for (int q = 0; q < 8; ++q) rnext[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (grow < M) {
          const float4* rp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(residual) + (long long)grow * ldr +
                                                             n0 + half * 128);
#pragma unroll
          for (int q = 0; q < 8; ++q) rnext[q] = rp[q];
        }
      }
      // ---- mainloop: one wgmma group per k-block, one group kept in flight ----
      {
        const int kb0 = kb_begin(chunk), kb1 = kb_end(chunk);
        auto issue = [&](bool first) {  // the four wgmma of the k-block in `stage`, as one group
          const uint64_t a_desc = a_desc0 + uint64_t(stage * (Cfg::A_BYTES >> 4));
          const uint64_t b_desc = b_desc0 + uint64_t(stage * (Cfg::B_BYTES >> 4));
          wgmma_fence_regs(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < Cfg::BLOCK_K / 16; ++k)
            wgmma_m64n256k16_ss(acc, a_desc + uint64_t(2 * k), b_desc + uint64_t(2 * k), (first && k == 0) ? 0u : 1u);
          wgmma_commit();
          wgmma_fence_regs(acc);
        };
        mbar_wait(&full_bar[stage], phase);
        issue(true);
        int prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        for (int kb = kb0 + 1; kb < kb1; ++kb) {
          mbar_wait(&full_bar[stage], phase);  // TMA bytes (both W halves) have landed
          issue(false);
          wgmma_wait<1>();  // the previous k-block has retired: its smem slot goes back to the producer(s)
          release(prev);
          prev = stage;
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        release(prev);
      }
      if constexpr (!Cfg::ROW_WISE) {
        // ---- column-wise epilogue from the accumulator fragments: rows frow and frow + 8, columns 8 j + 2 (lane % 4), + 1 ----
        // Box b = the warpgroup's 64 rows x columns [b * BOX_COLS, (b + 1) * BOX_COLS) of the tile, 128 bytes per row, in
        // the 128B-swizzled layout of the TMA store (16-byte chunk q of row r at q ^ (r % 8)).  Boxes alternate between
        // two staging buffers: before the barrier that publishes box b, thread 0 waits until the store of box b - 1 has
        // read its buffer, which box b + 1 is written into.
        constexpr int BOX_COLS = 128 / int(sizeof(OutT));
        constexpr int BOXES = Cfg::BLOCK_N / BOX_COLS;
        constexpr int BOX_BYTES = 64 * 128;
        constexpr int NBUF = Cfg::CD_BYTES / BOX_BYTES;
        static_assert(NBUF >= 2 && BOXES % NBUF == 0, "staging buffers must alternate the same way in every tile");
        const int fcol = 2 * (lane & 3);                     // first of this thread's two columns in each 8-column group
        const int grow_lo = m0 + cwg * 64 + frow, grow_hi = grow_lo + 8;
        if (fold_in) named_bar_sync(bar_id, 128);  // ln_sm of this tile is complete
        // split-K: the bias belongs to split 0, the later splits add their bare partial products
        const bool with_bias = !(kEpi == EPI_BIAS_ACCUM && chunk > 0);
        // fl(acc + bias) or the LnFold rstd * (acc - mean * c) + b', then the activation or the residual add
        auto epi = [&](float v, float b, float c, float2 ln, int grow, int col) -> float {
          float f = fold_in ? fmaf(ln.y, fmaf(-ln.x, c, v), b) : v + b;
          if constexpr (kEpi == EPI_BIAS_RELU) f = fmaxf(f, 0.0f);
          if constexpr (kEpi == EPI_BIAS_SILU) f = silu_fast(f);
          if constexpr (kEpi == EPI_BIAS_TANH) {
            // tanh(f), written in silu_fast's h = f / 2 form: h + h == f for every normal f, and with it ptxas allocates
            // the four tanh instantiations without spills (a plain tanh_approx(f) spills 8-48 bytes at the 168-register cap)
            const float h = 0.5f * f;
            f = tanh_approx(h + h);
          }
          if constexpr (kEpi == EPI_BIAS_RESIDUAL) {
            if (grow < M) {
              if constexpr (sizeof(OutT) == 4) f += reinterpret_cast<const float*>(residual)[(long long)grow * ldr + col];
              else f += __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(residual)[(long long)grow * ldr + col]);
            }
          }
          return f;
        };
        // the 8-column group j of the tile: bias (and LnFold colsum) of this thread's two columns, then both rows
        auto group = [&](int j, float (&o)[4]) {
          const int col = n0 + 8 * j + fcol;
          const float2 b2 = with_bias ? __ldg(reinterpret_cast<const float2*>(bias + col)) : make_float2(0.f, 0.f);
          const float2 c2 = fold_in ? __ldg(reinterpret_cast<const float2*>(lf.colsum + col)) : make_float2(0.f, 0.f);
          // (mean, rstd) of rows frow, frow + 8, read where they are used: not held in registers across the epilogue
          const float2 ln_lo = fold_in ? ln_sm[frow] : make_float2(0.f, 1.f);
          const float2 ln_hi = fold_in ? ln_sm[frow + 8] : make_float2(0.f, 1.f);
          o[0] = epi(acc[4 * j + 0], b2.x, c2.x, ln_lo, grow_lo, col);
          o[1] = epi(acc[4 * j + 1], b2.y, c2.y, ln_lo, grow_lo, col + 1);
          o[2] = epi(acc[4 * j + 2], b2.x, c2.x, ln_hi, grow_hi, col);
          o[3] = epi(acc[4 * j + 3], b2.y, c2.y, ln_hi, grow_hi, col + 1);
        };
        const uint32_t cd_base = smem_u32(smem_cd_wg);
#pragma unroll
        for (int b = 0; b < BOXES; ++b) {
          const uint32_t buf = cd_base + (b % NBUF) * BOX_BYTES;
          if constexpr (sizeof(OutT) == 2) {
            // stmatrix x4 per 16 columns: matrices (rows 0-7, j), (rows 8-15, j), (rows 0-7, j + 1), (rows 8-15, j + 1)
            // of the warp's 16 rows; lane l addresses row l % 8 of matrix l / 8
            const int mrow = (warp_idx & 3) * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
            for (int p = 0; p < BOX_COLS / 16; ++p) {
              const int j = b * (BOX_COLS / 8) + 2 * p;
              float o0[4], o1[4];
              group(j, o0);
              group(j + 1, o1);
              const int q = 2 * p + (lane >> 4);
              stmatrix_x4(buf + mrow * 128 + ((q ^ (lane & 7)) << 4), pack_bf16x2(o0[0], o0[1]), pack_bf16x2(o0[2], o0[3]),
                          pack_bf16x2(o1[0], o1[1]), pack_bf16x2(o1[2], o1[3]));
            }
          } else {
            // 8 bytes per row and group: byte 4 fcol of the group's 32 bytes
#pragma unroll
            for (int jj = 0; jj < BOX_COLS / 8; ++jj) {
              float o[4];
              group(b * (BOX_COLS / 8) + jj, o);
              const int q = 2 * jj + ((lane >> 1) & 1);
              const uint32_t a = buf + frow * 128 + ((q ^ (frow & 7)) << 4) + 8 * (lane & 1);
              st_shared_v2(a, o[0], o[1]);
              st_shared_v2(a + 8 * 128, o[2], o[3]);
            }
          }
          fence_proxy_async_smem();
          if (t == 0) tma_store_wait_read<NBUF - 2>();
          named_bar_sync(bar_id, 128);
          if (t == 0) {
            const int c0 = n0 + b * BOX_COLS, r0 = m0 + cwg * 64;
            if constexpr (kEpi == EPI_BIAS_ACCUM) {
              // Ordered split-K: the splits of a tile add into C one after the other (x + p0, + p1, + p2 -- the same sum on
              // every run).  Split s waits for the counter its predecessor leaves after ITS adds have completed; the
              // predecessor is a lower-numbered item, so it is already running on another resident cluster or finished.
              int* flag = nullptr;
              if (k_splits > 1) {
                flag = splitk_flags + ((long long)(m_blk * num_n_tiles + n_blk) * kCtaGroup + int(cta_rank)) * 2 + cwg;
                if (b == 0 && chunk > 0) {
                  while (ld_acquire_gpu(flag) != chunk) __nanosleep(64);
                  fence_proxy_async_all();
                }
              }
              tma_reduce_add_2d(&tm_c, reinterpret_cast<const void*>(smem_cd_wg + (b % NBUF) * BOX_BYTES), c0, r0);
              tma_store_commit();
              if (k_splits > 1 && b == BOXES - 1) {
                tma_store_wait_all<0>();  // this split's adds have been performed
                fence_proxy_async_all();
                __threadfence();
                st_release_gpu(flag, chunk == k_splits - 1 ? 0 : chunk + 1);  // the last split re-arms the counter
              }
            } else {
              tma_store_2d(&tm_c, smem_cd_wg + (b % NBUF) * BOX_BYTES, c0, r0);
              tma_store_commit();
            }
          }
        }
        continue;
      }
      // fragments of piece s (columns 32 s .. 32 s + 31 of both column halves) -> trans[row][half * 32 + column]
      auto stage_piece = [&](int s) {
        named_bar_sync(bar_id, 128);  // the previous piece has been read by every thread
        float* tr = trans + frow * Cfg::TRANS_LD + 2 * (lane & 3);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 16 * hh + 4 * s + jj;
            *reinterpret_cast<float2*>(tr + 32 * hh + 8 * jj) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(tr + 8 * Cfg::TRANS_LD + 32 * hh + 8 * jj) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
          }
        named_bar_sync(bar_id, 128);
      };
      auto load_piece = [&](uint32_t (&v)[32]) {
        const float4* src = reinterpret_cast<const float4*>(trans + erow * Cfg::TRANS_LD + half * 32);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 x = src[i];
          v[4 * i] = __float_as_uint(x.x); v[4 * i + 1] = __float_as_uint(x.y);
          v[4 * i + 2] = __float_as_uint(x.z); v[4 * i + 3] = __float_as_uint(x.w);
        }
      };
      if constexpr (kEpi == EPI_TOPK) {
        // ---- running per-row top-KC over the whole sweep of n tiles (no C matrix is ever written) ----
        if (first_in_item) {
#pragma unroll
          for (int p = 0; p < KC; ++p) { tv[p] = -CUDART_INF_F; ti[p] = -1; }
          run_max = -CUDART_INF_F;
          run_sum = 0.f;
        }
        // each thread sweeps ITS column half of the row and keeps its own list: a row ends up with EPI_GROUPS lists per
        // n-chunk, merged by the caller's next kernel.
        // Candidates are not inserted where they are found: a thread PUSHES (value, column) of every element above its
        // current 16th value into a small queue in shared memory (the idle output staging buffer) and the warp drains all
        // 32 queues together when one fills up.  Inserting in place costs the whole warp ~80 instructions whenever ANY lane
        // qualifies (32 rows with independent insertion events -> ~2500 instructions per tile per warp on random logits);
        // drained together, a round of insertions serves every lane that has one pending.  Same elements, same order per
        // row, same result bit for bit.
        const bool cf_on = cf.thr != nullptr && grow < M;
        constexpr int kQ = 16;  // queue entries per thread; drained once any lane holds more than kQ - 8
        uint2* queue = reinterpret_cast<uint2*>(smem_cd_wg) + t;  // entry e of this thread at queue[e * 128]
        auto drain = [&]() {
          const int rounds = __reduce_max_sync(0xffffffffu, q_n);
          for (int r = 0; r < rounds; ++r) {
            if (r < q_n) {
              const uint2 e = queue[r * 128];
              const float x = __uint_as_float(e.x);
              if (x > tv[KC - 1]) topk_insert<KC>(tv, ti, x, int(e.y));
            }
          }
          q_n = 0;
        };
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          uint32_t v[32];
          stage_piece(s);
          load_piece(v);
          const int gcol = n0 + half * 128 + s * 32;
          if (gcol + 32 > N) {  // ragged last tile: columns >= N are zero-filled operands, not candidates
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (gcol + j >= N) v[j] = __float_as_uint(-CUDART_INF_F);
          }
          // maxima of the four 8-column groups: shared by the candidate pre-filter and the log-sum-exp
          float gm[4];
#pragma unroll
          for (int g8 = 0; g8 < 4; ++g8) {
            float mx = __uint_as_float(v[g8 * 8]);
#pragma unroll
            for (int j = 1; j < 8; ++j) mx = fmaxf(mx, __uint_as_float(v[g8 * 8 + j]));
            gm[g8] = mx;
          }
          if (lse_part != nullptr) {  // online log-sum-exp over every column of the row (fp32, like log_softmax)
            const float cm = fmaxf(fmaxf(gm[0], gm[1]), fmaxf(gm[2], gm[3]));
            if (cm > run_max) {
              run_sum *= __expf(run_max - cm);  // exp(-inf) = 0 on the first chunk
              run_max = cm;
            }
            if (run_max > -CUDART_INF_F) {
              float cs = 0.f;
#pragma unroll
              for (int j = 0; j < 32; ++j) cs += __expf(__uint_as_float(v[j]) - run_max);
              run_sum += cs;
            }
          }
          const float thr = tv[KC - 1];  // (stale between drains: a few extra pushes, rejected when drained)
          float t8[4] = {CUDART_INF_F, CUDART_INF_F, CUDART_INF_F, CUDART_INF_F};  // column filter off / rows beyond M: never hit
          if (cf_on) {
            const float4 tt = __ldg(reinterpret_cast<const float4*>(cf.thr8 + (gcol >> 3)));
            t8[0] = tt.x; t8[1] = tt.y; t8[2] = tt.z; t8[3] = tt.w;
          }
#pragma unroll
          for (int g8 = 0; g8 < 4; ++g8) {
            if (gm[g8] > t8[g8]) {  // column filter: some element of these 8 is above its COLUMN's threshold (rare)
              const float4 t0 = *reinterpret_cast<const float4*>(cf.thr + gcol + g8 * 8);  // (not __ldg: columns get closed)
              const float4 t1 = *reinterpret_cast<const float4*>(cf.thr + gcol + g8 * 8 + 4);
              const float th[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float x = __uint_as_float(v[g8 * 8 + j]);
                if (x > th[j]) {
                  const int col = gcol + g8 * 8 + j;
                  const int slot = atomicAdd(cf.cnt + col, 1);
                  if (slot < cf.cap) cf.buf[(long long)col * cf.cap + slot] = make_uint2(__float_as_uint(x), uint32_t(grow));
                  else cf.thr[col] = CUDART_INF_F;  // full: the caller redoes this column; stop collecting for it
                }
              }
            }
            if (gm[g8] > thr) {
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float x = __uint_as_float(v[g8 * 8 + j]);
                if (x > thr) {
                  queue[q_n * 128] = make_uint2(__float_as_uint(x), uint32_t(gcol + g8 * 8 + j));
                  ++q_n;
                }
              }
            }
            if (__any_sync(0xffffffffu, q_n > kQ - 8)) drain();
          }
        }
        if (last_in_item) drain();
        if (last_in_item && grow < M) {
          const long long slot = ((long long)grow * n_chunks + chunk) * Cfg::EPI_GROUPS + half;
#pragma unroll
          for (int p = 0; p < KC; ++p) {
            cand_val[slot * KC + p] = tv[p];
            cand_idx[slot * KC + p] = ti[p];
          }
          if (lse_part != nullptr) {
            lse_part[slot * 2] = run_max;
            lse_part[slot * 2 + 1] = run_sum;
          }
        }
        continue;
      }
      // ---- residual + LayerNorm statistics (EPI_BIAS_RESIDUAL_STATS, fp32 C): one row of 32 columns per thread and piece ----
      if constexpr (kEpi == EPI_BIAS_RESIDUAL_STATS) {
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          if (t == 0) tma_store_wait_read<0>();  // the staging buffer is free again (ordered by stage_piece's barrier)
          uint32_t v[32];
          stage_piece(s);
          load_piece(v);
          uint8_t* cd_row = smem_cd_wg + half * (64 * 128) + erow * 128;
          const int gcol = n0 + half * 128 + s * 32;
          float f[32];
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + gcol + j));
            f[j + 0] = __uint_as_float(v[j + 0]) + b4.x;
            f[j + 1] = __uint_as_float(v[j + 1]) + b4.y;
            f[j + 2] = __uint_as_float(v[j + 2]) + b4.z;
            f[j + 3] = __uint_as_float(v[j + 3]) + b4.w;
          }
          // x_new = x + (acc + bias): the residual chunk was fetched one piece ahead; fetch the next one now
          float4 rcur[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) rcur[q] = rnext[q];
          if (s + 1 < 4 && grow < M) {
            const float4* rp = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(residual) +
                                                               (long long)grow * ldr + gcol + 32);
#pragma unroll
            for (int q = 0; q < 8; ++q) rnext[q] = rp[q];
          }
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            f[4 * q + 0] += rcur[q].x; f[4 * q + 1] += rcur[q].y; f[4 * q + 2] += rcur[q].z; f[4 * q + 3] += rcur[q].w;
          }
          // running (mean, M2) of the row over this thread's half of the tile: two-pass inside the piece, Chan merge across
          float cs = 0.f;
#pragma unroll
          for (int j = 0; j < 32; ++j) cs += f[j];
          const float cm = cs * (1.0f / 32.0f);
          float cq = 0.f;
#pragma unroll
          for (int j = 0; j < 32; ++j) { const float dv = f[j] - cm; cq = fmaf(dv, dv, cq); }
          const float n_new = st_n + 32.f;
          const float dlt = cm - st_mean;
          st_mean = fmaf(dlt, 32.f / n_new, st_mean);
          st_m2 += cq + dlt * dlt * (st_n * 32.f / n_new);
          st_n = n_new;
          if (grow < M) {  // bf16 copy of the new residual stream: the A operand of the next (LayerNorm-folded) GEMM
            uint4* hp = reinterpret_cast<uint4*>(lf.h_out + (long long)grow * lf.ldh + gcol);
#pragma unroll
            for (int q = 0; q < 4; ++q)
              hp[q] = make_uint4(pack_bf16x2(f[8 * q], f[8 * q + 1]), pack_bf16x2(f[8 * q + 2], f[8 * q + 3]),
                                 pack_bf16x2(f[8 * q + 4], f[8 * q + 5]), pack_bf16x2(f[8 * q + 6], f[8 * q + 7]));
            if (s == 3)  // this thread's half of the tile row: kLnPartCols columns
              reinterpret_cast<float2*>(lf.stats_out)[((long long)grow * num_n_tiles + n_blk) * Cfg::EPI_GROUPS + half] =
                  make_float2(st_mean, st_m2);
          }
          // 128B-swizzled staging row: logical 16B chunk q lives at physical chunk q ^ (row % 8)
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int phys = q ^ (erow & 7);
            *reinterpret_cast<float4*>(cd_row + phys * 16) = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
          }
          fence_proxy_async_smem();  // both halves' [64 x 128 B] chunks are complete: two TMA stores
          named_bar_sync(bar_id, 128);
          if (t == 0) {
            const int c0 = n0 + s * 32, r0 = m0 + cwg * 64;
            tma_store_2d(&tm_c, smem_cd_wg, c0, r0);
            tma_store_2d(&tm_c, smem_cd_wg + 64 * 128, c0 + 128, r0);
            tma_store_commit();
          }
        }
      }
    }
    if (t == 0) tma_store_wait_all<0>();
  }

  // ===================== teardown =====================
  if (kCtaGroup == 2) cluster_sync_all();  // no CTA exits while its peer may still multicast into it or arrive on its barriers
}

// ----------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess || !p) {
      set_last_error("cuTensorMapEncodeTiled driver entry point not available");
      return nullptr;
    }
    fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }
  return fn;
}

// 2-D row-major tensor [rows, cols] with leading dimension ld (elements); box = [box_rows, box_cols];
// inner box extent must be exactly 128 bytes (SWIZZLE_128B).
int make_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, long long rows, long long cols, long long ld,
                 int box_rows, int box_cols) {
  PFN_tmapEncodeTiled enc = get_encode_fn();
  if (!enc) return -3;
  CUtensorMapDataType dt = (elem_bytes == 2) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * (cuuint64_t)elem_bytes};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  if (box_cols * elem_bytes != 128) {
    set_last_error("make_tmap_2d: inner box must span 128 bytes");
    return -1;
  }
  CUresult r = enc(out, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld cols=%lld ld=%lld elem=%d)", (int)r,
                   rows, cols, ld, elem_bytes);
    return -3;
  }
  return 0;
}

template <int kCtaGroup, int kEpi, typename OutT>
static int launch_inst(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const float* bias,
                       const void* residual, long long ldr, int M, int N, int K, int num_sms, cudaStream_t stream,
                       float* cand_val = nullptr, int* cand_idx = nullptr, float* lse_part = nullptr,
                       int n_chunks = 1, const LnFold& lf = LnFold(), const ColFilter& cf = ColFilter(), int k_splits = 1,
                       int* splitk_flags = nullptr) {
  using Cfg = GemmCfg<kCtaGroup, kEpi>;
  auto kern = gemm_bf16_wgmma_kernel<kCtaGroup, kEpi, OutT>;
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set)) {
    SB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  }
  const int tile_m = Cfg::BLOCK_M * kCtaGroup;
  const long long num_m_tiles = (M + tile_m - 1) / tile_m;
  const long long num_tiles = num_m_tiles * ((N + Cfg::BLOCK_N - 1) / Cfg::BLOCK_N);
  long long clusters = num_sms / kCtaGroup;
  if (clusters > num_tiles * k_splits) clusters = num_tiles * k_splits;
  if (kEpi == EPI_TOPK && clusters > num_m_tiles * n_chunks) clusters = num_m_tiles * n_chunks;  // whole items
  if (clusters < 1) clusters = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(clusters * kCtaGroup), 1, 1);
  cfg.blockDim = dim3(Cfg::THREADS, 1, 1);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCtaGroup;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (kCtaGroup == 2) {
    // the persistent grid (and the ordered split-K hand-over) needs every cluster resident at once
    int max_clusters = 0;
    SB_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&max_clusters, kern, &cfg));
    if (max_clusters < 1) {
      set_last_error("gemm_bf16: no 2-CTA cluster of the GEMM kernel fits on this device");
      return -2;
    }
    if (clusters > max_clusters) cfg.gridDim.x = (unsigned)(max_clusters * kCtaGroup);
  }
  SB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, ta, tb, tc, bias, reinterpret_cast<const OutT*>(residual), ldr, M, N, K,
                                   cand_val, cand_idx, lse_part, n_chunks, lf, cf, k_splits, splitk_flags));
  return 0;
}

// Number of n-chunks the top-k sweep is split into so that (m-blocks x chunks) fills the clusters.
int gemm_topk_chunks(int M, int N, int cta_group, int num_sms) {
  const int cg = (cta_group == 1) ? 1 : 2;
  const int clusters = (num_sms > 0 ? num_sms : device_sm_count()) / cg;
  const int num_m_tiles = (M + 128 * cg - 1) / (128 * cg);
  const int num_n_tiles = (N + 255) / 256;
  int want = clusters / num_m_tiles;
  if (want < 1) want = 1;
  if (want > num_n_tiles) want = num_n_tiles;
  const int tpc = (num_n_tiles + want - 1) / want;
  return (num_n_tiles + tpc - 1) / tpc;  // every chunk non-empty
}

// Per-row top-kTopkCandidates of A[M,K] . W[N,K]^T (bf16 operands, fp32 accumulate) without materialising
// the product.  Outputs are per (row, list) with gemm_topk_lists(n_chunks) = 2 * n_chunks lists per row (one per n-chunk and
// column half of the 256-column tiles; a list covers a disjoint subset of the columns): cand_val / cand_idx [M, lists, kTopkCandidates]
// sorted by value descending, and (optional) lse_part [M, lists, 2] = (max, sum exp(v - max)) over the list's columns.
int gemm_bf16_topk(const __nv_bfloat16* A, long long lda, const __nv_bfloat16* W, long long ldw, int M, int N, int K,
                   float* cand_val, int* cand_idx, float* lse_part, int n_chunks, int cta_group, int num_sms,
                   cudaStream_t stream, const ColFilter& cf) {
  if (M <= 0 || N <= 0) return 0;
  if (cf.thr != nullptr && (!cf.thr8 || !cf.cnt || !cf.buf || cf.cap <= 0)) {
    set_last_error("gemm_bf16_topk: column filter needs cnt, buf and a positive capacity");
    return -1;
  }
  if (K % 64 != 0 || K <= 0) {
    set_last_error("gemm_bf16_topk: K must be a positive multiple of 64 (got %d)", K);
    return -1;
  }
  const int num_n_tiles = (N + 255) / 256;
  if (n_chunks < 1 || n_chunks > num_n_tiles ||
      ((num_n_tiles + n_chunks - 1) / n_chunks) * (n_chunks - 1) >= num_n_tiles) {
    set_last_error("gemm_bf16_topk: invalid n_chunks=%d for %d n-tiles", n_chunks, num_n_tiles);
    return -1;
  }
  const int cg = (cta_group == 1) ? 1 : 2;
  CUtensorMap ta, tb;
  int rc;
  if ((rc = make_tmap_2d(&ta, A, 2, M, K, lda, 128, 64))) return rc;
  if ((rc = make_tmap_2d(&tb, W, 2, N, K, ldw, 256 / cg, 64))) return rc;
  const int sms = num_sms > 0 ? num_sms : device_sm_count();
  if (cg == 2)
    return launch_inst<2, EPI_TOPK, float>(ta, tb, ta /*unused*/, nullptr, nullptr, 0, M, N, K, sms, stream, cand_val,
                                           cand_idx, lse_part, n_chunks, LnFold(), cf);
  return launch_inst<1, EPI_TOPK, float>(ta, tb, ta /*unused*/, nullptr, nullptr, 0, M, N, K, sms, stream, cand_val,
                                         cand_idx, lse_part, n_chunks, LnFold(), cf);
}

int gemm_bf16(const GemmArgs& g, cudaStream_t stream) {
  if (g.M <= 0) return 0;
  if (g.allow_skinny && gemm_skinny_eligible(g) && !g.lf.stats_in && g.epi != EPI_BIAS_RESIDUAL_STATS)
    return gemm_skinny(g, stream);
  if (g.N % 256 != 0 || g.K % 64 != 0 || g.K <= 0 || g.N <= 0) {
    set_last_error("gemm_bf16: need N %% 256 == 0 and K %% 64 == 0 (got M=%d N=%d K=%d)", g.M, g.N, g.K);
    return -1;
  }
  if (g.epi == EPI_BIAS_RESIDUAL && !g.residual) {
    set_last_error("gemm_bf16: residual epilogue without residual pointer");
    return -1;
  }
  if (!g.bias) {
    set_last_error("gemm_bf16: bias pointer is required");
    return -1;
  }
  const int cg = (g.cta_group == 1) ? 1 : 2;
  const int out_bytes = g.out_fp32 ? 4 : 2;
  CUtensorMap ta, tb, tc;
  int rc;
  if ((rc = make_tmap_2d(&ta, g.A, 2, g.M, g.K, g.lda, 128, 64))) return rc;
  if ((rc = make_tmap_2d(&tb, g.W, 2, g.N, g.K, g.ldw, 256 / cg, 64))) return rc;
  if ((rc = make_tmap_2d(&tc, g.C, out_bytes, g.M, g.N, g.ldc, 64, 128 / out_bytes))) return rc;
  const int sms = g.num_sms > 0 ? g.num_sms : device_sm_count();
  int epi = g.epi;
  if (epi == EPI_BIAS_RESIDUAL && g.out_fp32 && g.residual == g.C && g.ldr == g.ldc) epi = EPI_BIAS_ACCUM;
  if (epi == EPI_BIAS_ACCUM && !g.out_fp32) {
    set_last_error("gemm_bf16: accumulate epilogue needs fp32 output");
    return -1;
  }

  // ---- LayerNorm folding (LnFold) ----
  if (g.lf.stats_in != nullptr) {  // consumer
    if ((epi != EPI_BIAS && epi != EPI_BIAS_RELU) || !g.lf.colsum || g.lf.chunks < 1 || g.lf.chunks > 8 ||
        g.K != kLnPartCols * g.lf.chunks) {
      set_last_error("gemm_bf16: folded LayerNorm input needs a bias / bias+ReLU epilogue and K = 128 * chunks <= 1024 "
                     "(K=%d chunks=%d)", g.K, g.lf.chunks);
      return -1;
    }
  }
  if (epi == EPI_BIAS_RESIDUAL_STATS) {  // producer
    if (!g.out_fp32 || !g.residual || !g.lf.h_out || !g.lf.stats_out || g.lf.ldh < g.N) {
      set_last_error("gemm_bf16: the residual+statistics epilogue needs fp32 C, a residual, h_out and stats_out");
      return -1;
    }
  } else if (g.lf.h_out != nullptr || g.lf.stats_out != nullptr) {
    set_last_error("gemm_bf16: h_out / stats_out are outputs of EPI_BIAS_RESIDUAL_STATS only");
    return -1;
  }

  // Ordered split-K for the accumulate epilogue when the tiles do not fill the machine (the decoder's FFN output
  // projection at 2 560 rows: 40 tile pairs on 66 SM pairs): pick the split count with the fewest k-blocks on the
  // critical path, ~8 k-blocks charged per item for its epilogue and hand-over.
  if (epi == EPI_BIAS_ACCUM && cg == 2 && g.splitk_flags != nullptr) {
    const long long tiles = (long long)((g.M + 255) / 256) * (g.N / 256);
    const long long clusters = sms / 2;
    const int num_kb = g.K / 64;
    int best = 1;
    double best_cost = 1e30;
    for (int ks = 1; ks <= 4; ++ks) {
      if (num_kb / ks < 8) break;
      const double cost = double((tiles * ks + clusters - 1) / clusters) * (double(num_kb) / ks + 8.0);
      if (cost < best_cost * 0.95) { best_cost = cost; best = ks; }  // a later candidate must win by 5 %
    }
    if (best > 1 && tiles * 2 * 2 <= g.splitk_flags_len)
      return launch_inst<2, EPI_BIAS_ACCUM, float>(ta, tb, tc, g.bias, g.residual, g.ldr, g.M, g.N, g.K, sms, stream, nullptr,
                                                   nullptr, nullptr, 1, LnFold(), ColFilter(), best, g.splitk_flags);
  }

#define SB_DISPATCH(CG, EPI, T)                                                                                   \
  return launch_inst<CG, EPI, T>(ta, tb, tc, g.bias, g.residual, g.ldr, g.M, g.N, g.K, sms, stream, nullptr, nullptr, \
                                 nullptr, 1, g.lf)
#define SB_DISPATCH_EPI(CG, T)                                              \
  switch (epi) {                                                            \
    case EPI_BIAS: SB_DISPATCH(CG, EPI_BIAS, T);                            \
    case EPI_BIAS_RELU: SB_DISPATCH(CG, EPI_BIAS_RELU, T);                  \
    case EPI_BIAS_SILU: SB_DISPATCH(CG, EPI_BIAS_SILU, T);                  \
    case EPI_BIAS_TANH: SB_DISPATCH(CG, EPI_BIAS_TANH, T);                  \
    case EPI_BIAS_RESIDUAL: SB_DISPATCH(CG, EPI_BIAS_RESIDUAL, T);          \
    case EPI_BIAS_ACCUM: SB_DISPATCH(CG, EPI_BIAS_ACCUM, float);            \
    case EPI_BIAS_RESIDUAL_STATS: SB_DISPATCH(CG, EPI_BIAS_RESIDUAL_STATS, float); \
    default: set_last_error("gemm_bf16: bad epilogue %d", epi); return -1;  \
  }
  if (cg == 2) {
    if (g.out_fp32) { SB_DISPATCH_EPI(2, float) } else { SB_DISPATCH_EPI(2, __nv_bfloat16) }
  } else {
    if (g.out_fp32) { SB_DISPATCH_EPI(1, float) } else { SB_DISPATCH_EPI(1, __nv_bfloat16) }
  }
#undef SB_DISPATCH
#undef SB_DISPATCH_EPI
  return -1;
}

}  // namespace sb
