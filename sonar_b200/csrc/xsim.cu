// xsim cosine k-NN + margin scoring over sentence embeddings (BASELINE.json config 5).
// Not part of the reference repository (README.md:5 only names the task); algorithm = public LASER
// xsim.py, restated in oracle/xsim.py (SURVEY.md Appendix D).
//
// Pipeline for knn(x[n,d], y[m,d], k):
//   1. l2_normalize: fp32 rows -> unit-norm bf16 rows (+ fp64 norms)                     [HBM-bound]
//   2. gemm_bf16_topk: wgmma GEMM x^ . y^T whose epilogue keeps, per column half of a tile, a running top-16 per row
//      in registers (32 candidates per row) -- the n x m similarity matrix is never written  [tensor-bound]
//   3. exact re-rank of the 16 best of those 32 (by bf16 score) in fp64 from the RAW fp32 embeddings
//      (cos = <x,y> / (|x||y|)), order (score desc, index asc), keep k                   [gather, L2/HBM]
// so the final neighbours/scores do not depend on bf16 rounding as long as the true top-k are among the
// 16 best bf16 candidates.

#include "../../include/sonar_b200.h"
#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>
#include <cmath>

namespace sb {

// one warp per row: y = x / |x| (bf16), norm (fp64)
__global__ void __launch_bounds__(256)
l2_normalize_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ xn, double* __restrict__ norm, long long n,
                    int d) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const float4* xr = reinterpret_cast<const float4*>(x + row * d);
  double s = 0.0;
  for (int c = lane; c < d / 4; c += 32) {
    const float4 v = xr[c];
    s += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const double nr = sqrt(s);
  const float inv = (float)(1.0 / fmax(nr, 1e-30));
  uint2* out = reinterpret_cast<uint2*>(xn + row * d);
  for (int c = lane; c < d / 4; c += 32) {
    const float4 v = xr[c];
    out[c] = make_uint2(pack_bf16x2(v.x * inv, v.y * inv), pack_bf16x2(v.z * inv, v.w * inv));
  }
  if (lane == 0) norm[row] = nr;
}

// one warp per x row: the KC (<= 32) bf16 candidates of the row's lists are first cut to the KEEP best by bf16 score (one
// candidate per lane, rank by 32 shuffles), those get their exact fp64 cosine, and the best k by (score desc, index asc)
// are written
template <int KC, int KEEP>
__global__ void __launch_bounds__(256)
rerank_kernel(const float* __restrict__ x, const float* __restrict__ y, const double* __restrict__ nx,
              const double* __restrict__ ny, const float* __restrict__ cand_val, const int* __restrict__ cand_idx, int n,
              int m, int d, int k, double* __restrict__ out_val, int* __restrict__ out_idx) {
  static_assert(KC <= 32 && KEEP <= KC, "one candidate per lane");
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)row * d);
  int cj = (lane < KC) ? cand_idx[(long long)row * KC + lane] : -1;
  float cv = (lane < KC) ? cand_val[(long long)row * KC + lane] : -CUDART_INF_F;
  if (cj < 0 || cj >= m) { cj = -1; cv = -CUDART_INF_F; }
  int pre = 0;  // rank of this lane's candidate by (bf16 score desc, index asc); invalid ones rank last
  for (int c = 0; c < 32; ++c) {
    const float ov = __shfl_sync(0xffffffffu, cv, c);
    const int oj = __shfl_sync(0xffffffffu, cj, c);
    if (oj >= 0 && (cj < 0 || ov > cv || (ov == cv && oj < cj))) ++pre;
  }
  unsigned keep = __ballot_sync(0xffffffffu, cj >= 0 && pre < KEEP);
  double my_score = -CUDART_INF;
  int my_idx = 0x7fffffff;
  while (keep) {
    const int c = __ffs(keep) - 1;
    keep &= keep - 1;
    const int j = __shfl_sync(0xffffffffu, cj, c);
    const float4* yr = reinterpret_cast<const float4*>(y + (long long)j * d);
    double dot = 0.0;
    for (int q = lane; q < d / 4; q += 32) {
      const float4 a = xr[q], b = yr[q];
      dot += (double)a.x * b.x + (double)a.y * b.y + (double)a.z * b.z + (double)a.w * b.w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (lane == c) {
      my_score = dot / fmax(nx[row] * ny[j], 1e-300);
      my_idx = j;
    }
  }
  // rank of lane's candidate among the rescored ones (the others hold -inf / INT_MAX and rank last)
  int rank = 0;
  for (int c = 0; c < 32; ++c) {
    const double s = __shfl_sync(0xffffffffu, my_score, c);
    const int i = __shfl_sync(0xffffffffu, my_idx, c);
    if (s > my_score || (s == my_score && i < my_idx)) ++rank;
  }
  const bool valid = my_idx != 0x7fffffff;
  if (valid && rank < k) {
    out_val[(long long)row * k + rank] = my_score;
    out_idx[(long long)row * k + rank] = my_idx;
  }
  const int nvalid = __popc(__ballot_sync(0xffffffffu, valid));
  if (lane >= nvalid && lane < k) {  // fewer than k candidates (m < k): the tail is (-inf, -1)
    out_val[(long long)row * k + lane] = -CUDART_INF;
    out_idx[(long long)row * k + lane] = -1;
  }
}

// one thread per x row: margin scoring over the forward candidates (LASER xsim)
__global__ void margin_predict_kernel(const double* __restrict__ val_xy, const int* __restrict__ idx_xy,
                                      const double* __restrict__ val_yx, int n, int m, int k, int mode,
                                      int* __restrict__ pred) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mode == 0) {  // absolute: plain top-1 cosine
    pred[i] = idx_xy[(long long)i * k];
    return;
  }
  double avg_x = 0.0;
  for (int c = 0; c < k; ++c) avg_x += val_xy[(long long)i * k + c];
  avg_x /= (double)k;
  double best = -CUDART_INF;
  int best_j = -1;
  for (int c = 0; c < k; ++c) {
    const int j = idx_xy[(long long)i * k + c];
    if (j < 0 || j >= m) continue;
    double avg_y = 0.0;
    for (int q = 0; q < k; ++q) avg_y += val_yx[(long long)j * k + q];
    avg_y /= (double)k;
    const double denom = (avg_x + avg_y) / 2.0;
    const double cs = val_xy[(long long)i * k + c];
    const double score = (mode == 1) ? cs / denom : cs - denom;
    if (score > best) {  // strict: first maximum wins (lowest candidate rank)
      best = score;
      best_j = j;
    }
  }
  pred[i] = best_j;
}

// bf16-similarity candidates per row handed to the exact re-rank: one n-chunk -> gemm_topk_lists(1) lists of 16
constexpr int kXsimCands = kTopkListsPerChunk * kTopkCandidates;
static_assert(kXsimCands <= 32, "rerank_kernel maps one candidate to one lane");

// Few query rows (fewer 256-row tile pairs than SM pairs): the key rows are split into up to 16 chunks swept by different
// clusters, each writing its own two candidate lists; merge_lists_kernel then keeps the 32 best of them per row.
static int xsim_chunks(int n, int m) {
  int c = gemm_topk_chunks(n, m, 2, 0 /* SM count of the device */);
  if (c > 16) {
    const int tiles = (m + 255) / 256, tpc = (tiles + 15) / 16;
    c = (tiles + tpc - 1) / tpc;
  }
  return c;
}

// one warp per row: the 32 best of `total` (<= 512) candidates by (bf16 score desc, index asc) -> out [n, 32]
__global__ void __launch_bounds__(256)
merge_lists_kernel(const float* __restrict__ cand_val, const int* __restrict__ cand_idx, int total, int n, int m,
                   float* __restrict__ out_val, int* __restrict__ out_idx) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const float* cv = cand_val + (long long)row * total;
  const int* ci = cand_idx + (long long)row * total;
  out_val[(long long)row * 32 + lane] = -CUDART_INF_F;
  out_idx[(long long)row * 32 + lane] = -1;
  __syncwarp();
  for (int a = lane; a < total; a += 32) {
    const int ia = ci[a];
    if (ia < 0 || ia >= m) continue;
    const float va = cv[a];
    int rank = 0;
    for (int b = 0; b < total && rank < 32; ++b) {
      const int ib = ci[b];
      if (ib < 0 || ib >= m) continue;
      const float vb = cv[b];
      if (vb > va || (vb == va && ib < ia)) ++rank;
    }
    if (rank < 32) {
      out_val[(long long)row * 32 + rank] = va;
      out_idx[(long long)row * 32 + rank] = ia;
    }
  }
}

struct XsimWs {
  int chunks;
  float* merged_val;  // [n, 32], only when chunks > 1
  int* merged_idx;
  __nv_bfloat16* xn;
  __nv_bfloat16* yn;
  double* nx;
  double* ny;
  float* cand_val;
  int* cand_idx;
  size_t bytes;
};

static XsimWs carve_xsim(int n, int m, int d, void* base) {
  Carver c(base);
  XsimWs w;
  w.xn = c.take<__nv_bfloat16>((size_t)n * d * 2);
  w.yn = c.take<__nv_bfloat16>((size_t)m * d * 2);
  w.nx = c.take<double>((size_t)n * 8);
  w.ny = c.take<double>((size_t)m * 8);
  w.chunks = xsim_chunks(n, m);
  const size_t per_row = (size_t)gemm_topk_lists(w.chunks) * kTopkCandidates;
  w.cand_val = c.take<float>((size_t)n * per_row * 4);
  w.cand_idx = c.take<int>((size_t)n * per_row * 4);
  w.merged_val = nullptr;
  w.merged_idx = nullptr;
  if (w.chunks > 1) {
    w.merged_val = c.take<float>((size_t)n * 32 * 4);
    w.merged_idx = c.take<int>((size_t)n * 32 * 4);
  }
  w.bytes = c.off;
  return w;
}


// ---- one-pass bidirectional k-NN: the reverse direction (for every y row its best x rows) comes out of the SAME x . y^T GEMM
// through the sweep epilogue's column filter (ColFilter, sonar_b200_internal.h) ----
constexpr int kColCap = 256;          // candidate slots per y row (expected hits = 16 * kSampleStride = 128, see below)
constexpr int kSampleStride = 8;      // the thresholds come from every 8th x row: a 1/8-size GEMM instead of a second full one
constexpr float kThrSlack = 1e-5f;    // the sampled rows themselves must pass (>) their own score again in the full sweep

// one warp per y row: threshold = the 16th best bf16 score among the SAMPLED x rows.  The plain search keeps a row's 16 best
// candidates by bf16 score and re-scores those exactly; a subset's 16th best cannot exceed the 16th best over all rows, so
// everything the plain search would keep passes the threshold: the one-pass result is the two-pass result by construction,
// for any data.  How many rows pass is distribution-free as well: about 16 x kSampleStride (order statistics of a 1/8 sample).
__global__ void __launch_bounds__(256)
col_threshold_kernel(const float* __restrict__ cand_val, const int* __restrict__ cand_idx, int lists, int m,
                     float* __restrict__ thr) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= m) return;
  const int total = lists * kTopkCandidates;  // <= 32
  float v = -CUDART_INF_F;
  if (lane < total && cand_idx[(long long)row * total + lane] >= 0) v = cand_val[(long long)row * total + lane];
  int rank = 0;  // number of strictly better candidates (ties: lower lane first)
  for (int c = 0; c < 32; ++c) {
    const float o = __shfl_sync(0xffffffffu, v, c);
    if (o > v || (o == v && c < lane)) ++rank;
  }
  if (rank == kTopkCandidates - 1) thr[row] = (v > -CUDART_INF_F) ? v - kThrSlack : -CUDART_INF_F;  // < 16 sampled rows: all pass
}

// thr8[g] = min of the thresholds of columns 8g .. 8g+7: the sweep epilogue tests a row's 8-column maximum against it first
__global__ void group_min8_kernel(const float* __restrict__ thr, float* __restrict__ thr8, long long groups) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= groups) return;
  const float4 a = *reinterpret_cast<const float4*>(thr + g * 8), b = *reinterpret_cast<const float4*>(thr + g * 8 + 4);
  thr8[g] = fminf(fminf(fminf(a.x, a.y), fminf(a.z, a.w)), fminf(fminf(b.x, b.y), fminf(b.z, b.w)));
}

__global__ void fill_f32_kernel(float* p, long long n, float v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// one warp per y row j: its candidate x rows (bf16 score above the threshold) -> the 16 best by bf16 score -> exact fp64
// cosine from the raw fp32 embeddings -> the best k by (score desc, index asc)
__global__ void __launch_bounds__(256)
col_rerank_kernel(const float* __restrict__ x, const float* __restrict__ y, const double* __restrict__ nx,
                  const double* __restrict__ ny, const int* __restrict__ col_cnt, const uint2* __restrict__ col_buf, int n,
                  int m, int d, int k, double* __restrict__ out_val, int* __restrict__ out_idx, int* __restrict__ overflow) {
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= m) return;
  int cnt = col_cnt[j];
  if (cnt > kColCap) {  // more hits than slots (the threshold of this y row came out low): the caller redoes this row exactly
    if (lane == 0) atomicAdd(overflow, 1);
    if (lane < k) {
      out_val[(long long)j * k + lane] = -CUDART_INF;
      out_idx[(long long)j * k + lane] = -2;
    }
    return;
  }
  constexpr int PER = kColCap / 32;
  float cv[PER];
  int ci[PER];
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int p = q * 32 + lane;
    cv[q] = -CUDART_INF_F;
    ci[q] = 0x7fffffff;
    if (p < cnt) {
      const uint2 e = col_buf[(long long)j * kColCap + p];
      cv[q] = __uint_as_float(e.x);
      ci[q] = int(e.y);
    }
  }
  // 16 rounds of warp arg-max by (bf16 score desc, row asc): lane r keeps the r-th best candidate
  int sel = -1;
  for (int r = 0; r < kTopkCandidates; ++r) {
    float bv = -CUDART_INF_F;
    int bi = 0x7fffffff, bq = -1;
#pragma unroll
    for (int q = 0; q < PER; ++q)
      if (ci[q] != 0x7fffffff && (cv[q] > bv || (cv[q] == bv && ci[q] < bi))) { bv = cv[q]; bi = ci[q]; bq = q; }
    float wv = bv;
    int wi = bi;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, wv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, wi, o);
      if (ov > wv || (ov == wv && oi < wi)) { wv = ov; wi = oi; }
    }
    if (wi == 0x7fffffff) break;  // fewer than 16 candidates (warp-uniform)
    if (bq >= 0 && bi == wi) {    // row indices are unique within a column: exactly one lane owns the winner
#pragma unroll
      for (int q = 0; q < PER; ++q)
        if (q == bq) ci[q] = 0x7fffffff;
    }
    if (lane == r) sel = wi;
  }
  const float4* yr = reinterpret_cast<const float4*>(y + (long long)j * d);
  double my_score = -CUDART_INF;
  int my_idx = 0x7fffffff;
  for (int c = 0; c < kTopkCandidates; ++c) {
    const int i = __shfl_sync(0xffffffffu, sel, c);
    if (i < 0 || i >= n) continue;  // warp-uniform
    const float4* xr = reinterpret_cast<const float4*>(x + (long long)i * d);
    double dot = 0.0;
    for (int q = lane; q < d / 4; q += 32) {
      const float4 a = xr[q], b = yr[q];
      dot += (double)a.x * b.x + (double)a.y * b.y + (double)a.z * b.z + (double)a.w * b.w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    if (lane == c) {
      my_score = dot / fmax(nx[i] * ny[j], 1e-300);
      my_idx = i;
    }
  }
  int rank = 0;
  for (int c = 0; c < 32; ++c) {
    const double sv = __shfl_sync(0xffffffffu, my_score, c);
    const int iv = __shfl_sync(0xffffffffu, my_idx, c);
    if (sv > my_score || (sv == my_score && iv < my_idx)) ++rank;
  }
  const bool valid = my_idx != 0x7fffffff;
  if (valid && rank < k) {
    out_val[(long long)j * k + rank] = my_score;
    out_idx[(long long)j * k + rank] = my_idx;
  }
  const int nvalid = __popc(__ballot_sync(0xffffffffu, valid));
  if (lane >= nvalid && lane < k) {
    out_val[(long long)j * k + lane] = -CUDART_INF;
    out_idx[(long long)j * k + lane] = -1;
  }
}

struct XsimBidirWs {
  XsimWs base;
  float* s_val;   // [m, 32] sample-pass candidates of the y rows
  int* s_idx;
  float* thr;     // [m padded to 256]
  float* thr8;    // [m padded to 256, / 8] minimum over each 8 adjacent y rows
  int* cnt;       // [m]
  int* overflow;  // [1]
  uint2* buf;     // [m, kColCap]
  size_t bytes;
};

static XsimBidirWs carve_xsim_bidir(int n, int m, int d, void* base) {
  XsimBidirWs w;
  w.base = carve_xsim(n, m, d, base);
  Carver c(base);
  c.off = w.base.bytes;  // the reverse direction's buffers follow the forward layout
  const size_t mp = ((size_t)m + 255) / 256 * 256;
  w.s_val = c.take<float>((size_t)m * kXsimCands * 4);
  w.s_idx = c.take<int>((size_t)m * kXsimCands * 4);
  w.thr = c.take<float>(mp * 4);
  w.thr8 = c.take<float>(mp / 8 * 4);
  w.cnt = c.take<int>((size_t)m * 4);
  w.overflow = c.take<int>(256);
  w.buf = c.take<uint2>((size_t)m * kColCap * 8);
  w.bytes = c.off;
  return w;
}
}  // namespace sb

using namespace sb;

extern "C" {

int sb_xsim_workspace_bytes(int32_t n, int32_t m, int32_t d, size_t* bytes) {
  if (n <= 0 || m <= 0 || d <= 0 || !bytes) { set_last_error("sb_xsim_workspace_bytes: bad argument"); return SB_ERR_INVALID; }
  *bytes = carve_xsim(n, m, d, nullptr).bytes + kWorkspaceAlign;
  return SB_OK;
}

int sb_xsim_knn(const float* x, const float* y, int32_t n, int32_t m, int32_t d, int32_t k, double* out_val,
                int32_t* out_idx, void* workspace, size_t workspace_bytes, void* stream_v) {
  if (!x || !y || !out_val || !out_idx || !workspace) { set_last_error("sb_xsim_knn: null pointer"); return SB_ERR_INVALID; }
  if (n <= 0 || m <= 0) { set_last_error("sb_xsim_knn: empty input"); return SB_ERR_INVALID; }
  if (d <= 0 || d % 64 != 0) { set_last_error("sb_xsim_knn: embedding dim must be a multiple of 64 (got %d)", d); return SB_ERR_INVALID; }
  if (k <= 0 || k > kTopkCandidates) { set_last_error("sb_xsim_knn: k must be in [1, %d]", kTopkCandidates); return SB_ERR_INVALID; }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  XsimWs w;
  int rc = bind_workspace("sb_xsim_knn", workspace, workspace_bytes, &w, [&](void* p) { return carve_xsim(n, m, d, p); });
  if (rc) return rc;
  int sms = 0;
  if ((rc = require_hopper("sb_xsim_knn", &sms))) return rc;
  l2_normalize_kernel<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(x, w.xn, w.nx, n, d);
  l2_normalize_kernel<<<(unsigned)((m + 7) / 8), 256, 0, stream>>>(y, w.yn, w.ny, m, d);
  SB_CUDA_CHECK(cudaGetLastError());
  if ((rc = gemm_bf16_topk(w.xn, d, w.yn, d, n, m, d, w.cand_val, w.cand_idx, nullptr, w.chunks, 2, sms, stream)))
    return rc;
  const float* cv = w.cand_val;
  const int* ci = w.cand_idx;
  if (w.chunks > 1) {
    merge_lists_kernel<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(w.cand_val, w.cand_idx,
                                                                    gemm_topk_lists(w.chunks) * kTopkCandidates, n, m,
                                                                    w.merged_val, w.merged_idx);
    cv = w.merged_val;
    ci = w.merged_idx;
  }
  rerank_kernel<kXsimCands, kTopkCandidates><<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(x, y, w.nx, w.ny, cv, ci, n, m, d, k,
                                                                                          out_val, out_idx);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}


int sb_xsim_bidir_workspace_bytes(int32_t n, int32_t m, int32_t d, size_t* bytes) {
  if (n <= 0 || m <= 0 || d <= 0 || !bytes) { set_last_error("sb_xsim_bidir_workspace_bytes: bad argument"); return SB_ERR_INVALID; }
  *bytes = carve_xsim_bidir(n, m, d, nullptr).bytes + kWorkspaceAlign;
  return SB_OK;
}

int sb_xsim_knn_bidir(const float* x, const float* y, int32_t n, int32_t m, int32_t d, int32_t k, double* val_xy,
                      int32_t* idx_xy, double* val_yx, int32_t* idx_yx, int32_t* overflow_flag, void* workspace,
                      size_t workspace_bytes, void* stream_v) {
  if (!x || !y || !val_xy || !idx_xy || !val_yx || !idx_yx || !overflow_flag || !workspace) {
    set_last_error("sb_xsim_knn_bidir: null pointer");
    return SB_ERR_INVALID;
  }
  if (n <= 0 || m <= 0) { set_last_error("sb_xsim_knn_bidir: empty input"); return SB_ERR_INVALID; }
  if (d <= 0 || d % 64 != 0) { set_last_error("sb_xsim_knn_bidir: embedding dim must be a multiple of 64 (got %d)", d); return SB_ERR_INVALID; }
  if (k <= 0 || k > kTopkCandidates) { set_last_error("sb_xsim_knn_bidir: k must be in [1, %d]", kTopkCandidates); return SB_ERR_INVALID; }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  XsimBidirWs w;
  int rc = bind_workspace("sb_xsim_knn_bidir", workspace, workspace_bytes, &w,
                          [&](void* p) { return carve_xsim_bidir(n, m, d, p); });
  if (rc) return rc;
  int sms = 0;
  if ((rc = require_hopper("sb_xsim_knn_bidir", &sms))) return rc;
  l2_normalize_kernel<<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(x, w.base.xn, w.base.nx, n, d);
  l2_normalize_kernel<<<(unsigned)((m + 7) / 8), 256, 0, stream>>>(y, w.base.yn, w.base.ny, m, d);
  SB_CUDA_CHECK(cudaGetLastError());
  // (1) thresholds of the y rows from a strided sample of the x rows: y^ . xs^T with the usual running top-16 per row
  const int stride = n >= 512 * kSampleStride ? kSampleStride : (n >= 1024 ? n / 512 : 1);
  const int ns = (n + stride - 1) / stride;
  if ((rc = gemm_bf16_topk(w.base.yn, d, w.base.xn, (long long)stride * d, m, ns, d, w.s_val, w.s_idx, nullptr, 1, 2, sms,
                           stream)))
    return rc;
  const long long mp = ((long long)m + 255) / 256 * 256;
  fill_f32_kernel<<<(unsigned)((mp + 255) / 256), 256, 0, stream>>>(w.thr, mp, INFINITY);  // padding columns: never hit
  col_threshold_kernel<<<(unsigned)((m + 7) / 8), 256, 0, stream>>>(w.s_val, w.s_idx, gemm_topk_lists(1), m, w.thr);
  group_min8_kernel<<<(unsigned)((mp / 8 + 255) / 256), 256, 0, stream>>>(w.thr, w.thr8, mp / 8);
  SB_CUDA_CHECK(cudaGetLastError());
  SB_CUDA_CHECK(cudaMemsetAsync(w.cnt, 0, sizeof(int) * (size_t)m, stream));
  SB_CUDA_CHECK(cudaMemsetAsync(w.overflow, 0, sizeof(int), stream));
  // (2) ONE pass over x^ . y^T: per-row top-16 lists (forward direction) + per-column candidates above the thresholds
  ColFilter cf;
  cf.thr = w.thr; cf.thr8 = w.thr8; cf.cnt = w.cnt; cf.buf = w.buf; cf.cap = kColCap;
  rc = gemm_bf16_topk(w.base.xn, d, w.base.yn, d, n, m, d, w.base.cand_val, w.base.cand_idx, nullptr, 1, 2, sms, stream, cf);
  if (rc) return rc;
  rerank_kernel<kXsimCands, kTopkCandidates><<<(unsigned)((n + 7) / 8), 256, 0, stream>>>(
      x, y, w.base.nx, w.base.ny, w.base.cand_val, w.base.cand_idx, n, m, d, k, val_xy, idx_xy);
  col_rerank_kernel<<<(unsigned)((m + 7) / 8), 256, 0, stream>>>(x, y, w.base.nx, w.base.ny, w.cnt, w.buf, n, m, d, k, val_yx,
                                                                 idx_yx, w.overflow);
  SB_CUDA_CHECK(cudaGetLastError());
  SB_CUDA_CHECK(cudaMemcpyAsync(overflow_flag, w.overflow, sizeof(int), cudaMemcpyDeviceToDevice, stream));
  return SB_OK;
}

int sb_xsim_margin_predict(const double* val_xy, const int32_t* idx_xy, const double* val_yx, int32_t n, int32_t m,
                           int32_t k, int32_t margin_mode, int32_t* pred, void* stream_v) {
  if (!val_xy || !idx_xy || !pred || (margin_mode != 0 && !val_yx)) {
    set_last_error("sb_xsim_margin_predict: null pointer");
    return SB_ERR_INVALID;
  }
  if (margin_mode < 0 || margin_mode > 2 || n <= 0 || k <= 0) {
    set_last_error("sb_xsim_margin_predict: bad argument");
    return SB_ERR_INVALID;
  }
  margin_predict_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_v)>>>(
      val_xy, idx_xy, val_yx, n, m, k, margin_mode, pred);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

}  // extern "C"
