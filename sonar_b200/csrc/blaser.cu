// BLASER 2.0 translation-quality scoring over sentence embeddings (BlaserModel.forward, sonar/models/blaser/model.py:82-125):
//   F.normalize(src, mt[, ref]) -> featurize_input -> [Linear -> Tanh] x num_hidden -> Linear(K_last -> 1)
// One forward is: blaser_featurize_kernel (bf16 feature rows, the first GEMM's A operand), one wgmma GEMM per hidden layer
// with the tanh epilogue (the last one writes fp32), and blaser_output_kernel (the final dot product).  Every kernel does
// the same arithmetic in the same order for a row whatever the other rows are, so a pair's score does not depend on the
// batch it is scored in, bit for bit.

#include "common.cuh"
#include "sonar_b200_internal.h"

#include <algorithm>
#include <memory>
#include <new>
#include <vector>

using namespace sb;

namespace {

constexpr int kWarpsPerCta = 8;
constexpr float kNormEps = 1e-12f;  // F.normalize's default eps

__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ void store8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) =
      make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

__device__ __forceinline__ float sum_sq8(const float* p, float acc) {
  float v[8];
  load8(p, v);
#pragma unroll
  for (int i = 0; i < 8; ++i) acc = fmaf(v[i], v[i], acc);
  return acc;
}

// One warp per row; lane l handles the 8-column chunks l, l + 32, ... of E (16-byte loads and stores).
//   COMET (kQE = false): out[r] = [ref, mt, src*mt, ref*mt, |mt-src|, |mt-ref|]   (model.py:104-114)
//   QE    (kQE = true):  out[r] = [src, mt, src*mt, |mt-src|]                     (model.py:116-124), ref is never read
// With `normalize`, each input row is first divided by max(||row||_2, 1e-12) as F.normalize does (a zero row stays zero);
// the norms are fp32 sums of squares.
template <bool kQE, typename OutT>
__global__ void __launch_bounds__(kWarpsPerCta * 32) blaser_featurize_kernel(const float* __restrict__ src,
                                                                             const float* __restrict__ mt,
                                                                             const float* __restrict__ ref, long long ld,
                                                                             int rows, int E, int normalize,
                                                                             OutT* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* s = src + (long long)row * ld;
  const float* m = mt + (long long)row * ld;
  const float* r = kQE ? nullptr : ref + (long long)row * ld;
  const int chunks = E / 8;
  float ds = 1.f, dm = 1.f, dr = 1.f;
  if (normalize) {
    float ss = 0.f, sm = 0.f, sr = 0.f;
    for (int c = lane; c < chunks; c += 32) {
      ss = sum_sq8(s + 8 * c, ss);
      sm = sum_sq8(m + 8 * c, sm);
      if constexpr (!kQE) sr = sum_sq8(r + 8 * c, sr);
    }
    ds = fmaxf(sqrtf(warp_sum(ss)), kNormEps);
    dm = fmaxf(sqrtf(warp_sum(sm)), kNormEps);
    if constexpr (!kQE) dr = fmaxf(sqrtf(warp_sum(sr)), kNormEps);
  }
  OutT* o = out + (long long)row * (kQE ? 4 : 6) * E;
  for (int c = lane; c < chunks; c += 32) {
    float vs[8], vm[8], vr[8], f[8];
    load8(s + 8 * c, vs);
    load8(m + 8 * c, vm);
    if constexpr (!kQE) load8(r + 8 * c, vr);
    if (normalize) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        vs[i] = vs[i] / ds;
        vm[i] = vm[i] / dm;
        if constexpr (!kQE) vr[i] = vr[i] / dr;
      }
    }
    OutT* p = o + 8 * c;
    if constexpr (kQE) {
      store8(p, vs);
      store8(p + E, vm);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = vs[i] * vm[i];
      store8(p + 2 * E, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = fabsf(vm[i] - vs[i]);
      store8(p + 3 * E, f);
    } else {
      store8(p, vr);
      store8(p + E, vm);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = vs[i] * vm[i];
      store8(p + 2 * E, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = vr[i] * vm[i];
      store8(p + 3 * E, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = fabsf(vm[i] - vs[i]);
      store8(p + 4 * E, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = fabsf(vm[i] - vr[i]);
      store8(p + 5 * E, f);
    }
  }
}

// out[r] = h[r, :] . w + b, the final Linear(K -> 1): one warp per row, K % 128 == 0.  Lane l accumulates the float4s
// l, l + 32, ... in order, then a fixed butterfly adds the lanes: the same order for every row.
__global__ void __launch_bounds__(kWarpsPerCta * 32) blaser_output_kernel(const float* __restrict__ h, int rows, int K,
                                                                          const float* __restrict__ w,
                                                                          const float* __restrict__ b,
                                                                          float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4* hr = reinterpret_cast<const float4*>(h + (long long)row * K);
  const float4* w4 = reinterpret_cast<const float4*>(w);
  float acc = 0.f;
  for (int i = lane; i < K / 4; i += 32) {
    const float4 x = __ldg(hr + i), y = __ldg(w4 + i);
    acc = fmaf(x.x, y.x, acc);
    acc = fmaf(x.y, y.y, acc);
    acc = fmaf(x.z, y.z, acc);
    acc = fmaf(x.w, y.w, acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) out[row] = acc + __ldg(b);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int feature_width(int input_form, int E) { return (input_form == SB_BLASER_QE ? 4 : 6) * E; }

// Checks and launches the featurize kernel; `who` names the entry point in errors.
int blaser_featurize(const char* who, const float* src, const float* mt, const float* ref, long long ld, int rows, int E,
                     int input_form, int normalize, void* out, int out_fp32, cudaStream_t stream) {
  const bool qe = input_form == SB_BLASER_QE;
  if (!src || !mt || !out || (!qe && !ref)) {
    set_last_error("%s: null src, mt or out, or no ref for the COMET input form", who);
    return SB_ERR_INVALID;
  }
  if (input_form != SB_BLASER_COMET && input_form != SB_BLASER_QE) {
    set_last_error("%s: unknown input_form %d", who, input_form);
    return SB_ERR_INVALID;
  }
  if (E <= 0 || E % 16 != 0 || ld < E || ld % 4 != 0 || rows < 0) {
    set_last_error("%s: need E a positive multiple of 16, ld >= E and ld %% 4 == 0, rows >= 0 (got E=%d ld=%lld rows=%d)",
                   who, E, ld, rows);
    return SB_ERR_INVALID;
  }
  if (!aligned16(src) || !aligned16(mt) || (!qe && !aligned16(ref)) || !aligned16(out)) {
    set_last_error("%s: src, mt, ref and out must be 16-byte aligned", who);
    return SB_ERR_INVALID;
  }
  if (rows == 0) return SB_OK;
  const unsigned grid = (unsigned)((rows + kWarpsPerCta - 1) / kWarpsPerCta);
  const unsigned block = kWarpsPerCta * 32;
  if (qe && out_fp32)
    blaser_featurize_kernel<true, float><<<grid, block, 0, stream>>>(src, mt, nullptr, ld, rows, E, normalize, (float*)out);
  else if (qe)
    blaser_featurize_kernel<true, __nv_bfloat16><<<grid, block, 0, stream>>>(src, mt, nullptr, ld, rows, E, normalize,
                                                                             (__nv_bfloat16*)out);
  else if (out_fp32)
    blaser_featurize_kernel<false, float><<<grid, block, 0, stream>>>(src, mt, ref, ld, rows, E, normalize, (float*)out);
  else
    blaser_featurize_kernel<false, __nv_bfloat16><<<grid, block, 0, stream>>>(src, mt, ref, ld, rows, E, normalize,
                                                                              (__nv_bfloat16*)out);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

struct BlaserWs {
  __nv_bfloat16* x = nullptr;  // [rows, max(F, hidden widths but the last)]: the features, then every second hidden layer
  __nv_bfloat16* y = nullptr;  // [rows, max(hidden widths but the last)]
  float* h = nullptr;          // [rows, hidden_dims[last]] fp32: the last hidden layer
  size_t bytes = 0;
};

}  // namespace

struct SbBlaser {
  int input_form = 0, E = 0, F = 0;
  std::vector<int> dims;                   // hidden widths
  std::vector<const __nv_bfloat16*> w;     // [num_hidden] bf16 [dims[i], in_i]
  std::vector<const float*> b;             // [num_hidden] fp32 [dims[i]]
  const float* w_out = nullptr;            // fp32 [dims.back()]
  const float* b_out = nullptr;            // fp32 [1]
  int cta_group = 2, num_sms = 0;
  int inner_width = 0;                     // widest hidden layer that is not the last (0 with one hidden layer)
};

static BlaserWs blaser_carve(const SbBlaser* e, size_t rows, void* base) {
  Carver c(base);
  BlaserWs w;
  w.x = c.take<__nv_bfloat16>(rows * (size_t)std::max(e->F, e->inner_width) * 2);
  w.y = c.take<__nv_bfloat16>(rows * (size_t)e->inner_width * 2);
  w.h = c.take<float>(rows * (size_t)e->dims.back() * 4);
  w.bytes = c.off;
  return w;
}

extern "C" {

int sb_blaser_create(const SbBlaserConfig* cfg, const SbBlaserWeights* w, SbBlaser** out) {
  if (!cfg || !w || !out) { set_last_error("sb_blaser_create: null argument"); return SB_ERR_INVALID; }
  *out = nullptr;
  const int L = cfg->num_hidden;
  bool dims_ok = L >= 1 && cfg->hidden_dims != nullptr;
  for (int i = 0; dims_ok && i < L; ++i) dims_ok = cfg->hidden_dims[i] > 0 && cfg->hidden_dims[i] % 256 == 0;
  const bool form_ok = cfg->input_form == SB_BLASER_COMET || cfg->input_form == SB_BLASER_QE;
  if (!form_ok || !dims_ok || cfg->embedding_dim <= 0 || cfg->embedding_dim % 16 != 0 ||
      feature_width(cfg->input_form, cfg->embedding_dim) % 64 != 0 || cfg->cta_group < 0 || cfg->cta_group > 2) {
    set_last_error("sb_blaser_create: outside the engine's envelope (input_form COMET or QE, embedding_dim a positive "
                   "multiple of 16 whose feature width 4E (QE) or 6E (COMET) is a multiple of 64, num_hidden >= 1 hidden "
                   "widths that are positive multiples of 256, cta_group 0, 1 or 2); got input_form=%d embedding_dim=%d "
                   "num_hidden=%d", cfg->input_form, cfg->embedding_dim, L);
    return SB_ERR_INVALID;
  }
  if (!w->w || !w->b) { set_last_error("sb_blaser_create: missing weight array"); return SB_ERR_INVALID; }
  for (int i = 0; i <= L; ++i)
    if (!w->w[i] || !w->b[i]) {
      set_last_error("sb_blaser_create: layer %d has a null weight or bias pointer", i);
      return SB_ERR_INVALID;
    }
  if (!aligned16(w->w[L])) { set_last_error("sb_blaser_create: the output weight must be 16-byte aligned"); return SB_ERR_INVALID; }
  int num_sms = 0;
  if (int rc = require_hopper("sb_blaser_create", &num_sms)) return rc;
  std::unique_ptr<SbBlaser> e(new (std::nothrow) SbBlaser());
  if (!e) { set_last_error("out of host memory"); return SB_ERR_INVALID; }
  e->input_form = cfg->input_form;
  e->E = cfg->embedding_dim;
  e->F = feature_width(cfg->input_form, cfg->embedding_dim);
  e->dims.assign(cfg->hidden_dims, cfg->hidden_dims + L);
  for (int i = 0; i < L; ++i) {
    e->w.push_back(static_cast<const __nv_bfloat16*>(w->w[i]));
    e->b.push_back(w->b[i]);
    if (i + 1 < L) e->inner_width = std::max(e->inner_width, e->dims[i]);
  }
  e->w_out = static_cast<const float*>(w->w[L]);
  e->b_out = w->b[L];
  e->cta_group = cfg->cta_group == 1 ? 1 : 2;
  e->num_sms = cfg->num_sms > 0 ? cfg->num_sms : num_sms;
  *out = e.release();
  return SB_OK;
}

void sb_blaser_destroy(SbBlaser* e) { delete e; }

int sb_blaser_workspace_bytes(const SbBlaser* e, int32_t max_rows, size_t* bytes) {
  if (!e || !bytes || max_rows <= 0) { set_last_error("sb_blaser_workspace_bytes: bad argument"); return SB_ERR_INVALID; }
  *bytes = blaser_carve(e, (size_t)max_rows, nullptr).bytes + kWorkspaceAlign;
  return SB_OK;
}

int sb_blaser_forward(SbBlaser* e, const float* src, const float* mt, const float* ref, int64_t ld, int32_t rows,
                      float* scores, void* workspace, size_t workspace_bytes, void* stream_v) {
  if (!e || !scores || !workspace) { set_last_error("sb_blaser_forward: null argument"); return SB_ERR_INVALID; }
  if (rows < 0) { set_last_error("sb_blaser_forward: rows=%d", rows); return SB_ERR_INVALID; }
  if (rows == 0) return SB_OK;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  BlaserWs ws;
  int rc = bind_workspace("sb_blaser_forward", workspace, workspace_bytes, &ws,
                          [&](void* p) { return blaser_carve(e, (size_t)rows, p); });
  if (rc) return rc;
  if ((rc = blaser_featurize("sb_blaser_forward", src, mt, e->input_form == SB_BLASER_QE ? nullptr : ref, ld, rows, e->E,
                             e->input_form, 1, ws.x, 0, stream)))
    return rc;
  const int L = (int)e->dims.size();
  __nv_bfloat16* cur = ws.x;
  int K = e->F;
  for (int i = 0; i < L; ++i) {
    const bool last = i + 1 == L;
    __nv_bfloat16* nxt = cur == ws.x ? ws.y : ws.x;
    void* C = last ? static_cast<void*>(ws.h) : static_cast<void*>(nxt);
    GemmArgs g = gemm_args(cur, K, e->w[i], K, C, e->dims[i], last ? 1 : 0, e->b[i], rows, e->dims[i], K, EPI_BIAS_TANH,
                           e->num_sms);
    g.cta_group = e->cta_group;  // allow_skinny stays 0: the same summation order for every batch size
    if ((rc = gemm_bf16(g, stream))) return rc;
    cur = nxt;
    K = e->dims[i];
  }
  blaser_output_kernel<<<(unsigned)((rows + kWarpsPerCta - 1) / kWarpsPerCta), kWarpsPerCta * 32, 0, stream>>>(
      ws.h, rows, K, e->w_out, e->b_out, scores);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

int sb_blaser_featurize(const float* src, const float* mt, const float* ref, int64_t ld, int32_t rows, int32_t E,
                        int32_t input_form, int32_t normalize, void* out, int32_t out_fp32, void* stream) {
  int sms = 0;
  if (int rc = require_hopper("sb_blaser_featurize", &sms)) return rc;
  return blaser_featurize("sb_blaser_featurize", src, mt, input_form == SB_BLASER_QE ? nullptr : ref, ld, rows, E,
                          input_form, normalize != 0, out, out_fp32, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
