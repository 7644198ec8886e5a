// SONAR embedding -> text decoder, one incremental step at a time (BASELINE.json config 4).
//
// Reference: ConditionalTransformerDecoderModel.decode/project (sonar/nn/conditional_decoder_model.py:60-94),
// wiring sonar/models/sonar_text/factory.py:229-315 (pre-LN layers: causal self-attention with a KV cache,
// encoder-decoder attention, ReLU FFN; final LayerNorm; logits = h . E^T with the tied embedding matrix),
// driven one token at a time by fairseq2's BeamSearchSeq2SeqGenerator (sonar/inference_pipelines/text.py:305-346).
//
// The source is the sentence embedding as a SINGLE encoder position (sonar/models/sonar_translation/model.py:48-53),
// so every cross-attention softmax is over one key and equals 1: the layer's cross-attention output is the
// per-sentence constant  c_l = Wo_l (Wv_l e + bv_l) + bo_l  (q/k projections are dead compute).  sb_decoder_begin
// computes c_l once per sentence with two GEMMs per layer; each step then only adds it.
//
// Per step (R = sentences x beam rows, all at the same position t):
//   x = E[token] * sqrt(d) + pos[t]
//   24 x { h = LN(x); qkv = h Wqkv^T (wgmma GEMM); K/V appended to the cache; attention over positions 0..t
//          through a per-row ancestry table (beam reordering never moves the cache); x += o Wo^T + bo (TMA reduce-add);
//          x += c_l[sentence]; h = LN(x); x += W2 relu(W1 h + b1) + b2 }
//   h = LN_final(x);  logits = h E^T  -- never materialised: the wgmma GEMM's sweep epilogue keeps a running
//   top-16 and an online log-sum-exp per row over all 256 206 columns; a merge kernel turns the per-chunk partials
//   into the 16 best (log-prob, token) pairs per row plus log P(EOS).

#include "../../include/sonar_b200.h"
#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>
#include <memory>
#include <new>
#include <vector>

namespace sb {

// x[r,:] = E[token[r],:] * scale + pos[t,:]      (one warp per row)
__global__ void __launch_bounds__(256)
decode_embed_kernel(const int64_t* __restrict__ tokens, const __nv_bfloat16* __restrict__ embed, long long vocab,
                    const float* __restrict__ pos_row, int D, float scale, float* __restrict__ x, int R,
                    int* __restrict__ err_flag) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  long long id = tokens[r];
  if (id < 0 || id >= vocab) {
    if (lane == 0) atomicExch(err_flag, 1);
    id = 0;
  }
  const uint4* erow = reinterpret_cast<const uint4*>(embed + id * (long long)D);
  const float4* prow = reinterpret_cast<const float4*>(pos_row);
  float4* xrow = reinterpret_cast<float4*>(x + (long long)r * D);
  for (int c = lane; c < D / 8; c += 32) {
    const uint4 e = __ldg(erow + c);
    const float4 p0 = __ldg(prow + 2 * c), p1 = __ldg(prow + 2 * c + 1);
    const uint32_t w[4] = {e.x, e.y, e.z, e.w};
    float f[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&w[q]);
      f[2 * q] = __low2float(v);
      f[2 * q + 1] = __high2float(v);
    }
    xrow[2 * c] = make_float4(fmaf(f[0], scale, p0.x), fmaf(f[1], scale, p0.y), fmaf(f[2], scale, p0.z), fmaf(f[3], scale, p0.w));
    xrow[2 * c + 1] = make_float4(fmaf(f[4], scale, p1.x), fmaf(f[5], scale, p1.y), fmaf(f[6], scale, p1.z), fmaf(f[7], scale, p1.w));
  }
}

// x[r,:] += c[r / beam, :], then h[r,:] = LayerNorm(x[r,:]) in bf16: the collapsed cross-attention residual and the FFN
// LayerNorm in one pass over the row (D = 128 * nvec, nvec <= kMaxVec).
__global__ void __launch_bounds__(256)
add_const_layernorm_kernel(float* __restrict__ x, const float* __restrict__ c, int R, int beam, int D,
                           const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                           __nv_bfloat16* __restrict__ h) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const int nvec = D / 128;
  float4 v[kMaxVec], cv[kMaxVec];
  load_row(x + (long long)r * D, nvec, lane, v);
  load_row(c + (long long)(r / beam) * D, nvec, lane, cv);
  float4* xr = reinterpret_cast<float4*>(x + (long long)r * D);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i)
    if (i < nvec) {
      v[i].x += cv[i].x; v[i].y += cv[i].y; v[i].z += cv[i].z; v[i].w += cv[i].w;
      xr[i * 32 + lane] = v[i];
    }
  normalize_row(v, nvec, lane, D, gamma, beta, eps);
  uint2* hr = reinterpret_cast<uint2*>(h + (long long)r * D);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i)
    if (i < nvec) hr[i * 32 + lane] = make_uint2(pack_bf16x2(v[i].x, v[i].y), pack_bf16x2(v[i].z, v[i].w));
}

// fp32 [n, D] -> bf16 (plain cast; A operand of the cross-attention constant GEMMs)
__global__ void cast_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, long long n) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i + 3 < n) {
    const float4 v = *reinterpret_cast<const float4*>(in + i);
    *reinterpret_cast<uint2*>(out + i) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  } else {
    for (long long j = i; j < n; ++j) out[j] = __float2bfloat16_rn(in[j]);
  }
}

// Incremental causal self-attention: one warp per (row, head).  Appends this step's K/V to the cache at
// position t (physical row r) and attends over positions 0..t, where position t' < t of hypothesis r lives in
// physical cache row table[r, t'] (its ancestor at that step).
// The warp walks the keys FOUR at a time: lane group g = lane/8 owns keys g, g+4, ..., and inside a group each lane
// owns 8 of the 64 head dims, so every K and V access is one 16-byte load per lane and 128 contiguous bytes per group.
// Each group keeps its own online-softmax state (max, sum, 8 accumulators per lane); the four states are merged
// with two shuffle rounds at the end.  HBM-bound: 2 x 128 B per (hypothesis, head, cached position).
constexpr int kMaxDecodeLen = 512;  // positions <= the decoder's position table

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&w[e]);
    f[2 * e] = __low2float(b);
    f[2 * e + 1] = __high2float(b);
  }
}

__global__ void __launch_bounds__(128)
decode_attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ kcache,
                        __nv_bfloat16* __restrict__ vcache, const int32_t* __restrict__ table, int t, int Tmax, int H,
                        __nv_bfloat16* __restrict__ out) {
  const int r = blockIdx.y;
  const int h = blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (h >= H) return;
  const int D = H * 64;
  const __nv_bfloat16* row = qkv + (long long)r * 3 * D + h * 64;
  {  // append this step's K / V (2 dims per lane) to the cache
    const long long own = ((long long)r * Tmax + t) * D + h * 64 + lane * 2;
    *reinterpret_cast<__nv_bfloat162*>(kcache + own) = *reinterpret_cast<const __nv_bfloat162*>(row + D + lane * 2);
    *reinterpret_cast<__nv_bfloat162*>(vcache + own) = *reinterpret_cast<const __nv_bfloat162*>(row + 2 * D + lane * 2);
  }
  const int grp = lane >> 3, sub = lane & 7;
  float q8[8];
  unpack8(*reinterpret_cast<const uint4*>(row + sub * 8), q8);
  __syncwarp();  // the row appended above is read back below by other lanes of this warp
  const int nk = t + 1;
  const int32_t* trow = table + (long long)r * Tmax;
  const float sl2 = 0.125f * 1.4426950408889634f;
  float m = -CUDART_INF_F, l = 0.f;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  // 16 keys per pass (4 per 8-lane group): the ancestry-table entries, then all eight 16-byte K / V loads of a lane are
  // in flight before the first dot product -- the loop is bound by loaded HBM latency, not by arithmetic.
  constexpr int U = 4;
  for (int base = 0; base < nk; base += 4 * U) {
    int tpv[U];
    bool val[U];
    int prow[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      tpv[u] = base + 4 * u + grp;
      val[u] = tpv[u] < nk;
      prow[u] = (val[u] && tpv[u] != t) ? __ldg(trow + tpv[u]) : r;
    }
    uint4 kq[U], vq[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long off = ((long long)prow[u] * Tmax + (val[u] ? tpv[u] : t)) * D + h * 64 + sub * 8;
      kq[u] = vq[u] = make_uint4(0u, 0u, 0u, 0u);
      if (val[u]) {
        kq[u] = *reinterpret_cast<const uint4*>(kcache + off);
        vq[u] = *reinterpret_cast<const uint4*>(vcache + off);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float k8[8], v8[8];
      unpack8(kq[u], k8);
      unpack8(vq[u], v8);
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) s = fmaf(q8[e], k8[e], s);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      if (val[u]) {  // uniform inside each 8-lane group
        const float mn = fmaxf(m, s);
        const float corr = exp2f((m - mn) * sl2);  // m = -inf on the group's first key -> 0
        const float pj = exp2f((s - mn) * sl2);
        l = l * corr + pj;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = fmaf(pj, v8[e], acc[e] * corr);
        m = mn;
      }
    }
  }
  // merge the four group states (a group that saw no key has m = -inf, l = 0)
  float M = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
  M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 16));
  const float sc = (m == -CUDART_INF_F) ? 0.f : exp2f((m - M) * sl2);
  l *= sc;
  l += __shfl_xor_sync(0xffffffffu, l, 8);
  l += __shfl_xor_sync(0xffffffffu, l, 16);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float a = acc[e] * sc;
    a += __shfl_xor_sync(0xffffffffu, a, 8);
    a += __shfl_xor_sync(0xffffffffu, a, 16);
    acc[e] = a;
  }
  if (grp == 0) {
    const float inv = 1.0f / l;
    *reinterpret_cast<uint4*>(out + (long long)r * D + h * 64 + sub * 8) =
        make_uint4(pack_bf16x2(acc[0] * inv, acc[1] * inv), pack_bf16x2(acc[2] * inv, acc[3] * inv),
                   pack_bf16x2(acc[4] * inv, acc[5] * inv), pack_bf16x2(acc[6] * inv, acc[7] * inv));
  }
}

// Merge the per-chunk partials of the vocabulary GEMM: one warp per row.
//   lse = log sum_j exp(logit_j) over all columns; out: 16 best (logit - lse, token), order (value desc, token asc);
//   eos_lprob = <h, E[eos]> - lse (needed when the generator must force EOS and EOS is not among the 16).
template <int KC>
__global__ void __launch_bounds__(256)
vocab_merge_kernel(const float* __restrict__ cand_val, const int* __restrict__ cand_idx, const float* __restrict__ lse_part,
                   int n_chunks, const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ embed, int D,
                   int eos_idx, int R, float* __restrict__ out_lprob, int* __restrict__ out_tok,
                   float* __restrict__ out_eos, const int64_t* __restrict__ probe_tokens, long long vocab,
                   float* __restrict__ out_probe) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  // ---- log-sum-exp ----
  float M = -CUDART_INF_F;
  for (int c = lane; c < n_chunks; c += 32) M = fmaxf(M, lse_part[((long long)r * n_chunks + c) * 2]);
  M = warp_max(M);
  float S = 0.f;
  for (int c = lane; c < n_chunks; c += 32) {
    const float mc = lse_part[((long long)r * n_chunks + c) * 2];
    const float sc = lse_part[((long long)r * n_chunks + c) * 2 + 1];
    if (mc > -CUDART_INF_F) S += sc * __expf(mc - M);
  }
  S = warp_sum(S);
  const float lse = M + logf(S);
  // ---- top-KC of the n_chunks*KC candidates: every lane keeps a strided slice, then KC rounds of warp arg-max ----
  const int total = n_chunks * KC;
  const float* cv = cand_val + (long long)r * total;
  const int* ci = cand_idx + (long long)r * total;
  unsigned long long taken0 = 0ull, taken1 = 0ull;  // lane-local bitmap over its slice (slice <= 128 entries: n_lists <= 256)
  for (int k = 0; k < KC; ++k) {
    float bv = -CUDART_INF_F;
    int bi = 0x7fffffff, bpos = -1;
    int s = 0;
    for (int p = lane; p < total; p += 32, ++s) {
      if (((s < 64) ? taken0 : taken1) & (1ull << (s & 63))) continue;
      const float v = cv[p];
      const int i = ci[p];
      if (i < 0) continue;
      if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; bpos = s; }
    }
    // warp arg-max by (value desc, token asc)
    float wv = bv;
    int wi = bi;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, wv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, wi, o);
      if (ov > wv || (ov == wv && oi < wi)) { wv = ov; wi = oi; }
    }
    if (bpos >= 0 && bv == wv && bi == wi) {  // token ids are unique -> exactly one lane
      if (bpos < 64) taken0 |= (1ull << bpos); else taken1 |= (1ull << (bpos - 64));
    }
    if (lane == 0) {
      const bool valid = wi != 0x7fffffff;
      out_lprob[(long long)r * KC + k] = valid ? (wv - lse) : -CUDART_INF_F;
      out_tok[(long long)r * KC + k] = valid ? wi : -1;
    }
  }
  // ---- log P(EOS) ----
  float dot = 0.f;
  const __nv_bfloat16* hr = h + (long long)r * D;
  const __nv_bfloat16* er = embed + (long long)eos_idx * D;
  for (int q = lane * 2; q < D; q += 64) {
    const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(hr + q);
    const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(er + q);
    dot += __low2float(a) * __low2float(b) + __high2float(a) * __high2float(b);
  }
  dot = warp_sum(dot);
  if (lane == 0) out_eos[r] = dot - lse;
  // ---- log P(probe token): the prompt scores the generator's prefill accumulates ----
  if (probe_tokens != nullptr) {
    long long pt = probe_tokens[r];
    if (pt < 0 || pt >= vocab) pt = 0;  // out-of-range ids are reported by decode_embed_kernel when they are fed back
    const __nv_bfloat16* pr = embed + pt * (long long)D;
    float pd = 0.f;
    for (int q = lane * 2; q < D; q += 64) {
      const __nv_bfloat162 a = *reinterpret_cast<const __nv_bfloat162*>(hr + q);
      const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(pr + q);
      pd += __low2float(a) * __low2float(b) + __high2float(a) * __high2float(b);
    }
    pd = warp_sum(pd);
    if (lane == 0) out_probe[r] = pd - lse;
  }
}

// ---------------------------------------------------------------------------------------------
// launches: sb_decoder_step and the kernel-level entry points below call the same functions
// ---------------------------------------------------------------------------------------------
namespace {

// x [R, D] fp32 = E[tokens] * scale + pos_row; ids outside [0, vocab) set *err_flag and embed row 0
int decoder_embed(const int64_t* tokens, const __nv_bfloat16* embed, long long vocab, const float* pos_row, int D, float scale,
                  float* x, int R, int* err_flag, cudaStream_t stream) {
  decode_embed_kernel<<<(unsigned)((R + 7) / 8), 256, 0, stream>>>(tokens, embed, vocab, pos_row, D, scale, x, R, err_flag);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

// The limits of decode_attention_kernel, with the caller's name in the message: one CTA row per hypothesis (grid y),
// positions up to the position table, heads in 256-column groups of the residual stream.
int check_decoder_attention(const char* who, int t, int Tmax, int R, int H) {
  if (t < 0 || t >= Tmax) { set_last_error("%s: position %d outside [0,%d)", who, t, Tmax); return SB_ERR_INVALID; }
  if (Tmax > kMaxDecodeLen) { set_last_error("%s: max_len %d > %d", who, Tmax, kMaxDecodeLen); return SB_ERR_INVALID; }
  if (R <= 0 || R > 65535) { set_last_error("%s: too many rows (%d)", who, R); return SB_ERR_INVALID; }
  if (H <= 0 || (64 * H) % 256 != 0) { set_last_error("%s: model_dim 64 * %d is not a multiple of 256", who, H); return SB_ERR_INVALID; }
  return SB_OK;
}

// qkv bf16 [R, 3D]; caches bf16 [R, Tmax, D] of one layer; table int32 [R, Tmax]; out bf16 [R, D]
int decoder_attention(const __nv_bfloat16* qkv, __nv_bfloat16* kcache, __nv_bfloat16* vcache, const int32_t* table, int t,
                      int R, int Tmax, int H, __nv_bfloat16* out, cudaStream_t stream) {
  decode_attention_kernel<<<dim3((unsigned)((H + 3) / 4), (unsigned)R), 128, 0, stream>>>(qkv, kcache, vcache, table, t, Tmax,
                                                                                        H, out);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

// x [R, D] fp32 += c[r / beam]; h [R, D] bf16 = LayerNorm(x)
int decoder_add_const_layernorm(float* x, const float* c, int R, int beam, int D, const float* gamma, const float* beta,
                                float eps, __nv_bfloat16* h, cudaStream_t stream) {
  add_const_layernorm_kernel<<<(unsigned)((R + 7) / 8), 256, 0, stream>>>(x, c, R, beam, D, gamma, beta, eps, h);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

// The vocabulary head: the top-k sweep of h [R, D] . embed [V, D]^T over n_chunks column chunks into the scratch
// (cand_val / cand_idx [R, lists, 16], lse_part [R, lists, 2], lists = gemm_topk_lists(n_chunks) <= 256), then the merge.
int decoder_vocab_head(const __nv_bfloat16* h, const __nv_bfloat16* embed, int R, int V, int D, int eos_idx,
                       const int64_t* probe_tokens, int n_chunks, float* cand_val, int* cand_idx, float* lse_part,
                       float* out_lprob, int* out_tok, float* out_eos, float* out_probe, int num_sms, cudaStream_t stream) {
  if (int rc = gemm_bf16_topk(h, D, embed, D, R, V, D, cand_val, cand_idx, lse_part, n_chunks, 2, num_sms, stream)) return rc;
  vocab_merge_kernel<kTopkCandidates><<<(unsigned)((R + 7) / 8), 256, 0, stream>>>(
      cand_val, cand_idx, lse_part, gemm_topk_lists(n_chunks), h, embed, D, eos_idx, R, out_lprob, out_tok, out_eos,
      probe_tokens, (long long)V, out_probe);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

}  // namespace
}  // namespace sb

using namespace sb;

struct SbDecoder {
  SbDecoderConfig cfg;
  const void* embed;
  const float* pos_table;
  const float* final_ln_g;
  const float* final_ln_b;
  std::vector<SbDecoderLayerWeights> layers;
  InputFlag err_flag;  // token id out of range, cleared by sb_decoder_check_inputs
  int num_sms;
};

namespace {

constexpr long long kSplitkFlags = 4096;  // >= 4 * (tile pairs of an [R, D] residual GEMM) whenever splitting can pay

struct DecWs {
  int* splitk_flags;      // [kSplitkFlags] hand-over counters of the split-K residual GEMMs (zeroed by sb_decoder_begin)
  float* x;               // [R, D] fp32 residual stream of the current step
  __nv_bfloat16* h;       // [R, D]
  __nv_bfloat16* qkv;     // [R, 3D]
  __nv_bfloat16* f;       // [R, F]
  float* cross;           // [L, N, D] per-sentence cross-attention constants
  __nv_bfloat16* ebf;     // [N, D] bf16 sentence embeddings
  __nv_bfloat16* vtmp;    // [N, D]
  float* cand_val;        // [R, n_lists, 16]   n_lists = gemm_topk_lists(n_chunks)
  int* cand_idx;
  float* lse_part;        // [R, n_lists, 2]
  __nv_bfloat16* kcache;  // [L, R, Tmax, D]
  __nv_bfloat16* vcache;
  int n_chunks;
  size_t bytes;
};

DecWs carve_dec(const SbDecoder* d, int N, int beam, int Tmax, void* base) {
  const size_t D = d->cfg.model_dim, F = d->cfg.ffn_inner_dim, L = d->cfg.num_layers;
  const size_t R = (size_t)N * beam;
  Carver c(base);
  DecWs w;
  w.n_chunks = gemm_topk_chunks((int)R, (int)d->cfg.vocab_size, 2, d->num_sms);
  w.splitk_flags = c.take<int>(kSplitkFlags * sizeof(int));
  w.x = c.take<float>(R * D * 4);
  w.h = c.take<__nv_bfloat16>(R * D * 2);
  w.qkv = c.take<__nv_bfloat16>(R * 3 * D * 2);
  w.f = c.take<__nv_bfloat16>(R * F * 2);
  w.cross = c.take<float>(L * (size_t)N * D * 4);
  w.ebf = c.take<__nv_bfloat16>((size_t)N * D * 2);
  w.vtmp = c.take<__nv_bfloat16>((size_t)N * D * 2);
  const size_t n_lists = (size_t)gemm_topk_lists(w.n_chunks);
  w.cand_val = c.take<float>(R * n_lists * kTopkCandidates * 4);
  w.cand_idx = c.take<int>(R * n_lists * kTopkCandidates * 4);
  w.lse_part = c.take<float>(R * n_lists * 2 * 4);
  w.kcache = c.take<__nv_bfloat16>(L * R * (size_t)Tmax * D * 2);
  w.vcache = c.take<__nv_bfloat16>(L * R * (size_t)Tmax * D * 2);
  w.bytes = c.off;
  return w;
}

int check_ws(const char* who, const SbDecoder* d, int N, int beam, int Tmax, void* workspace, size_t workspace_bytes,
             DecWs* out) {
  if (!d || !workspace) { set_last_error("%s: null argument", who); return SB_ERR_INVALID; }
  if (N <= 0 || beam <= 0 || Tmax <= 0 || Tmax > d->cfg.pos_rows) {
    set_last_error("%s: bad N=%d beam=%d max_len=%d (position table has %d rows)", who, N, beam, Tmax, d->cfg.pos_rows);
    return SB_ERR_INVALID;
  }
  auto carve = [&](void* p) { return carve_dec(d, N, beam, Tmax, p); };
  if (int rc = bind_workspace(who, workspace, workspace_bytes, out, carve)) return rc;
  if (gemm_topk_lists(out->n_chunks) > 256) { set_last_error("%s: vocabulary split into too many chunks", who); return SB_ERR_INVALID; }
  return SB_OK;
}

}  // namespace

extern "C" {

int sb_decoder_create(const SbDecoderConfig* cfg, const SbDecoderWeights* w, SbDecoder** out) {
  if (!cfg || !w || !out) { set_last_error("sb_decoder_create: null argument"); return SB_ERR_INVALID; }
  *out = nullptr;
  const int D = cfg->model_dim, H = cfg->num_heads, F = cfg->ffn_inner_dim;
  if (D <= 0 || D % 256 != 0 || D > 1024 || H <= 0 || D != H * 64 || F <= 0 || F % 256 != 0) {
    set_last_error("sb_decoder_create: need model_dim %% 256 == 0 (<= 1024), head_dim 64, ffn %% 256 == 0");
    return SB_ERR_INVALID;
  }
  static_assert(128 * kMaxVec >= 1024, "add_const_layernorm_kernel holds a row of up to 1024 columns in registers");
  if (cfg->input_dim != D) {
    set_last_error("sb_decoder_create: input_dim (%d) must equal model_dim (%d)", cfg->input_dim, D);
    return SB_ERR_INVALID;
  }
  if (cfg->num_layers < 0 || cfg->pos_rows <= 0 || cfg->vocab_size <= 0 || cfg->eos_idx < 0 ||
      cfg->eos_idx >= cfg->vocab_size) {
    set_last_error("sb_decoder_create: bad num_layers / pos_rows / vocab_size / eos_idx");
    return SB_ERR_INVALID;
  }
  if (!w->embed || !w->pos_table || !w->final_ln_g || !w->final_ln_b || (cfg->num_layers > 0 && !w->layers)) {
    set_last_error("sb_decoder_create: missing weight pointer");
    return SB_ERR_INVALID;
  }
  for (int i = 0; i < cfg->num_layers; ++i)
    if (has_null_pointer(w->layers[i])) {
      set_last_error("sb_decoder_create: layer %d has a null weight pointer", i);
      return SB_ERR_INVALID;
    }
  int num_sms = 0;
  if (int rc = require_hopper("sb_decoder_create", &num_sms)) return rc;
  std::unique_ptr<SbDecoder> d(new (std::nothrow) SbDecoder());
  if (!d) { set_last_error("out of host memory"); return SB_ERR_INVALID; }
  d->cfg = *cfg;
  d->embed = w->embed;
  d->pos_table = w->pos_table;
  d->final_ln_g = w->final_ln_g;
  d->final_ln_b = w->final_ln_b;
  d->layers.assign(w->layers, w->layers + cfg->num_layers);
  d->num_sms = num_sms;
  if (int rc = d->err_flag.create("sb_decoder_create")) return rc;
  *out = d.release();
  return SB_OK;
}

void sb_decoder_destroy(SbDecoder* d) { delete d; }

int sb_decoder_workspace_bytes(const SbDecoder* d, int32_t num_sentences, int32_t beam, int32_t max_len, size_t* bytes) {
  if (!d || !bytes || num_sentences <= 0 || beam <= 0 || max_len <= 0) {
    set_last_error("sb_decoder_workspace_bytes: bad argument");
    return SB_ERR_INVALID;
  }
  *bytes = carve_dec(d, num_sentences, beam, max_len, nullptr).bytes + kWorkspaceAlign;
  return SB_OK;
}

int sb_decoder_begin(SbDecoder* d, const float* embeddings, int32_t N, int32_t beam, int32_t max_len, void* workspace,
                     size_t workspace_bytes, void* stream_v) {
  DecWs w;
  int rc = check_ws("sb_decoder_begin", d, N, beam, max_len, workspace, workspace_bytes, &w);
  if (rc) return rc;
  if (!embeddings) { set_last_error("sb_decoder_begin: null embeddings"); return SB_ERR_INVALID; }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const int D = d->cfg.model_dim;
  SB_CUDA_CHECK(cudaMemsetAsync(w.splitk_flags, 0, kSplitkFlags * sizeof(int), stream));
  const long long n = (long long)N * D;
  cast_bf16_kernel<<<(unsigned)((n / 4 + 255) / 256 + 1), 256, 0, stream>>>(embeddings, w.ebf, n);
  SB_CUDA_CHECK(cudaGetLastError());
  for (int li = 0; li < d->cfg.num_layers; ++li) {
    const SbDecoderLayerWeights& L = d->layers[li];
    // v = e Wv^T + bv  (bf16), c = v Wo^T + bo (fp32)
    GemmArgs v = gemm_args(w.ebf, D, L.cross_wv, D, w.vtmp, D, 0, L.cross_bv, N, D, D, EPI_BIAS, d->num_sms);
    v.allow_skinny = 1;
    if ((rc = gemm_bf16(v, stream))) return rc;
    GemmArgs c = gemm_args(w.vtmp, D, L.cross_wo, D, w.cross + (size_t)li * N * D, D, 1, L.cross_bo, N, D, D, EPI_BIAS,
                           d->num_sms);
    c.allow_skinny = 1;
    if ((rc = gemm_bf16(c, stream))) return rc;
  }
  return SB_OK;
}

int sb_decoder_step(SbDecoder* d, const int64_t* tokens, const int32_t* table, int32_t t, int32_t N, int32_t beam,
                    int32_t max_len, float* out_lprob, int32_t* out_tok, float* out_eos_lprob,
                    const int64_t* probe_tokens, float* out_probe_lprob, void* workspace, size_t workspace_bytes,
                    void* stream_v) {
  DecWs w;
  int rc = check_ws("sb_decoder_step", d, N, beam, max_len, workspace, workspace_bytes, &w);
  if (rc) return rc;
  if (!tokens || !table || !out_lprob || !out_tok || !out_eos_lprob) { set_last_error("sb_decoder_step: null pointer"); return SB_ERR_INVALID; }
  if ((probe_tokens != nullptr) != (out_probe_lprob != nullptr)) {
    set_last_error("sb_decoder_step: probe_tokens and out_probe_lprob go together");
    return SB_ERR_INVALID;
  }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const int D = d->cfg.model_dim, F = d->cfg.ffn_inner_dim, H = d->cfg.num_heads;
  const int R = N * beam;
  if ((rc = check_decoder_attention("sb_decoder_step", t, max_len, R, H))) return rc;
  const __nv_bfloat16* embed = reinterpret_cast<const __nv_bfloat16*>(d->embed);
  if ((rc = decoder_embed(tokens, embed, d->cfg.vocab_size, d->pos_table + (size_t)t * D, D, d->cfg.embed_scale, w.x, R,
                          d->err_flag.dev, stream)))
    return rc;
  // Every GEMM of a step may take the weight-streaming path; the residual ones may split K when their tiles leave SM
  // pairs idle (2 560 rows).
  auto gemm = [&](GemmArgs g) {
    g.allow_skinny = 1;
    g.splitk_flags = w.splitk_flags;
    g.splitk_flags_len = kSplitkFlags;
    return gemm_bf16(g, stream);
  };
  const size_t layer_stride = (size_t)R * max_len * D;
  for (int li = 0; li < d->cfg.num_layers; ++li) {
    const SbDecoderLayerWeights& L = d->layers[li];
    if ((rc = layernorm_bf16(w.x, L.ln1_g, L.ln1_b, d->cfg.ln_eps, w.h, R, D, stream))) return rc;
    if ((rc = gemm(gemm_args(w.h, D, L.wqkv, D, w.qkv, 3 * D, 0, L.bqkv, R, 3 * D, D, EPI_BIAS, d->num_sms)))) return rc;
    if ((rc = decoder_attention(w.qkv, w.kcache + li * layer_stride, w.vcache + li * layer_stride, table, t, R, max_len, H, w.h,
                                stream)))
      return rc;
    if ((rc = gemm(gemm_args(w.h, D, L.wo, D, w.x, D, 1, L.bo, R, D, D, EPI_BIAS_RESIDUAL, d->num_sms)))) return rc;
    if ((rc = decoder_add_const_layernorm(w.x, w.cross + (size_t)li * N * D, R, beam, D, L.ln3_g, L.ln3_b, d->cfg.ln_eps, w.h,
                                          stream)))
      return rc;
    if ((rc = gemm(gemm_args(w.h, D, L.w1, D, w.f, F, 0, L.b1, R, F, D, EPI_BIAS_RELU, d->num_sms)))) return rc;
    if ((rc = gemm(gemm_args(w.f, F, L.w2, F, w.x, D, 1, L.b2, R, D, F, EPI_BIAS_RESIDUAL, d->num_sms)))) return rc;
  }
  if ((rc = layernorm_bf16(w.x, d->final_ln_g, d->final_ln_b, d->cfg.ln_eps, w.h, R, D, stream))) return rc;
  return decoder_vocab_head(w.h, embed, R, (int)d->cfg.vocab_size, D, d->cfg.eos_idx, probe_tokens, w.n_chunks, w.cand_val,
                            w.cand_idx, w.lse_part, out_lprob, out_tok, out_eos_lprob, out_probe_lprob, d->num_sms, stream);
}

int sb_decoder_check_inputs(SbDecoder* d, void* stream_v) {
  if (!d) { set_last_error("sb_decoder_check_inputs: null argument"); return SB_ERR_INVALID; }
  return d->err_flag.check("sb_decoder_step", reinterpret_cast<cudaStream_t>(stream_v));
}

int sb_decoder_embed(const int64_t* tokens, const void* embed, int64_t vocab, const float* pos_row, int32_t D, float scale,
                     float* x, int32_t R, int32_t* err_flag, void* stream) {
  if (!tokens || !embed || !pos_row || !x || !err_flag) { set_last_error("sb_decoder_embed: null argument"); return SB_ERR_INVALID; }
  if (R <= 0 || vocab <= 0 || D <= 0 || D % 8 != 0) {
    set_last_error("sb_decoder_embed: bad argument (R %d, vocab %lld, D %d)", R, (long long)vocab, D);
    return SB_ERR_INVALID;
  }
  return decoder_embed(tokens, static_cast<const __nv_bfloat16*>(embed), vocab, pos_row, D, scale, x, R, err_flag,
                       reinterpret_cast<cudaStream_t>(stream));
}

int sb_decoder_attention(const void* qkv, void* kcache, void* vcache, const int32_t* table, int32_t t, int32_t R,
                         int32_t Tmax, int32_t H, void* out, void* stream) {
  if (!qkv || !kcache || !vcache || !table || !out) { set_last_error("sb_decoder_attention: null argument"); return SB_ERR_INVALID; }
  if (int rc = check_decoder_attention("sb_decoder_attention", t, Tmax, R, H)) return rc;
  return decoder_attention(static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(kcache),
                           static_cast<__nv_bfloat16*>(vcache), table, t, R, Tmax, H, static_cast<__nv_bfloat16*>(out),
                           reinterpret_cast<cudaStream_t>(stream));
}

int sb_decoder_add_const_layernorm(float* x, const float* c, int32_t R, int32_t beam, int32_t D, const float* gamma,
                                   const float* beta, float eps, void* h, void* stream) {
  if (!x || !c || !gamma || !beta || !h) { set_last_error("sb_decoder_add_const_layernorm: null argument"); return SB_ERR_INVALID; }
  if (R <= 0 || beam <= 0 || D <= 0 || D % 128 != 0 || D > 128 * kMaxVec) {
    set_last_error("sb_decoder_add_const_layernorm: bad argument (R %d, beam %d, D %d; D a multiple of 128 <= %d)", R, beam, D,
                   128 * kMaxVec);
    return SB_ERR_INVALID;
  }
  return decoder_add_const_layernorm(x, c, R, beam, D, gamma, beta, eps, static_cast<__nv_bfloat16*>(h),
                                     reinterpret_cast<cudaStream_t>(stream));
}

int sb_decoder_vocab_chunks(int32_t R, int64_t V, int32_t* n_chunks) {
  if (!n_chunks || R <= 0 || V <= 0 || V > INT32_MAX) { set_last_error("sb_decoder_vocab_chunks: bad argument"); return SB_ERR_INVALID; }
  int sms = 0;
  if (int rc = require_hopper("sb_decoder_vocab_chunks", &sms)) return rc;
  *n_chunks = gemm_topk_chunks(R, (int)V, 2, sms);
  return SB_OK;
}

int sb_decoder_vocab_head(const void* h, const void* embed, int32_t R, int64_t V, int32_t D, int32_t eos_idx,
                          const int64_t* probe_tokens, int32_t n_chunks, float* cand_val, int32_t* cand_idx, float* lse_part,
                          float* out_lprob, int32_t* out_tok, float* out_eos, float* out_probe, void* stream) {
  if (!h || !embed || !cand_val || !cand_idx || !lse_part || !out_lprob || !out_tok || !out_eos ||
      (probe_tokens != nullptr) != (out_probe != nullptr)) {
    set_last_error("sb_decoder_vocab_head: null argument (probe_tokens and out_probe go together)");
    return SB_ERR_INVALID;
  }
  if (R <= 0 || V <= 0 || V > INT32_MAX || D <= 0 || eos_idx < 0 || eos_idx >= V || n_chunks < 0) {
    set_last_error("sb_decoder_vocab_head: bad argument (R %d, V %lld, D %d, eos %d, n_chunks %d)", R, (long long)V, D, eos_idx,
                   n_chunks);
    return SB_ERR_INVALID;
  }
  int sms = 0;
  if (int rc = require_hopper("sb_decoder_vocab_head", &sms)) return rc;
  if (n_chunks == 0) n_chunks = gemm_topk_chunks(R, (int)V, 2, sms);
  if (gemm_topk_lists(n_chunks) > 256) {  // the merge kernel's per-lane bitmap covers 128 entries: 256 lists of 16
    set_last_error("sb_decoder_vocab_head: %d chunks give %d candidate lists (at most 256)", n_chunks, gemm_topk_lists(n_chunks));
    return SB_ERR_INVALID;
  }
  return decoder_vocab_head(static_cast<const __nv_bfloat16*>(h), static_cast<const __nv_bfloat16*>(embed), R, (int)V, D, eos_idx,
                            probe_tokens, n_chunks, cand_val, cand_idx, lse_part, out_lprob, out_tok, out_eos, out_probe, sms,
                            reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
