// HBM-bound kernels of the SONAR text-encoder path: embedding frontend, LayerNorm,
// final LayerNorm + sequence pooling.  All are one-warp-per-token-row with 16-byte
// vectorised, fully coalesced accesses and fp32 statistics.
//
// Reference semantics:
//   frontend ..... sonar/models/sonar_text/factory.py:73-100  (embed * sqrt(d) + sinusoid, no LN, dropout off)
//   layer norms .. factory.py:117,122-128 (eps 1e-5, affine)
//   pooling ...... sonar/models/sonar_text/model.py:86-128 (static_pooling MAX / MEAN / LAST)

#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>

namespace sb {


// ----------------------------------------------------------------------------
// embedding frontend
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
embed_kernel(const int64_t* __restrict__ ids, long long ids_stride, const int32_t* __restrict__ cu, int S,
             const __nv_bfloat16* __restrict__ embed, long long vocab, const float* __restrict__ pos_table, int D,
             float scale, float* __restrict__ x, int* __restrict__ err_flag, int pos_offset,
             __nv_bfloat16* __restrict__ h_out, float* __restrict__ stats_out) {
  const int b = blockIdx.x;
  const int pos = blockIdx.y * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int start = cu[b];
  const int len = cu[b + 1] - start;
  if (pos >= len || pos >= S) return;
  long long id = ids[(long long)b * ids_stride + pos];
  if (id < 0 || id >= vocab) {
    if (lane == 0) atomicExch(err_flag, 1);
    id = 0;
  }
  const uint4* erow = reinterpret_cast<const uint4*>(embed + id * (long long)D);
  const float4* prow = reinterpret_cast<const float4*>(pos_table + (long long)(pos + pos_offset) * D);
  float4* xrow = reinterpret_cast<float4*>(x + (long long)(start + pos) * D);
  // LnFold producer side (optional): bf16 copy of the row and (mean, M2) of each kLnPartCols (128)-column chunk -- iteration
  // k of the loop below covers columns [256k, 256k + 256) with 8 columns per lane, so each HALF warp reduces one chunk
  uint4* hrow = h_out ? reinterpret_cast<uint4*>(h_out + (long long)(start + pos) * D) : nullptr;
  for (int c = lane; c < D / 8; c += 32) {
    const uint4 e = __ldg(erow + c);
    const float4 p0 = __ldg(prow + 2 * c), p1 = __ldg(prow + 2 * c + 1);
    const __nv_bfloat162 e0 = *reinterpret_cast<const __nv_bfloat162*>(&e.x);
    const __nv_bfloat162 e1 = *reinterpret_cast<const __nv_bfloat162*>(&e.y);
    const __nv_bfloat162 e2 = *reinterpret_cast<const __nv_bfloat162*>(&e.z);
    const __nv_bfloat162 e3 = *reinterpret_cast<const __nv_bfloat162*>(&e.w);
    float4 o0, o1;
    o0.x = fmaf(__low2float(e0), scale, p0.x);
    o0.y = fmaf(__high2float(e0), scale, p0.y);
    o0.z = fmaf(__low2float(e1), scale, p0.z);
    o0.w = fmaf(__high2float(e1), scale, p0.w);
    o1.x = fmaf(__low2float(e2), scale, p1.x);
    o1.y = fmaf(__high2float(e2), scale, p1.y);
    o1.z = fmaf(__low2float(e3), scale, p1.z);
    o1.w = fmaf(__high2float(e3), scale, p1.w);
    xrow[2 * c] = o0;
    xrow[2 * c + 1] = o1;
    if (hrow != nullptr) {
      hrow[c] = make_uint4(pack_bf16x2(o0.x, o0.y), pack_bf16x2(o0.z, o0.w), pack_bf16x2(o1.x, o1.y), pack_bf16x2(o1.z, o1.w));
      float hs = (o0.x + o0.y) + (o0.z + o0.w) + (o1.x + o1.y) + (o1.z + o1.w);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) hs += __shfl_xor_sync(0xffffffffu, hs, o);  // stays inside each 16-lane half
      const float mean = hs * (1.0f / 128.0f);
      float q = 0.f;
      q = fmaf(o0.x - mean, o0.x - mean, q); q = fmaf(o0.y - mean, o0.y - mean, q);
      q = fmaf(o0.z - mean, o0.z - mean, q); q = fmaf(o0.w - mean, o0.w - mean, q);
      q = fmaf(o1.x - mean, o1.x - mean, q); q = fmaf(o1.y - mean, o1.y - mean, q);
      q = fmaf(o1.z - mean, o1.z - mean, q); q = fmaf(o1.w - mean, o1.w - mean, q);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      if ((lane & 15) == 0)
        reinterpret_cast<float2*>(stats_out)[(long long)(start + pos) * (D / 128) + 2 * (c >> 5) + (lane >> 4)] =
            make_float2(mean, q);
    }
  }
}

int embed_tokens(const int64_t* ids, long long ids_stride, const int32_t* cu_seqlens, int B, int S,
                 const __nv_bfloat16* embed, long long vocab, const float* pos_table, int pos_rows, int D, float scale,
                 float* x, int* err_flag, cudaStream_t stream, int pos_offset, __nv_bfloat16* h_out, float* stats_out) {
  if (B <= 0 || S <= 0) return 0;
  if (D % 8 != 0) { set_last_error("embed_tokens: D must be a multiple of 8"); return -1; }
  if ((h_out != nullptr) != (stats_out != nullptr) || (h_out != nullptr && D % 256 != 0)) {
    set_last_error("embed_tokens: h_out and stats_out go together and need D %% 256 == 0");
    return -1;
  }
  if (S + pos_offset > pos_rows || pos_offset < 0) {
    set_last_error("embed_tokens: positions [%d,%d) exceed the position table (%d rows)", pos_offset, S + pos_offset, pos_rows);
    return -1;
  }
  dim3 grid((unsigned)B, (unsigned)((S + 7) / 8), 1);
  embed_kernel<<<grid, 256, 0, stream>>>(ids, ids_stride, cu_seqlens, S, embed, vocab, pos_table, D, scale, x,
                                         err_flag, pos_offset, h_out, stats_out);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// LnFold weight preparation (once, at create): one warp per output row n of W [N, K]
//   Wf[n,k] = bf16(W[n,k] * gamma[k]);  colsum[n] = sum_k Wf[n,k];  bias_f[n] = bias[n] + sum_k W[n,k] * beta[k]
__global__ void __launch_bounds__(256)
fold_layernorm_kernel(const __nv_bfloat16* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ gamma,
                      const float* __restrict__ beta, int N, int K, __nv_bfloat16* __restrict__ Wf,
                      float* __restrict__ colsum, float* __restrict__ bias_f) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  const __nv_bfloat16* w = W + (long long)n * K;
  __nv_bfloat16* wf = Wf + (long long)n * K;
  double cs = 0.0, bs = 0.0;
  for (int k = lane; k < K; k += 32) {
    const float wv = __bfloat162float(w[k]);
    const __nv_bfloat16 r = __float2bfloat16_rn(wv * gamma[k]);
    wf[k] = r;
    cs += (double)__bfloat162float(r);
    bs += (double)wv * (double)beta[k];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cs += __shfl_xor_sync(0xffffffffu, cs, o);
    bs += __shfl_xor_sync(0xffffffffu, bs, o);
  }
  if (lane == 0) {
    colsum[n] = (float)cs;
    bias_f[n] = (float)((double)bias[n] + bs);
  }
}

int fold_layernorm_weights(const __nv_bfloat16* W, const float* bias, const float* gamma, const float* beta, int N, int K,
                           __nv_bfloat16* Wf, float* colsum, float* bias_f, cudaStream_t stream) {
  fold_layernorm_kernel<<<(unsigned)((N + 7) / 8), 256, 0, stream>>>(W, bias, gamma, beta, N, K, Wf, colsum, bias_f);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

__global__ void __launch_bounds__(256)
layernorm_bf16_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                      float eps, __nv_bfloat16* __restrict__ y, long long T, int D) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= T) return;
  const int nvec = D / 128;
  float4 v[kMaxVec];
  load_row(x + row * D, nvec, lane, v);
  normalize_row(v, nvec, lane, D, gamma, beta, eps);
  uint2* yrow = reinterpret_cast<uint2*>(y + row * D);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i)
    if (i < nvec) yrow[i * 32 + lane] = make_uint2(pack_bf16x2(v[i].x, v[i].y), pack_bf16x2(v[i].z, v[i].w));
}

// y32 = LN(x) in fp32 (may alias x: every row is read into registers before it is written) and/or a bf16 copy
__global__ void __launch_bounds__(256)
layernorm_dual_kernel(const float* x, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                      float* y32, __nv_bfloat16* __restrict__ y16, long long T, int D) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= T) return;
  const int nvec = D / 128;
  float4 v[kMaxVec];
  load_row(x + row * D, nvec, lane, v);
  normalize_row(v, nvec, lane, D, gamma, beta, eps);
  if (y32 != nullptr) {
    float4* r = reinterpret_cast<float4*>(y32 + row * D);
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i)
      if (i < nvec) r[i * 32 + lane] = v[i];
  }
  if (y16 != nullptr) {
    uint2* r = reinterpret_cast<uint2*>(y16 + row * D);
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i)
      if (i < nvec) r[i * 32 + lane] = make_uint2(pack_bf16x2(v[i].x, v[i].y), pack_bf16x2(v[i].z, v[i].w));
  }
}

// x[b, :] = v, xb[b, :] = bf16(v) for every b < B: the single decoder position both attention poolers start from
__global__ void broadcast_rows_kernel(const float* __restrict__ v, float* __restrict__ x, __nv_bfloat16* __restrict__ xb,
                                      int B, int D) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * D) return;
  const float f = v[i % D];
  x[i] = f;
  xb[i] = __float2bfloat16_rn(f);
}

int broadcast_rows(const float* v, float* x, __nv_bfloat16* xb, int B, int D, cudaStream_t stream) {
  broadcast_rows_kernel<<<(unsigned)(((long long)B * D + 255) / 256), 256, 0, stream>>>(v, x, xb, B, D);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int layernorm_bf16(const float* x, const float* gamma, const float* beta, float eps, __nv_bfloat16* y, long long T,
                   int D, cudaStream_t stream) {
  if (T <= 0) return 0;
  if (D % 128 != 0 || D > 128 * kMaxVec) {
    set_last_error("layernorm_bf16: D must be a multiple of 128 and <= %d (got %d)", 128 * kMaxVec, D);
    return -1;
  }
  const long long blocks = (T + 7) / 8;
  layernorm_bf16_kernel<<<(unsigned)blocks, 256, 0, stream>>>(x, gamma, beta, eps, y, T, D);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int layernorm_dual(const float* x, const float* gamma, const float* beta, float eps, float* y32, __nv_bfloat16* y16,
                   long long T, int D, cudaStream_t stream) {
  if (T <= 0) return 0;
  if (D % 128 != 0 || D > 128 * kMaxVec) {
    set_last_error("layernorm_dual: D must be a multiple of 128 and <= %d (got %d)", 128 * kMaxVec, D);
    return -1;
  }
  layernorm_dual_kernel<<<(unsigned)((T + 7) / 8), 256, 0, stream>>>(x, gamma, beta, eps, y32, y16, T, D);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ----------------------------------------------------------------------------
// final LayerNorm + pooling: one CTA per sequence, warps stride over its tokens,
// fp32 accumulation, fixed-order cross-warp combine (deterministic, independent of
// which other sequences share the batch).
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ln_pool_kernel(const float* __restrict__ x, const int32_t* __restrict__ cu, int D, const float* __restrict__ gamma,
               const float* __restrict__ beta, float eps, int apply_ln, int pool_mode, float* __restrict__ out,
               float* __restrict__ encoded_padded, int S_padded) {
  __shared__ float4 part[8][32 * kMaxVec];  // 32 KB
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int start = cu[b];
  const int len = cu[b + 1] - start;
  const int nvec = D / 128;
  const float init = (pool_mode == POOL_MAX) ? -CUDART_INF_F : 0.f;
  float4 acc[kMaxVec];
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) acc[i] = make_float4(init, init, init, init);

  for (int t = warp; t < len; t += 8) {
    float4 v[kMaxVec];
    load_row(x + (long long)(start + t) * D, nvec, lane, v);
    if (apply_ln) normalize_row(v, nvec, lane, D, gamma, beta, eps);
    if (encoded_padded != nullptr && t < S_padded) {
      float4* erow = reinterpret_cast<float4*>(encoded_padded + ((long long)b * S_padded + t) * D);
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i)
        if (i < nvec) erow[i * 32 + lane] = v[i];
    }
    if (pool_mode == POOL_MEAN) {
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i)
        if (i < nvec) { acc[i].x += v[i].x; acc[i].y += v[i].y; acc[i].z += v[i].z; acc[i].w += v[i].w; }
    } else if (pool_mode == POOL_MAX) {
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i)
        if (i < nvec) {
          acc[i].x = fmaxf(acc[i].x, v[i].x); acc[i].y = fmaxf(acc[i].y, v[i].y);
          acc[i].z = fmaxf(acc[i].z, v[i].z); acc[i].w = fmaxf(acc[i].w, v[i].w);
        }
    } else if (t == len - 1) {  // POOL_LAST
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i)
        if (i < nvec) acc[i] = v[i];
    }
  }
  if (encoded_padded != nullptr) {  // zero the padded tail of this sequence
    for (int t = len + warp; t < S_padded; t += 8) {
      float4* erow = reinterpret_cast<float4*>(encoded_padded + ((long long)b * S_padded + t) * D);
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i)
        if (i < nvec) erow[i * 32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i)
    if (i < nvec) part[warp][i * 32 + lane] = acc[i];
  __syncthreads();
  // weights = 1 / (seq_len + 1e-7) in the tensor dtype (model.py:118-121)
  const float w = 1.0f / (float(len) + 1e-7f);
  for (int c = threadIdx.x; c < nvec * 32; c += 256) {
    float4 r = part[0][c];
    for (int k = 1; k < 8; ++k) {
      const float4 p = part[k][c];
      if (pool_mode == POOL_MAX) {
        r.x = fmaxf(r.x, p.x); r.y = fmaxf(r.y, p.y); r.z = fmaxf(r.z, p.z); r.w = fmaxf(r.w, p.w);
      } else {  // MEAN: ordered sum; LAST: exactly one warp holds non-zero data
        r.x += p.x; r.y += p.y; r.z += p.z; r.w += p.w;
      }
    }
    if (pool_mode == POOL_MEAN) { r.x *= w; r.y *= w; r.z *= w; r.w *= w; }
    reinterpret_cast<float4*>(out + (long long)b * D)[c] = r;
  }
}

int ln_pool(const float* x, const int32_t* cu_seqlens, int B, int D, const float* gamma, const float* beta,
            float eps, int apply_ln, int pool_mode, float* out, float* encoded_padded, int S_padded,
            cudaStream_t stream) {
  if (B <= 0) return 0;
  if (D % 128 != 0 || D > 128 * kMaxVec) {
    set_last_error("ln_pool: D must be a multiple of 128 and <= %d (got %d)", 128 * kMaxVec, D);
    return -1;
  }
  if (pool_mode != POOL_MAX && pool_mode != POOL_MEAN && pool_mode != POOL_LAST) {
    set_last_error("ln_pool: unsupported pooling mode %d", pool_mode);
    return -1;
  }
  if (apply_ln && (!gamma || !beta)) { set_last_error("ln_pool: LayerNorm requested without parameters"); return -1; }
  ln_pool_kernel<<<(unsigned)B, 256, 0, stream>>>(x, cu_seqlens, D, gamma, beta, eps, apply_ln, pool_mode, out,
                                                  encoded_padded, S_padded);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace sb
