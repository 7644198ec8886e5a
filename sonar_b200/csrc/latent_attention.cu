// The attention pooler of the text and speech encoders (AttentionPooler, sonar_b200_internal.h): its single-query latent
// cross-attention, the create-time weight absorption behind it and the layer loop around it (reference:
// AttentionEncoderOutputPooler, sonar/nn/encoder_pooler.py:47-89, built by SonarTextEncoderFactory.create_attention_pooler,
// sonar/models/sonar_text/factory.py:155-226, and by the speech factory; fairseq2's encoder-decoder attention with ONE
// decoder position).
//
// For head h (head dim 64, scale 1/8), memory row m_t (final-LayerNormed token state, width D) and pooler query q:
//   score_t = q_h . (W_k,h m_t + b_k,h) / 8 = (W_k,h^T q_h) . m_t / 8 + const      (softmax cancels the constant)
//   out_h   = sum_t p_t (W_v,h m_t + b_v,h) = W_v,h (sum_t p_t m_t) + b_v,h         (sum_t p_t = 1)
// so the keys AND the values of every head are the memory rows themselves: 16 query rows (qt_h = W_k,h^T q_h, computed by
// one GEMM with the absorbed weights) attend over width-D keys, and the memory is read once per pooler layer; no [T, .]
// projection is ever written.  W_v is absorbed into the output projection (W_o blockdiag(W_v,h)).

#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>

namespace sb {
namespace {

constexpr int kLaThreads = 256;  // 8 warps
constexpr int kLaKeys = 16;      // keys per shared-memory tile (one k-step of the P . M product)
constexpr int kLaRows = 16;      // query rows = heads (<= 16), padded with zero rows: one mma M-tile

// Byte offset of 16-byte chunk `c` of row `r` in a [rows, D] bf16 tile whose row pitch is 2D bytes.  The chunk index is
// XORed with the row's low three bits, so the eight rows one ldmatrix phase reads hit eight different bank groups.
__device__ __forceinline__ uint32_t la_off(int r, int c, int D) { return r * (D * 2) + ((c ^ (r & 7)) << 4); }

__device__ __forceinline__ void la_cp16(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void la_ldsm4(uint32_t a, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void la_ldsm4t(uint32_t a, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}

// Shared memory: Q [16, D] | two key stages [16, D] | partial scores [4 column quarters][16][16] fp32
inline size_t la_smem_bytes(int D) { return (size_t)3 * kLaRows * D * 2 + 4 * kLaRows * kLaKeys * 4; }

// One CTA per sentence.  Each 16-key tile of the sentence's memory rows reaches shared memory once (cp.async, double
// buffered) and feeds both products on the tensor cores (mma.sync m16n8k16):
//   scores S[16 x 16] = Q . M^T: warp w computes key half (w & 1) over column quarter (w >> 1); the four quarters meet in
//   shared memory;
//   every warp then runs the same online softmax (identical inputs, identical m / l) and accumulates O += P . M over its
//   own D/8 columns.
// An empty sentence writes zeros.  u[b, h, :] = softmax_t(qt[b, h, :] . m_t / 8) . m for h < Hd.
template <int DQ>  // D = 256 * DQ
__global__ void __launch_bounds__(kLaThreads, 2)
pool_latent_attention_kernel(const __nv_bfloat16* __restrict__ qt, const __nv_bfloat16* __restrict__ mem,
                             const int32_t* __restrict__ cu, int Hd, __nv_bfloat16* __restrict__ u) {
  constexpr int D = 256 * DQ;
  constexpr int kChunks = D / 8;       // 16-byte chunks per row
  constexpr int kNT = D / 64;          // 8-column n-tiles of P . M per warp (a warp owns D/8 columns)
  constexpr int kKSteps = D / 64;      // k16 steps of a column quarter in Q . M^T
  constexpr int kTileBytes = kLaRows * D * 2;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem), sM0 = sQ + kTileBytes;
  float* sS = reinterpret_cast<float*>(smem + 3 * kTileBytes);
  const int b = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int start = cu[b], len = cu[b + 1] - start;
  const int g = lane >> 2, q4 = lane & 3;
  const int col0 = warp * (D / 8);  // this warp's output columns

  if (len <= 0) {
    for (int i = tid; i < Hd * kChunks; i += kLaThreads)
      reinterpret_cast<uint4*>(u + (long long)b * Hd * D)[i] = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  const int ntiles = (len + kLaKeys - 1) / kLaKeys;
  // rows past the sentence (or past Hd) are zero-filled: a masked key then contributes 0 * 0, never 0 * garbage
  auto load_tile = [&](int tile, uint32_t dst) {
#pragma unroll 1
    for (int i = 0; i < kLaKeys * kChunks / kLaThreads; ++i) {
      const int idx = i * kLaThreads + tid, r = idx / kChunks, c = idx % kChunks;
      const int key = tile * kLaKeys + r;
      const bool ok = key < len;
      la_cp16(dst + la_off(r, c, D), mem + (long long)(start + (ok ? key : 0)) * D + c * 8, ok);
    }
  };
#pragma unroll
  for (int i = 0; i < kLaRows * kChunks / kLaThreads; ++i) {
    const int idx = i * kLaThreads + tid, r = idx / kChunks, c = idx % kChunks;
    const bool ok = r < Hd;
    la_cp16(sQ + la_off(r, c, D), qt + ((long long)b * Hd + (ok ? r : 0)) * D + c * 8, ok);
  }
  load_tile(0, sM0);
  asm volatile("cp.async.commit_group;" ::: "memory");

  float o[kNT][4];
#pragma unroll
  for (int j = 0; j < kNT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_run[2] = {0.f, 0.f};  // rows g and g + 8
  const float sl2 = 0.125f * 1.4426950408889634f;
  const int kh = warp & 1, cq = warp >> 1;  // score work: key half, column quarter

  for (int tile = 0; tile < ntiles; ++tile) {
    const uint32_t sM = sM0 + (tile & 1) * kTileBytes;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();  // tile (and Q) visible to all; every warp is done with the other stage and with sS
    if (tile + 1 < ntiles) load_tile(tile + 1, sM0 + ((tile + 1) & 1) * kTileBytes);
    asm volatile("cp.async.commit_group;" ::: "memory");

    // ---- partial scores: keys [8 kh, 8 kh + 8) over columns [cq D/4, (cq + 1) D/4) ----
    float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int ks = 0; ks < kKSteps; ks += 2) {
      const int c0 = cq * (kChunks / 4) + ks * 2;  // first 16-byte chunk of this k-step pair
      uint32_t a0[4], a1[4], bm[4];
      la_ldsm4(sQ + la_off(lane & 15, c0 + (lane >> 4), D), a0[0], a0[1], a0[2], a0[3]);
      la_ldsm4(sQ + la_off(lane & 15, c0 + 2 + (lane >> 4), D), a1[0], a1[1], a1[2], a1[3]);
      la_ldsm4(sM + la_off(kh * 8 + (lane & 7), c0 + (lane >> 3), D), bm[0], bm[1], bm[2], bm[3]);
      mma_m16n8k16_bf16(s, a0, bm[0], bm[1]);
      mma_m16n8k16_bf16(s, a1, bm[2], bm[3]);
    }
    {
      float* dst = sS + cq * kLaRows * kLaKeys;
      *reinterpret_cast<float2*>(dst + g * kLaKeys + kh * 8 + 2 * q4) = make_float2(s[0], s[1]);
      *reinterpret_cast<float2*>(dst + (g + 8) * kLaKeys + kh * 8 + 2 * q4) = make_float2(s[2], s[3]);
    }
    __syncthreads();

    // ---- online softmax (every warp, same values): this thread's A-fragment entries of P ----
    // a0: (g, 2q4..+1)  a1: (g+8, 2q4..+1)  a2: (g, 8+2q4..+1)  a3: (g+8, 8+2q4..+1)
    float t[2][4];  // [row half][col 2q4, 2q4+1, 8+2q4, 9+2q4]
#pragma unroll
    for (int rh = 0; rh < 2; ++rh)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int row = g + rh * 8, col = (e >> 1) * 8 + 2 * q4 + (e & 1);
        float v = 0.f;
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) v += sS[(qq * kLaRows + row) * kLaKeys + col];
        t[rh][e] = (tile * kLaKeys + col < len) ? v * sl2 : -CUDART_INF_F;
      }
    uint32_t pa[4];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      float mx = fmaxf(fmaxf(t[rh][0], t[rh][1]), fmaxf(t[rh][2], t[rh][3]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m_run[rh], mx);  // finite: key tile*16 < len is always valid
      const float corr = exp2f(m_run[rh] - mn);
      m_run[rh] = mn;
      float p[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) p[e] = exp2f(t[rh][e] - mn);
      l_run[rh] = l_run[rh] * corr + ((p[0] + p[1]) + (p[2] + p[3]));
#pragma unroll
      for (int j = 0; j < kNT; ++j) { o[j][2 * rh] *= corr; o[j][2 * rh + 1] *= corr; }
      pa[rh] = pack_bf16x2(p[0], p[1]);
      pa[2 + rh] = pack_bf16x2(p[2], p[3]);
    }

    // ---- O[:, col0 .. col0 + D/8) += P . M ----
#pragma unroll
    for (int j = 0; j < kNT; j += 2) {
      uint32_t b0, b1, b2, b3;
      la_ldsm4t(sM + la_off(((lane >> 3) & 1) * 8 + (lane & 7), (col0 + j * 8) / 8 + (lane >> 4), D), b0, b1, b2, b3);
      mma_m16n8k16_bf16(o[j], pa, b0, b1);
      mma_m16n8k16_bf16(o[j + 1], pa, b2, b3);
    }
  }

  // ---- normalise and store rows < Hd ----
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    float l = l_run[rh];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = g + rh * 8;
    if (row < Hd) {
      const float inv = 1.0f / l;
      __nv_bfloat16* dst = u + ((long long)b * Hd + row) * D + col0 + 2 * q4;
#pragma unroll
      for (int j = 0; j < kNT; ++j)
        *reinterpret_cast<uint32_t*>(dst + j * 8) = pack_bf16x2(o[j][2 * rh] * inv, o[j][2 * rh + 1] * inv);
    }
  }
}

template <int DQ>
int launch_latent(const __nv_bfloat16* qt, const __nv_bfloat16* mem, const int32_t* cu, int B, int Hd, __nv_bfloat16* u,
                  cudaStream_t stream) {
  const size_t smem = la_smem_bytes(256 * DQ);
  static bool attr_set[64] = {};
  if (first_use_on_device(attr_set))
    SB_CUDA_CHECK(cudaFuncSetAttribute(pool_latent_attention_kernel<DQ>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
  pool_latent_attention_kernel<DQ><<<(unsigned)B, kLaThreads, smem, stream>>>(qt, mem, cu, Hd, u);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// create-time weight absorption (fp32 accumulation of the bf16 weights, one bf16 rounding of the product)
// ---------------------------------------------------------------------------------------------
// For every head h and 64 x 64 block (x, y):  out[h*soh + x*sox + y*soy] = bf16(sum_j P[(64h+j)*spj + x*spx] *
//                                                                                     Q[(64h+j)*sqj + y*sqy])
__global__ void __launch_bounds__(256)
absorb_heads_kernel(const __nv_bfloat16* __restrict__ P, long long spj, long long spx, const __nv_bfloat16* __restrict__ Q,
                    long long sqj, long long sqy, __nv_bfloat16* __restrict__ out, long long soh, long long sox,
                    long long soy) {
  __shared__ float sp[64][65], sq[64][65];
  const int h = blockIdx.z, x0 = blockIdx.x * 64, y0 = blockIdx.y * 64, tid = threadIdx.x;
  for (int i = tid; i < 64 * 64; i += 256) {
    const int j = i / 64, c = i % 64;
    const long long row = 64ll * h + j;
    sp[j][c] = __bfloat162float(P[row * spj + (x0 + c) * spx]);
    sq[j][c] = __bfloat162float(Q[row * sqj + (y0 + c) * sqy]);
  }
  __syncthreads();
  const int tx = tid % 16, ty = tid / 16;  // 4 x 4 outputs per thread: x = tx + 16 a, y = ty + 16 c
  float acc[4][4] = {};
  for (int j = 0; j < 64; ++j)
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(sp[j][tx + 16 * a], sq[j][ty + 16 * c], acc[a][c]);
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c)
      out[h * soh + (long long)(x0 + tx + 16 * a) * sox + (long long)(y0 + ty + 16 * c) * soy] = __float2bfloat16_rn(acc[a][c]);
}

// out[gi*X + x] = sum_{j < J} P[(gi*J + j)*spj + x*spx] * v[gi*J + j]  (+ add[gi*X + x]), fp64 accumulation
__global__ void __launch_bounds__(256)
absorb_bias_kernel(const __nv_bfloat16* __restrict__ P, long long spj, long long spx, const float* __restrict__ v, int J,
                   int X, int groups, const float* __restrict__ add, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= (long long)groups * X) return;
  const int gi = (int)(i / X), x = (int)(i % X);
  double s = add ? (double)add[i] : 0.0;
  for (int j = 0; j < J; ++j)
    s += (double)__bfloat162float(P[((long long)gi * J + j) * spj + (long long)x * spx]) * (double)v[gi * J + j];
  out[i] = (float)s;
}

}  // namespace

int pool_latent_attention(const __nv_bfloat16* qt, const __nv_bfloat16* mem, const int32_t* cu_seqlens, int B, int Hd, int D,
                          __nv_bfloat16* u, cudaStream_t stream) {
  if (B <= 0) return 0;
  if (Hd < 1 || Hd > kLaRows) { set_last_error("pool_latent_attention: 1 <= heads <= 16 required (got %d)", Hd); return -1; }
  switch (D) {
    case 256: return launch_latent<1>(qt, mem, cu_seqlens, B, Hd, u, stream);
    case 512: return launch_latent<2>(qt, mem, cu_seqlens, B, Hd, u, stream);
    case 768: return launch_latent<3>(qt, mem, cu_seqlens, B, Hd, u, stream);
    case 1024: return launch_latent<4>(qt, mem, cu_seqlens, B, Hd, u, stream);
    default: set_last_error("pool_latent_attention: width must be 256, 512, 768 or 1024 (got %d)", D); return -1;
  }
}

// Absorbs the cross-attention projections of one pooler layer (kv width D, pooler width E = 64 Hd) into the
// AttentionPooler::Layer weights wqk / bqk / wvo / bvo.
static int absorb_pooler_weights(const SbPoolerLayerWeights& P, int D, int E, __nv_bfloat16* wqk, float* bqk,
                                 __nv_bfloat16* wvo, float* bvo, cudaStream_t stream) {
  const int Hd = E / 64;
  const auto* wq = reinterpret_cast<const __nv_bfloat16*>(P.ca_wq);
  const auto* wk = reinterpret_cast<const __nv_bfloat16*>(P.ca_wkv);
  const auto* wv = wk + (long long)E * D;
  const auto* wo = reinterpret_cast<const __nv_bfloat16*>(P.ca_wo);
  // wqk [Hd*D, E]: row h*D + d = sum_j W_k[64h+j, d] W_q[64h+j, :];  bqk[h*D + d] = sum_j W_k[64h+j, d] b_q[64h+j]
  absorb_heads_kernel<<<dim3(D / 64, E / 64, Hd), 256, 0, stream>>>(wk, D, 1, wq, E, 1, wqk, (long long)D * E, E, 1);
  SB_CUDA_CHECK(cudaGetLastError());
  absorb_bias_kernel<<<(unsigned)(((long long)Hd * D + 255) / 256), 256, 0, stream>>>(wk, D, 1, P.ca_bq, 64, D, Hd, nullptr,
                                                                                      bqk);
  SB_CUDA_CHECK(cudaGetLastError());
  // wvo [E, Hd*D]: column h*D + d = sum_j W_o[:, 64h+j] W_v[64h+j, d];  bvo = W_o b_v + b_o
  absorb_heads_kernel<<<dim3(D / 64, E / 64, Hd), 256, 0, stream>>>(wv, D, 1, wo, 1, E, wvo, D, 1, (long long)Hd * D);
  SB_CUDA_CHECK(cudaGetLastError());
  absorb_bias_kernel<<<(unsigned)((E + 255) / 256), 256, 0, stream>>>(wo, 1, E, P.ca_bkv + E, E, E, 1, P.ca_bo, bvo);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int AttentionPooler::create(const char* who, const SbPoolerLayerWeights* w, int num_layers, const float* q0,
                            const void* proj_w, const float* proj_b, int D, int E, int F, float eps, int num_sms,
                            int cta_group, int allow_skinny) {
  if (!q0 || !proj_w || !proj_b || (num_layers > 0 && !w)) {
    set_last_error("%s: attention pooling needs pooler_q0, proj_w, proj_b and pooler", who);
    return SB_ERR_INVALID;
  }
  for (int i = 0; i < num_layers; ++i)
    if (has_null_pointer(w[i])) {
      set_last_error("%s: pooler layer %d has a null weight pointer", who, i);
      return SB_ERR_INVALID;
    }
  this->q0 = q0; this->proj_w = proj_w; this->proj_b = proj_b;
  this->D = D; this->E = E; this->F = F; this->eps = eps;
  this->num_sms = num_sms; this->cta_group = cta_group; this->allow_skinny = allow_skinny;
  layers.resize(num_layers);
  for (int i = 0; i < num_layers; ++i) layers[i].w = w[i];
  // absorbed cross-attention weights of every layer; the caller's weights are not modified
  const size_t HdD = (size_t)(E / 64) * D, Es = E;
  int rc = absorbed.alloc(who, "absorbed pooler weights", [&](Carver& c) {
    for (Layer& l : layers) {
      l.wqk = c.take<__nv_bfloat16>(HdD * Es * 2, 256);
      l.bqk = c.take<float>(HdD * 4, 256);
      l.wvo = c.take<__nv_bfloat16>(Es * HdD * 2, 256);
      l.bvo = c.take<float>(Es * 4, 256);
    }
  });
  if (rc) return rc;
  for (const Layer& l : layers)
    if ((rc = absorb_pooler_weights(l.w, D, E, l.wqk, l.bqk, l.wvo, l.bvo, nullptr))) return rc;
  return sync_prepared(who, "absorbing the pooler weights");
}

AttentionPooler::Ws AttentionPooler::take(Carver& c, size_t B) const {
  const size_t Ds = D, Es = E, Fs = F, HdD = (size_t)(E / 64) * D;
  Ws w;
  w.px = c.take<float>(B * (Ds > Es ? Ds : Es) * 4);
  w.ph = c.take<__nv_bfloat16>(B * Es * 2);
  w.pt = c.take<__nv_bfloat16>(B * (Fs > Es ? Fs : Es) * 2);
  w.qt = c.take<__nv_bfloat16>(B * HdD * 2);
  w.u = c.take<__nv_bfloat16>(B * HdD * 2);
  return w;
}

int AttentionPooler::forward(const Ws& w, const __nv_bfloat16* mem, const int32_t* cu_seqlens, int B, float* out,
                             cudaStream_t stream) const {
  const int Hd = E / 64, HdD = Hd * D;
  auto gemm = [&](const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int fp32,
                  const float* bias, int N, int K, int epi) {
    GemmArgs g = gemm_args(A, lda, W, ldw, C, ldc, fp32, bias, B, N, K, epi, num_sms);
    g.cta_group = cta_group;
    g.allow_skinny = allow_skinny;
    return gemm_bf16(g, stream);
  };
  int rc;
  if ((rc = broadcast_rows(q0, w.px, w.ph, B, E, stream))) return rc;
  for (const Layer& l : layers) {
    const SbPoolerLayerWeights& P = l.w;
    // self-attention over the single query token == Wo(Wv x + bv) + bo
    if ((rc = gemm(w.ph, E, P.sa_wv, E, w.pt, E, 0, P.sa_bv, E, E, EPI_BIAS))) return rc;
    if ((rc = gemm(w.pt, E, P.sa_wo, E, w.px, E, 1, P.sa_bo, E, E, EPI_BIAS_RESIDUAL))) return rc;
    if ((rc = layernorm_dual(w.px, P.sa_ln_g, P.sa_ln_b, eps, w.px, w.ph, B, E, stream))) return rc;
    // cross-attention over the sequence on the absorbed form
    if ((rc = gemm(w.ph, E, l.wqk, E, w.qt, HdD, 0, l.bqk, HdD, E, EPI_BIAS))) return rc;
    if ((rc = pool_latent_attention(w.qt, mem, cu_seqlens, B, Hd, D, w.u, stream))) return rc;
    if ((rc = gemm(w.u, HdD, l.wvo, HdD, w.px, E, 1, l.bvo, E, HdD, EPI_BIAS_RESIDUAL))) return rc;
    if ((rc = layernorm_dual(w.px, P.ca_ln_g, P.ca_ln_b, eps, w.px, w.ph, B, E, stream))) return rc;
    // ReLU FFN
    if ((rc = gemm(w.ph, E, P.w1, E, w.pt, F, 0, P.b1, F, E, EPI_BIAS_RELU))) return rc;
    if ((rc = gemm(w.pt, F, P.w2, F, w.px, E, 1, P.b2, E, F, EPI_BIAS_RESIDUAL))) return rc;
    if ((rc = layernorm_dual(w.px, P.ffn_ln_g, P.ffn_ln_b, eps, w.px, w.ph, B, E, stream))) return rc;
  }
  return gemm(w.ph, E, proj_w, E, out, E, 1, proj_b, E, E, EPI_BIAS);
}

}  // namespace sb
