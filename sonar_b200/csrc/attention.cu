// Bidirectional multi-head self-attention over PACKED variable-length sequences
// (no padded tokens exist in HBM, so there is no mask tensor: keys t >= len are simply
// never visited).  softmax(q k^T / sqrt(64)) v, head_dim 64, fp32 softmax/accumulate.
//
// Reference semantics: fairseq2 StandardMultiheadAttention + create_default_sdpa
// (sonar/models/sonar_text/factory.py:130-141) = F.scaled_dot_product_attention with
// a key-padding mask, scale 1/sqrt(head_dim), no causal mask (SURVEY App. A.2, F4).
//
// NOT on the product path any more (attention_tc.cu handles every length on wgmma); kept as `impl = 1` of
// sb_attention: an independent second implementation for tests and A/B timing.
// mma.sync.m16n8k16 bf16 (legacy tensor path), flash-style online softmax.
// One CTA = one (sequence, head, 128-query block); 8 warps x 16 query rows; K/V are
// streamed in 64-key blocks through swizzled shared memory with cp.async.
// At S=128 this op is ~1.2% of the encoder FLOPs and HBM-bound (reads 6 B/token/dim,
// writes 2); the wgmma kernel is described in DESIGN.md.

#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>

namespace sb {

namespace {

constexpr int kHeadDim = 64;
constexpr int kQBlock = 128;
constexpr int kKBlock = 64;

__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* gsrc, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                                  uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// smem tile: rows of 64 bf16 (128 B); 16-byte chunk c of row r is stored at chunk c ^ (r & 7)
__device__ __forceinline__ uint32_t tile_off(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

__global__ void __launch_bounds__(256)
attention_packed_kernel(const __nv_bfloat16* __restrict__ qkv, const int32_t* __restrict__ cu, int H,
                        __nv_bfloat16* __restrict__ out) {
  __shared__ __align__(128) uint8_t sQ[kQBlock * 128];
  __shared__ __align__(128) uint8_t sK[kKBlock * 128];
  __shared__ __align__(128) uint8_t sV[kKBlock * 128];

  const int qblk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int start = cu[b];
  const int len = cu[b + 1] - start;
  const int q0 = qblk * kQBlock;
  if (q0 >= len) return;
  const int D = H * kHeadDim;
  const long long row_stride = 3ll * D;  // elements
  const __nv_bfloat16* qbase = qkv + (long long)start * row_stride + h * kHeadDim;
  const __nv_bfloat16* kbase = qbase + D;
  const __nv_bfloat16* vbase = qbase + 2 * D;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t sQa = smem_u32(sQ), sKa = smem_u32(sK), sVa = smem_u32(sV);

  // ---- stage the Q block (rows beyond the sequence are zero-filled) ----
  for (int i = tid; i < kQBlock * 8; i += 256) {
    const int r = i >> 3, c = i & 7;
    const bool ok = (q0 + r) < len;
    cp_async_16(sQa + tile_off(r, c), qbase + (long long)(ok ? q0 + r : 0) * row_stride + c * 8, ok);
  }
  cp_async_commit();
  cp_async_wait_all();
  __syncthreads();

  // Q fragments for this warp's 16 rows: 4 k-steps of 16
  uint32_t qf[4][4];
  {
    const int r = warp * 16 + (lane & 15);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const int c = kk * 2 + (lane >> 4);
      ldmatrix_x4(sQa + tile_off(r, c), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
    }
  }

  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
  float m_run[2] = {-CUDART_INF_F, -CUDART_INF_F};
  float l_run[2] = {0.f, 0.f};
  const float sl2 = 0.125f * 1.4426950408889634f;  // 1/sqrt(64) * log2(e)

  const int nkb = (len + kKBlock - 1) / kKBlock;
  for (int kb = 0; kb < nkb; ++kb) {
    const int k0 = kb * kKBlock;
    __syncthreads();  // previous block's K/V fully consumed
    for (int i = tid; i < kKBlock * 8; i += 256) {
      const int r = i >> 3, c = i & 7;
      const bool ok = (k0 + r) < len;
      const long long g = (long long)(ok ? k0 + r : 0) * row_stride + c * 8;
      cp_async_16(sKa + tile_off(r, c), kbase + g, ok);
      cp_async_16(sVa + tile_off(r, c), vbase + g, ok);
    }
    cp_async_commit();
    cp_async_wait_all();
    __syncthreads();

    // ---- S = Q K^T for 16 rows x 64 keys ----
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of 8-key tiles
        const int mtx = lane >> 3;      // which 8x8 matrix this lane addresses
        const int key = (jp * 2 + (mtx >> 1)) * 8 + (lane & 7);
        const int c = kk * 2 + (mtx & 1);
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4(sKa + tile_off(key, c), b0, b1, b2, b3);
        mma_bf16_16816(s[jp * 2], qf[kk], b0, b1);
        mma_bf16_16816(s[jp * 2 + 1], qf[kk], b2, b3);
      }
    }

    // ---- mask keys beyond the sequence, online softmax ----
    const int kcol = k0 + (lane & 3) * 2;
    float mx[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kcol + j * 8 + (e & 1);
        if (key >= len) s[j][e] = -CUDART_INF_F;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[j][e]);
      }
    }
    float corr[2], mnew[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      mnew[r] = fmaxf(m_run[r], mx[r]);  // finite: key k0 < len always exists in a visited block
      corr[r] = exp2f((m_run[r] - mnew[r]) * sl2);
      m_run[r] = mnew[r];
      l_run[r] *= corr[r];
    }
    uint32_t pf[4][4];  // P as A-fragments: 4 k-steps of 16 keys
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = exp2f((s[j][0] - mnew[0]) * sl2);
      const float p1 = exp2f((s[j][1] - mnew[0]) * sl2);
      const float p2 = exp2f((s[j][2] - mnew[1]) * sl2);
      const float p3 = exp2f((s[j][3] - mnew[1]) * sl2);
      ls[0] += p0 + p1;
      ls[1] += p2 + p3;
      pf[j >> 1][(j & 1) * 2 + 0] = pack_bf16x2(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p2, p3);
      o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1];
    }
    l_run[0] += ls[0];
    l_run[1] += ls[1];

    // ---- O += P V ----
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of 8-wide d tiles
        const int mtx = lane >> 3;
        const int key = kk * 16 + (mtx & 1) * 8 + (lane & 7);
        const int c = jp * 2 + (mtx >> 1);
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(sVa + tile_off(key, c), b0, b1, b2, b3);
        mma_bf16_16816(o[jp * 2], pf[kk], b0, b1);
        mma_bf16_16816(o[jp * 2 + 1], pf[kk], b2, b3);
      }
    }
  }

  // ---- finalise: O /= l, stage through this warp's (now dead) Q rows, coalesced store ----
  float inv[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = l_run[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv[r] = 1.0f / l;
  }
  __syncwarp();
  {
    const int r0 = warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int byte_in_chunk = (lane & 3) * 4;
      *reinterpret_cast<uint32_t*>(sQ + tile_off(r0, j) + byte_in_chunk) = pack_bf16x2(o[j][0] * inv[0], o[j][1] * inv[0]);
      *reinterpret_cast<uint32_t*>(sQ + tile_off(r0 + 8, j) + byte_in_chunk) =
          pack_bf16x2(o[j][2] * inv[1], o[j][3] * inv[1]);
    }
  }
  __syncwarp();
  __nv_bfloat16* obase = out + (long long)start * D + h * kHeadDim;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = i * 32 + lane;  // 16 rows x 8 chunks
    const int r = warp * 16 + (idx >> 3), c = idx & 7;
    if (q0 + r < len)
      *reinterpret_cast<uint4*>(obase + (long long)(q0 + r) * D + c * 8) = *reinterpret_cast<const uint4*>(sQ + tile_off(r, c));
  }
}

}  // namespace

int attention_packed(const __nv_bfloat16* qkv, const int32_t* cu_seqlens, int B, int max_len, int H,
                     long long total_tokens, int impl, int num_sms, __nv_bfloat16* out, cudaStream_t stream) {
  if (B <= 0 || max_len <= 0) return 0;
  if (H <= 0 || H > 65535 || B > 65535) {
    set_last_error("attention_packed: unsupported B=%d H=%d", B, H);
    return -1;
  }
  // impl 0 (auto) and 2: the wgmma kernel, any sequence length (128-key tiles with online softmax beyond 128 tokens);
  // impl 1 keeps the mma.sync flash kernel below reachable for A/B measurements and as a second implementation in tests
  if (impl != 1) return attention_packed_tc(qkv, cu_seqlens, B, H, total_tokens, out, num_sms, stream);
  dim3 grid((unsigned)((max_len + kQBlock - 1) / kQBlock), (unsigned)H, (unsigned)B);
  attention_packed_kernel<<<grid, 256, 0, stream>>>(qkv, cu_seqlens, H, out);
  SB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace sb
