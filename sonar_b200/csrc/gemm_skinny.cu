// Skinny GEMM for a handful of rows (M <= 64): C[M,N] = epi(A[M,K] . W[N,K]^T + bias).
//
// The decoder's beam step at the pipelines' default batch (5 sentences x beam 5 = 25 hypothesis rows) and the speech
// pooler's single-query layers multiply a few activation rows with full weight matrices.  The 128 x 256 wgmma tiles of
// gemm_wgmma.cu spend a whole tile's MMA time on mostly-zero rows and put only N/256 CTA pairs on the machine, so a
// [25 x 8192] . [8192 x 1024] product takes ~50 us.  This path is the opposite design point: the work is streaming W once
// from HBM, so every CTA owns 8 rows of W (one n8 tile -> N/8 CTAs cover the SMs), its 8 warps split K, each lane pulls
// 16 contiguous bytes of "its" W row and of the activation rows straight from global memory, and the products run on
// mma.sync m16n8k16 with the activations as the A operand.  The K order inside a 32-element chunk is permuted identically
// for both operands (lane t owns elements 8t..8t+7), which a dot product does not see and which makes every load a full
// 16-byte vector.  The 8 per-warp partial tiles are summed through shared memory in warp order (deterministic) and the
// epilogue (bias, ReLU / SiLU, in-place fp32 residual) is applied once.
#include "common.cuh"
#include "sonar_b200_internal.h"

namespace sb {
namespace {

// The kernel is bound by loaded HBM latency (~2 us), so what matters is bytes in flight.  A CTA's 8 warps cover 1024
// elements of K in one shot (8 rows x 2 KB of W, all loads issued before the first mma); longer K is split over a
// thread-block CLUSTER of K/1024 CTAs along grid.y whose partial tiles meet in the leader CTA's shared memory (DSMEM
// stores + one cluster barrier) and are summed there in rank order -- still deterministic, still one launch.
constexpr int kSkinnyWarps = 8;
constexpr int kSkinnyThreads = kSkinnyWarps * 32;
constexpr int kSkinnyMaxSplit = 8;  // portable cluster size

__device__ __forceinline__ void st_shared_cluster_f32(const float* local_addr, uint32_t cta, float v) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "st.shared::cluster.f32 [ra], %2;\n\t"
      "}\n" ::"r"(smem_u32(local_addr)),
      "r"(cta), "f"(v)
      : "memory");
}

// MT = number of 16-row activation tiles (M <= 16 * MT); UNROLL = 32-element chunks in flight per lane;
// gridDim.y = cluster size = number of K splits (1..8)
template <int MT, int UNROLL, typename OutT>
__global__ void __launch_bounds__(kSkinnyThreads)
gemm_skinny_kernel(const __nv_bfloat16* __restrict__ A, long long lda, const __nv_bfloat16* __restrict__ W, long long ldw,
                   OutT* C, long long ldc, const float* __restrict__ bias, int M, int N, int K, int epi) {
  __shared__ float part[kSkinnyWarps][MT * 16][8 + 1];
  __shared__ float split_part[kSkinnyMaxSplit][MT * 16][8];  // leader CTA: one partial tile per cluster rank
  const int nsplit = gridDim.y;
  const uint32_t rank = (nsplit > 1) ? cluster_ctarank() : 0u;
  if (nsplit > 1) cluster_sync_all();  // every CTA of the cluster is running before anyone stores into the leader's shared memory
  const int n0 = blockIdx.x * 8;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int kslice = K / (kSkinnyWarps * nsplit);  // multiple of 32 (host checks)
  const int kbeg = (int(rank) * kSkinnyWarps + warp) * kslice;
  const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
  const __nv_bfloat16* wrow = W + (long long)(n0 + g) * ldw + kbeg + 8 * t;
  const __nv_bfloat16* arow[MT][2];
  bool aok[MT][2];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = i * 16 + hh * 8 + g;
      aok[i][hh] = r < M;
      arow[i][hh] = A + (long long)(aok[i][hh] ? r : 0) * lda + kbeg + 8 * t;
    }
  float acc[MT][4];
#pragma unroll
  for (int i = 0; i < MT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  constexpr int kUnroll = UNROLL;
  for (int k = 0; k < kslice; k += 32 * kUnroll) {
    uint4 w4[kUnroll], a4[kUnroll][MT][2];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const bool in = k + 32 * u < kslice;
      w4[u] = in ? __ldg(reinterpret_cast<const uint4*>(wrow + k + 32 * u)) : zero4;
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          a4[u][i][hh] = (in && aok[i][hh]) ? __ldg(reinterpret_cast<const uint4*>(arow[i][hh] + k + 32 * u)) : zero4;
    }
    asm volatile("" ::: "memory");  // scheduling fence: every load of the pass is issued before the first mma consumes one
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
#pragma unroll
      for (int i = 0; i < MT; ++i) {
        const uint32_t lo[4] = {a4[u][i][0].x, a4[u][i][1].x, a4[u][i][0].y, a4[u][i][1].y};
        const uint32_t hi[4] = {a4[u][i][0].z, a4[u][i][1].z, a4[u][i][0].w, a4[u][i][1].w};
        mma_m16n8k16_bf16(acc[i], lo, w4[u].x, w4[u].y);
        mma_m16n8k16_bf16(acc[i], hi, w4[u].z, w4[u].w);
      }
  }
  // accumulator fragment: c0,c1 -> (row g, cols 2t,2t+1); c2,c3 -> (row g+8, cols 2t,2t+1)
#pragma unroll
  for (int i = 0; i < MT; ++i) {
    part[warp][i * 16 + g][2 * t] = acc[i][0];
    part[warp][i * 16 + g][2 * t + 1] = acc[i][1];
    part[warp][i * 16 + g + 8][2 * t] = acc[i][2];
    part[warp][i * 16 + g + 8][2 * t + 1] = acc[i][3];
  }
  __syncthreads();
  if (nsplit > 1) {
    // every CTA of the cluster reduces its 8 warps in order and drops the tile into slot `rank` of the leader's buffer
    for (int o = tid; o < MT * 16 * 8; o += kSkinnyThreads) {
      const int r = o >> 3, c = o & 7;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kSkinnyWarps; ++w) v += part[w][r][c];
      st_shared_cluster_f32(&split_part[rank][r][c], 0u, v);
    }
    cluster_sync_all();  // release/acquire at cluster scope: the leader sees every slot
    if (rank != 0) return;
  }
  for (int o = tid; o < MT * 16 * 8; o += kSkinnyThreads) {
    const int r = o >> 3, c = o & 7;
    if (r >= M) continue;
    float v = 0.f;
    if (nsplit > 1) {
      for (int q = 0; q < nsplit; ++q) v += split_part[q][r][c];  // rank order: bitwise reproducible
    } else {
#pragma unroll
      for (int w = 0; w < kSkinnyWarps; ++w) v += part[w][r][c];  // fixed order: bitwise reproducible
    }
    if (bias) v += bias[n0 + c];
    if (epi == EPI_BIAS_RELU) v = fmaxf(v, 0.f);
    if (epi == EPI_BIAS_SILU) v = silu_fast(v);
    OutT* dst = C + (long long)r * ldc + n0 + c;
    if constexpr (sizeof(OutT) == 4) {
      if (epi == EPI_BIAS_RESIDUAL || epi == EPI_BIAS_ACCUM) v = *dst + v;  // same rounding as the wgmma path: fl(x + fl(acc + bias))
      *dst = v;
    } else {
      *dst = __float2bfloat16_rn(v);
    }
  }
}

template <int MT, int UNROLL>
int launch_skinny(const GemmArgs& g, cudaStream_t stream) {
  // K splits: one CTA per 1024 elements of K (cluster along grid.y, at most 8), each warp's slice a multiple of 32
  int nsplit = g.K / 1024;
  if (nsplit > kSkinnyMaxSplit) nsplit = kSkinnyMaxSplit;
  while (nsplit > 1 && g.K % (nsplit * kSkinnyWarps * 32) != 0) --nsplit;
  if (nsplit < 1) nsplit = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(g.N / 8), (unsigned)nsplit, 1);
  cfg.blockDim = dim3(kSkinnyThreads, 1, 1);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = (unsigned)nsplit;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e;
  if (g.out_fp32)
    e = cudaLaunchKernelEx(&cfg, gemm_skinny_kernel<MT, UNROLL, float>, g.A, g.lda, g.W, g.ldw,
                           reinterpret_cast<float*>(g.C), g.ldc, g.bias, g.M, g.N, g.K, g.epi);
  else
    e = cudaLaunchKernelEx(&cfg, gemm_skinny_kernel<MT, UNROLL, __nv_bfloat16>, g.A, g.lda, g.W, g.ldw,
                           reinterpret_cast<__nv_bfloat16*>(g.C), g.ldc, g.bias, g.M, g.N, g.K, g.epi);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("gemm_skinny launch failed: %s", cudaGetErrorString(e));
    return -2;
  }
  return 0;
}

}  // namespace

bool gemm_skinny_eligible(const GemmArgs& g) {
  if (g.M <= 0 || g.M > 64 || g.N % 8 != 0 || g.K % 256 != 0) return false;
  if (g.lda % 8 != 0 || g.ldw % 8 != 0) return false;  // 16-byte vector loads
  if ((reinterpret_cast<uintptr_t>(g.A) | reinterpret_cast<uintptr_t>(g.W)) & 15) return false;
  switch (g.epi) {
    case EPI_BIAS:
    case EPI_BIAS_RELU:
    case EPI_BIAS_SILU:
      return true;
    case EPI_BIAS_RESIDUAL:
    case EPI_BIAS_ACCUM:  // only the in-place fp32 form x += A.W^T + b
      return g.out_fp32 && (g.epi == EPI_BIAS_ACCUM || (g.residual == g.C && g.ldr == g.ldc));
    default:
      return false;
  }
}

int gemm_skinny(const GemmArgs& g, cudaStream_t stream) {
  if (g.M <= 16) return launch_skinny<1, 4>(g, stream);
  if (g.M <= 32) return launch_skinny<2, 4>(g, stream);
  return launch_skinny<4, 4>(g, stream);
}

}  // namespace sb
