// The LASER2 text encoder (LaserLstmEncoder, sonar/nn/laser_lstm_encoder.py:60-116; `laser2` config,
// sonar/models/laser2_text/config.py:28-38): embedding gather -> num_layers x [ input GEMM (gemm_bf16) -> recurrent kernel ]
// -> max over time, which the last layer's recurrent kernel keeps in registers.
//
// Per layer and direction, with gate order i, f, g, o in the stacked [4H, in] matrices of torch.nn.LSTM:
//   G   = X . W_ih^T + (b_ih + b_hh)                  all T packed tokens at once, bf16 [T, dirs * 4H]
//   z   = G[token of step s] + h_{s-1} . W_hh^T
//   c_s = sigmoid(z_f) c_{s-1} + sigmoid(z_i) tanh(z_g),   h_s = sigmoid(z_o) tanh(c_s),   h_{-1} = c_{-1} = 0
// Sequence b runs over its own len_b positions; the reverse direction visits position len_b - 1 - s at step s.
//
// Recurrent kernel (H = 512): one 16-CTA thread-block cluster owns one direction and one tile of 64 sequences for the
// whole sequence.  CTA c owns hidden units [32c, 32c + 32) of all four gates, i.e. 128 gate columns; its 128 x 512 slice of
// W_hh (128 KB) stays in shared memory for every step, next to the full h_{s-1} [64 x 512] bf16 of the tile (64 KB).
// The engine repacks W_ih / W_hh rows at create so that CTA c's i / f / g / o columns are adjacent (lstm_gate_row); G
// comes out of the input GEMM in the same order.  One step:
//   wgmma m64n128k16 x 32 (h_{s-1} . W_hh,slice^T) -> cluster barrier arrive (done reading h) -> gates from the
//   accumulators + G (prefetched one step ahead) -> c in fp32 registers -> own slice of h_s into the local h buffer ->
//   wait (every CTA done reading) -> DSMEM copy of the 4 KB slice into the 15 peers -> arrive / wait (h_s complete).
// Each accumulator row depends on its own h row only, so a row's result does not depend on its tile neighbours.
// Both shared-memory operands use the unswizzled K-major core-matrix layout (8 rows x 16 bytes), in which CTA c's slice
// of h (k in [32c, 32c + 32)) is one contiguous 4 KB block.

#include "../../include/sonar_b200.h"

#include "common.cuh"
#include "sonar_b200_internal.h"

#include <math_constants.h>

#include <algorithm>
#include <memory>
#include <new>
#include <numeric>
#include <vector>

namespace sb {
namespace {

constexpr int kLstmH = 512;                      // hidden size: the only one the recurrent kernel supports
constexpr int kLstmCtas = 16;                    // CTAs per cluster
constexpr int kLstmUnits = kLstmH / kLstmCtas;   // hidden units per CTA (32)
constexpr int kLstmCols = 4 * kLstmUnits;        // gate columns per CTA (128)
constexpr int kLstmRows = 64;                    // sequences per tile (the wgmma M)
constexpr int kLstmThreads = 128;                // one warpgroup
constexpr int kLstmWBytes = kLstmCols * kLstmH * 2;  // 128 KB
constexpr int kLstmHBytes = kLstmRows * kLstmH * 2;  // 64 KB
constexpr int kLstmSmem = kLstmWBytes + kLstmHBytes;
// core-matrix strides: h [k/8][r/8][r%8][k%8], W [k/8][n/8][n%8][k%8]
constexpr uint32_t kHKGroup = (kLstmRows / 8) * 128;  // 1024 B between k-groups of h
constexpr uint32_t kWKGroup = (kLstmCols / 8) * 128;  // 2048 B between k-groups of W
constexpr int kSliceBytes = (kLstmUnits / 8) * kHKGroup;  // 4 KB: one CTA's h slice

struct LstmArgs {
  const __nv_bfloat16* G;  // [T, ldg]; direction d's 4H columns start at d * 4H, in lstm_gate_row order
  long long ldg;
  const __nv_bfloat16* Whh;  // [dirs, 4H, H], rows in lstm_gate_row order
  const int32_t* cu;         // [B + 1]
  const int32_t* tile_seqs;  // [tiles * 64] sequence index or -1
  __nv_bfloat16* Y;          // [T, ldy], direction d at columns d * H (null with pool)
  long long ldy;
  float* pool;  // [B, ldp] max over time, direction d at columns d * H (null with Y)
  long long ldp;
  const uint8_t* pad;   // [T] 1 = the token's id is pad_idx (pool only; null = none is)
  const uint8_t* tail;  // [B] 1 = a position >= len_b holds another id (pool only; null = none does)
  float pad_value;
};

// Unswizzled K-major wgmma descriptor: LBO = bytes between the two core matrices of a k16 step, SBO = bytes between
// 8-row groups.
__device__ __forceinline__ uint64_t lstm_desc(uint32_t addr, uint32_t lbo, uint32_t sbo) {
  return uint64_t((addr >> 4) & 0x3FFFu) | (uint64_t((lbo >> 4) & 0x3FFFu) << 16) | (uint64_t((sbo >> 4) & 0x3FFFu) << 32);
}

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// 16 bytes to the same shared-memory offset in CTA `cta` of the cluster
__device__ __forceinline__ void st_cluster_v4(uint32_t local_addr, uint32_t cta, const int4& v) {
  asm volatile(
      "{\n\t"
      ".reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "st.shared::cluster.v4.b32 [ra], {%2, %3, %4, %5};\n\t"
      "}\n" ::"r"(local_addr),
      "r"(cta), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
      : "memory");
}

// 1 / (1 + e^-x) with the SFU exponential and reciprocal (no IEEE-division slow path: no function call in this kernel)
__device__ __forceinline__ float lstm_sigmoid(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }

__device__ __forceinline__ float2 bf16x2_to_float2(uint32_t u) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
}

// Thread t of the warpgroup (warp w, lane l, q = l % 4) owns rows r_i = 16 w + l / 4 + 8 i (i = 0, 1) and hidden units
// 32 c + 8 j + 2 q + e (j = 0..3, e = 0, 1): the accumulator columns gate * 32 + 8 j + 2 q + e, i.e. accumulator pairs
// d[4 (4 gate + j) + 2 i + e].  Its G values for one step: g[(4 i + gate) * 4 + j] = the bf16 pair of units (e = 0, 1).
template <bool kPool>
__global__ void __launch_bounds__(kLstmThreads, 1) lstm_recurrent_kernel(const LstmArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ int s_len[4];
  uint8_t* w_s = smem;
  uint8_t* h_s = smem + kLstmWBytes;
  const int c = (int)cluster_ctarank();
  const int tile = blockIdx.y, dir = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 3;

  // W_hh slice -> shared memory (once)
  {
    const int4* wg = reinterpret_cast<const int4*>(a.Whh + ((size_t)dir * 4 * kLstmH + (size_t)c * kLstmCols) * kLstmH);
    for (int i = tid; i < kLstmCols * (kLstmH / 8); i += kLstmThreads) {
      const int n = i / (kLstmH / 8), kg = i % (kLstmH / 8);
      *reinterpret_cast<int4*>(w_s + kg * kWKGroup + (n >> 3) * 128 + (n & 7) * 16) = __ldg(wg + i);
    }
    for (int i = tid; i < kLstmHBytes / 16; i += kLstmThreads) reinterpret_cast<int4*>(h_s)[i] = make_int4(0, 0, 0, 0);
  }
  int seq[2], len[2], base[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = 16 * warp + (lane >> 2) + 8 * i;
    seq[i] = a.tile_seqs[(size_t)tile * kLstmRows + r];
    base[i] = seq[i] >= 0 ? a.cu[seq[i]] : 0;
    len[i] = seq[i] >= 0 ? a.cu[seq[i] + 1] - base[i] : 0;
  }
  {
    const int m = __reduce_max_sync(0xffffffffu, max(len[0], len[1]));
    if (lane == 0) s_len[warp] = m;
  }
  fence_proxy_async_smem();  // the generic-proxy writes above -> visible to wgmma
  __syncthreads();
  const int steps = max(max(s_len[0], s_len[1]), max(s_len[2], s_len[3]));  // identical in every CTA of the cluster

  // this thread's G pairs at step s (zeros for a finished row) and, for the pool, whether that token is a pad id
  const __nv_bfloat16* g_col = a.G + (size_t)dir * 4 * kLstmH + (size_t)c * kLstmCols + 2 * q;
  auto load_g = [&](int s, uint32_t (&g)[32], bool (&padded)[2]) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const bool live = s < len[i];
      const long long tok = base[i] + (dir ? len[i] - 1 - s : s);
      const uint32_t* p = reinterpret_cast<const uint32_t*>(g_col + (live ? tok : 0) * a.ldg);
#pragma unroll
      for (int gate = 0; gate < 4; ++gate)
#pragma unroll
        for (int j = 0; j < 4; ++j) g[(4 * i + gate) * 4 + j] = live ? __ldg(p + (gate * 32 + 8 * j) / 2) : 0u;
      if (kPool) padded[i] = live && a.pad != nullptr && a.pad[tok] != 0;
    }
  };

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  float cst[16], hmax[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) { cst[i] = 0.f; hmax[i] = -CUDART_INF_F; }
  uint32_t g_next[32];
  bool pad_next[2] = {false, false};
  load_g(0, g_next, pad_next);

  const uint32_t h_addr = smem_u32(h_s), w_addr = smem_u32(w_s);
  const uint32_t slice_addr = h_addr + (uint32_t)c * kSliceBytes;
  cluster_sync_all();  // every CTA of the cluster is running and has zeroed its h

  for (int s = 0; s < steps; ++s) {
    if (s > 0) cluster_wait();  // h_{s-1} is complete in every CTA
    fence_proxy_async_smem();
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kLstmH / 16; ++kk)
      wgmma_m64n128k16_ss(acc, lstm_desc(h_addr + kk * 2 * kHKGroup, kHKGroup, 128),
                          lstm_desc(w_addr + kk * 2 * kWKGroup, kWKGroup, 128), kk > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    cluster_arrive();  // this CTA has finished reading h_{s-1}

    uint32_t g[32];
    bool padded[2];
#pragma unroll
    for (int i = 0; i < 32; ++i) g[i] = g_next[i];
    padded[0] = pad_next[0];
    padded[1] = pad_next[1];
    if (s + 1 < steps) load_g(s + 1, g_next, pad_next);

#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (s >= len[i]) continue;  // a finished row keeps its state and writes nothing
      const int r = 16 * warp + (lane >> 2) + 8 * i;
      const long long tok = base[i] + (dir ? len[i] - 1 - s : s);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float hv[2];
        const float2 gi = bf16x2_to_float2(g[(4 * i + 0) * 4 + j]), gf = bf16x2_to_float2(g[(4 * i + 1) * 4 + j]);
        const float2 gg = bf16x2_to_float2(g[(4 * i + 2) * 4 + j]), go = bf16x2_to_float2(g[(4 * i + 3) * 4 + j]);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float zi = acc[4 * (0 + j) + 2 * i + e] + (e ? gi.y : gi.x);
          const float zf = acc[4 * (4 + j) + 2 * i + e] + (e ? gf.y : gf.x);
          const float zg = acc[4 * (8 + j) + 2 * i + e] + (e ? gg.y : gg.x);
          const float zo = acc[4 * (12 + j) + 2 * i + e] + (e ? go.y : go.x);
          float& cc = cst[8 * i + 2 * j + e];
          cc = lstm_sigmoid(zf) * cc + lstm_sigmoid(zi) * tanhf(zg);
          hv[e] = lstm_sigmoid(zo) * tanhf(cc);
          if (kPool && !padded[i]) hmax[8 * i + 2 * j + e] = fmaxf(hmax[8 * i + 2 * j + e], hv[e]);
        }
        const uint32_t packed = pack_bf16x2(hv[0], hv[1]);
        *reinterpret_cast<uint32_t*>(h_s + (c * 4 + j) * kHKGroup + (r >> 3) * 128 + (r & 7) * 16 + q * 4) = packed;
        if (!kPool)
          *reinterpret_cast<uint32_t*>(a.Y + tok * a.ldy + (size_t)dir * kLstmH + c * kLstmUnits + 8 * j + 2 * q) = packed;
      }
    }
    __syncthreads();  // the own slice of h_s is complete
    cluster_wait();   // every CTA has finished reading h_{s-1}
    if (s + 1 < steps) {
      const int4 v0 = *reinterpret_cast<const int4*>(h_s + c * kSliceBytes + tid * 16);
      const int4 v1 = *reinterpret_cast<const int4*>(h_s + c * kSliceBytes + (tid + kLstmThreads) * 16);
#pragma unroll 1
      for (int p = 1; p < kLstmCtas; ++p) {
        const uint32_t peer = (uint32_t)((c + p) % kLstmCtas);
        st_cluster_v4(slice_addr + tid * 16, peer, v0);
        st_cluster_v4(slice_addr + (tid + kLstmThreads) * 16, peer, v1);
      }
    }
    cluster_arrive();  // this CTA's slice of h_s is in every CTA
  }
  if (steps > 0) cluster_wait();  // no CTA leaves while a peer may still write into its shared memory

  if (kPool) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (seq[i] < 0) continue;
      const bool tail = a.tail != nullptr && a.tail[seq[i]] != 0;
      float* o = a.pool + (size_t)seq[i] * a.ldp + (size_t)dir * kLstmH + c * kLstmUnits + 2 * q;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 v = make_float2(hmax[8 * i + 2 * j], hmax[8 * i + 2 * j + 1]);
        if (tail) { v.x = fmaxf(v.x, a.pad_value); v.y = fmaxf(v.y, a.pad_value); }
        *reinterpret_cast<float2*>(o + 8 * j) = v;
      }
    }
  }
}

// X[cu[b] + t, :] = E[ids[b, t], :] (bf16, width D a multiple of 8), pad[cu[b] + t] = (ids[b, t] == pad_idx) for t < len_b,
// tail[b] = any ids[b, t] != pad_idx for len_b <= t < S; an id outside [0, vocab) sets *err and gathers zeros.
__global__ void laser_embed_kernel(const int64_t* __restrict__ ids, long long stride, const int32_t* __restrict__ cu, int S,
                                   const int4* __restrict__ E, long long vocab, int D, long long pad_idx, int4* __restrict__ X,
                                   uint8_t* __restrict__ pad, uint8_t* __restrict__ tail, int* err) {
  const int b = blockIdx.x;
  const int base = cu[b], len = cu[b + 1] - base;
  const int chunks = D / 8;
  const int64_t* row = ids + (size_t)b * stride;
  for (int i = threadIdx.x; i < len * chunks; i += blockDim.x) {
    const int t = i / chunks, k = i % chunks;
    const long long id = row[t];
    const bool ok = id >= 0 && id < vocab;
    if (!ok) atomicExch(err, 1);
    X[(size_t)(base + t) * chunks + k] = ok ? __ldg(E + id * chunks + k) : make_int4(0, 0, 0, 0);
    if (k == 0) pad[base + t] = id == pad_idx;
  }
  int keep = 0;
  for (int t = len + threadIdx.x; t < S; t += blockDim.x) keep |= row[t] != pad_idx;
  keep = __syncthreads_or(keep);
  if (threadIdx.x == 0) tail[b] = keep != 0;
}

// dst row n <- src row lstm_gate_row(n) of a [4H, K] bf16 matrix, for `dirs` stacked matrices
__device__ __forceinline__ int lstm_gate_row(int n) {
  const int cta = n / kLstmCols, gate = (n % kLstmCols) / kLstmUnits, u = n % kLstmUnits;
  return gate * kLstmH + cta * kLstmUnits + u;
}

__global__ void lstm_repack_rows_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int K) {
  const int n = blockIdx.x;
  const __nv_bfloat16* s = src + (size_t)lstm_gate_row(n) * K;
  for (int k = threadIdx.x; k < K; k += blockDim.x) dst[(size_t)n * K + k] = s[k];
}

__global__ void lstm_repack_bias_kernel(const float* __restrict__ b_ih, const float* __restrict__ b_hh, float* __restrict__ dst) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < 4 * kLstmH) dst[n] = b_ih[lstm_gate_row(n)] + b_hh[lstm_gate_row(n)];
}

template <bool kPool>
int lstm_prepare() {
  static bool done[64];
  if (first_use_on_device(done)) {
    SB_CUDA_CHECK(cudaFuncSetAttribute(lstm_recurrent_kernel<kPool>, cudaFuncAttributeMaxDynamicSharedMemorySize, kLstmSmem));
    SB_CUDA_CHECK(cudaFuncSetAttribute(lstm_recurrent_kernel<kPool>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  }
  return SB_OK;
}

void lstm_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int tiles, int dirs, cudaStream_t stream) {
  *cfg = cudaLaunchConfig_t{};
  cfg->gridDim = dim3(kLstmCtas, tiles, dirs);
  cfg->blockDim = dim3(kLstmThreads, 1, 1);
  cfg->dynamicSmemBytes = kLstmSmem;
  cfg->stream = stream;
  attr->id = cudaLaunchAttributeClusterDimension;
  attr->val.clusterDim.x = kLstmCtas;
  attr->val.clusterDim.y = 1;
  attr->val.clusterDim.z = 1;
  cfg->attrs = attr;
  cfg->numAttrs = 1;
}

int lstm_recurrent(const LstmArgs& a, int tiles, int dirs, cudaStream_t stream) {
  if (tiles <= 0 || tiles > 65535 || dirs < 1 || dirs > 2) {
    set_last_error("lstm_recurrent: bad grid (%d tiles, %d directions)", tiles, dirs);
    return SB_ERR_INVALID;
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr;
  lstm_launch_config(&cfg, &attr, tiles, dirs, stream);
  if (a.pool) {
    if (int rc = lstm_prepare<true>()) return rc;
    SB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, lstm_recurrent_kernel<true>, a));
  } else {
    if (int rc = lstm_prepare<false>()) return rc;
    SB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, lstm_recurrent_kernel<false>, a));
  }
  return SB_OK;
}

// SB_ERR_CUDA unless at least one 16-CTA cluster of the recurrent kernel fits on the device
int lstm_check_cluster_fit(const char* who) {
  for (int pool = 0; pool < 2; ++pool) {
    if (int rc = pool ? lstm_prepare<true>() : lstm_prepare<false>()) return rc;
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr;
    lstm_launch_config(&cfg, &attr, 1, 1, nullptr);
    int n = 0;
    const cudaError_t e = pool ? cudaOccupancyMaxActiveClusters(&n, lstm_recurrent_kernel<true>, &cfg)
                               : cudaOccupancyMaxActiveClusters(&n, lstm_recurrent_kernel<false>, &cfg);
    if (e != cudaSuccess || n < 1) {
      set_last_error("%s: the LSTM recurrent kernel's %d-CTA cluster (%d KB of shared memory per CTA) does not fit on this "
                     "device (cudaOccupancyMaxActiveClusters: %d, %s)", who, kLstmCtas, kLstmSmem / 1024, n,
                     cudaGetErrorString(e));
      return SB_ERR_CUDA;
    }
  }
  return SB_OK;
}

struct LaserWs {
  int32_t* cu;         // [B + 1]
  int32_t* tile_seqs;  // [tiles * 64]
  uint8_t* pad;        // [T]
  uint8_t* tail;       // [B]
  __nv_bfloat16* xy;   // [T, max(E, dirs * H)]: layer 0's embeddings, then every layer's output
  __nv_bfloat16* g;    // [T, dirs * 4H]
  size_t bytes;
};

int lstm_tiles(long long B) { return (int)((B + kLstmRows - 1) / kLstmRows); }

bool aligned_to(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

}  // namespace
}  // namespace sb

using namespace sb;

struct SbLaser2 {
  SbLaser2Config cfg;
  int dirs = 1;
  const void* embed = nullptr;
  WeightPool packed;  // behind every repacked weight below
  std::vector<__nv_bfloat16*> w_ih;  // per layer [dirs * 4H, in_l], rows in lstm_gate_row order per direction
  std::vector<float*> bias;          // per layer [dirs * 4H] = b_ih + b_hh, same order
  std::vector<__nv_bfloat16*> w_hh;  // per layer [dirs, 4H, H], same order
  InputFlag err_flag;
  int num_sms = 0;
  static constexpr int kMaxBatch = 32768;
  static constexpr int kSlotInts = (kMaxBatch + 1) + kMaxBatch + kLstmRows;
  StagingRing staging;  // cu_seqlens, then the length-sorted tiles
};

static LaserWs laser_carve(const SbLaser2* e, long long B, long long T, void* base) {
  const size_t H = kLstmH, dirs = e->dirs;
  const size_t width = std::max<size_t>((size_t)e->cfg.embed_dim, dirs * H);
  const size_t T_ = (size_t)std::max(T, 1ll);
  Carver c(base);
  LaserWs w;
  w.cu = c.take<int32_t>(sizeof(int32_t) * (size_t)(B + 1));
  w.tile_seqs = c.take<int32_t>(sizeof(int32_t) * (size_t)lstm_tiles(B) * kLstmRows);
  w.pad = c.take<uint8_t>(T_);
  w.tail = c.take<uint8_t>((size_t)B);
  w.xy = c.take<__nv_bfloat16>(T_ * width * 2);
  w.g = c.take<__nv_bfloat16>(T_ * dirs * 4 * H * 2);
  w.bytes = c.off;
  return w;
}

extern "C" {

int sb_laser2_create(const SbLaser2Config* cfg, const SbLaser2Weights* w, SbLaser2** out) {
  if (!cfg || !w || !out) { set_last_error("sb_laser2_create: null argument"); return SB_ERR_INVALID; }
  *out = nullptr;
  if (cfg->hidden_size != kLstmH || cfg->embed_dim <= 0 || cfg->embed_dim % 64 != 0 || cfg->num_layers < 1 ||
      (cfg->bidirectional != 0 && cfg->bidirectional != 1) || cfg->vocab_size <= 0) {
    set_last_error("sb_laser2_create: outside the engine's envelope (hidden_size 512, embed_dim a positive multiple of 64, "
                   "num_layers >= 1, bidirectional 0 or 1, vocab_size >= 1); got hidden_size=%d embed_dim=%d num_layers=%d "
                   "bidirectional=%d vocab_size=%lld", cfg->hidden_size, cfg->embed_dim, cfg->num_layers, cfg->bidirectional,
                   (long long)cfg->vocab_size);
    return SB_ERR_INVALID;
  }
  const int dirs = cfg->bidirectional ? 2 : 1, L = cfg->num_layers;
  if (!w->embed || !w->layers) { set_last_error("sb_laser2_create: missing weight pointer"); return SB_ERR_INVALID; }
  if (!aligned_to(w->embed, 16)) {  // the gather reads the table as int4
    set_last_error("sb_laser2_create: the embedding table must be 16-byte aligned");
    return SB_ERR_INVALID;
  }
  for (int i = 0; i < L * dirs; ++i)
    if (has_null_pointer(w->layers[i])) {
      set_last_error("sb_laser2_create: layer %d direction %d has a null weight pointer", i / dirs, i % dirs);
      return SB_ERR_INVALID;
    }
  int num_sms = 0;
  if (int rc = require_hopper("sb_laser2_create", &num_sms)) return rc;
  if (int rc = lstm_check_cluster_fit("sb_laser2_create")) return rc;
  std::unique_ptr<SbLaser2> e(new (std::nothrow) SbLaser2());
  if (!e) { set_last_error("out of host memory"); return SB_ERR_INVALID; }
  e->cfg = *cfg;
  e->dirs = dirs;
  e->embed = w->embed;
  e->num_sms = cfg->num_sms > 0 ? cfg->num_sms : num_sms;
  if (int rc = e->staging.create("sb_laser2_create", SbLaser2::kSlotInts)) return rc;
  if (int rc = e->err_flag.create("sb_laser2_create")) return rc;
  // repacked weights: W_ih / W_hh rows and the summed bias in the recurrent kernel's gate order (the caller's weights are
  // not modified)
  const size_t G4 = 4 * kLstmH;
  e->w_ih.resize(L);
  e->bias.resize(L);
  e->w_hh.resize(L);
  int rc = e->packed.alloc("sb_laser2_create", "repacked LSTM weights", [&](Carver& c) {
    for (int l = 0; l < L; ++l) {
      const size_t in = l == 0 ? (size_t)cfg->embed_dim : (size_t)dirs * kLstmH;
      e->w_ih[l] = c.take<__nv_bfloat16>(dirs * G4 * in * 2, 256);
      e->bias[l] = c.take<float>(dirs * G4 * 4, 256);
      e->w_hh[l] = c.take<__nv_bfloat16>(dirs * G4 * kLstmH * 2, 256);
    }
  });
  if (rc) return rc;
  for (int l = 0; l < L; ++l) {
    const int in = l == 0 ? cfg->embed_dim : dirs * kLstmH;
    for (int d = 0; d < dirs; ++d) {
      const SbLstmLayerWeights& lw = w->layers[l * dirs + d];
      lstm_repack_rows_kernel<<<(unsigned)G4, 256>>>(reinterpret_cast<const __nv_bfloat16*>(lw.w_ih), e->w_ih[l] + d * G4 * in, in);
      lstm_repack_rows_kernel<<<(unsigned)G4, 256>>>(reinterpret_cast<const __nv_bfloat16*>(lw.w_hh),
                                                     e->w_hh[l] + d * G4 * kLstmH, kLstmH);
      lstm_repack_bias_kernel<<<(unsigned)(G4 / 256), 256>>>(lw.b_ih, lw.b_hh, e->bias[l] + d * G4);
    }
  }
  if ((rc = sync_prepared("sb_laser2_create", "repacking the LSTM weights"))) return rc;
  *out = e.release();
  return SB_OK;
}

void sb_laser2_destroy(SbLaser2* e) { delete e; }

int sb_laser2_workspace_bytes(const SbLaser2* e, int32_t max_batch, int64_t max_tokens, size_t* bytes) {
  if (!e || !bytes || max_batch <= 0 || max_tokens <= 0) {
    set_last_error("sb_laser2_workspace_bytes: bad argument");
    return SB_ERR_INVALID;
  }
  *bytes = laser_carve(e, max_batch, max_tokens, nullptr).bytes + kWorkspaceAlign;
  return SB_OK;
}

int sb_laser2_forward(SbLaser2* e, const int64_t* ids, int64_t ids_row_stride, const int32_t* seq_lens_host, int32_t B,
                      int32_t S, float* out, void* workspace, size_t workspace_bytes, void* stream_v) {
  if (!e || !ids || !out || !workspace) { set_last_error("sb_laser2_forward: null argument"); return SB_ERR_INVALID; }
  if (B <= 0 || S <= 0) { set_last_error("sb_laser2_forward: empty batch (B=%d, S=%d)", B, S); return SB_ERR_INVALID; }
  if (B > SbLaser2::kMaxBatch) {
    set_last_error("sb_laser2_forward: batch of %d sequences exceeds %d", B, SbLaser2::kMaxBatch);
    return SB_ERR_INVALID;
  }
  if (ids_row_stride < S) { set_last_error("sb_laser2_forward: ids_row_stride < seq_len"); return SB_ERR_INVALID; }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const int dirs = e->dirs, H = kLstmH, tiles = lstm_tiles(B);

  // cu_seqlens (a packed LSTM sequence cannot be empty) and the length-sorted tiles on the host, staged through a pinned ring
  int32_t* cu_h;
  long long T;
  int rc = e->staging.acquire(&cu_h);
  if (!rc) rc = host_cu_seqlens("sb_laser2_forward", seq_lens_host, B, S, 1, cu_h, &T);
  if (rc) return rc;
  int32_t* tiles_h = cu_h + (B + 1);
  // longest first, so that a tile runs about as many steps as its rows need; ties keep the input order
  std::iota(tiles_h, tiles_h + B, 0);
  std::stable_sort(tiles_h, tiles_h + B, [&](int x, int y) { return cu_h[x + 1] - cu_h[x] > cu_h[y + 1] - cu_h[y]; });
  std::fill(tiles_h + B, tiles_h + (size_t)tiles * kLstmRows, -1);

  LaserWs w;
  rc = bind_workspace("sb_laser2_forward", workspace, workspace_bytes, &w, [&](void* p) { return laser_carve(e, B, T, p); });
  if (rc) return rc;
  SB_CUDA_CHECK(cudaMemcpyAsync(w.cu, cu_h, sizeof(int32_t) * (B + 1), cudaMemcpyHostToDevice, stream));
  SB_CUDA_CHECK(cudaMemcpyAsync(w.tile_seqs, tiles_h, sizeof(int32_t) * (size_t)tiles * kLstmRows, cudaMemcpyHostToDevice,
                                stream));
  if ((rc = e->staging.record(stream))) return rc;

  const int E = e->cfg.embed_dim;
  laser_embed_kernel<<<B, 128, 0, stream>>>(ids, ids_row_stride, w.cu, S, reinterpret_cast<const int4*>(e->embed),
                                            e->cfg.vocab_size, E, e->cfg.pad_idx, reinterpret_cast<int4*>(w.xy), w.pad,
                                            w.tail, e->err_flag.dev);
  SB_CUDA_CHECK(cudaGetLastError());
  const int N = dirs * 4 * H;
  for (int l = 0; l < e->cfg.num_layers; ++l) {
    const int in = l == 0 ? E : dirs * H;
    GemmArgs g = gemm_args(w.xy, in, e->w_ih[l], in, w.g, N, 0, e->bias[l], (int)T, N, in, EPI_BIAS, e->num_sms);
    if ((rc = gemm_bf16(g, stream))) return rc;
    LstmArgs a{};
    a.G = w.g; a.ldg = N;
    a.Whh = e->w_hh[l];
    a.cu = w.cu; a.tile_seqs = w.tile_seqs;
    if (l + 1 < e->cfg.num_layers) {
      a.Y = w.xy; a.ldy = dirs * H;
    } else {
      a.pool = out; a.ldp = dirs * H;
      a.pad = w.pad; a.tail = w.tail; a.pad_value = e->cfg.padding_value;
    }
    if ((rc = lstm_recurrent(a, tiles, dirs, stream))) return rc;
  }
  return SB_OK;
}

int sb_laser2_check_inputs(SbLaser2* e, void* stream_v) {
  if (!e) { set_last_error("sb_laser2_check_inputs: null argument"); return SB_ERR_INVALID; }
  return e->err_flag.check("sb_laser2_forward", reinterpret_cast<cudaStream_t>(stream_v));
}

int sb_laser2_layer_weights(const SbLaser2* e, int32_t layer, const void** w_ih, const float** bias, const void** w_hh) {
  if (!e || !w_ih || !bias || !w_hh || layer < 0 || layer >= e->cfg.num_layers) {
    set_last_error("sb_laser2_layer_weights: null argument or layer %d outside [0, %d)", layer, e ? e->cfg.num_layers : 0);
    return SB_ERR_INVALID;
  }
  *w_ih = e->w_ih[layer];
  *bias = e->bias[layer];
  *w_hh = e->w_hh[layer];
  return SB_OK;
}

int sb_laser2_embed(const int64_t* ids, int64_t ids_row_stride, const int32_t* cu_seqlens, int32_t B, int32_t S,
                    const void* table, int64_t vocab, int32_t D, int64_t pad_idx, void* x, uint8_t* pad_mask,
                    uint8_t* tail_keep, int32_t* err_flag, void* stream) {
  if (!ids || !cu_seqlens || !table || !x || !pad_mask || !tail_keep || !err_flag) {
    set_last_error("sb_laser2_embed: null pointer");
    return SB_ERR_INVALID;
  }
  if (B <= 0 || S <= 0 || ids_row_stride < S || vocab <= 0 || D <= 0 || D % 8 != 0) {
    set_last_error("sb_laser2_embed: bad shape (B=%d, S=%d, ids_row_stride=%lld, vocab=%lld, D=%d; D a positive multiple of 8)",
                   B, S, (long long)ids_row_stride, (long long)vocab, D);
    return SB_ERR_INVALID;
  }
  if (!aligned_to(table, 16) || !aligned_to(x, 16)) {  // rows move as int4
    set_last_error("sb_laser2_embed: table and x must be 16-byte aligned");
    return SB_ERR_INVALID;
  }
  int sms = 0;
  if (int rc = require_hopper("sb_laser2_embed", &sms)) return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  laser_embed_kernel<<<B, 128, 0, s>>>(ids, ids_row_stride, cu_seqlens, S, reinterpret_cast<const int4*>(table), vocab, D,
                                       pad_idx, reinterpret_cast<int4*>(x), pad_mask, tail_keep, err_flag);
  SB_CUDA_CHECK(cudaGetLastError());
  return SB_OK;
}

int sb_lstm_recurrent(const void* G, int64_t ldg, const void* w_hh, const int32_t* cu_seqlens, const int32_t* tile_seqs,
                      int32_t num_tiles, int32_t num_dirs, void* y, int64_t ldy, float* pool_out, int64_t ldp,
                      const uint8_t* pad_mask, const uint8_t* tail_keep, float padding_value, void* stream) {
  if (!G || !w_hh || !cu_seqlens || !tile_seqs || (!y) == (!pool_out)) {
    set_last_error("sb_lstm_recurrent: null pointer, or not exactly one of y / pool_out");
    return SB_ERR_INVALID;
  }
  if (num_dirs < 1 || num_dirs > 2) { set_last_error("sb_lstm_recurrent: num_dirs %d (1 or 2)", num_dirs); return SB_ERR_INVALID; }
  // the kernel loads G in bf16 pairs, stores y in bf16 pairs and the pool in fp32 pairs, and copies W_hh in 16-byte pieces
  const long long width = (long long)num_dirs * kLstmH;
  const long long ld_out = y ? ldy : ldp;
  if (ldg < 4 * width || ldg % 2 != 0 || ld_out < width || ld_out % 2 != 0) {
    set_last_error("sb_lstm_recurrent: leading dimensions must be even with ldg >= %lld and %s >= %lld (got ldg=%lld, %s=%lld)",
                   4 * width, y ? "ldy" : "ldp", width, (long long)ldg, y ? "ldy" : "ldp", ld_out);
    return SB_ERR_INVALID;
  }
  if (!aligned_to(G, 4) || !aligned_to(w_hh, 16) || (y && !aligned_to(y, 4)) || (pool_out && !aligned_to(pool_out, 8))) {
    set_last_error("sb_lstm_recurrent: G and y must be 4-byte aligned, pool_out 8-byte aligned and w_hh 16-byte aligned");
    return SB_ERR_INVALID;
  }
  int sms = 0;
  if (int rc = require_hopper("sb_lstm_recurrent", &sms)) return rc;
  LstmArgs a{};
  a.G = reinterpret_cast<const __nv_bfloat16*>(G); a.ldg = ldg;
  a.Whh = reinterpret_cast<const __nv_bfloat16*>(w_hh);
  a.cu = cu_seqlens; a.tile_seqs = tile_seqs;
  a.Y = reinterpret_cast<__nv_bfloat16*>(y); a.ldy = ldy;
  a.pool = pool_out; a.ldp = ldp;
  a.pad = pad_mask; a.tail = tail_keep; a.pad_value = padding_value;
  return lstm_recurrent(a, num_tiles, num_dirs, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
