// Internal (C++) interfaces shared by the sonar_b200 CUDA translation units.
// The public C ABI is include/sonar_b200.h.
#pragma once

#include "../../include/sonar_b200.h"

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

namespace sb {

// EPI_BIAS_ACCUM (internal): C += A.W^T + bias with the add done by TMA reduce-add at L2; chosen
// automatically for EPI_BIAS_RESIDUAL when the residual aliases a fp32 C (the encoder's x += ... case).
// Bit-identical to EPI_BIAS_RESIDUAL: both compute fl32(x + fl32(acc + bias)).
// EPI_TOPK (internal): no C at all -- the epilogue keeps a running per-row top-k of the product (xsim mining).
// EPI_BIAS_SILU: x*sigmoid(x) (the Conformer's swish FFN activation)
// EPI_BIAS_TANH: tanh(x) (BLASER's hidden layers)
// EPI_BIAS_RESIDUAL_STATS (internal): fp32 C = residual + A.W^T + bias, plus the bf16 copy and row statistics of LnFold
enum EpiMode { EPI_BIAS = 0, EPI_BIAS_RELU = 1, EPI_BIAS_RESIDUAL = 2, EPI_BIAS_ACCUM = 3, EPI_TOPK = 4, EPI_BIAS_SILU = 5,
               EPI_BIAS_RESIDUAL_STATS = 6, EPI_BIAS_TANH = 7 };
constexpr int kTopkCandidates = 16;  // bf16-similarity candidates per row handed to the exact fp64 re-rank
enum PoolMode { POOL_MAX = 1, POOL_MEAN = 2, POOL_LAST = 3 };  // = reference `Pooling` enum values (model.py:23-27)

void set_last_error(const char* fmt, ...);

// SM count of the current device in *num_sms, after checking that a device exists and is a Hopper GPU (compute
// capability 9.x), which the sm_90a kernels need.  SB_ERR_CUDA, with `who` in the message, otherwise.
int require_hopper(const char* who, int* num_sms);

// True if any pointer of a weight struct made of device pointers only (SbLayerWeights, SbDecoderLayerWeights,
// SbConformerLayerWeights, SbPoolerLayerWeights) is null.
template <class Weights>
bool has_null_pointer(const Weights& w) {
  static_assert(sizeof(Weights) % sizeof(void*) == 0, "a weight struct holds pointers only");
  for (size_t i = 0; i < sizeof(Weights) / sizeof(void*); ++i) {
    const void* p;
    memcpy(&p, reinterpret_cast<const char*>(&w) + i * sizeof(void*), sizeof(void*));
    if (!p) return true;
  }
  return false;
}

// ---- workspaces: one caller-owned device buffer per call, carved into the engine's buffers ----
// Every buffer starts on a kWorkspaceAlign boundary.  The *_workspace_bytes functions add kWorkspaceAlign bytes of slack
// to the carved size, so that the caller's pointer can be rounded up to that boundary.
constexpr size_t kWorkspaceAlign = 1024;

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Bump allocator: take() returns the next buffer and starts the one after it on an `align` boundary.  A null base only
// sizes the layout; `off` is then the number of bytes it needs.
struct Carver {
  uintptr_t base;
  size_t off = 0;
  explicit Carver(void* p) : base(reinterpret_cast<uintptr_t>(p)) {}
  template <class T>
  T* take(size_t bytes, size_t align = kWorkspaceAlign) {
    T* p = reinterpret_cast<T*>(base + off);
    off = align_up(off + bytes, align);
    return p;
  }
};

// Where a workspace's first buffer starts: the caller's pointer rounded up to kWorkspaceAlign.
inline void* workspace_base(void* workspace) {
  return reinterpret_cast<void*>((reinterpret_cast<uintptr_t>(workspace) + kWorkspaceAlign - 1) &
                                 ~uintptr_t(kWorkspaceAlign - 1));
}

// *ws = carve(workspace_base(workspace)); SB_ERR_INVALID, with `who` in the message, if the layout needs more than the
// caller's workspace_bytes.
template <class Layout, class Carve>
int bind_workspace(const char* who, void* workspace, size_t workspace_bytes, Layout* ws, Carve&& carve) {
  void* base = workspace_base(workspace);
  *ws = carve(base);
  const size_t need = (reinterpret_cast<uintptr_t>(base) - reinterpret_cast<uintptr_t>(workspace)) + ws->bytes;
  if (need > workspace_bytes) {
    set_last_error("%s: workspace too small (%zu bytes given, %zu needed)", who, workspace_bytes, need);
    return SB_ERR_INVALID;
  }
  return SB_OK;
}

// ---- what an engine handle owns: each type frees it in its destructor, also after a failed create(), so none is copied ----
struct NoCopy {
  NoCopy() = default;
  NoCopy(const NoCopy&) = delete;
  NoCopy& operator=(const NoCopy&) = delete;
};

// Pinned host ring through which a forward stages its per-batch host data (cu_seqlens, ...) for its H2D copies without
// synchronising with the stream: kSlots slots of `slot_ints` int32, one event per slot.
struct StagingRing : NoCopy {
  static constexpr int kSlots = 8;
  int32_t* pinned = nullptr;
  size_t slot_ints = 0;
  cudaEvent_t ev[kSlots];
  int num_ev = 0;  // ev[0 .. num_ev) exist
  unsigned next_slot = 0;
  ~StagingRing();
  int create(const char* who, size_t slot_ints);  // errors name `who`
  // *slot = the next slot, once the copies that read it last have completed (this blocks only while kSlots forwards are
  // in flight).  The caller writes it, enqueues the copies that read it, then calls record().
  int acquire(int32_t** slot);
  // The slot acquire() returned stays in use until the work enqueued on `stream` so far has completed.
  int record(cudaStream_t stream);
};

// cu[0] = 0, cu[b + 1] = lens[0] + ... + lens[b] for the B host lengths (every one S when lens is null), and *T = cu[B].
// SB_ERR_INVALID, naming `who` and the offending index, unless each length lies in [min_len, S] and the total fits in int32.
int host_cu_seqlens(const char* who, const int32_t* lens, int B, int S, int min_len, int32_t* cu, long long* T);

// Device flag (256 bytes, zeroed at create) that an engine's embedding kernel sets on a token id outside the vocabulary.
// It stays set over any number of forwards until check() reads it.
struct InputFlag : NoCopy {
  int32_t* dev = nullptr;
  ~InputFlag() { cudaFree(dev); }
  int create(const char* who);
  // Reads and clears the flag, synchronises `stream`: SB_ERR_INPUT, naming `forward`, if it was set since the last check.
  int check(const char* forward, cudaStream_t stream);
};

// One device allocation behind the weights an engine prepares at create (LayerNorm-folded, repacked, absorbed).
struct WeightPool : NoCopy {
  void* base = nullptr;
  ~WeightPool() { cudaFree(base); }
  // Sizes the pool by running layout(Carver&) on a null base, allocates it (nothing for zero bytes) and runs layout on it,
  // which sets the caller's pointers.  SB_ERR_CUDA, "<who>: cudaMalloc of N bytes for the <what> failed", on failure.
  template <class Layout>
  int alloc(const char* who, const char* what, Layout&& layout) {
    Carver sizing(nullptr);
    layout(sizing);
    if (sizing.off && cudaMalloc(&base, sizing.off) != cudaSuccess) {
      base = nullptr;
      set_last_error("%s: cudaMalloc of %zu bytes for the %s failed", who, sizing.off, what);
      return SB_ERR_CUDA;
    }
    Carver c(base);
    layout(c);
    return SB_OK;
  }
};

// Synchronises after the kernels that prepared an engine's weights: SB_ERR_CUDA, "<who>: <what> failed: <error>", on failure.
int sync_prepared(const char* who, const char* what);

// cudaFuncSetAttribute is per device: returns true the first time `flags` (a per-call-site static array of 64 bools)
// is consulted for the current device.
inline bool first_use_on_device(bool (&flags)[64]) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return true;
  if (flags[dev]) return false;
  flags[dev] = true;
  return true;
}

// LayerNorm FOLDED into the GEMMs on either side of it (the text encoder's default schedule; no LayerNorm kernel runs).
//   LN(x) . W^T + b  =  rstd * (x . W'^T  -  mean * c)  +  b'      with  W' = W diag(gamma),  c[n] = sum_k W'[n,k],
//                                                                        b' = b + W beta          (prepared once at create)
// so the GEMM that CONSUMES a LayerNorm runs on the un-normalised bf16 copy of the residual stream and applies the
// per-row (mean, rstd) in its epilogue (`stats_in`, `colsum`), and the GEMM that PRODUCES the residual stream
// (EPI_BIAS_RESIDUAL_STATS) emits, next to x, that bf16 copy (`h_out`) and per-row partial statistics (`stats_out`):
// one (mean, M2) pair per kLnPartCols columns of the row (one column half of a 256-column tile), merged by
// the consumer with Chan's formula (no E[x^2]-mean^2 cancellation).  Saves the LayerNorm kernel's read of x and one of
// the two passes over h per LayerNorm.
constexpr int kLnPartCols = 128;
struct LnFold {
  const float* stats_in = nullptr;  // [M, chunks, 2] (mean, M2) of `chunks` disjoint kLnPartCols-column subsets of the input rows
  const float* colsum = nullptr;    // [N] c[n]
  int chunks = 0;                   // K / kLnPartCols of the LayerNorm the consumer folds (<= 8)
  float eps = 0.f;
  __nv_bfloat16* h_out = nullptr;   // producer: [M, N] bf16 copy of the new residual stream, leading dimension ldh
  long long ldh = 0;
  float* stats_out = nullptr;       // producer: [M, N / kLnPartCols, 2]
};

// SM count of the current device (what `num_sms = 0` means everywhere); 1 if the query fails, so a grid is never empty
inline int device_sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1)
    return 1;
  return n;
}

struct GemmArgs {
  const __nv_bfloat16* A = nullptr;  // [M,K] row-major, ld = lda
  long long lda = 0;
  const __nv_bfloat16* W = nullptr;  // [N,K] row-major (nn.Linear layout), ld = ldw
  long long ldw = 0;
  void* C = nullptr;  // [M,N] bf16 or fp32
  long long ldc = 0;
  int out_fp32 = 0;
  const float* bias = nullptr;     // [N] fp32
  const void* residual = nullptr;  // [M,N] same dtype as C (may alias C), ld = ldr
  long long ldr = 0;
  int M = 0, N = 0, K = 0;
  int epi = EPI_BIAS;  // EpiMode
  int cta_group = 2;   // 1 or 2
  int num_sms = 0;     // 0 -> device_sm_count()
  LnFold lf;           // LayerNorm folding (see above); default = off
  // Opt-in to the weight-streaming path for M <= 64 (gemm_skinny.cu).  It sums K in a different order than the wgmma
  // tiles, so a caller that promises results independent of the batch size across the M = 64 boundary (the text
  // encoder: bitwise batch-composition invariance) leaves it off; the decoder step and the speech pooler turn it on.
  int allow_skinny = 0;
  // Ordered split-K of the accumulate epilogue (x += A.W^T + b with few tiles): zero-initialised device counters, one per
  // (tile, CTA of the pair, epilogue warpgroup); the kernel leaves them zero.  nullptr = never split.  Changes the
  // summation order (deterministically), so only callers that do not promise batch-size-independent bits pass it.
  int* splitk_flags = nullptr;
  long long splitk_flags_len = 0;
};

// C = epi(A . W^T + bias) with every option off; the residual epilogues add C itself (x += ...).  Callers set LnFold,
// split-K counters, the skinny path or a residual other than C on the value returned.
inline GemmArgs gemm_args(const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int out_fp32,
                          const float* bias, int M, int N, int K, int epi, int num_sms) {
  GemmArgs g;
  g.A = static_cast<const __nv_bfloat16*>(A); g.lda = lda;
  g.W = static_cast<const __nv_bfloat16*>(W); g.ldw = ldw;
  g.C = C; g.ldc = ldc; g.out_fp32 = out_fp32; g.bias = bias;
  if (epi == EPI_BIAS_RESIDUAL || epi == EPI_BIAS_RESIDUAL_STATS) { g.residual = C; g.ldr = ldc; }
  g.M = M; g.N = N; g.K = K; g.epi = epi;
  g.num_sms = num_sms;
  return g;
}

int gemm_bf16(const GemmArgs& g, cudaStream_t stream);

// M <= 64 rows: weight-streaming mma.sync path (gemm_skinny.cu); gemm_bf16 dispatches to it when eligible
bool gemm_skinny_eligible(const GemmArgs& g);
int gemm_skinny(const GemmArgs& g, cudaStream_t stream);

// Column filter of the top-k sweep (xsim: both k-NN directions from ONE pass over x . y^T): next to the per-row lists, every
// element above its column's threshold is appended to that column's candidate buffer -- entry = (bf16 product as fp32 bits,
// row index); `cnt[col]` counts the hits (beyond `cap` they are dropped and the column's threshold is raised to +inf so that
// degenerate inputs -- every product above its threshold -- cannot turn the sweep into a stream of atomics: the caller checks
// cnt > cap).
// `thr` must be readable up to the next multiple of 256 columns (pad with +inf); `thr8[g]` = min(thr[8g .. 8g+7]) lets the
// epilogue reject 8 columns of a row with one compare against the maximum it already has.
struct ColFilter {
  float* thr = nullptr;        // [N padded to 256]; nullptr = no column filter.  A column that fills up is closed (+inf)
  const float* thr8 = nullptr; // [N padded to 256, / 8]
  int* cnt = nullptr;          // [N]
  uint2* buf = nullptr;        // [N, cap]
  int cap = 0;
};

int gemm_topk_chunks(int M, int N, int cta_group, int num_sms);
// candidate lists per row that gemm_bf16_topk writes for a given n_chunks (two column halves per n-chunk)
constexpr int kTopkListsPerChunk = 2;
inline int gemm_topk_lists(int n_chunks) { return kTopkListsPerChunk * n_chunks; }
int gemm_bf16_topk(const __nv_bfloat16* A, long long lda, const __nv_bfloat16* W, long long ldw, int M, int N, int K,
                   float* cand_val, int* cand_idx, float* lse_part, int n_chunks, int cta_group, int num_sms,
                   cudaStream_t stream, const ColFilter& cf = ColFilter());

int make_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, long long rows, long long cols, long long ld,
                 int box_rows, int box_cols);

// x[cu[b]+t, :] = E[ids[b,t], :] * scale + pos[t, :]   (fp32 out)
int embed_tokens(const int64_t* ids, long long ids_stride, const int32_t* cu_seqlens, int B, int S,
                 const __nv_bfloat16* embed, long long vocab, const float* pos_table, int pos_rows, int D, float scale,
                 float* x, int* err_flag, cudaStream_t stream, int pos_offset = 0, __nv_bfloat16* h_out = nullptr,
                 float* stats_out = nullptr);  // h_out / stats_out: LnFold producer outputs (bf16 copy + row statistics)

// LnFold weight preparation: Wf = bf16(W diag(gamma)), colsum[n] = sum_k Wf[n,k], bias_f = bias + W beta
int fold_layernorm_weights(const __nv_bfloat16* W, const float* bias, const float* gamma, const float* beta, int N, int K,
                           __nv_bfloat16* Wf, float* colsum, float* bias_f, cudaStream_t stream);

// y = LN(x) * gamma + beta, fp32 in, bf16 out, one warp per row
int layernorm_bf16(const float* x, const float* gamma, const float* beta, float eps, __nv_bfloat16* y, long long T,
                   int D, cudaStream_t stream);

// LN with an fp32 result (y32 may alias x) and/or a bf16 copy (either may be null)
int layernorm_dual(const float* x, const float* gamma, const float* beta, float eps, float* y32, __nv_bfloat16* y16,
                   long long T, int D, cudaStream_t stream);

// softmax(q k^T / sqrt(64)) v over packed sequences of any length on wgmma (attention_tc.cu); qkv [T, 3*D] bf16
// (q | k | v), out [T, D] bf16
int attention_packed(const __nv_bfloat16* qkv, const int32_t* cu_seqlens, int B, int H, long long total_tokens, int num_sms,
                     __nv_bfloat16* out, cudaStream_t stream);

// Transformer-XL relative-position attention of the Conformer blocks on wgmma (attention_relpos_tc.cu):
// score(i,j) = ((q_i+u).k_j + (q_i+v).p[S_center-1-i+j]) / 8; qu / qv = [T, D] bf16 scratch for the biased queries.
// At most kRelposTcMaxBatch utterances: cu_seqlens and the query-tile prefix are staged in shared memory.
constexpr int kRelposTcMaxBatch = 2047;
int attention_relpos_tc(const __nv_bfloat16* qkv, const __nv_bfloat16* p, const float* u_bias, const float* v_bias,
                        const int32_t* cu_seqlens, int B, int H, long long total_tokens, int Npad, int S_center,
                        __nv_bfloat16* qu, __nv_bfloat16* qv, __nv_bfloat16* out, int num_sms, cudaStream_t stream);

// x [B, D] fp32 and xb [B, D] bf16 = B copies of the fp32 row v [D] (the attention poolers' single query position)
int broadcast_rows(const float* v, float* x, __nv_bfloat16* xb, int B, int D, cudaStream_t stream);

// Latent cross-attention of the attention pooler (latent_attention.cu).  u [B, Hd, D] bf16 = softmax_t(qt[b, h, :] .
// mem[t, :] / 8) . mem over the rows t of sequence b in the packed memory mem [T, D] bf16; qt [B, Hd, D] bf16; Hd <= 16;
// D in {256, 512, 768, 1024}; an empty sequence gives zeros.
int pool_latent_attention(const __nv_bfloat16* qt, const __nv_bfloat16* mem, const int32_t* cu_seqlens, int B, int Hd, int D,
                          __nv_bfloat16* u, cudaStream_t stream);

// The attention pooler of the text and speech encoders (latent_attention.cu; AttentionEncoderOutputPooler,
// sonar/nn/encoder_pooler.py:47-89): one query row per sequence (px fp32 / ph bf16 [B, E], starting from q0) runs the
// POST-LN decoder layers
//   [ self-attention over itself = Wo (Wv x + bv) + bo -> LN -> absorbed query GEMM (qt [B, Hd*D]) -> latent
//     cross-attention over the memory (pool_latent_attention) -> absorbed output GEMM (+residual) -> LN -> ReLU FFN -> LN ]
// and projection_out (+bias) writes out [B, E] fp32.  Memory width D, pooler width E = 64 Hd (both multiples of 256,
// <= 1024; the engines check that), FFN width F.  The GEMMs run with the owning engine's GEMM policy.
struct AttentionPooler {
  struct Layer {
    SbPoolerLayerWeights w;          // the caller's weights (copied at create)
    __nv_bfloat16* wqk = nullptr;    // [Hd*D, E]  absorbed W_k,h^T W_q,h: qt_h = W_k,h^T (W_q,h x + b_q,h)
    float* bqk = nullptr;            // [Hd*D]
    __nv_bfloat16* wvo = nullptr;    // [E, Hd*D]  absorbed W_o blockdiag(W_v,h)
    float* bvo = nullptr;            // [E]        W_o b_v + b_o (the key bias drops out: softmax is shift-invariant)
  };
  struct Ws {  // the pooler's workspace buffers
    float* px = nullptr;          // [B, max(D, E)] fp32 pooler state (the text encoder's `encoded` scatter uses its first B*D)
    __nv_bfloat16* ph = nullptr;  // [B, E] bf16 copy of px
    __nv_bfloat16* pt = nullptr;  // [B, max(F, E)]
    __nv_bfloat16* qt = nullptr;  // [B, Hd*D] absorbed queries
    __nv_bfloat16* u = nullptr;   // [B, Hd*D] latent attention output
  };
  std::vector<Layer> layers;
  WeightPool absorbed;  // behind every layer's absorbed weights
  const float* q0 = nullptr;      // fp32 [E]
  const void* proj_w = nullptr;   // bf16 [E, E]
  const float* proj_b = nullptr;  // fp32 [E]
  int D = 0, E = 0, F = 0;
  float eps = 0.f;
  int num_sms = 0, cta_group = 2, allow_skinny = 0;  // GEMM policy

  // Checks the weight pointers, copies the layers and absorbs their cross-attention weights into one allocation of
  // num_layers * (2 Hd D E * 2 + (Hd D + E) * 4) bytes, then synchronises the device.  Errors name `who`.
  int create(const char* who, const SbPoolerLayerWeights* w, int num_layers, const float* q0, const void* proj_w,
             const float* proj_b, int D, int E, int F, float eps, int num_sms, int cta_group, int allow_skinny);
  Ws take(Carver& c, size_t B) const;  // the next buffers of a workspace layout, for B sequences
  // out [B, E] fp32 from the memory mem [T, D] bf16 packed by cu_seqlens [B + 1]
  int forward(const Ws& w, const __nv_bfloat16* mem, const int32_t* cu_seqlens, int B, float* out, cudaStream_t stream) const;
};

// optional final LayerNorm + pooling over packed sequences -> out [B, D] fp32;
// optionally also scatters the (normalised) rows to a padded [B, S, D] fp32 tensor.
int ln_pool(const float* x, const int32_t* cu_seqlens, int B, int D, const float* gamma, const float* beta,
            float eps, int apply_ln, int pool_mode, float* out, float* encoded_padded, int S_padded,
            cudaStream_t stream);

}  // namespace sb
