// C ABI (include/sonar_b200.h) + the per-batch schedule of the SONAR text encoder:
//   embed -> 24 x [LN -> QKV GEMM -> attention -> out-proj GEMM(+residual)
//                  -> LN -> FFN1 GEMM(+ReLU) -> FFN2 GEMM(+residual)] -> final LN + pool
// following SonarTextTransformerEncoderModel.forward (sonar/models/sonar_text/model.py:130-143)
// with the `basic` wiring of sonar/models/sonar_text/factory.py:72-153.
//
// HBM layout of one batch (all buffers inside the caller's workspace):
//   tokens are PACKED: row cu_seqlens[b] + t holds token t of sentence b, so padded
//   positions never exist on the device (the reference computes them and masks them).
//   x   fp32 [T, D]   residual stream (fp32 so 48 residual adds do not accumulate bf16 rounding)
//   h   bf16 [T, D]   GEMM A operands: bf16 copy of x (LayerNorm folded into the GEMMs) or LayerNorm output; attention output
//   qkv bf16 [T, 3D]  fused q|k|v projections (its first [T, D] doubles as the bf16 copy of x behind the out-projection)
//   f   bf16 [T, F]   FFN inner activations
//
// Schedule with cfg.ln_fold = 1, 5 launches per layer, no LayerNorm kernel:
//   embed -> x, h = bf16(x), row stats
//   24 x [ QKV GEMM (folds LN1: stats + gamma/beta prepared into W', c, b') -> attention (wgmma) ->
//          out-proj GEMM (+residual; emits x, bf16(x), stats) -> FFN1 GEMM (folds LN2, +ReLU) ->
//          FFN2 GEMM (+residual; emits x, bf16(x), stats) ] -> final LN + pool
// cfg.ln_fold = 0 (what the Python wrapper selects by default: measured faster, see bench.py `ab_layernorm_schedule`) keeps
// the classic schedule: separate LayerNorm kernels, residual adds by TMA reduce-add, 7 launches per layer.
//
// Attention pooling (SB_POOL_ATTENTION, factory.py:155-226): the final LayerNorm writes x in place and its bf16 copy h, the
// memory of the attention pooler (AttentionPooler, latent_attention.cu), which writes out [B, E].

#include "../../include/sonar_b200.h"
#include <stdlib.h>

#include "common.cuh"
#include "sonar_b200_internal.h"

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <vector>

namespace sb {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int require_hopper(const char* who, int* num_sms) {
  int n_gpu = 0, dev = 0, major = 0, minor = 0;
  if (cudaGetDeviceCount(&n_gpu) != cudaSuccess || n_gpu == 0) {
    set_last_error("%s: no CUDA device (this engine has no CPU path)", who);
    return SB_ERR_CUDA;
  }
  SB_CUDA_CHECK(cudaGetDevice(&dev));
  SB_CUDA_CHECK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  SB_CUDA_CHECK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9) {
    set_last_error("%s: the sm_90a kernels need a Hopper H100-class GPU (found sm_%d%d)", who, major, minor);
    return SB_ERR_CUDA;
  }
  SB_CUDA_CHECK(cudaDeviceGetAttribute(num_sms, cudaDevAttrMultiProcessorCount, dev));
  return SB_OK;
}

StagingRing::~StagingRing() {
  for (int i = 0; i < num_ev; ++i) cudaEventDestroy(ev[i]);
  if (pinned) cudaFreeHost(pinned);
}

int StagingRing::create(const char* who, size_t slot_ints) {
  this->slot_ints = slot_ints;
  if (cudaMallocHost(reinterpret_cast<void**>(&pinned), sizeof(int32_t) * kSlots * slot_ints) != cudaSuccess) {
    pinned = nullptr;
    set_last_error("%s: cudaMallocHost failed", who);
    return SB_ERR_CUDA;
  }
  for (; num_ev < kSlots; ++num_ev)
    if (cudaEventCreateWithFlags(&ev[num_ev], cudaEventDisableTiming) != cudaSuccess) {
      set_last_error("%s: cudaEventCreate failed", who);
      return SB_ERR_CUDA;
    }
  return SB_OK;
}

int StagingRing::acquire(int32_t** slot) {
  const unsigned i = next_slot++ % kSlots;
  SB_CUDA_CHECK(cudaEventSynchronize(ev[i]));  // before the host writes the slot
  *slot = pinned + (size_t)i * slot_ints;
  return SB_OK;
}

int StagingRing::record(cudaStream_t stream) {
  SB_CUDA_CHECK(cudaEventRecord(ev[(next_slot - 1) % kSlots], stream));
  return SB_OK;
}

int host_cu_seqlens(const char* who, const int32_t* lens, int B, int S, int min_len, int32_t* cu, long long* T) {
  *T = 0;
  cu[0] = 0;
  for (int b = 0; b < B; ++b) {
    const int len = lens ? lens[b] : S;
    if (len < min_len || len > S) {
      set_last_error("%s: seq_lens[%d]=%d outside [%d,%d]", who, b, len, min_len, S);
      return SB_ERR_INVALID;
    }
    if ((*T += len) > 0x7fffffffll) {
      set_last_error("%s: too many tokens (seq_lens[0..%d] sum to more than 2^31 - 1)", who, b);
      return SB_ERR_INVALID;
    }
    cu[b + 1] = (int32_t)*T;
  }
  return SB_OK;
}

int InputFlag::create(const char* who) {
  if (cudaMalloc(reinterpret_cast<void**>(&dev), 256) != cudaSuccess || cudaMemset(dev, 0, 256) != cudaSuccess) {
    set_last_error("%s: cudaMalloc of the input-check flag failed", who);
    return SB_ERR_CUDA;
  }
  return SB_OK;
}

int InputFlag::check(const char* forward, cudaStream_t stream) {
  int32_t flag = 0;
  SB_CUDA_CHECK(cudaMemcpyAsync(&flag, dev, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
  SB_CUDA_CHECK(cudaMemsetAsync(dev, 0, sizeof(int32_t), stream));  // sticky until read: covers every forward since
  SB_CUDA_CHECK(cudaStreamSynchronize(stream));
  if (flag != 0) {
    set_last_error("token id outside [0, vocab_size) in a batch passed to %s since the last check", forward);
    return SB_ERR_INPUT;
  }
  return SB_OK;
}

int sync_prepared(const char* who, const char* what) {
  if (cudaDeviceSynchronize() != cudaSuccess) {
    set_last_error("%s: %s failed: %s", who, what, cudaGetErrorString(cudaGetLastError()));
    return SB_ERR_CUDA;
  }
  return SB_OK;
}

struct Workspace {
  int32_t* cu;
  float* ln_stats;  // [T, D/128, 2] per-row LayerNorm partials (LnFold)
  float* x;
  __nv_bfloat16* h;
  __nv_bfloat16* qkv;
  __nv_bfloat16* f;
  AttentionPooler::Ws pool;  // attention pooling only
  size_t bytes;
};

}  // namespace sb

using namespace sb;

struct FoldedLayer {  // LnFold weights of one layer (device memory owned by the handle)
  __nv_bfloat16* wqkv = nullptr;
  __nv_bfloat16* w1 = nullptr;
  float* cqkv = nullptr;
  float* bqkv = nullptr;
  float* c1 = nullptr;
  float* b1 = nullptr;
};

struct SbEncoder {
  SbEncoderConfig cfg;
  int out_dim;  // width of `out`: embedding_dim with attention pooling, model_dim otherwise
  std::vector<FoldedLayer> folded;
  WeightPool fold_pool;  // behind all FoldedLayer pointers
  InputFlag err_flag;    // token id out of range, cleared by sb_encoder_check_inputs
  const void* embed;
  const float* pos_table;
  const float* final_ln_g;
  const float* final_ln_b;
  std::vector<SbLayerWeights> layers;
  AttentionPooler pooler;  // attention pooling only
  int num_sms;
  static constexpr int kSlotInts = 32768 + 8;
  StagingRing staging;  // cu_seqlens
  // optional in-step timing of the dominant kernel (FFN inner-projection GEMM of the middle layer)
  cudaEvent_t prof_start = nullptr, prof_stop = nullptr;
};

static Workspace carve(const SbEncoder* e, int32_t max_batch, int64_t max_tokens, void* base) {
  const size_t D = e->cfg.model_dim, F = e->cfg.ffn_inner_dim;
  const size_t T = (size_t)(max_tokens > 0 ? max_tokens : 1);
  Carver c(base);
  Workspace w;
  w.cu = c.take<int32_t>(sizeof(int32_t) * ((size_t)max_batch + 1));
  w.ln_stats = c.take<float>(T * (D / kLnPartCols) * 2 * sizeof(float));
  w.x = c.take<float>(T * D * 4);
  w.h = c.take<__nv_bfloat16>(T * D * 2);
  w.qkv = c.take<__nv_bfloat16>(T * 3 * D * 2);
  w.f = c.take<__nv_bfloat16>(T * F * 2);
  w.pool = {};
  if (e->cfg.pooling == SB_POOL_ATTENTION) w.pool = e->pooler.take(c, (size_t)max_batch);
  w.bytes = c.off;
  return w;
}

extern "C" {

const char* sb_last_error(void) { return g_err; }
int sb_version(void) { return 113; }

int sb_encoder_create(const SbEncoderConfig* cfg, const SbEncoderWeights* w, SbEncoder** out) {
  if (!cfg || !w || !out) { set_last_error("sb_encoder_create: null argument"); return SB_ERR_INVALID; }
  *out = nullptr;
  const int D = cfg->model_dim, H = cfg->num_heads, F = cfg->ffn_inner_dim;
  if (D <= 0 || D % 256 != 0 || D > 1024) {
    set_last_error("sb_encoder_create: model_dim must be a multiple of 256 and <= 1024 (got %d)", D);
    return SB_ERR_INVALID;
  }
  if (H <= 0 || D != H * 64) {
    set_last_error("sb_encoder_create: head_dim must be 64 (model_dim=%d, num_heads=%d)", D, H);
    return SB_ERR_INVALID;
  }
  if (F <= 0 || F % 256 != 0) { set_last_error("sb_encoder_create: ffn_inner_dim must be a multiple of 256"); return SB_ERR_INVALID; }
  if (cfg->ln_fold < 0 || cfg->ln_fold > 2) { set_last_error("sb_encoder_create: ln_fold must be 0, 1 or 2"); return SB_ERR_INVALID; }
  if (cfg->num_layers < 0 || cfg->pos_rows <= 0 || cfg->vocab_size <= 0) {
    set_last_error("sb_encoder_create: bad num_layers / pos_rows / vocab_size");
    return SB_ERR_INVALID;
  }
  const bool attn_pool = cfg->pooling == SB_POOL_ATTENTION;
  if (cfg->pooling != SB_POOL_MAX && cfg->pooling != SB_POOL_MEAN && cfg->pooling != SB_POOL_LAST && !attn_pool) {
    set_last_error("sb_encoder_create: unsupported pooling %d", cfg->pooling);
    return SB_ERR_INVALID;
  }
  const int E = cfg->embedding_dim;
  if (attn_pool) {
    if (E <= 0 || E % 256 != 0 || E > 1024 || E != 64 * cfg->pooler_heads) {
      set_last_error("sb_encoder_create: attention pooling needs embedding_dim = 64 * pooler_heads, a multiple of 256 and "
                     "<= 1024 (embedding_dim=%d, pooler_heads=%d)", E, cfg->pooler_heads);
      return SB_ERR_INVALID;
    }
    if (cfg->pooler_ffn_inner_dim <= 0 || cfg->pooler_ffn_inner_dim % 256 != 0 || cfg->pooler_layers < 1) {
      set_last_error("sb_encoder_create: attention pooling needs pooler_layers >= 1 and pooler_ffn_inner_dim a multiple of 256 "
                     "(got %d, %d)", cfg->pooler_layers, cfg->pooler_ffn_inner_dim);
      return SB_ERR_INVALID;
    }
  } else if (E != 0 && E != D) {
    set_last_error("sb_encoder_create: embedding_dim (%d) != model_dim (%d) needs attention pooling", E, D);
    return SB_ERR_INVALID;
  }
  if (!w->embed || !w->pos_table || !w->final_ln_g || !w->final_ln_b || (cfg->num_layers > 0 && !w->layers)) {
    set_last_error("sb_encoder_create: missing weight pointer");
    return SB_ERR_INVALID;
  }
  for (int i = 0; i < cfg->num_layers; ++i)
    if (has_null_pointer(w->layers[i])) {
      set_last_error("sb_encoder_create: layer %d has a null weight pointer", i);
      return SB_ERR_INVALID;
    }
  int num_sms = 0;
  if (int rc = require_hopper("sb_encoder_create", &num_sms)) return rc;
  std::unique_ptr<SbEncoder> e(new (std::nothrow) SbEncoder());
  if (!e) { set_last_error("out of host memory"); return SB_ERR_INVALID; }
  e->cfg = *cfg;
  e->embed = w->embed;
  e->pos_table = w->pos_table;
  e->final_ln_g = w->final_ln_g;
  e->final_ln_b = w->final_ln_b;
  e->layers.assign(w->layers, w->layers + cfg->num_layers);
  e->out_dim = attn_pool ? E : D;
  e->num_sms = cfg->num_sms > 0 ? cfg->num_sms : num_sms;
  if (int rc = e->staging.create("sb_encoder_create", SbEncoder::kSlotInts)) return rc;
  if (int rc = e->err_flag.create("sb_encoder_create")) return rc;
  if (cfg->ln_fold && cfg->num_layers > 0) {
    // LayerNorm folding (LnFold): W' = W diag(gamma), c = row sums of W', b' = b + W beta for the two GEMMs that consume a
    // LayerNorm in every layer; prepared once here (the caller's weights are not modified)
    const size_t D_ = D, F_ = F;
    e->folded.resize(cfg->num_layers);
    int rc = e->fold_pool.alloc("sb_encoder_create", "LayerNorm-folded weights", [&](Carver& c) {
      for (FoldedLayer& f : e->folded) {
        f.wqkv = c.take<__nv_bfloat16>(3 * D_ * D_ * 2, 256);
        f.w1 = c.take<__nv_bfloat16>(F_ * D_ * 2, 256);
        f.cqkv = c.take<float>(3 * D_ * 4, 256);
        f.bqkv = c.take<float>(3 * D_ * 4, 256);
        f.c1 = c.take<float>(F_ * 4, 256);
        f.b1 = c.take<float>(F_ * 4, 256);
      }
    });
    if (rc) return rc;
    for (int i = 0; i < cfg->num_layers; ++i) {
      const FoldedLayer& f = e->folded[i];
      const SbLayerWeights& l = e->layers[i];
      rc = fold_layernorm_weights(reinterpret_cast<const __nv_bfloat16*>(l.wqkv), l.bqkv, l.ln1_g, l.ln1_b, 3 * D, D,
                                  f.wqkv, f.cqkv, f.bqkv, nullptr);
      if (!rc)
        rc = fold_layernorm_weights(reinterpret_cast<const __nv_bfloat16*>(l.w1), l.b1, l.ln2_g, l.ln2_b, F, D, f.w1, f.c1,
                                    f.b1, nullptr);
      if (rc) return rc;
    }
    if ((rc = sync_prepared("sb_encoder_create", "folding the LayerNorm weights"))) return rc;
  }
  if (attn_pool)
    if (int rc = e->pooler.create("sb_encoder_create", w->pooler, cfg->pooler_layers, w->pooler_q0, w->proj_w, w->proj_b,
                                  D, E, cfg->pooler_ffn_inner_dim, cfg->ln_eps, e->num_sms, cfg->cta_group == 1 ? 1 : 2, 0))
      return rc;
  *out = e.release();
  return SB_OK;
}

void sb_encoder_destroy(SbEncoder* e) { delete e; }

int sb_encoder_workspace_bytes(const SbEncoder* enc, int32_t max_batch, int64_t max_tokens, size_t* bytes) {
  if (!enc || !bytes || max_batch <= 0 || max_tokens <= 0) {
    set_last_error("sb_encoder_workspace_bytes: bad argument");
    return SB_ERR_INVALID;
  }
  *bytes = carve(enc, max_batch, max_tokens, nullptr).bytes + kWorkspaceAlign;
  return SB_OK;
}

int sb_encoder_forward(SbEncoder* e, const int64_t* ids, int64_t ids_row_stride, const int32_t* seq_lens_host,
                       int32_t B, int32_t S, float* out, float* encoded, void* workspace, size_t workspace_bytes,
                       void* stream_v) {
  if (!e || !ids || !out || !workspace) { set_last_error("sb_encoder_forward: null argument"); return SB_ERR_INVALID; }
  if (B <= 0 || S <= 0) { set_last_error("sb_encoder_forward: empty batch (B=%d, S=%d)", B, S); return SB_ERR_INVALID; }
  if (S > e->cfg.pos_rows) {
    set_last_error("sb_encoder_forward: seq_len %d exceeds the encoder's max_seq_len %d", S, e->cfg.pos_rows);
    return SB_ERR_INVALID;
  }
  if (B + 1 > SbEncoder::kSlotInts) { set_last_error("sb_encoder_forward: batch too large (%d)", B); return SB_ERR_INVALID; }
  if (ids_row_stride < S) { set_last_error("sb_encoder_forward: ids_row_stride < seq_len"); return SB_ERR_INVALID; }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  const int D = e->cfg.model_dim, F = e->cfg.ffn_inner_dim, H = e->cfg.num_heads;

  // ---- cu_seqlens on the host, staged through a pinned ring ----
  int32_t* cu_h;
  long long T;
  int rc = e->staging.acquire(&cu_h);
  if (!rc) rc = host_cu_seqlens("sb_encoder_forward", seq_lens_host, B, S, 0, cu_h, &T);
  if (rc) return rc;
  Workspace w;
  rc = bind_workspace("sb_encoder_forward", workspace, workspace_bytes, &w, [&](void* p) { return carve(e, B, T, p); });
  if (rc) return rc;
  SB_CUDA_CHECK(cudaMemcpyAsync(w.cu, cu_h, sizeof(int32_t) * (B + 1), cudaMemcpyHostToDevice, stream));
  if ((rc = e->staging.record(stream))) return rc;
  const bool attn_pool = e->cfg.pooling == SB_POOL_ATTENTION;
  if (T == 0) {
    if (!attn_pool) {
      SB_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)B * D, stream));
      return SB_OK;
    }
    if (encoded) SB_CUDA_CHECK(cudaMemsetAsync(encoded, 0, sizeof(float) * (size_t)B * S * D, stream));
    return e->pooler.forward(w.pool, w.h, w.cu, B, out, stream);
  }

  const bool fold = e->cfg.ln_fold != 0 && e->cfg.num_layers > 0;  // LN1 (attention block) folded into FFN2 -> QKV
  const bool fold2 = fold && e->cfg.ln_fold == 1;                   // LN2 (FFN block) folded into out-proj -> FFN1 as well
  __nv_bfloat16* hn = w.qkv;  // [T, D] view of the (dead after attention) qkv buffer: bf16(x) behind the out-projection
  if ((rc = embed_tokens(ids, ids_row_stride, w.cu, B, S, reinterpret_cast<const __nv_bfloat16*>(e->embed),
                         e->cfg.vocab_size, e->pos_table, e->cfg.pos_rows, D, e->cfg.embed_scale, w.x, e->err_flag.dev,
                         stream, 0, fold ? w.h : nullptr, fold ? w.ln_stats : nullptr)))
    return rc;

  const int cta_group = (e->cfg.cta_group == 1) ? 1 : 2;
  const int M = (int)T;
  LnFold consume;  // what a LayerNorm-consuming GEMM needs
  consume.stats_in = w.ln_stats;
  consume.chunks = D / kLnPartCols;
  consume.eps = e->cfg.ln_eps;
  for (int li = 0; li < e->cfg.num_layers; ++li) {
    const SbLayerWeights& L = e->layers[li];
    const FoldedLayer* f = fold ? &e->folded[li] : nullptr;
    // --- self-attention block: x += Wo . SDPA(LN1(x)) + bo ---
    if (!fold)
      if ((rc = layernorm_bf16(w.x, L.ln1_g, L.ln1_b, e->cfg.ln_eps, w.h, T, D, stream))) return rc;
    GemmArgs qkv = gemm_args(w.h, D, fold ? f->wqkv : L.wqkv, D, w.qkv, 3 * D, 0, fold ? f->bqkv : L.bqkv, M, 3 * D, D,
                             EPI_BIAS, e->num_sms);
    qkv.cta_group = cta_group;
    if (fold) { qkv.lf = consume; qkv.lf.colsum = f->cqkv; }
    if ((rc = gemm_bf16(qkv, stream))) return rc;
    if ((rc = attention_packed(w.qkv, w.cu, B, H, T, e->num_sms, w.h, stream))) return rc;
    GemmArgs proj = gemm_args(w.h, D, L.wo, D, w.x, D, 1, L.bo, M, D, D, EPI_BIAS_RESIDUAL, e->num_sms);
    proj.cta_group = cta_group;
    if (fold2) {  // emits x, hn = bf16(x) and the statistics LN2 needs
      proj.epi = EPI_BIAS_RESIDUAL_STATS;
      proj.lf.h_out = hn; proj.lf.ldh = D; proj.lf.stats_out = w.ln_stats;
    }
    if ((rc = gemm_bf16(proj, stream))) return rc;
    // --- feed-forward block: x += W2 . relu(W1 . LN2(x) + b1) + b2 ---
    if (!fold2)
      if ((rc = layernorm_bf16(w.x, L.ln2_g, L.ln2_b, e->cfg.ln_eps, w.h, T, D, stream))) return rc;
    GemmArgs ffn1 = gemm_args(fold2 ? hn : w.h, D, fold2 ? f->w1 : L.w1, D, w.f, F, 0, fold2 ? f->b1 : L.b1, M, F, D,
                              EPI_BIAS_RELU, e->num_sms);
    ffn1.cta_group = cta_group;
    if (fold2) { ffn1.lf = consume; ffn1.lf.colsum = f->c1; }
    const bool prof = e->prof_start && li == e->cfg.num_layers / 2;
    if (prof) SB_CUDA_CHECK(cudaEventRecord(e->prof_start, stream));
    if ((rc = gemm_bf16(ffn1, stream))) return rc;
    if (prof) SB_CUDA_CHECK(cudaEventRecord(e->prof_stop, stream));
    GemmArgs ffn2 = gemm_args(w.f, F, L.w2, F, w.x, D, 1, L.b2, M, D, F, EPI_BIAS_RESIDUAL, e->num_sms);
    ffn2.cta_group = cta_group;
    if (fold && li + 1 < e->cfg.num_layers) {  // emits x, h = bf16(x) and the statistics the next layer's LN1 needs
      ffn2.epi = EPI_BIAS_RESIDUAL_STATS;
      ffn2.lf.h_out = w.h; ffn2.lf.ldh = D; ffn2.lf.stats_out = w.ln_stats;
    }
    if ((rc = gemm_bf16(ffn2, stream))) return rc;
  }
  if (!attn_pool)
    return ln_pool(w.x, w.cu, B, D, e->final_ln_g, e->final_ln_b, e->cfg.ln_eps, 1, e->cfg.pooling, out, encoded, S,
                   stream);
  // final LayerNorm in place + its bf16 copy (the pooler's memory); `encoded` is scattered from the normalised rows
  if ((rc = layernorm_dual(w.x, e->final_ln_g, e->final_ln_b, e->cfg.ln_eps, w.x, w.h, T, D, stream))) return rc;
  if (encoded)
    if ((rc = ln_pool(w.x, w.cu, B, D, nullptr, nullptr, e->cfg.ln_eps, 0, POOL_LAST, w.pool.px, encoded, S, stream)))
      return rc;
  return e->pooler.forward(w.pool, w.h, w.cu, B, out, stream);
}

int sb_encoder_forward_host(SbEncoder* e, const int64_t* ids_host, const int32_t* seq_lens_host, int32_t B,
                            int32_t S, float* out_host, int64_t* ids_staging, float* out_staging, void* workspace,
                            size_t workspace_bytes, void* stream_v) {
  if (!e || !ids_host || !out_host || !ids_staging || !out_staging) {
    set_last_error("sb_encoder_forward_host: null argument");
    return SB_ERR_INVALID;
  }
  if (B <= 0 || S <= 0) { set_last_error("sb_encoder_forward_host: empty batch"); return SB_ERR_INVALID; }
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_v);
  SB_CUDA_CHECK(cudaMemcpyAsync(ids_staging, ids_host, sizeof(int64_t) * (size_t)B * S, cudaMemcpyHostToDevice, stream));
  int rc = sb_encoder_forward(e, ids_staging, S, seq_lens_host, B, S, out_staging, nullptr, workspace, workspace_bytes,
                              stream_v);
  if (rc) return rc;
  SB_CUDA_CHECK(cudaMemcpyAsync(out_host, out_staging, sizeof(float) * (size_t)B * e->out_dim,
                                cudaMemcpyDeviceToHost, stream));
  SB_CUDA_CHECK(cudaStreamSynchronize(stream));
  return SB_OK;
}

int sb_encoder_profile_ffn1(SbEncoder* e, void* start_event, void* stop_event) {
  if (!e || (!start_event) != (!stop_event)) { set_last_error("sb_encoder_profile_ffn1: bad argument"); return SB_ERR_INVALID; }
  e->prof_start = reinterpret_cast<cudaEvent_t>(start_event);
  e->prof_stop = reinterpret_cast<cudaEvent_t>(stop_event);
  return SB_OK;
}

int sb_encoder_check_inputs(SbEncoder* e, void* stream_v) {
  if (!e) { set_last_error("sb_encoder_check_inputs: null argument"); return SB_ERR_INVALID; }
  return e->err_flag.check("sb_encoder_forward", reinterpret_cast<cudaStream_t>(stream_v));
}

// ---------------------------------------------------------------------------------------------
// kernel-level entry points
// ---------------------------------------------------------------------------------------------
int sb_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc, int32_t out_fp32,
                 const float* bias, const void* residual, int64_t ldr, int32_t M, int32_t N, int32_t K, int32_t epi,
                 int32_t cta_group, void* stream) {
  if (!A || !W || !C) { set_last_error("sb_gemm_bf16: null pointer"); return SB_ERR_INVALID; }
  int sms = 0;
  if (int rc = require_hopper("sb_gemm_bf16", &sms)) return rc;
  GemmArgs g = gemm_args(A, lda, W, ldw, C, ldc, out_fp32, bias, M, N, K, epi, sms);
  g.residual = residual; g.ldr = ldr;
  g.cta_group = cta_group == 1 ? 1 : 2;
  g.allow_skinny = (cta_group == 0);  // 0 = automatic: M <= 64 may take the weight-streaming path
  return gemm_bf16(g, reinterpret_cast<cudaStream_t>(stream));
}

int sb_fold_layernorm(const void* W, const float* bias, const float* gamma, const float* beta, int32_t N, int32_t K,
                      void* Wf, float* colsum, float* bias_f, void* stream) {
  if (!W || !bias || !gamma || !beta || !Wf || !colsum || !bias_f || N <= 0 || K <= 0) {
    set_last_error("sb_fold_layernorm: bad argument");
    return SB_ERR_INVALID;
  }
  return fold_layernorm_weights(reinterpret_cast<const __nv_bfloat16*>(W), bias, gamma, beta, N, K,
                                reinterpret_cast<__nv_bfloat16*>(Wf), colsum, bias_f, reinterpret_cast<cudaStream_t>(stream));
}

int sb_gemm_ln_consumer(const void* A, int64_t lda, const void* Wf, int64_t ldw, void* C, int64_t ldc, const float* bias_f,
                        const float* colsum, const float* stats, float eps, int32_t M, int32_t N, int32_t K, int32_t relu,
                        void* stream) {
  if (!A || !Wf || !C || !bias_f || !colsum || !stats) { set_last_error("sb_gemm_ln_consumer: null pointer"); return SB_ERR_INVALID; }
  int sms = 0;
  if (int rc = require_hopper("sb_gemm_ln_consumer", &sms)) return rc;
  GemmArgs g = gemm_args(A, lda, Wf, ldw, C, ldc, 0, bias_f, M, N, K, relu ? EPI_BIAS_RELU : EPI_BIAS, sms);
  g.lf.stats_in = stats; g.lf.colsum = colsum; g.lf.chunks = K / kLnPartCols; g.lf.eps = eps;
  return gemm_bf16(g, reinterpret_cast<cudaStream_t>(stream));
}

int sb_gemm_residual_stats(const void* A, int64_t lda, const void* W, int64_t ldw, float* x, int64_t ldx, const float* bias,
                           void* h_out, int64_t ldh, float* stats_out, int32_t M, int32_t N, int32_t K, void* stream) {
  if (!A || !W || !x || !bias || !h_out || !stats_out) { set_last_error("sb_gemm_residual_stats: null pointer"); return SB_ERR_INVALID; }
  int sms = 0;
  if (int rc = require_hopper("sb_gemm_residual_stats", &sms)) return rc;
  GemmArgs g = gemm_args(A, lda, W, ldw, x, ldx, 1, bias, M, N, K, EPI_BIAS_RESIDUAL_STATS, sms);
  g.lf.h_out = reinterpret_cast<__nv_bfloat16*>(h_out); g.lf.ldh = ldh; g.lf.stats_out = stats_out;
  return gemm_bf16(g, reinterpret_cast<cudaStream_t>(stream));
}

int sb_gemm_residual_splitk(const void* A, int64_t lda, const void* W, int64_t ldw, float* x, int64_t ldx, const float* bias,
                            int32_t M, int32_t N, int32_t K, int32_t* counters, int64_t n_counters, void* stream) {
  if (!A || !W || !x || !bias || !counters) { set_last_error("sb_gemm_residual_splitk: null pointer"); return SB_ERR_INVALID; }
  int sms = 0;
  if (int rc = require_hopper("sb_gemm_residual_splitk", &sms)) return rc;
  GemmArgs g = gemm_args(A, lda, W, ldw, x, ldx, 1, bias, M, N, K, EPI_BIAS_RESIDUAL, sms);
  g.splitk_flags = counters;
  g.splitk_flags_len = n_counters;
  return gemm_bf16(g, reinterpret_cast<cudaStream_t>(stream));
}

int sb_layernorm(const float* x, const float* gamma, const float* beta, float eps, void* y, int64_t T, int32_t D,
                 void* stream) {
  if (!x || !gamma || !beta || !y) { set_last_error("sb_layernorm: null pointer"); return SB_ERR_INVALID; }
  return layernorm_bf16(x, gamma, beta, eps, reinterpret_cast<__nv_bfloat16*>(y), T, D,
                        reinterpret_cast<cudaStream_t>(stream));
}

int sb_layernorm_dual(const float* x, const float* gamma, const float* beta, float eps, float* y32, void* y16, int64_t T,
                      int32_t D, void* stream) {
  if (!x || !gamma || !beta || (!y32 && !y16)) { set_last_error("sb_layernorm_dual: null pointer"); return SB_ERR_INVALID; }
  return layernorm_dual(x, gamma, beta, eps, y32, reinterpret_cast<__nv_bfloat16*>(y16), T, D,
                        reinterpret_cast<cudaStream_t>(stream));
}

int sb_attention(const void* qkv, const int32_t* cu_seqlens, int32_t B, int32_t H, int64_t total_tokens, void* out,
                 void* stream) {
  if (!qkv || !cu_seqlens || !out) { set_last_error("sb_attention: null pointer"); return SB_ERR_INVALID; }
  int sms = 0;
  if (int rc = require_hopper("sb_attention", &sms)) return rc;
  return attention_packed(reinterpret_cast<const __nv_bfloat16*>(qkv), cu_seqlens, B, H, total_tokens, sms,
                          reinterpret_cast<__nv_bfloat16*>(out), reinterpret_cast<cudaStream_t>(stream));
}

int sb_embed(const int64_t* ids, int64_t ids_row_stride, const int32_t* cu_seqlens, int32_t B, int32_t S,
             const void* embed, int64_t vocab, const float* pos_table, int32_t pos_rows, int32_t D, float scale,
             float* x, int32_t* err_flag, void* h_out, float* stats_out, void* stream) {
  if (!ids || !cu_seqlens || !embed || !pos_table || !x || !err_flag) {
    set_last_error("sb_embed: null pointer");
    return SB_ERR_INVALID;
  }
  return embed_tokens(ids, ids_row_stride, cu_seqlens, B, S, reinterpret_cast<const __nv_bfloat16*>(embed), vocab,
                      pos_table, pos_rows, D, scale, x, err_flag, reinterpret_cast<cudaStream_t>(stream), 0,
                      reinterpret_cast<__nv_bfloat16*>(h_out), stats_out);
}

int sb_pool_latent_attention(const void* qt, const void* mem, const int32_t* cu_seqlens, int32_t B, int32_t Hd, int32_t D,
                             void* u, void* stream) {
  if (!qt || !mem || !cu_seqlens || !u) { set_last_error("sb_pool_latent_attention: null pointer"); return SB_ERR_INVALID; }
  int sms = 0;
  if (int rc = require_hopper("sb_pool_latent_attention", &sms)) return rc;
  return pool_latent_attention(reinterpret_cast<const __nv_bfloat16*>(qt), reinterpret_cast<const __nv_bfloat16*>(mem),
                               cu_seqlens, B, Hd, D, reinterpret_cast<__nv_bfloat16*>(u), reinterpret_cast<cudaStream_t>(stream));
}

int sb_pool(const float* x, const int32_t* cu_seqlens, int32_t B, int32_t D, const float* gamma, const float* beta,
            float eps, int32_t apply_ln, int32_t pool_mode, float* out, float* encoded_padded, int32_t S_padded,
            void* stream) {
  if (!x || !cu_seqlens || !out) { set_last_error("sb_pool: null pointer"); return SB_ERR_INVALID; }
  return ln_pool(x, cu_seqlens, B, D, gamma, beta, eps, apply_ln, pool_mode, out, encoded_padded, S_padded,
                 reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
