/* sonar_b200 -- C ABI of the Hopper-native SONAR text-embedding hot path.
 *
 * Plain C, no torch / CUDA types in the signatures: device buffers are `void*` /
 * typed raw pointers, the stream is an opaque `void*` (a `cudaStream_t`).
 * Every entry point returns 0 on success or a negative code and never throws;
 * `sb_last_error()` gives the message (thread-local).  No hidden device
 * allocations happen inside `sb_encoder_forward`; the caller owns all buffers.
 *
 * The reference (facebookresearch/SONAR) has NO native interface for this path --
 * it reaches fairseq2 Python modules.  Each entry point therefore cites the Python
 * interface it replaces:
 *
 *   sb_encoder_create / sb_encoder_forward
 *       <- SonarTextTransformerEncoderModel.forward(SequenceBatch) -> SonarEncoderOutput
 *          (sonar/models/sonar_text/model.py:130-143; built by
 *           SonarTextEncoderFactory.create_model, sonar/models/sonar_text/factory.py:72-120),
 *          called from TextToEmbeddingModelPipeline.predict via `.map(self.model)`
 *          (sonar/inference_pipelines/text.py:231-247).
 *   seq_lens / padded ids layout
 *       <- Collater(pad_idx) + extract_sequence_batch (text.py:241-242,
 *          sonar/inference_pipelines/utils.py:18-21): ids int64 [B,S] right-padded,
 *          PaddingMask(seq_lens).
 *   sb_pool
 *       <- SonarTextTransformerEncoderModel.static_pooling (model.py:86-128).
 *   SB_POOL_ATTENTION / sb_pool_latent_attention
 *       <- the attention pooler of SonarTextEncoderFactory.create_attention_pooler (factory.py:155-226).
 *   weight layout
 *       <- fairseq2 state-dict names mapped in sonar/models/sonar_text/handler.py:71-92
 *          (nn.Linear [out,in] row-major).
 */
#ifndef SONAR_B200_H_
#define SONAR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_OK 0
#define SB_ERR_INVALID (-1)  /* bad argument / unsupported shape */
#define SB_ERR_CUDA (-2)     /* CUDA runtime error */
#define SB_ERR_DRIVER (-3)   /* driver entry point / tensor-map failure */
#define SB_ERR_INPUT (-4)    /* device-side input check failed (e.g. token id out of range) */

/* Reference `Pooling` enum values (sonar/models/sonar_text/model.py:23-27). */
#define SB_POOL_MAX 1
#define SB_POOL_MEAN 2
#define SB_POOL_LAST 3
#define SB_POOL_ATTENTION 4 /* trainable attention pooler (SonarTextEncoderFactory.create_attention_pooler, factory.py:155-226) */

/* GEMM epilogues */
#define SB_EPI_BIAS 0
#define SB_EPI_BIAS_RELU 1
#define SB_EPI_BIAS_RESIDUAL 2
#define SB_EPI_BIAS_SILU 5
#define SB_EPI_BIAS_TANH 7

typedef struct SbEncoder SbEncoder;

/* Mirrors the fields of SonarTextEncoderConfig that reach the math
 * (sonar/models/sonar_text/config.py:14-84). */
typedef struct SbEncoderConfig {
  int32_t model_dim;     /* 1024 (multiple of 256, <= 1024; head_dim must be 64) */
  int32_t num_layers;    /* 24 */
  int32_t num_heads;     /* 16 */
  int32_t ffn_inner_dim; /* 8192 (multiple of 256) */
  int64_t vocab_size;    /* 256206 */
  int32_t pos_rows;      /* rows of the sinusoidal table = max_seq_len + pad_idx + 1 = 514 */
  int32_t pooling;       /* SB_POOL_* ; `basic` = SB_POOL_MEAN */
  float ln_eps;          /* 1e-5 */
  float embed_scale;     /* sqrt(model_dim) unless no_scale_embedding */
  int32_t cta_group;     /* 0/2 = CTA pairs (2-CTA clusters, W tile multicast; default), 1 = single CTAs */
  int32_t num_sms;       /* 0 = query the device */
  int32_t ln_fold;       /* 1 = fold every encoder-layer LayerNorm into the GEMMs around it (no LayerNorm kernel runs:
                          *     the residual GEMMs emit per-row statistics + a bf16 copy of the stream, the QKV / FFN1 GEMMs
                          *     apply (mean, rstd) in their epilogue on weights pre-multiplied by gamma; sb_encoder_create
                          *     prepares those weights in device memory it owns -- the caller's weights are not modified);
                          * 2 = fold only the attention-block LayerNorm (FFN2 emits, QKV applies); the FFN-block LayerNorm
                          *     stays a kernel (the out-projection is HBM-bound, its epilogue has no slack for the extra work);
                          * 0 = separate LayerNorm kernels */
  /* Attention pooling (pooling = SB_POOL_ATTENTION; the four fields are ignored otherwise, except embedding_dim):
   * one BOS query through `pooler_layers` POST-LN decoder layers cross-attending the final-LayerNormed token states,
   * then projection_out (with bias) -> [batch, embedding_dim] (factory.py:155-226). */
  int32_t embedding_dim;        /* width E of `out`: multiple of 256, <= 1024, = 64 * pooler_heads; without attention
                                 * pooling it must be 0 or model_dim (0 = model_dim) */
  int32_t pooler_layers;        /* num_decoder_layers (24 for `basic`), >= 1 */
  int32_t pooler_heads;         /* num_decoder_attn_heads (head dim 64, <= 16 heads) */
  int32_t pooler_ffn_inner_dim; /* decoder_ffn_inner_dim, or ffn_inner_dim when that is None (multiple of 256) */
} SbEncoderConfig;

/* All pointers are DEVICE pointers and stay owned by the caller (must outlive the handle).
 * Matrices: bf16, row-major [out_features, in_features].  Vectors: fp32. */
typedef struct SbLayerWeights {
  const void* wqkv;   /* bf16 [3*D, D] = rows of q_proj | k_proj | v_proj */
  const float* bqkv;  /* [3*D] */
  const void* wo;     /* bf16 [D, D]   self_attn.output_proj */
  const float* bo;    /* [D] */
  const void* w1;     /* bf16 [F, D]   ffn.inner_proj */
  const float* b1;    /* [F] */
  const void* w2;     /* bf16 [D, F]   ffn.output_proj */
  const float* b2;    /* [D] */
  const float* ln1_g; /* self_attn_layer_norm */
  const float* ln1_b;
  const float* ln2_g; /* ffn_layer_norm */
  const float* ln2_b;
} SbLayerWeights;

typedef struct SbEncoderWeights {
  const void* embed;           /* bf16 [vocab, D]  encoder_frontend.embed.weight */
  const float* pos_table;      /* fp32 [pos_rows, D]; row t = sinusoid of position t + pad_idx + 1 */
  const float* final_ln_g;     /* layer_norm.weight */
  const float* final_ln_b;     /* layer_norm.bias */
  const SbLayerWeights* layers; /* HOST array of num_layers entries (copied at create) */
  /* attention pooling only (NULL otherwise); E = embedding_dim.  pooler[i] uses SbPoolerLayerWeights (declared with the
   * speech encoder below) with every matrix [E, E] except ca_wkv = bf16 [2E, D] (k_proj | v_proj of
   * encoder_decoder_attn, whose inputs are the D-wide token states), ca_bkv [2E], w1 [F_pool, E], w2 [E, F_pool] */
  const float* pooler_q0;       /* fp32 [E] = pooler.decoder_frontend.embed.weight[0] * sqrt(E) + pos[0] */
  const void* proj_w;           /* pooler.projection_out.weight bf16 [E, E] */
  const float* proj_b;          /* pooler.projection_out.bias [E] */
  const struct SbPoolerLayerWeights* pooler; /* HOST array of pooler_layers entries (copied at create) */
} SbEncoderWeights;

const char* sb_last_error(void);
int sb_version(void);

/* Allocates the handle's own device memory (a 256-byte input-check flag; with cfg->ln_fold the folded copies of the QKV and
 * FFN inner-projection weights, ~22 MB per layer; with attention pooling the absorbed cross-attention weights of every pooler
 * layer, 2 * Hd * D * E * 2 + (Hd * D + E) * 4 bytes = 64 MB per layer at D = E = 1024, 16 heads) and synchronises the
 * device once.  sb_encoder_forward never allocates. */
int sb_encoder_create(const SbEncoderConfig* cfg, const SbEncoderWeights* w, SbEncoder** out);
void sb_encoder_destroy(SbEncoder* enc);

/* Bytes of device workspace needed for a batch of <= max_batch sequences holding
 * <= max_tokens real (unpadded) tokens in total. */
int sb_encoder_workspace_bytes(const SbEncoder* enc, int32_t max_batch, int64_t max_tokens, size_t* bytes);

/* One pass of the hot path.
 *   ids            DEVICE int64 [batch, ids_row_stride >= seq_len], right-padded (any pad value)
 *   seq_lens_host  HOST int32 [batch] true lengths (1..seq_len); NULL = every row is full (no padding_mask)
 *   out            DEVICE fp32 [batch, embedding_dim] sentence embeddings
 *   encoded        DEVICE fp32 [batch, seq_len, model_dim] or NULL (final-LayerNormed states, padded rows zeroed)
 * Asynchronous on `stream` (does not synchronise). */
int sb_encoder_forward(SbEncoder* enc, const int64_t* ids, int64_t ids_row_stride, const int32_t* seq_lens_host,
                       int32_t batch, int32_t seq_len, float* out, float* encoded, void* workspace,
                       size_t workspace_bytes, void* stream);

/* Same, but `ids_host` / `out_host` are HOST buffers (pinned for full speed); performs the
 * H2D copy of the ids, the forward and the D2H copy of the embeddings on `stream`, then
 * synchronises the stream.  `ids_staging` is DEVICE int64 [batch*seq_len], `out_staging`
 * DEVICE fp32 [batch*embedding_dim] (caller-owned). */
int sb_encoder_forward_host(SbEncoder* enc, const int64_t* ids_host, const int32_t* seq_lens_host, int32_t batch,
                            int32_t seq_len, float* out_host, int64_t* ids_staging, float* out_staging,
                            void* workspace, size_t workspace_bytes, void* stream);

/* Measurement hook: every following forward records the two caller-owned CUDA events (cudaEvent_t, timing enabled)
 * around the FFN inner-projection GEMM of the middle layer -- the dominant kernel -- on the forward's stream, so its
 * duration can be read INSIDE a real step.  Pass NULL, NULL to switch it off. */
int sb_encoder_profile_ffn1(SbEncoder* enc, void* start_event, void* stop_event);

/* Reads and clears the handle's sticky device-side input flag (token id out of range in a forward since the last check);
 * synchronises `stream`.  Returns SB_OK or SB_ERR_INPUT. */
int sb_encoder_check_inputs(SbEncoder* enc, void* stream);

/* ---- individual kernels (used by the parity tests and the micro-benchmarks) ---- */

/* LayerNorm folding (the schedule behind SbEncoderConfig.ln_fold; replaces F.layer_norm + F.linear pairs of the pre-LN
 * encoder layer, sonar/models/sonar_text/factory.py:122-153):
 *   LN(x; gamma, beta) . W^T + b  =  rstd * (x . Wf^T - mean * colsum) + bias_f
 * sb_fold_layernorm prepares Wf = bf16(W diag(gamma)) [N,K], colsum[n] = sum_k Wf[n,k], bias_f = bias + W beta;
 * sb_gemm_residual_stats computes x += A . W^T + bias (fp32, in place) and emits h_out = bf16(x) plus stats_out
 *   [M, N/128, 2] = (mean, M2) of N/128 disjoint 128-column subsets of the new rows (one per epilogue warpgroup and tile);
 * sb_gemm_ln_consumer computes C (bf16) = [relu](rstd * (A . Wf^T - mean * colsum) + bias_f) with A = the bf16 copy and
 *   (mean, rstd) merged from `stats` [M, K/128, 2].  K = a multiple of 128, <= 1024. */
int sb_fold_layernorm(const void* W, const float* bias, const float* gamma, const float* beta, int32_t N, int32_t K,
                      void* Wf, float* colsum, float* bias_f, void* stream);
int sb_gemm_ln_consumer(const void* A, int64_t lda, const void* Wf, int64_t ldw, void* C, int64_t ldc, const float* bias_f,
                        const float* colsum, const float* stats, float eps, int32_t M, int32_t N, int32_t K, int32_t relu,
                        void* stream);
int sb_gemm_residual_stats(const void* A, int64_t lda, const void* W, int64_t ldw, float* x, int64_t ldx, const float* bias,
                           void* h_out, int64_t ldh, float* stats_out, int32_t M, int32_t N, int32_t K, void* stream);

/* x += A . W^T + bias (fp32, in place) as the decoder step issues it (the residual additions of
 * fairseq2's StandardTransformerDecoderLayer, reached from sonar/models/sonar_text/factory.py:263-301): when the
 * [M/256, N/256] tile pairs leave SM pairs idle (2 560 hypothesis rows x 1 024 columns = 40 tiles on 74 pairs) the K
 * dimension is split into up to 4 slices run by different SM pairs, which add into x ONE AFTER THE OTHER (hand-over through
 * `counters`, >= 4 * tiles zero-initialised device ints that the call leaves zero): x + p0, + p1, + p2 -- the same bits on
 * every run.  With enough tiles it is the plain accumulate epilogue. */
int sb_gemm_residual_splitk(const void* A, int64_t lda, const void* W, int64_t ldw, float* x, int64_t ldx, const float* bias,
                            int32_t M, int32_t N, int32_t K, int32_t* counters, int64_t n_counters, void* stream);

/* C[M,N] = epi(A[M,K] * W[N,K]^T + bias[N]) ; A, W bf16 row-major; C bf16 (out_fp32=0) or fp32;
 * residual (SB_EPI_BIAS_RESIDUAL) has C's dtype and may alias C.  N % 256 == 0, K % 64 == 0.
 * cta_group: 2 = CTA-pair tiles (2-CTA clusters), 1 = single-CTA tiles, 0 = automatic (paired tiles, except that M <= 64 with
 * K % 256 == 0 takes the weight-streaming mma.sync path the decoder step uses; then only N % 8 == 0 is required). */
int sb_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, void* C, int64_t ldc, int32_t out_fp32,
                 const float* bias, const void* residual, int64_t ldr, int32_t M, int32_t N, int32_t K, int32_t epi,
                 int32_t cta_group, void* stream);

/* y[T,D] (bf16) = LayerNorm(x[T,D] fp32) */
int sb_layernorm(const float* x, const float* gamma, const float* beta, float eps, void* y, int64_t T, int32_t D,
                 void* stream);

/* packed self-attention: qkv bf16 [total_tokens, 3*64*H], cu_seqlens DEVICE int32 [B+1], out bf16 [total_tokens, 64*H].
 * The wgmma kernel of the encoder: any sequence length (128-key tiles with online softmax beyond 128 tokens). */
int sb_attention(const void* qkv, const int32_t* cu_seqlens, int32_t B, int32_t H, int64_t total_tokens, void* out,
                 void* stream);

/* y32 fp32 [T,D] and / or y16 bf16 [T,D] = LayerNorm(x[T,D] fp32), either output may be NULL; y32 may alias x (the
 * in-place final / pooler LayerNorm of the attention pooling path).  D a multiple of 128, <= 1024. */
int sb_layernorm_dual(const float* x, const float* gamma, const float* beta, float eps, float* y32, void* y16, int64_t T,
                      int32_t D, void* stream);

/* x[cu[b]+t,:] = embed[ids[b,t],:]*scale + pos[t,:] for t < min(len_b, S) (ids past a sentence's length are not read);
 * err_flag DEVICE int32 (set to 1 on an id outside [0, vocab); that row embeds id 0).  h_out / stats_out (both or
 * neither, D % 256 == 0): the LnFold outputs the encoder's first LayerNorm-consuming GEMM reads -- h_out bf16 [T, D] =
 * bf16(x), stats_out fp32 [T, D/128, 2] = (mean, M2) of each 128-column chunk of the row of x. */
int sb_embed(const int64_t* ids, int64_t ids_row_stride, const int32_t* cu_seqlens, int32_t B, int32_t S,
             const void* embed, int64_t vocab, const float* pos_table, int32_t pos_rows, int32_t D, float scale,
             float* x, int32_t* err_flag, void* h_out, float* stats_out, void* stream);

/* (optional LayerNorm +) pooling of packed rows x fp32 [T,D] -> out fp32 [B,D] */
int sb_pool(const float* x, const int32_t* cu_seqlens, int32_t B, int32_t D, const float* gamma, const float* beta,
            float eps, int32_t apply_ln, int32_t pool_mode, float* out, float* encoded_padded, int32_t S_padded,
            void* stream);

/* The attention pooler's cross-attention on the absorbed form (see SbEncoderWeights.pooler): qt DEVICE bf16 [B, Hd, D]
 * (Hd <= 16 absorbed queries per sentence), mem DEVICE bf16 [total_tokens, D] packed rows (row cu_seqlens[b] + t),
 * cu_seqlens DEVICE int32 [B+1]; u DEVICE bf16 [B, Hd, D] = softmax_t(qt[b,h,:] . mem[t,:] / 8) . mem over sentence b's
 * rows (zeros for an empty sentence).  D in {256, 512, 768, 1024}. */
int sb_pool_latent_attention(const void* qt, const void* mem, const int32_t* cu_seqlens, int32_t B, int32_t Hd, int32_t D,
                             void* u, void* stream);

/* The speech encoder's kernels, launched as sb_speech_encoder_forward launches them.  Packed rows: utterance b owns rows
 * cu_seqlens[b] .. cu_seqlens[b+1] - 1 (cu_seqlens DEVICE int32 [B+1]).
 *
 * Transformer-XL relative-position self-attention of a Conformer block, D = 64 * H in {256, 512, 768, 1024}:
 *   out[i] = sum_j softmax_j(((q_i + u) . k_j + (q_i + v) . p[S_center - 1 - i + j]) / 8) v_j   over the keys j of i's utterance
 * qkv bf16 [total_tokens, 3D] (q | k | v), p bf16 [Npad, D] = r_proj of the relative-position table (row k <-> relative
 * position S_center - 1 - k), u_bias / v_bias fp32 [D], out bf16 [total_tokens, D].  S_center = the longest utterance,
 * Npad = roundup(2 * S_center - 1, 256).  impl 0 = the wgmma kernel (B <= 2047; qu, qv bf16 [total_tokens, D] scratch),
 * impl 1 = the mma.sync kernel (vp fp32 [H, Npad] scratch). */
int sb_attention_relpos(const void* qkv, const void* p, const float* u_bias, const float* v_bias, const int32_t* cu_seqlens,
                        int32_t B, int32_t H, int64_t total_tokens, int32_t Npad, int32_t S_center, int32_t impl, void* qu,
                        void* qv, float* vp, void* out, void* stream);
/* The convolution module between its pointwise convolutions: g bf16 [total, 2D] (value | gate) -> out bf16 [total, D] =
 * SiLU(bn_scale * depthwise_conv(value * sigmoid(gate)) + bn_shift), 31 taps dw fp32 [D, 31], zero outside each utterance;
 * max_len = the longest utterance, D a multiple of 64. */
int sb_conformer_conv(const void* g, const int32_t* cu_seqlens, int32_t B, int32_t max_len, int32_t D, const float* dw,
                      const float* bn_scale, const float* bn_shift, void* out, void* stream);
/* The w2v-BERT frontend's first step: row cu_seqlens[b] + t of out (bf16 [total, 192]) = LayerNorm(160) of fbank frames
 * 2t, 2t+1 of utterance b (fbank DEVICE fp32 [B, padded_frames, 80]), columns 160..191 zero; max_len = the longest
 * utterance (2 * max_len <= padded_frames). */
int sb_speech_frontend(const float* fbank, int32_t padded_frames, const int32_t* cu_seqlens, int32_t B, int32_t max_len,
                       const float* gamma, const float* beta, float eps, void* out, void* stream);

/* ---- embedding -> text decoder, one incremental step at a time (BASELINE.json config 4) ----
 * Replaces ConditionalTransformerDecoderModel.decode + project (sonar/nn/conditional_decoder_model.py:60-94,
 * built by SonarTextDecoderFactory, sonar/models/sonar_text/factory.py:229-315) as driven by fairseq2's
 * BeamSearchSeq2SeqGenerator inside EmbeddingToTextModelPipeline.predict (sonar/inference_pipelines/text.py:305-346).
 * State-dict names: sonar/models/sonar_text/handler.py:136-158. */
typedef struct SbDecoder SbDecoder;

typedef struct SbDecoderConfig {
  int32_t model_dim;     /* 1024 */
  int32_t num_layers;    /* 24 */
  int32_t num_heads;     /* 16 */
  int32_t ffn_inner_dim; /* 8192 */
  int32_t input_dim;     /* dimensionality of the sentence embedding; must equal model_dim */
  int64_t vocab_size;    /* 256206 */
  int32_t pos_rows;      /* rows of the sinusoidal table (max_seq_len + pad_idx + 1) */
  int32_t eos_idx;       /* 3 */
  float ln_eps;          /* 1e-5 */
  float embed_scale;     /* sqrt(model_dim) */
} SbDecoderConfig;

/* DEVICE pointers, caller-owned; matrices bf16 [out,in], vectors fp32.  The encoder-decoder attention attends
 * over ONE key (the sentence embedding), so only its v_proj / output_proj reach the result. */
typedef struct SbDecoderLayerWeights {
  const void* wqkv;      /* bf16 [3D, D] self_attn q|k|v */
  const float* bqkv;
  const void* wo;        /* self_attn.output_proj */
  const float* bo;
  const void* cross_wv;  /* encoder_decoder_attn.v_proj [D, input_dim] */
  const float* cross_bv;
  const void* cross_wo;  /* encoder_decoder_attn.output_proj */
  const float* cross_bo;
  const void* w1;        /* ffn.inner_proj */
  const float* b1;
  const void* w2;        /* ffn.output_proj */
  const float* b2;
  const float* ln1_g;    /* self_attn_layer_norm */
  const float* ln1_b;
  const float* ln3_g;    /* ffn_layer_norm */
  const float* ln3_b;
} SbDecoderLayerWeights;

typedef struct SbDecoderWeights {
  const void* embed;       /* bf16 [vocab, D] decoder_frontend.embed.weight == final_proj.weight (tied) */
  const float* pos_table;  /* fp32 [pos_rows, D] */
  const float* final_ln_g; /* decoder.layer_norm */
  const float* final_ln_b;
  const SbDecoderLayerWeights* layers; /* HOST array */
} SbDecoderWeights;

/* Allocates the handle's 256-byte input-check flag; sb_decoder_begin and sb_decoder_step never allocate. */
int sb_decoder_create(const SbDecoderConfig* cfg, const SbDecoderWeights* w, SbDecoder** out);
void sb_decoder_destroy(SbDecoder* dec);
/* workspace for num_sentences x beam hypotheses of at most max_len positions (holds the KV caches) */
int sb_decoder_workspace_bytes(const SbDecoder* dec, int32_t num_sentences, int32_t beam, int32_t max_len, size_t* bytes);
/* start a batch: embeddings DEVICE fp32 [num_sentences, model_dim]; precomputes the per-layer cross-attention constants */
int sb_decoder_begin(SbDecoder* dec, const float* embeddings, int32_t num_sentences, int32_t beam, int32_t max_len,
                     void* workspace, size_t workspace_bytes, void* stream);
/* one decoding step at position t for all R = num_sentences*beam rows (row = sentence*beam + beam_slot):
 *   tokens  DEVICE int64 [R]           input token of every hypothesis at position t
 *   table   DEVICE int32 [R, max_len]  table[r, t'] = physical cache row holding position t' < t of hypothesis r
 *   out_lprob / out_tok DEVICE [R, 16] the 16 most probable next tokens (fp32 log-softmax over the whole vocabulary),
 *                                      ordered by (log-prob desc, token asc)
 *   out_eos_lprob DEVICE fp32 [R]      log P(eos)
 *   probe_tokens  DEVICE int64 [R] or NULL; with it out_probe_lprob DEVICE fp32 [R] = log P(probe_tokens[r]) -- the
 *                                      prompt-token scores fairseq2's generator accumulates while prefilling [fs2 _prefill] */
int sb_decoder_step(SbDecoder* dec, const int64_t* tokens, const int32_t* table, int32_t t, int32_t num_sentences,
                    int32_t beam, int32_t max_len, float* out_lprob, int32_t* out_tok, float* out_eos_lprob,
                    const int64_t* probe_tokens, float* out_probe_lprob, void* workspace, size_t workspace_bytes,
                    void* stream);
/* Reads and clears the handle's sticky device-side input flag (token id outside [0, vocab_size) in a step since the last
 * check; sb_decoder_begin leaves it as it is); synchronises `stream`.  Returns SB_OK or SB_ERR_INPUT. */
int sb_decoder_check_inputs(SbDecoder* dec, void* stream);

/* The decoder step's kernels, launched as sb_decoder_step launches them (R hypothesis rows, DEVICE pointers).
 *
 * Embedding: x fp32 [R, D] = embed[tokens[r]] * scale + pos_row (bf16 [vocab, D], fp32 [D] = the position's row of the
 * table, D a multiple of 8); an id outside [0, vocab) sets *err_flag (int32) to 1 and embeds row 0. */
int sb_decoder_embed(const int64_t* tokens, const void* embed, int64_t vocab, const float* pos_row, int32_t D, float scale,
                     float* x, int32_t R, int32_t* err_flag, void* stream);
/* Cached causal self-attention at position t of one layer, D = 64 * H a multiple of 256:
 *   qkv bf16 [R, 3D] (q | k | v of position t); kcache / vcache bf16 [R, Tmax, D]; table int32 [R, Tmax]
 *   (table[r, t'] = the cache row holding position t' < t of hypothesis r).  Writes k and v of row r to cache row r at
 *   position t, then out bf16 [R, D] = softmax(q . k / 8) . v over positions 0..t.  t in [0, Tmax), Tmax <= 512, R <= 65535. */
int sb_decoder_attention(const void* qkv, void* kcache, void* vcache, const int32_t* table, int32_t t, int32_t R,
                         int32_t Tmax, int32_t H, void* out, void* stream);
/* x fp32 [R, D] += c[r / beam] (c fp32 [R / beam, D], one row per sentence); h bf16 [R, D] = LayerNorm(x) * gamma + beta;
 * D a multiple of 128, at most 1024. */
int sb_decoder_add_const_layernorm(float* x, const float* c, int32_t R, int32_t beam, int32_t D, const float* gamma,
                                   const float* beta, float eps, void* h, void* stream);
/* n-chunks sb_decoder_step splits the vocabulary sweep into for R rows; the head's scratch holds 2 * n_chunks lists. */
int sb_decoder_vocab_chunks(int32_t R, int64_t V, int32_t* n_chunks);
/* The vocabulary head: logits = h . embed^T (h bf16 [R, D], embed bf16 [V, D], never materialised) ->
 *   out_lprob fp32 / out_tok int32 [R, 16]: the 16 best (logit - logsumexp, token), ordered by (value desc, token asc);
 *   when V < 16 the last 16 - V entries are (-inf, -1);
 *   out_eos fp32 [R] = log P(eos_idx); probe_tokens int64 [R] or NULL, with it out_probe fp32 [R] = log P(probe_tokens[r])
 *   (an id outside [0, V) scores token 0).
 * Caller-owned scratch with L = 2 * n_chunks lists: cand_val fp32 / cand_idx int32 [R, L, 16], lse_part fp32 [R, L, 2].
 * n_chunks = 0 takes the step's own split (sb_decoder_vocab_chunks); a positive count is used as given, and refused if
 * some chunk would get no 256-column tile or L > 256. */
int sb_decoder_vocab_head(const void* h, const void* embed, int32_t R, int64_t V, int32_t D, int32_t eos_idx,
                          const int64_t* probe_tokens, int32_t n_chunks, float* cand_val, int32_t* cand_idx, float* lse_part,
                          float* out_lprob, int32_t* out_tok, float* out_eos, float* out_probe, void* stream);

/* ---- speech feature frontend (BASELINE.json config 3, rows a9/a10) ----
 * Replaces fairseq2n WaveformToFbankConverter(num_mel_bins=80, waveform_scale=2**15, channel_last=True,
 * standardize=True) + Collater(pad_value=0, pad_to_multiple=2) (sonar/inference_pipelines/speech.py:120-127,139,
 * 283-290,444).  16 kHz mono input. */
size_t sb_fbank_tables_bytes(void);
/* fills a HOST buffer of sb_fbank_tables_bytes() (window, FFT twiddles, mel filters); upload it to the device once */
int sb_fbank_build_tables(void* host_buf);
/* waves DEVICE fp32 packed samples in [-1,1]; wave_offsets DEVICE int64 [B+1]; frame_offsets DEVICE int32 [B+1]
 * (cumulative frame counts, frames_b = 1 + (samples_b - 400) / 160); tables DEVICE (see above);
 * raw_out DEVICE fp32 [total_frames, 80] scratch; out DEVICE fp32 [B, padded_frames, 80] standardised, zero padded */
int sb_fbank(const float* waves, const int64_t* wave_offsets, const int32_t* frame_offsets, int32_t B,
             int32_t total_frames, const void* tables, float* raw_out, float* out, int32_t padded_frames, void* stream);

/* ---- speech encoder: w2v-BERT Conformer stack + attention pooler (BASELINE.json config 3, rows a11/a12) ----
 * Replaces SonarSpeechEncoderModel.forward (sonar/models/sonar_speech/model.py:59-77; factory.py:53-152;
 * sonar/nn/encoder_pooler.py:70-83); parameter names per sonar/models/sonar_speech/handler.py:63-100. */
typedef struct SbSpeechEncoder SbSpeechEncoder;

typedef struct SbSpeechConfig {
  int32_t model_dim;            /* 1024 */
  int32_t num_layers;           /* 24 Conformer blocks */
  int32_t num_heads;            /* 16 */
  int32_t ffn_inner_dim;        /* 4096 */
  int32_t conv_kernel;          /* 31 */
  int32_t pooler_layers;        /* 3 (english) / 6 (non_english) */
  int32_t pooler_ffn_inner_dim; /* 4096 */
  float ln_eps;                 /* 1e-5 */
  int32_t attn_impl;            /* relative-position attention: 0 = wgmma kernel, 1 = mma.sync kernel (the Python wrapper's
                                 * default) */
} SbSpeechConfig;

/* every field is a DEVICE pointer (matrices bf16 [out,in]; vectors fp32) */
typedef struct SbConformerLayerWeights {
  const float* ffn1_ln_g; const float* ffn1_ln_b;
  const void* ffn1_w1; const float* ffn1_b1; const void* ffn1_w2 /* x0.5 */; const float* ffn1_b2 /* x0.5 */;
  const float* attn_ln_g; const float* attn_ln_b;
  const void* wqkv; const float* bqkv; const void* wo; const float* bo;
  const void* wr;            /* self_attn.sdpa.r_proj.weight */
  const float* u_bias;       /* [H*64] */
  const float* v_bias;
  const float* conv_ln_g; const float* conv_ln_b;
  const void* pw1;           /* conv.pointwise_conv1 [2D, D] */
  const float* dw;           /* conv.depthwise_conv  fp32 [D, 31] */
  const float* bn_scale;     /* gamma / sqrt(running_var + eps) */
  const float* bn_shift;     /* beta - running_mean * bn_scale */
  const void* pw2;           /* conv.pointwise_conv2 [D, D] */
  const float* ffn2_ln_g; const float* ffn2_ln_b;
  const void* ffn2_w1; const float* ffn2_b1; const void* ffn2_w2 /* x0.5 */; const float* ffn2_b2 /* x0.5 */;
  const float* ln_g; const float* ln_b;   /* the block's final layer_norm */
} SbConformerLayerWeights;

typedef struct SbPoolerLayerWeights {
  const void* sa_wv; const float* sa_bv; const void* sa_wo; const float* sa_bo;
  const float* sa_ln_g; const float* sa_ln_b;
  const void* ca_wq; const float* ca_bq;
  const void* ca_wkv /* [2D, D] = k_proj | v_proj */; const float* ca_bkv;
  const void* ca_wo; const float* ca_bo;
  const float* ca_ln_g; const float* ca_ln_b;
  const void* w1; const float* b1; const void* w2; const float* b2;
  const float* ffn_ln_g; const float* ffn_ln_b;
} SbPoolerLayerWeights;

typedef struct SbSpeechWeights {
  const float* front_ln_g;  /* encoder_frontend.post_extract_layer_norm [160] */
  const float* front_ln_b;
  const void* front_w;      /* encoder_frontend.model_dim_proj, bf16 [D, 192] (columns 160..191 zero) */
  const float* front_b;
  const float* final_ln_g;  /* layer_norm (re-homed stack LayerNorm) */
  const float* final_ln_b;
  const float* pooler_q0;   /* fp32 [D] = embed[bos] * sqrt(D) + pos[0] */
  const void* proj_w;       /* encoder_pooler.projection_out.weight bf16 [D, D] */
  const float* zeros;       /* fp32 zeros, >= max(2D, relpos rows) entries (bias of the bias-free projections) */
  const SbConformerLayerWeights* layers; /* HOST arrays */
  const SbPoolerLayerWeights* pooler;
} SbSpeechWeights;

/* Allocates the handle's own memory: on the device the absorbed cross-attention weights of every pooler layer (as for
 * sb_encoder_create with E = D and Hd = num_heads: 2 * Hd * D * D * 2 + (Hd * D + D) * 4 bytes = 64 MB per layer at
 * D = 1024, so 192 MB for `english` and 384 MB for `non_english`), on the host a pinned ring of 8 x 65 536 int32 through
 * which the forwards stage their lengths.  Synchronises the device once.  sb_speech_encoder_forward never allocates. */
int sb_speech_encoder_create(const SbSpeechConfig* cfg, const SbSpeechWeights* w, SbSpeechEncoder** out);
void sb_speech_encoder_destroy(SbSpeechEncoder* enc);
int sb_speech_encoder_workspace_bytes(const SbSpeechEncoder* enc, int32_t batch, int64_t total_positions,
                                      int32_t max_positions, size_t* bytes);
/* fbank DEVICE fp32 [batch, padded_frames, 80] (sb_fbank output); lens_host HOST int32 [batch] positions per utterance
 * (= frames // 2) in 1..padded_frames / 2; relpos_table DEVICE bf16 [relpos_rows, D] with
 * relpos_rows = roundup(2*max_len - 1, 256), row k = sinusoid of relative position (max_len - 1 - k), zero rows after
 * 2*max_len - 1; out DEVICE fp32 [batch, D]; encoded_packed DEVICE fp32 [total_positions, D] or NULL.
 * batch <= 65535.  Asynchronous on `stream` (does not synchronise). */
int sb_speech_encoder_forward(SbSpeechEncoder* enc, const float* fbank, int32_t padded_frames, const int32_t* lens_host,
                              int32_t batch, const void* relpos_table, int32_t relpos_rows, float* out,
                              float* encoded_packed, void* workspace, size_t workspace_bytes, void* stream);

/* ---- xsim cosine k-NN / margin mining over sentence embeddings (BASELINE.json config 5) ----
 * Not a reference interface: the reference only ever does normalize + matmul
 * (tests/integration_tests/test_text_sonar.py:42,51); algorithm = public LASER xsim (SURVEY App. D). */

int sb_xsim_workspace_bytes(int32_t n, int32_t m, int32_t d, size_t* bytes);

/* k nearest rows of y[m,d] (cosine) for every row of x[n,d]; x, y DEVICE fp32 row-major (raw, un-normalised).
 * out_val DEVICE fp64 [n,k] exact cosines, out_idx DEVICE int32 [n,k]; sorted by (cosine desc, index asc).
 * Candidates come from a bf16 wgmma GEMM with a fused running top-16, then are re-scored in fp64. */
int sb_xsim_knn(const float* x, const float* y, int32_t n, int32_t m, int32_t d, int32_t k, double* out_val,
                int32_t* out_idx, void* workspace, size_t workspace_bytes, void* stream);

/* Both k-NN directions from ONE pass over x^ . y^T (SURVEY §8(e): "row top-k and simultaneously per-column partial top-k"):
 * val_xy / idx_xy [n,k] as sb_xsim_knn; val_yx / idx_yx [m,k] = for every y row its k nearest x rows (exact fp64 cosines,
 * int32 row indices).  The reverse direction's candidates are the elements of the product above a per-column threshold:
 * the 16th best bf16 score of that y row against every 8th x row (a 1/8-size GEMM).  sb_xsim_knn keeps the 16 best bf16
 * scores of a row and re-scores them exactly, and a subset's 16th best never exceeds the 16th best over all rows, so the
 * result equals sb_xsim_knn(y, x) for any data; about 16 * 8 = 128 rows pass per column whatever the score distribution.
 * A y row that collects more than its 256 slots (heavy ties / duplicates) is marked idx_yx[j, :] = -2 and counted in
 * *overflow_flag (DEVICE int): the caller recomputes those rows with sb_xsim_knn(y[rows], x) (sonar_b200/xsim.py::knn_bidir
 * does). */
int sb_xsim_bidir_workspace_bytes(int32_t n, int32_t m, int32_t d, size_t* bytes);
int sb_xsim_knn_bidir(const float* x, const float* y, int32_t n, int32_t m, int32_t d, int32_t k, double* val_xy,
                      int32_t* idx_xy, double* val_yx, int32_t* idx_yx, int32_t* overflow_flag, void* workspace,
                      size_t workspace_bytes, void* stream);

/* pred[i] = forward candidate of row i with the best margin score.
 * margin_mode 0 = absolute, 1 = ratio, 2 = distance; val_yx = fp64 [m,k] k-NN cosines of y rows among x. */
int sb_xsim_margin_predict(const double* val_xy, const int32_t* idx_xy, const double* val_yx, int32_t n, int32_t m,
                           int32_t k, int32_t margin_mode, int32_t* pred, void* stream);

/* ---- beam search bookkeeping (one step, one launch) ----
 * The state transition of fairseq2's BeamSearchSeq2SeqGenerator [fs2] as the reference drives it
 * (sonar/inference_pipelines/text.py:315-333): from the decoder step's 16 best continuations per hypothesis
 * (lp / tok [N*beam,16], eos_lp [N*beam]) select the 2*beam best per sentence (score desc, then beam*vocab+token asc),
 * retire the EOS-terminated ones ranked inside the beam into fin_* until the sentence owns `beam` hypotheses (slot
 * CAP = 2*beam is scratch), and let the first `beam` others continue: seqs [N,beam,Tmax], the KV-cache ancestry table [N*beam,Tmax], tokens [N*beam], cum / alive
 * [N,beam] and done [N] are updated in place (alive / done: one byte per flag).  t = position of the step's input token,
 * g = number of tokens generated before this step; EOS is forbidden while g < eos_block (= min_gen_len - 1: fairseq2's
 * `step_nr < min_seq_len - 1`); score_div = (P+g)^len_penalty with P the prompt length (fairseq2 normalises by
 * seq_len - 1 counting prompt and EOS).  beam <= 7. */
int sb_beam_step(const float* lp, const int32_t* tok, const float* eos_lp, int64_t* seqs, int32_t* table,
                 int64_t* tokens, float* cum, uint8_t* alive, uint8_t* done, float* fin_score, int64_t* fin_seq,
                 int64_t* fin_len, int64_t* fin_count, int32_t N, int32_t beam, int32_t Tmax, int32_t t, int32_t g,
                 int32_t eos_block, int32_t max_gen, int64_t vocab, int32_t eos, int32_t unk, int32_t pad,
                 float unk_penalty, float score_div, int32_t normalize, void* stream);

/* ---- LASER2 text encoder: embedding + bidirectional multi-layer LSTM + max over time ----
 * Replaces LaserLstmEncoder.forward(seqs, seq_lens) (sonar/nn/laser_lstm_encoder.py:60-116) built from the `laser2` config
 * (sonar/models/laser2_text/config.py:28-38); parameter names are the module's own (embed_tokens.weight,
 * lstm.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}[_reverse]), with no converter (sonar/models/laser2_text/handler.py). */
typedef struct SbLaser2 SbLaser2;

typedef struct SbLaser2Config {
  int64_t vocab_size;    /* 50004 */
  int64_t pad_idx;       /* 1: positions holding this id are left out of the max (-inf) */
  int32_t embed_dim;     /* 320 (model_dim; a positive multiple of 64) */
  int32_t hidden_size;   /* 512 (the only supported value) */
  int32_t num_layers;    /* 5 (>= 1) */
  int32_t bidirectional; /* 1 (0 or 1) */
  float padding_value;   /* 0.0: the value positions t >= len_b contribute to the max unless their id is pad_idx */
  int32_t num_sms;       /* 0 = query the device */
} SbLaser2Config;

/* One torch.nn.LSTM layer and direction; DEVICE pointers, caller-owned, gate order i, f, g, o. */
typedef struct SbLstmLayerWeights {
  const void* w_ih;   /* bf16 [4H, in]  weight_ih_l{k}[_reverse]; in = embed_dim for k = 0, else H * (1 + bidirectional) */
  const void* w_hh;   /* bf16 [4H, H]   weight_hh_l{k}[_reverse] */
  const float* b_ih;  /* [4H] */
  const float* b_hh;  /* [4H] */
} SbLstmLayerWeights;

typedef struct SbLaser2Weights {
  const void* embed;                /* bf16 [vocab, embed_dim]  embed_tokens.weight, 16-byte aligned (read as 16-byte rows) */
  const SbLstmLayerWeights* layers; /* HOST array of num_layers * (1 + bidirectional) entries: entry k * dirs + d is layer k,
                                     * direction d (d = 1: the _reverse weights); copied at create */
} SbLaser2Weights;

/* Allocates the handle's own device memory (a 256-byte input-check flag and the weights repacked into the recurrent kernel's
 * gate order with b_ih + b_hh summed: 57 MB for `laser2`; the caller's weights are not modified) and a pinned host staging
 * ring, and synchronises the device once.  Fails with SB_ERR_CUDA when one 16-CTA cluster of the recurrent kernel does not
 * fit on the device. */
int sb_laser2_create(const SbLaser2Config* cfg, const SbLaser2Weights* w, SbLaser2** out);
void sb_laser2_destroy(SbLaser2* enc);
/* Bytes of device workspace for <= max_batch sequences holding <= max_tokens real tokens in total. */
int sb_laser2_workspace_bytes(const SbLaser2* enc, int32_t max_batch, int64_t max_tokens, size_t* bytes);
/* ids            DEVICE int64 [batch, ids_row_stride >= seq_len], right-padded with any value
 * seq_lens_host  HOST int32 [batch] lengths in 1..seq_len (NULL = all seq_len); a zero length is SB_ERR_INVALID, as
 *                pack_padded_sequence refuses it
 * out            DEVICE fp32 [batch, H * (1 + bidirectional)] = max over t < seq_len of the [fwd | bwd] outputs, where a
 *                position t >= len_b contributes padding_value and a position whose id is pad_idx contributes -inf
 * batch <= 32768.  Asynchronous on `stream`; never allocates. */
int sb_laser2_forward(SbLaser2* enc, const int64_t* ids, int64_t ids_row_stride, const int32_t* seq_lens_host, int32_t batch,
                      int32_t seq_len, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* Checks the sticky device-side flag (token id outside [0, vocab_size)) of the forwards since the last check; synchronises
 * `stream`.  Returns SB_OK or SB_ERR_INPUT. */
int sb_laser2_check_inputs(SbLaser2* enc, void* stream);
/* Read-only view of the handle's repacked weights of layer `layer` (DEVICE pointers owned by the handle, valid until
 * sb_laser2_destroy; rows in the gate order of sb_lstm_recurrent, direction d at rows d * 4H):
 *   w_ih  bf16 [dirs * 4H, in] (in = embed_dim for layer 0, else dirs * H), bias fp32 [dirs * 4H] = b_ih + b_hh,
 *   w_hh  bf16 [dirs * 4H, H].
 * sb_laser2_forward is sb_laser2_embed, then per layer sb_gemm_bf16 (bias epilogue) on these and sb_lstm_recurrent. */
int sb_laser2_layer_weights(const SbLaser2* enc, int32_t layer, const void** w_ih, const float** bias, const void** w_hh);

/* The embedding gather of sb_laser2_forward alone.
 *   ids        DEVICE int64 [B, ids_row_stride >= S]; cu_seqlens DEVICE int32 [B + 1] with lengths in 0..S
 *   table      DEVICE bf16 [vocab, D], D a positive multiple of 8, 16-byte aligned
 *   x          DEVICE bf16 [cu[B], D], 16-byte aligned: row cu[b] + t = table[ids[b, t]] for t < len_b
 *   pad_mask   DEVICE uint8 [cu[B]]: 1 where ids[b, t] == pad_idx, t < len_b
 *   tail_keep  DEVICE uint8 [B]: 1 if some ids[b, t] != pad_idx with len_b <= t < S (positions >= S are not read)
 *   err_flag   DEVICE int32: set to 1 (never cleared) when an id lies outside [0, vocab); that row of x is zero. */
int sb_laser2_embed(const int64_t* ids, int64_t ids_row_stride, const int32_t* cu_seqlens, int32_t B, int32_t S,
                    const void* table, int64_t vocab, int32_t D, int64_t pad_idx, void* x, uint8_t* pad_mask,
                    uint8_t* tail_keep, int32_t* err_flag, void* stream);

/* The LSTM recurrence alone (H = 512), for one layer and `num_dirs` directions.  Gate order: row / column
 * d * 4H + 128 c + 32 gate + u of the operands below is gate `gate` (i, f, g, o) of hidden unit 32 c + u of direction d.
 *   G          DEVICE bf16 [T, ldg] input pre-activations X . W_ih^T + b_ih + b_hh of the packed tokens; 4-byte aligned,
 *              ldg even and >= num_dirs * 4H (only the first num_dirs * 4H columns are read)
 *   w_hh       DEVICE bf16 [num_dirs * 4H, H] in the gate order above, 16-byte aligned
 *   cu_seqlens DEVICE int32 [B + 1]: the tokens of sequence b are rows cu[b] .. cu[b + 1] - 1
 *   tile_seqs  DEVICE int32 [num_tiles * 64]: the sequences of each 64-row tile, -1 = empty row; a tile may be all -1
 * and exactly one of
 *   y          DEVICE bf16 [T, ldy]: h_t of direction d at columns d * H (the reverse direction runs from the last token);
 *              4-byte aligned, ldy even and >= num_dirs * H; only the tokens of sequences in tile_seqs and only the first
 *              num_dirs * H columns are written
 *   pool_out   DEVICE fp32 [B, ldp]: max over the sequence's tokens of h_t, skipping tokens with pad_mask[token] != 0
 *              (DEVICE uint8 [T] or NULL), then max with padding_value where tail_keep[b] != 0 (DEVICE uint8 [B] or NULL);
 *              -inf when nothing is left; 8-byte aligned, ldp even and >= num_dirs * H; only the rows of sequences named in
 *              tile_seqs and only the first num_dirs * H columns are written.
 * A leading dimension or an alignment outside these rules is SB_ERR_INVALID, refused before any launch. */
int sb_lstm_recurrent(const void* G, int64_t ldg, const void* w_hh, const int32_t* cu_seqlens, const int32_t* tile_seqs,
                      int32_t num_tiles, int32_t num_dirs, void* y, int64_t ldy, float* pool_out, int64_t ldp,
                      const uint8_t* pad_mask, const uint8_t* tail_keep, float padding_value, void* stream);

/* ---- BLASER 2.0: translation-quality scores from sentence embeddings ----
 * Replaces BlaserModel.forward / featurize_input (sonar/models/blaser/model.py:82-125) of the `basic_ref` (COMET) and
 * `basic_qe` (QE) configs (sonar/models/blaser/config.py:43-67), in eval mode (dropout off):
 *   F.normalize each input row -> features -> [Linear -> Tanh] x num_hidden -> Linear(hidden_dims[last] -> 1)
 * with the features (model.py:99-124)
 *   COMET: [ref, mt, src*mt, ref*mt, |mt-src|, |mt-ref|]  (6E)      QE: [src, mt, src*mt, |mt-src|]  (4E).
 * The features and the hidden layers but the last are bf16, the last hidden layer and the score fp32.  A pair's score does
 * not depend on the other pairs of the call or their number, bit for bit. */
#define SB_BLASER_COMET 0
#define SB_BLASER_QE 1

typedef struct SbBlaser SbBlaser;

typedef struct SbBlaserConfig {
  int32_t input_form;         /* SB_BLASER_COMET | SB_BLASER_QE */
  int32_t embedding_dim;      /* E = 1024; a positive multiple of 16 with a feature width (4E QE, 6E COMET) that is a
                               * multiple of 64 */
  int32_t num_hidden;         /* >= 1 (the positive entries of the reference's hidden_dims) */
  const int32_t* hidden_dims; /* HOST [num_hidden], each a positive multiple of 256 ([3072, 1536]); copied at create */
  int32_t cta_group;          /* GEMM tiles: 0/2 = CTA pairs, 1 = single CTAs */
  int32_t num_sms;            /* 0 = query the device */
} SbBlaserConfig;

/* HOST arrays of num_hidden + 1 DEVICE pointers (caller-owned, must outlive the handle), in the order of the module's
 * Linear layers (mlp.<i>.weight / .bias):
 *   w[i], i < num_hidden: bf16 [hidden_dims[i], in_i] (in_0 = the feature width)      b[i]: fp32 [hidden_dims[i]]
 *   w[num_hidden]: fp32 [hidden_dims[num_hidden - 1]] (the output layer's single row, 16-byte aligned)  b: fp32 [1] */
typedef struct SbBlaserWeights {
  const void* const* w;
  const float* const* b;
} SbBlaserWeights;

/* Allocates no device memory and does not synchronise. */
int sb_blaser_create(const SbBlaserConfig* cfg, const SbBlaserWeights* w, SbBlaser** out);
void sb_blaser_destroy(SbBlaser* model);
/* Bytes of device workspace for <= max_rows pairs: max_rows * (F * 2 + max(inner hidden widths) * 2 + hidden_dims[last] * 4)
 * plus alignment (about 1.6 GB for 65 536 pairs of `basic_ref`). */
int sb_blaser_workspace_bytes(const SbBlaser* model, int32_t max_rows, size_t* bytes);
/* src, mt, ref  DEVICE fp32 [rows, ld] embeddings (ld >= E, ld % 4 == 0, 16-byte aligned); ref is not read for QE and may
 *               be NULL there
 * scores        DEVICE fp32 [rows]
 * Asynchronous on `stream`; never allocates; rows = 0 does nothing. */
int sb_blaser_forward(SbBlaser* model, const float* src, const float* mt, const float* ref, int64_t ld, int32_t rows,
                      float* scores, void* workspace, size_t workspace_bytes, void* stream);
/* The featurization alone: out DEVICE [rows, 6E] (COMET) or [rows, 4E] (QE), fp32 (out_fp32 = 1) or bf16, of the inputs
 * as given (normalize = 0, BlaserModel.featurize_input) or after F.normalize (normalize = 1, what forward feeds the first
 * Linear).  E a positive multiple of 16; the other arguments as for sb_blaser_forward. */
int sb_blaser_featurize(const float* src, const float* mt, const float* ref, int64_t ld, int32_t rows, int32_t E,
                        int32_t input_form, int32_t normalize, void* out, int32_t out_fp32, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SONAR_B200_H_ */
