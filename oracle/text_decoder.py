"""CPU oracle for the SONAR embedding->text decoder + beam search (BASELINE.json config 4).
TEST INFRASTRUCTURE ONLY (see oracle/text_encoder.py for the import rule).

Restates:
* ``ConditionalTransformerDecoderModel.decode / project`` -- ``sonar/nn/conditional_decoder_model.py:60-94``
* the decoder wiring -- ``sonar/models/sonar_text/factory.py:229-315`` (pre-LN layers with self-attention,
  encoder-decoder attention over ``input_dim`` keys, ReLU FFN; stack ``norm_order=PRE`` => final LayerNorm;
  ``TiedProjection`` to the embedding matrix, no bias), config ``config.py:197-219``
* state-dict names -- ``sonar/models/sonar_text/handler.py:136-158``
* how the pipeline drives it -- ``sonar/inference_pipelines/text.py:272-346``: the sentence embedding is the
  single encoder position ``[N,1,1024]`` (``sonar/models/sonar_translation/model.py:48-53,81-95``), so every
  cross-attention softmax is over ONE key and equals 1.
* fairseq2 ``BeamSearchSeq2SeqGenerator`` [fs2] (SURVEY App. C / F8), written out in ``beam_search`` below.

Pinning: the layer maths is pinned against HuggingFace ``M2M100Decoder`` (independent implementation of the same
fairseq lineage) through ``tests/golden/m2m100_decoder_small.pt`` (``tests/golden/make_m2m100_golden.py``).
The beam-search bookkeeping restates fairseq2 0.4 from two independent recollections of its source (fairseq2 is not
installable here; the reference's own pins -- exact output strings, ``tests/integration_tests/test_text_sonar.py:107-118`` --
need real weights).  It is cross-checked against HuggingFace ``generate(num_beams=...)`` on a tiny M2M100 decoder in the
regime where the two algorithms coincide (``tests/test_beam_vs_hf.py``); every divergence is listed there.
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from .text_encoder import sinusoidal_table


@dataclass
class OracleDecoderConfig:
    """Fields of ``SonarTextDecoderConfig`` that reach the maths; defaults = arch ``basic`` (config.py:197-219)."""

    model_dim: int = 1024
    vocab_size: int = 256206
    max_seq_len: int = 512
    pad_idx: int = 1
    num_layers: int = 24
    num_heads: int = 16
    ffn_inner_dim: int = 8192
    input_dim: Optional[int] = None
    ln_eps: float = 1e-5


def make_synthetic_decoder_state_dict(cfg: OracleDecoderConfig, seed: int = 2, weight_std: float = 0.02) -> Dict[str, Tensor]:
    g = torch.Generator().manual_seed(seed)
    d, f = cfg.model_dim, cfg.ffn_inner_dim
    kv = cfg.input_dim or d

    def rn(*shape, std=weight_std):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    sd: Dict[str, Tensor] = {"decoder_frontend.embed.weight": rn(cfg.vocab_size, d, std=d ** -0.5)}
    for i in range(cfg.num_layers):
        p = f"decoder.layers.{i}."
        for attn, kdim in (("self_attn", d), ("encoder_decoder_attn", kv)):
            sd[p + f"{attn}.q_proj.weight"] = rn(d, d)
            sd[p + f"{attn}.k_proj.weight"] = rn(d, kdim)
            sd[p + f"{attn}.v_proj.weight"] = rn(d, kdim)
            sd[p + f"{attn}.output_proj.weight"] = rn(d, d)
            for n in ("q_proj", "k_proj", "v_proj", "output_proj"):
                sd[p + f"{attn}.{n}.bias"] = rn(d)
            sd[p + f"{attn}_layer_norm.weight"] = 1.0 + rn(d)
            sd[p + f"{attn}_layer_norm.bias"] = rn(d)
        sd[p + "ffn.inner_proj.weight"] = rn(f, d)
        sd[p + "ffn.inner_proj.bias"] = rn(f)
        sd[p + "ffn.output_proj.weight"] = rn(d, f)
        sd[p + "ffn.output_proj.bias"] = rn(d)
        sd[p + "ffn_layer_norm.weight"] = 1.0 + rn(d)
        sd[p + "ffn_layer_norm.bias"] = rn(d)
    sd["decoder.layer_norm.weight"] = 1.0 + rn(d)
    sd["decoder.layer_norm.bias"] = rn(d)
    sd["final_proj.weight"] = sd["decoder_frontend.embed.weight"]  # TiedProjection (factory.py:306-307)
    return sd


def attention_core(q: Tensor, k: Tensor, v: Tensor, mask: Optional[Tensor]) -> Tensor:
    """softmax(q . k / sqrt(head_dim) + mask) . v of q [B, H, S, hd], k / v [B, H, T, hd] -> [B, S, H * hd]."""
    b, h, s, hd = q.shape
    a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
    return a.transpose(1, 2).reshape(b, s, h * hd)


class OracleTextDecoder:
    """Teacher-forced full-sequence forward of the decoder (causal self-attention), fp32/fp64 on CPU."""

    def __init__(self, cfg: OracleDecoderConfig, state_dict: Dict[str, Tensor], dtype: torch.dtype = torch.float32):
        self.cfg = cfg
        self.dtype = dtype
        self.sd = {k: v.to(dtype) for k, v in state_dict.items()}
        self.pos = sinusoidal_table(cfg.max_seq_len + cfg.pad_idx + 1, cfg.model_dim, cfg.pad_idx)

    def _mha(self, p: str, q_in: Tensor, kv_in: Tensor, mask: Optional[Tensor]) -> Tensor:
        sd, h = self.sd, self.cfg.num_heads
        b, s, d = q_in.shape
        t = kv_in.shape[1]
        hd = d // h
        q = F.linear(q_in, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"]).view(b, s, h, hd).transpose(1, 2)
        k = F.linear(kv_in, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"]).view(b, t, h, hd).transpose(1, 2)
        v = F.linear(kv_in, sd[p + "v_proj.weight"], sd[p + "v_proj.bias"]).view(b, t, h, hd).transpose(1, 2)
        return F.linear(attention_core(q, k, v, mask), sd[p + "output_proj.weight"], sd[p + "output_proj.bias"])

    @torch.no_grad()
    def hidden(self, tokens: Tensor, encoder_output: Tensor) -> Tensor:
        """tokens int64 [B,S] (no padding), encoder_output [B,T,input_dim] (T = 1 for SONAR) -> final-LN states [B,S,D]."""
        cfg, sd = self.cfg, self.sd
        b, s = tokens.shape
        d = cfg.model_dim
        x = F.embedding(tokens, sd["decoder_frontend.embed.weight"]) * math.sqrt(d)
        x = (x.float() + self.pos[:s][None]).to(self.dtype)
        enc = encoder_output.to(self.dtype)
        causal = torch.full((s, s), -torch.inf, dtype=self.dtype).triu(1)
        for i in range(cfg.num_layers):
            p = f"decoder.layers.{i}."
            y = F.layer_norm(x, (d,), sd[p + "self_attn_layer_norm.weight"], sd[p + "self_attn_layer_norm.bias"], cfg.ln_eps)
            x = x + self._mha(p + "self_attn.", y, y, causal)
            y = F.layer_norm(x, (d,), sd[p + "encoder_decoder_attn_layer_norm.weight"],
                             sd[p + "encoder_decoder_attn_layer_norm.bias"], cfg.ln_eps)
            x = x + self._mha(p + "encoder_decoder_attn.", y, enc, None)
            y = F.layer_norm(x, (d,), sd[p + "ffn_layer_norm.weight"], sd[p + "ffn_layer_norm.bias"], cfg.ln_eps)
            y = F.relu(F.linear(y, sd[p + "ffn.inner_proj.weight"], sd[p + "ffn.inner_proj.bias"]))
            x = x + F.linear(y, sd[p + "ffn.output_proj.weight"], sd[p + "ffn.output_proj.bias"])
        return F.layer_norm(x, (d,), sd["decoder.layer_norm.weight"], sd["decoder.layer_norm.bias"], cfg.ln_eps)

    @torch.no_grad()
    def logits(self, tokens: Tensor, encoder_output: Tensor) -> Tensor:
        return F.linear(self.hidden(tokens, encoder_output), self.sd["final_proj.weight"])

    @torch.no_grad()
    def step_lprobs(self, tokens: Tensor, encoder_output: Tensor) -> Tensor:
        """fp32 log-probabilities of the NEXT token after ``tokens`` [B,S] -> [B,V] (full recompute, no cache)."""
        return torch.log_softmax(self.logits(tokens, encoder_output)[:, -1].float(), dim=-1)


# ----------------------------------------------------------------------------------------------------------
# beam search (fairseq2 0.4 BeamSearchSeq2SeqGenerator + StandardBeamSearchAlgorithm semantics, SURVEY App. C)
#
# Written in fairseq2's own terms (``step_nr`` = absolute index of the position being generated, prompt included)
# so each rule can be read against ``fairseq2/generation/beam_search.py`` [fs2]:
#   _prefill         the cumulative log-prob of prompt tokens 1..P-1 seeds every hypothesis score
#                    (``step_scores[:, 1:P] = cumsum(lprob(prompt[s] | prompt[:s]))``)
#   _step            PAD never; UNK -= unk_penalty; EOS forbidden while ``step_nr < min_seq_len - 1`` with
#                    ``min_seq_len = P + min_gen_len`` (so ``min_gen_len=1`` allows an immediate EOS); on the last
#                    step (``step_nr == max_seq_len - 1``) everything but EOS is -inf
#   algorithm.step   scores = lprobs + cumulative score; top ``min(2*beam, V)`` over beam x V (first step: one beam)
#   _search_beam     EOS candidates count only inside the top ``beam`` ranks; they are finished in rank order and the
#                    sentence is closed the moment it owns ``beam`` hypotheses (later EOS candidates of that step are
#                    dropped); the next beam = the first ``beam`` non-EOS candidates
#   _finish_sequence score /= (seq_len - 1) ** len_penalty with seq_len = step_nr + 1 counting prompt and EOS
#                    ("the first step's score is always 0, do not include it in the normalisation")
# ----------------------------------------------------------------------------------------------------------
@dataclass
class BeamSearchConfig:
    beam_size: int = 5
    min_gen_len: int = 1
    max_gen_len: int = 128      # generated tokens incl. EOS, prompt excluded (README.md:83 passes max_seq_len explicitly)
    normalize_scores: bool = True
    len_penalty: float = 1.0
    unk_penalty: float = 0.0
    pad_idx: int = 0            # tokenizer pad (NLLB: 0); never generated
    unk_idx: int = 1
    eos_idx: int = 3
    # fairseq2 always scores the prompt (True).  False drops that per-sentence constant: HuggingFace's forced-BOS generation
    # behaves that way, so tests/test_beam_vs_hf.py can pin every OTHER rule (divisor, EOS handling, closing) against it.
    score_prompt: bool = True


def beam_search_step(lprobs: Tensor, cum: Tensor, step: int, cfg: BeamSearchConfig, first: bool):
    """One expansion.  lprobs [N, beam, V] fp32 (already constrained), cum [N, beam] running sums.
    -> (cand_score [N, 2*beam], cand_beam, cand_token) sorted by score desc; ties by flat index asc."""
    n, beam, v = lprobs.shape
    total = lprobs + cum[:, :, None]
    if first:  # all beams are copies of the prompt: expand beam 0 only
        total = total.clone()
        total[:, 1:, :] = -torch.inf
    k = min(2 * beam, beam * v - 1)
    flat = total.reshape(n, beam * v)
    # stable order: score desc, flat index asc (torch.topk is not stable -> sort explicitly)
    order = torch.argsort(-flat, dim=1, stable=True)[:, :k]
    score = torch.gather(flat, 1, order)
    return score, order // v, order % v


def constrain_lprobs(lprobs: Tensor, gen_len: int, cfg: BeamSearchConfig) -> Tensor:
    """gen_len = number of tokens generated so far (0 at the first expansion) = step_nr - P."""
    lp = lprobs.clone()
    if gen_len >= cfg.max_gen_len - 1:  # step_nr == max_seq_len - 1: the last allowed token must be EOS
        eos = lp[..., cfg.eos_idx].clone()
        lp[...] = -torch.inf
        lp[..., cfg.eos_idx] = eos
        return lp
    lp[..., cfg.pad_idx] = -torch.inf
    if cfg.unk_penalty:
        lp[..., cfg.unk_idx] -= cfg.unk_penalty
    if gen_len < cfg.min_gen_len - 1:  # step_nr < min_seq_len - 1
        lp[..., cfg.eos_idx] = -torch.inf
    return lp


def beam_search(lprob_fn, prompt: Tensor, n: int, cfg: BeamSearchConfig,
                dropped_eos: Optional[List[int]] = None) -> List[List[Tuple[float, List[int]]]]:
    """``lprob_fn(tokens [R,S]) -> [R,V]`` next-token log-probs for R = n*beam rows laid out sentence-major.
    ``prompt`` int64 [P] (SONAR target mode: [</s>, __lang__]).  Returns, per sentence, its finished hypotheses
    sorted best first as (score, generated tokens incl. the final EOS).  ``dropped_eos`` (optional, length n) counts per
    sentence the in-beam EOS candidates that arrived when the sentence already owned ``beam`` hypotheses (fairseq2 drops them;
    HuggingFace would let them compete -- tests/test_beam_vs_hf.py uses the count to recognise that divergence)."""
    beam = cfg.beam_size
    P = prompt.numel()
    seqs = prompt[None, None, :].repeat(n, beam, 1)  # [N, beam, S]
    cum = torch.zeros(n, beam)
    for p in range(1, P if cfg.score_prompt else 1):  # _prefill: score of the prompt itself
        lp = lprob_fn(seqs[:, :, :p].reshape(n * beam, -1)).reshape(n, beam, -1).float()
        cum = cum + lp[:, :, int(prompt[p])]
    finished: List[List[Tuple[float, List[int]]]] = [[] for _ in range(n)]
    done = [False] * n
    alive = torch.ones(n, beam, dtype=torch.bool)
    for gen_len in range(cfg.max_gen_len):
        step_nr = P + gen_len
        lp = lprob_fn(seqs.reshape(n * beam, -1)).reshape(n, beam, -1).float()
        lp = constrain_lprobs(lp, gen_len, cfg)
        lp = torch.where(alive[:, :, None], lp, torch.full_like(lp, -torch.inf))
        score, cbeam, ctok = beam_search_step(lp, cum, gen_len, cfg, first=(gen_len == 0))
        new_seqs = torch.empty(n, beam, seqs.shape[2] + 1, dtype=torch.int64)
        new_cum = torch.full((n, beam), -torch.inf)
        new_alive = torch.zeros(n, beam, dtype=torch.bool)
        for i in range(n):
            if done[i]:
                new_seqs[i] = torch.cat([seqs[i], torch.full((beam, 1), cfg.pad_idx)], 1)
                continue
            slot = 0
            for r in range(score.shape[1]):
                s = float(score[i, r])
                if s == -math.inf:
                    break
                b, t = int(cbeam[i, r]), int(ctok[i, r])
                if t == cfg.eos_idx:
                    # only EOS candidates ranked inside the beam finish a hypothesis, and only until the sentence owns `beam`
                    if r < beam and len(finished[i]) >= beam and dropped_eos is not None:
                        dropped_eos[i] += 1
                    if r < beam and len(finished[i]) < beam:
                        toks = seqs[i, b, P:].tolist() + [t]
                        # IEEE float32 division, like the product (torch / CUDA)
                        fs = float(torch.tensor(s, dtype=torch.float32) /
                                   torch.tensor(float(step_nr) ** cfg.len_penalty, dtype=torch.float32)) \
                            if cfg.normalize_scores else s
                        finished[i].append((fs, toks))
                    continue
                if slot < beam:
                    new_seqs[i, slot] = torch.cat([seqs[i, b], torch.tensor([t])])
                    new_cum[i, slot] = s
                    new_alive[i, slot] = True
                    slot += 1
            for sl in range(slot, beam):
                new_seqs[i, sl] = torch.cat([seqs[i, 0], torch.tensor([cfg.pad_idx])])
            if len(finished[i]) >= beam:
                done[i] = True
                new_alive[i] = False
        seqs, cum, alive = new_seqs, new_cum, new_alive
        if all(done) or not bool(alive.any()):
            break
    out = []
    for i in range(n):
        # stable sort: score desc, earlier-finished first on ties
        out.append(sorted(finished[i], key=lambda h: -h[0])[:beam])
    return out


# ------------------------------------------------------------------------------------------------
# Sampling (fairseq2 SamplingSeq2SeqGenerator + TopKSampler / TopPSampler [fs2], restated from the documented behaviour;
# PARITY UNPINNED: fairseq2 is not installable and HuggingFace's samplers draw from another random stream).  The subset the
# sampler keeps is taken over the WHOLE vocabulary here -- sonar_b200/sampling.py sees 16 candidates per row and must agree
# whenever the subset lies inside them.
# ------------------------------------------------------------------------------------------------
@dataclass
class SamplingConfig:
    top_k: Optional[int] = None   # exactly one of top_k / top_p
    top_p: Optional[float] = None
    num_gens: int = 1
    min_gen_len: int = 1
    max_gen_len: int = 128
    normalize_scores: bool = True
    len_penalty: float = 1.0
    pad_idx: int = 0
    eos_idx: int = 3


def sampling_search(lprob_fn, prompt: Tensor, n: int, cfg: SamplingConfig, uniforms: Tensor
                    ) -> List[List[Tuple[float, List[int]]]]:
    """``lprob_fn(tokens [R,S]) -> [R,V]`` for R = n * num_gens rows (input-major); ``uniforms`` fp32 [max_gen_len, R]: the
    number in [0, 1) row r consumes at generation step g.  -> per input its ``num_gens`` hypotheses in generation order as
    (score, generated tokens incl. the final EOS); score = sum of the sampled tokens' log-probs, / step_nr ** len_penalty
    when normalised."""
    G = cfg.num_gens
    R = n * G
    P = prompt.numel()
    seqs = [[int(v) for v in prompt] for _ in range(R)]
    cum = [torch.zeros((), dtype=torch.float32) for _ in range(R)]
    out: List[Optional[Tuple[float, List[int]]]] = [None] * R
    for g in range(cfg.max_gen_len):
        live = [r for r in range(R) if out[r] is None]
        if not live:
            break
        lp = lprob_fn(torch.tensor([seqs[r] for r in live], dtype=torch.int64)).float()
        for row, r in enumerate(live):
            if g >= cfg.max_gen_len - 1:
                t, l = cfg.eos_idx, lp[row, cfg.eos_idx]
            else:
                probs = lp[row].exp()
                probs[cfg.pad_idx] = 0.0
                if g < cfg.min_gen_len - 1:
                    probs[cfg.eos_idx] = 0.0
                order = torch.argsort(probs, descending=True, stable=True)  # probability desc, token asc
                ps = probs[order]
                if cfg.top_k is not None:
                    w = ps.clone()
                    w[cfg.top_k:] = 0.0
                else:
                    w = ps.masked_fill((ps.cumsum(0) - ps) > cfg.top_p, 0.0)
                kept = int((w > 0).sum())
                cdf = w[:kept].cumsum(0)
                u = uniforms[g, r].float() * cdf[-1]
                pick = min(int((cdf <= u).sum()), kept - 1)
                t = int(order[pick])
                l = lp[row, t]
            seqs[r].append(t)
            cum[r] = cum[r] + l
            if t == cfg.eos_idx:
                s = cum[r] / torch.tensor(float(P + g) ** cfg.len_penalty, dtype=torch.float32) if cfg.normalize_scores else cum[r]
                out[r] = (float(s), seqs[r][P:])
    return [[out[i * G + j] for j in range(G)] for i in range(n)]
