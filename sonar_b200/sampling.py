"""Sampling generation over the CUDA decoder -- the ``sampler=`` branch of ``EmbeddingToTextModelPipeline.predict``
(``sonar/inference_pipelines/text.py:313-320``): fairseq2's ``SamplingSeq2SeqGenerator`` with a ``TopKSampler`` or
``TopPSampler`` [fs2].  fairseq2 is not installable here, so the semantics below are restated from its documented
behaviour and are **parity unpinned** against it (``oracle/text_decoder.py::sampling_search`` is the CPU restatement the
tests hold this file to; the token subsets the two samplers keep are pinned against HuggingFace's ``TopKLogitsWarper`` /
``TopPLogitsWarper``, ``tests/test_oracle_decoder.py``):

* every step turns the next-token distribution into probabilities, zeroes PAD, zeroes EOS while the hypothesis is shorter
  than ``min_gen_len``, lets the sampler keep a subset (the ``k`` most probable tokens / the smallest prefix of the
  descending order whose mass reaches ``p``), renormalises over that subset and draws one token; the last allowed
  position is forced to EOS;
* ``num_gens`` independent hypotheses per input; with ``compute_scores`` a hypothesis scores the sum of the log-probs of
  its sampled tokens, divided by ``step_nr ** len_penalty`` when ``normalize_scores`` (same divisor as beam search), and
  the hypotheses of an input are returned best first; without it they come in generation order with ``score=None``.

The decoder step hands back the 16 most probable tokens of a row with their exact log-probabilities over the whole
vocabulary (``sb_decoder_step``), which is all top-k sampling needs for ``k <= 14`` (PAD and EOS may have to be dropped
from the 16) and all nucleus sampling needs whenever the nucleus lies inside those 16 tokens; a nucleus that reaches
beyond them is reported as an error after the call instead of being truncated silently.  The draw itself is an inverse-CDF
lookup of one uniform number per row from a seeded ``torch.Generator`` -- a few [rows, 16] tensor ops per step, no host
synchronisation inside the loop except the periodic "everything finished" check.
"""

from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import torch
from torch import Tensor

from .generation import NEG_INF, Hypothesis, Seq2SeqGeneratorOutput
from .text_decoder import TOPK, B200TextDecoderModel


class Sampler:
    """Keeps a subset of the candidates: ``weights(probs)`` gets probabilities sorted descending along dim 1 (zeros for
    forbidden tokens) and returns (unnormalised sampling weights, rows whose subset may reach beyond the candidates)."""

    def weights(self, probs: Tensor) -> Tuple[Tensor, Optional[Tensor]]:
        raise NotImplementedError


class TopKSampler(Sampler):
    def __init__(self, k: int) -> None:
        if k < 1:
            raise ValueError("`k` must be greater than or equal to 1")
        if k > TOPK - 2:
            raise ValueError(f"`k` must be <= {TOPK - 2} (the decoder step returns the top-{TOPK} tokens per row and PAD / EOS "
                             "may have to be dropped from them)")
        self.k = k

    def weights(self, probs: Tensor) -> Tuple[Tensor, Optional[Tensor]]:
        w = probs.clone()
        w[:, self.k:] = 0.0
        return w, None


class TopPSampler(Sampler):
    def __init__(self, p: float) -> None:
        if not 0.0 < p <= 1.0:
            raise ValueError("`p` must be in (0, 1]")
        self.p = p

    def weights(self, probs: Tensor) -> Tuple[Tensor, Optional[Tensor]]:
        before = probs.cumsum(1) - probs  # mass of the strictly more probable tokens
        w = probs.masked_fill(before > self.p, 0.0)
        # every candidate kept and still short of p: the nucleus continues among tokens the step did not return
        short = (before[:, -1] + probs[:, -1] < self.p) & (probs[:, -1] > 0)
        return w, short


class SamplingSeq2SeqGenerator:
    def __init__(self, model: B200TextDecoderModel, sampler: Sampler, *, num_gens: int = 1, min_gen_len: int = 1,
                 max_gen_len: Tuple[int, int] = (1, 128), max_seq_len: Optional[int] = None, echo_prompt: bool = False,
                 compute_scores: bool = False, normalize_scores: bool = True, temperature: float = 1.0,
                 unk_penalty: float = 0.0, len_penalty: float = 1.0, pad_idx: int = 0, sync_every: int = 8,
                 generator: Optional[torch.Generator] = None,
                 uniform_fn: Optional[Callable[[int, int], Tensor]] = None) -> None:
        """``generator``: the ``torch.Generator`` (on the model's device) the uniform numbers come from; ``uniform_fn(step,
        rows)`` replaces it (tests feed the numbers the oracle consumed)."""
        if num_gens < 1:
            raise ValueError("`num_gens` must be greater than or equal to 1")
        if min_gen_len < 1:
            raise ValueError("`min_gen_len` must be greater than or equal to 1")
        if temperature != 1.0:
            raise NotImplementedError("temperature != 1.0 (the step returns log-probabilities normalised at temperature 1)")
        if unk_penalty != 0.0:
            raise NotImplementedError("unk_penalty with sampling")
        self.model, self.sampler = model, sampler
        self.num_gens, self.min_gen_len, self.max_gen_len, self.max_seq_len = num_gens, min_gen_len, max_gen_len, max_seq_len
        self.echo_prompt, self.compute_scores, self.normalize_scores = echo_prompt, compute_scores, normalize_scores
        self.len_penalty, self.pad_idx, self.sync_every = len_penalty, pad_idx, sync_every
        self.generator, self.uniform_fn = generator, uniform_fn

    def _uniform(self, step: int, rows: int, dev: torch.device) -> Tensor:
        if self.uniform_fn is not None:
            return self.uniform_fn(step, rows).to(dev, torch.float32)
        return torch.rand((rows,), generator=self.generator, device=dev, dtype=torch.float32)

    @torch.inference_mode()
    def __call__(self, source_seqs: Tensor, source_padding_mask, prompt_seqs: Tensor, prompt_padding_mask=None
                 ) -> Seq2SeqGeneratorOutput:
        m = self.model
        dev = m.device
        vi = m.target_vocab_info
        eos, pad = vi.eos_idx, self.pad_idx
        if source_seqs.dim() == 2:
            source_seqs = source_seqs[:, None, :]
        N, G = source_seqs.shape[0], self.num_gens
        R = N * G
        prompt = prompt_seqs.to(dev).long()
        if prompt.dim() == 1:
            prompt = prompt[None].expand(N, -1)
        P = prompt.shape[1]
        model_max = m.max_target_seq_len
        max_total = min(self.max_seq_len or model_max, model_max)
        max_gen = min(int(self.max_gen_len[0] * source_seqs.shape[1] + self.max_gen_len[1]), max_total - P)
        if max_gen < 1:
            raise ValueError("`max_seq_len` leaves no room to generate after the prompt")
        min_gen = min(self.min_gen_len, max_gen)
        Tmax = P + max_gen
        # one decoder row per (input, generation): `beam` = num_gens rows that never exchange history
        m.begin(source_seqs[:, 0], G, Tmax)
        table = torch.arange(R, dtype=torch.int32, device=dev)[:, None].expand(R, Tmax).contiguous()
        seqs = torch.full((R, Tmax), pad, dtype=torch.int64, device=dev)
        seqs[:, :P] = prompt.repeat_interleave(G, 0)
        cum = torch.zeros((R,), dtype=torch.float32, device=dev)
        score = torch.full((R,), NEG_INF, dtype=torch.float32, device=dev)
        length = torch.full((R,), Tmax, dtype=torch.int64, device=dev)
        done = torch.zeros((R,), dtype=torch.bool, device=dev)
        beyond = torch.zeros((), dtype=torch.bool, device=dev)
        for p in range(P - 1):  # prefill: the prompt feeds the KV cache
            m.step(seqs[:, p].contiguous(), table, p)
        tokens = seqs[:, P - 1].contiguous()
        ar = torch.arange(R, device=dev)
        for g in range(max_gen):
            t = P - 1 + g
            lp, tok, eos_lp = m.step(tokens, table, t)
            tok = tok.long()
            if g >= max_gen - 1:  # the last allowed token must be EOS
                new_tok = torch.full((R,), eos, dtype=torch.int64, device=dev)
                new_lp = eos_lp.clone()
            else:
                probs = lp.exp().masked_fill((tok < 0) | (tok == pad), 0.0)
                if g < min_gen - 1:
                    probs = probs.masked_fill(tok == eos, 0.0)
                order = torch.argsort(probs, dim=1, descending=True, stable=True)  # candidates arrive (value desc, token asc)
                probs = torch.gather(probs, 1, order)
                w, short = self.sampler.weights(probs)
                if short is not None:
                    beyond |= (short & ~done).any()
                cdf = w.cumsum(1)
                u = self._uniform(g, R, dev) * cdf[:, -1]
                pick = (cdf <= u[:, None]).sum(1)
                last = (w > 0).to(torch.int64).cumsum(1).argmax(1)  # last kept candidate (rounding at the top of the CDF)
                pick = torch.minimum(pick, last)
                sel = torch.gather(order, 1, pick[:, None])
                new_tok = torch.gather(tok, 1, sel)[:, 0]
                new_lp = torch.gather(lp, 1, sel)[:, 0]
            live = ~done
            seqs[:, t + 1] = torch.where(live, new_tok, seqs[:, t + 1])
            cum = torch.where(live, cum + new_lp, cum)
            ends = live & (new_tok == eos)
            div = torch.full((), float(P + g) ** self.len_penalty, dtype=torch.float32, device=dev)
            score = torch.where(ends, cum / div if self.normalize_scores else cum, score)
            length = torch.where(ends, torch.full_like(length, t + 2), length)
            done = done | ends
            tokens = torch.where(done, torch.full_like(new_tok, pad), new_tok)
            if (g + 1) % self.sync_every == 0 and bool(done.all()):
                break
        m.check_inputs()
        if bool(beyond):
            raise ValueError(f"top-p sampling: a nucleus reached beyond the {TOPK} most probable tokens the decoder step returns; "
                             "use a smaller `p` or TopKSampler")
        seqs_c, len_c, score_c = seqs.cpu(), length.cpu(), score.cpu()
        start = 0 if self.echo_prompt else P
        out: List[List[Hypothesis]] = []
        for i in range(N):
            hyps = [Hypothesis(seq=seqs_c[r, start:int(len_c[r])].clone(),
                               score=float(score_c[r]) if self.compute_scores else None)
                    for r in range(i * G, (i + 1) * G)]
            if self.compute_scores:
                hyps.sort(key=lambda h: -h.score)  # stable: generation order on ties
            out.append(hyps)
        return Seq2SeqGeneratorOutput(out)
