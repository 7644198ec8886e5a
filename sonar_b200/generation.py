"""Beam search over the CUDA decoder -- the part of fairseq2's ``BeamSearchSeq2SeqGenerator`` [fs2] that
``EmbeddingToTextModelPipeline.predict`` drives (``sonar/inference_pipelines/text.py:315-333``), with the same
constructor keywords (``beam_size=5, min_gen_len=1, max_gen_len=(1,128), max_seq_len, normalize_scores=True,
len_penalty=1.0, unk_penalty=0.0``; SURVEY App. C / F8).

All bookkeeping is vectorised ``torch`` on the device (a few [N, 2*beam] tensors per step) with NO host
synchronisation inside the loop except an "all sentences finished" check every few steps; the model step itself is
one C-ABI call.  Ordering rule everywhere: score descending, then (beam * vocab + token) ascending -- the rule the
oracle (``oracle/text_decoder.py::beam_search_step``) defines.
"""

from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple, Union

import torch
from torch import Tensor

from . import _lib
from .text_decoder import TOPK, B200TextDecoderModel

NEG_INF = float("-inf")


@dataclass
class Hypothesis:
    seq: Tensor            # generated tokens (prompt stripped unless echo_prompt), final EOS included
    score: Optional[float]


@dataclass
class Seq2SeqGeneratorOutput:
    hypotheses: List[List[Hypothesis]]


def select_candidates(total: Tensor, tok: Tensor, vocab: int, k: int):
    """total fp32 [N, B, C] candidate scores, tok int64 [N, B, C] -> the k best per sentence as
    (score [N,k], beam [N,k], token [N,k]) ordered by (score desc, beam*vocab+token asc)."""
    n, b, c = total.shape
    flat = total.reshape(n, b * c)
    beam_id = torch.arange(b, device=total.device)[None, :, None].expand(n, b, c).reshape(n, b * c)
    ftok = tok.reshape(n, b * c)
    key2 = beam_id * vocab + ftok
    o1 = torch.argsort(key2, dim=1, stable=True)
    o2 = torch.argsort(torch.gather(flat, 1, o1), dim=1, descending=True, stable=True)[:, :k]
    sel = torch.gather(o1, 1, o2)
    return torch.gather(flat, 1, sel), torch.gather(beam_id, 1, sel), torch.gather(ftok, 1, sel)


class _DecodeState:
    """Persistent device tensors of one beam search (shapes fixed by N, beam, Tmax): every step updates them IN PLACE so that
    a step can be captured once as a CUDA graph and replayed."""

    def __init__(self, N: int, B: int, Tmax: int, dev: torch.device):
        R, CAP = N * B, 2 * B
        self.N, self.B, self.Tmax, self.CAP = N, B, Tmax, CAP
        self.seqs = torch.empty((N, B, Tmax), dtype=torch.int64, device=dev)
        self.table = torch.empty((R, Tmax), dtype=torch.int32, device=dev)
        self.tokens = torch.empty((R,), dtype=torch.int64, device=dev)
        self.cum = torch.empty((N, B), dtype=torch.float32, device=dev)
        self.alive = torch.empty((N, B), dtype=torch.bool, device=dev)
        self.done = torch.empty((N,), dtype=torch.bool, device=dev)
        self.fin_score = torch.empty((N, CAP + 1), dtype=torch.float32, device=dev)
        self.fin_seq = torch.empty((N, CAP + 1, Tmax), dtype=torch.int64, device=dev)
        self.fin_len = torch.empty((N, CAP + 1), dtype=torch.int64, device=dev)
        self.fin_count = torch.empty((N,), dtype=torch.int64, device=dev)
        self.ar_n = torch.arange(N, device=dev)
        self.rank = torch.arange(2 * B, device=dev)[None, :]
        self.row_ids = torch.arange(R, device=dev, dtype=torch.int32)[:, None]

    def reset(self, prompt: Tensor, pad: int) -> None:
        P = prompt.shape[1]
        self.seqs.fill_(pad)
        self.seqs[:, :, :P] = prompt[:, None, :]
        self.table.copy_(self.row_ids.expand_as(self.table))
        self.cum.zero_()
        self.alive.fill_(True)
        self.done.fill_(False)
        self.fin_score.fill_(NEG_INF)
        self.fin_seq.fill_(pad)
        self.fin_len.zero_()
        self.fin_count.zero_()


class _GraphEntry:
    """CUDA graphs of the decode steps of one (shape, search-parameter) configuration; they bake the addresses of the state
    tensors and of the decoder workspace."""

    def __init__(self, state: _DecodeState, ws_ptr: int):
        self.state = state
        self.ws_ptr = ws_ptr
        self.graphs = {}
        self.pool = torch.cuda.graph_pool_handle()
        self.stream = torch.cuda.Stream(device=state.seqs.device)


_MAX_GRAPH_ENTRIES = 8


class BeamSearchSeq2SeqGenerator:
    def __init__(self, model: B200TextDecoderModel, *, beam_size: int = 5, min_gen_len: int = 1,
                 max_gen_len: Tuple[int, int] = (1, 128), max_seq_len: Optional[int] = None, echo_prompt: bool = False,
                 normalize_scores: bool = True, temperature: float = 1.0, unk_penalty: float = 0.0,
                 len_penalty: float = 1.0, pad_idx: int = 0, sync_every: int = 8,
                 cuda_graphs: Optional[bool] = None, fused_beam_step: Optional[bool] = None) -> None:
        """``cuda_graphs``: replay each decode step (the ~290 engine launches + the beam bookkeeping) as one CUDA graph.
        A small batch -- the pipelines' default ``batch_size=5`` is 25 hypotheses -- is launch-bound otherwise.  ``None``
        (default) turns it on for up to 512 hypothesis rows unless ``SONAR_B200_DECODE_GRAPHS=0``; graphs are captured the
        first time a (batch shape, step) is seen and cached on the model, so only repeated shapes benefit.
        ``fused_beam_step``: run the bookkeeping of a step as the single ``sb_beam_step`` kernel instead of the ~60 torch
        ops below (same state transition bit for bit; the torch ops remain the definition the CPU tests check against the
        oracle).  ``None`` = on for CUDA models unless ``SONAR_B200_FUSED_BEAM=0``."""
        if beam_size < 1:
            raise ValueError("`beam_size` must be greater than or equal to 1")
        # the decoder step returns the TOPK best tokens per row BEFORE the generator masks PAD, masks EOS (min length) and
        # demotes UNK: the exact 2*beam best of the constrained distribution lie inside the raw top 2*beam + (#tokens touched)
        need = 2 * beam_size + 2 + (1 if unk_penalty != 0.0 else 0)
        if need > TOPK:
            raise ValueError(f"`beam_size` must be <= {(TOPK - 2 - (1 if unk_penalty != 0.0 else 0)) // 2} "
                             f"(the decoder step returns the top-{TOPK} tokens per row; 2*beam_size + {need - 2 * beam_size} "
                             f"of them are needed{' with an UNK penalty' if unk_penalty != 0.0 else ''})")
        if min_gen_len < 1:
            raise ValueError("`min_gen_len` must be greater than or equal to 1")
        if temperature != 1.0:
            raise NotImplementedError("temperature != 1.0")
        self.model = model
        self.beam_size = beam_size
        self.min_gen_len = min_gen_len
        self.max_gen_len = max_gen_len
        self.max_seq_len = max_seq_len
        self.echo_prompt = echo_prompt
        self.normalize_scores = normalize_scores
        self.unk_penalty = unk_penalty
        self.len_penalty = len_penalty
        self.pad_idx = pad_idx
        self.sync_every = sync_every
        self.cuda_graphs = cuda_graphs
        self.fused_beam_step = fused_beam_step

    def _advance(self, st: _DecodeState, g: int, P: int, min_gen: int, max_gen: int) -> None:
        """One decode step: position t = P-1+g of every live hypothesis -> the next beam, all state updated in place.
        fairseq2 names [fs2]: ``step_nr = P + g`` is the absolute index of the token being generated; EOS is forbidden while
        ``step_nr < min_seq_len - 1`` (``min_seq_len = P + min_gen``), forced when ``step_nr == max_seq_len - 1``; a finished
        hypothesis scores ``cum / step_nr ** len_penalty`` (``seq_len - 1``: prompt and EOS counted, first step excluded)."""
        m = self.model
        vi = m.target_vocab_info
        eos, unk, pad, V = vi.eos_idx, vi.unk_idx, self.pad_idx, vi.size
        N, B, Tmax, CAP = st.N, st.B, st.Tmax, st.CAP
        R = N * B
        dev = st.seqs.device
        t = P - 1 + g  # position of the input token; the new token lands at t + 1
        lp, tok, eos_lp = m.step(st.tokens, st.table, t)
        fused = self.fused_beam_step
        if fused is None:
            fused = os.environ.get("SONAR_B200_FUSED_BEAM", "1") != "0"
        if fused and dev.type == "cuda" and B <= 7 and TOPK == 16:
            div = float(P + g) ** self.len_penalty
            with torch.cuda.device(dev):
                rc = m._lib.sb_beam_step(
                    lp.data_ptr(), tok.data_ptr(), eos_lp.data_ptr(), st.seqs.data_ptr(), st.table.data_ptr(),
                    st.tokens.data_ptr(), st.cum.data_ptr(), st.alive.data_ptr(), st.done.data_ptr(),
                    st.fin_score.data_ptr(), st.fin_seq.data_ptr(), st.fin_len.data_ptr(), st.fin_count.data_ptr(),
                    N, B, Tmax, t, g, min_gen - 1, max_gen, V, eos, unk, pad, float(self.unk_penalty), div,
                    1 if self.normalize_scores else 0, torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(rc, "sb_beam_step")
            return
        lp = lp.view(N, B, TOPK)
        tok = tok.view(N, B, TOPK).long()
        lp = lp.masked_fill((tok < 0) | (tok == pad), NEG_INF)
        if self.unk_penalty:
            lp = torch.where(tok == unk, lp - self.unk_penalty, lp)
        if g < min_gen - 1:
            lp = lp.masked_fill(tok == eos, NEG_INF)
        if g >= max_gen - 1:  # the last allowed token must be EOS
            lp = torch.full_like(lp, NEG_INF)
            lp[:, :, 0] = eos_lp.view(N, B)
            tok = tok.clone()
            tok[:, :, 0] = eos
        total = (st.cum[:, :, None] + lp).masked_fill(~st.alive[:, :, None], NEG_INF)
        if g == 0:
            total[:, 1:, :] = NEG_INF  # all beams are copies of the prompt
        c_score, c_beam, c_tok = select_candidates(total, tok, V, 2 * B)

        valid = c_score > NEG_INF
        is_eos = (c_tok == eos) & valid
        # ---- finalise EOS candidates ranked inside the beam ----
        fin_mask = is_eos & (st.rank < B) & ~st.done[:, None]
        fin_pos = st.fin_count[:, None] + torch.cumsum(fin_mask, 1) - 1
        fin_ok = fin_mask & (fin_pos < B)  # the sentence closes the moment it owns `beam` hypotheses
        dest = torch.where(fin_ok, fin_pos, torch.full_like(fin_pos, CAP))
        # divisor as a 0-dim tensor: IEEE division on every device (a Python-scalar divisor becomes a multiplication by the
        # reciprocal in torch's CUDA kernel, one ulp away from the CPU result and from sb_beam_step)
        fscore = c_score / torch.full((), float(P + g) ** self.len_penalty, dtype=torch.float32, device=dev) \
            if self.normalize_scores else c_score
        st.fin_score.scatter_(1, dest, torch.where(fin_ok, fscore, torch.full_like(fscore, NEG_INF)))
        cand_seqs = torch.gather(st.seqs, 1, c_beam[:, :, None].expand(N, 2 * B, Tmax)).clone()
        cand_seqs[:, :, t + 1] = c_tok
        st.fin_seq.scatter_(1, dest[:, :, None].expand(N, 2 * B, Tmax), cand_seqs)
        st.fin_len.scatter_(1, dest, torch.full_like(dest, t + 2))
        st.fin_score[:, CAP] = NEG_INF
        st.fin_count.add_(fin_mask.sum(1))
        # ---- next beam: the first B non-EOS candidates ----
        keep = valid & ~is_eos & ~st.done[:, None]
        kpos = torch.cumsum(keep, 1) - 1
        keep_ok = keep & (kpos < B)
        kdest = torch.where(keep_ok, kpos, torch.full_like(kpos, B))
        new_cum = torch.full((N, B + 1), NEG_INF, dtype=torch.float32, device=dev).scatter_(
            1, kdest, torch.where(keep_ok, c_score, torch.full_like(c_score, NEG_INF)))[:, :B]
        new_alive = torch.zeros((N, B + 1), dtype=torch.bool, device=dev).scatter_(1, kdest, keep_ok)[:, :B]
        new_src = torch.zeros((N, B + 1), dtype=torch.int64, device=dev).scatter_(1, kdest, c_beam)[:, :B]
        new_tok = torch.full((N, B + 1), pad, dtype=torch.int64, device=dev).scatter_(1, kdest, c_tok)[:, :B]
        new_src = torch.where(new_alive, new_src, torch.zeros_like(new_src))
        new_tok = torch.where(new_alive, new_tok, torch.full_like(new_tok, pad))
        st.done.logical_or_(st.fin_count >= B)
        new_alive = new_alive & ~st.done[:, None]
        new_seqs = torch.gather(st.seqs, 1, new_src[:, :, None].expand(N, B, Tmax))
        st.seqs.copy_(new_seqs)
        st.seqs[:, :, t + 1] = new_tok
        src_row = (st.ar_n[:, None] * B + new_src).reshape(R)
        new_table = st.table.index_select(0, src_row)
        st.table.copy_(new_table)
        st.table[:, t] = src_row.to(torch.int32)
        st.cum.copy_(new_cum)
        st.alive.copy_(new_alive)
        st.tokens.copy_(new_tok.reshape(R))

    def _graph_entry(self, key, N: int, B: int, Tmax: int) -> _GraphEntry:
        m = self.model
        cache = m.__dict__.setdefault("_decode_graph_cache", {})
        ws_ptr = m._workspace.data_ptr()
        ent = cache.get(key)
        if ent is not None and ent.ws_ptr != ws_ptr:  # the workspace moved: the captured addresses are stale
            del cache[key]
            ent = None
        if ent is None:
            while len(cache) >= _MAX_GRAPH_ENTRIES:
                cache.pop(next(iter(cache)))
            ent = _GraphEntry(_DecodeState(N, B, Tmax, m.device), ws_ptr)
            cache[key] = ent
        else:  # most recently used last
            cache[key] = cache.pop(key)
        return ent

    @torch.inference_mode()
    def __call__(self, source_seqs: Tensor, source_padding_mask, prompt_seqs: Tensor, prompt_padding_mask=None
                 ) -> Seq2SeqGeneratorOutput:
        m = self.model
        dev = m.device
        if source_seqs.dim() == 2:
            source_seqs = source_seqs[:, None, :]  # DummyEncoderModel + encode(): [N,1,D] (model.py:48-53)
        N = source_seqs.shape[0]
        B = self.beam_size
        R = N * B
        prompt = prompt_seqs.to(dev).long()
        if prompt.dim() == 1:
            prompt = prompt[None].expand(N, -1)
        P = prompt.shape[1]
        model_max = m.max_target_seq_len
        max_total = min(self.max_seq_len or model_max, model_max)
        src_len = source_seqs.shape[1]
        max_gen = min(int(self.max_gen_len[0] * src_len + self.max_gen_len[1]), max_total - P)
        if max_gen < 1:
            raise ValueError("`max_seq_len` leaves no room to generate after the prompt")
        min_gen = min(self.min_gen_len, max_gen)
        Tmax = P + max_gen
        m.begin(source_seqs[:, 0], B, Tmax)

        use_graphs = self.cuda_graphs
        if use_graphs is None:
            use_graphs = R <= 512 and os.environ.get("SONAR_B200_DECODE_GRAPHS", "1") != "0"
        use_graphs = bool(use_graphs) and torch.device(dev).type == "cuda"  # (CPU only in the host-logic tests)
        ent = None
        if use_graphs:
            key = (N, B, Tmax, P, min_gen, max_gen, self.unk_penalty, self.len_penalty, self.normalize_scores, self.pad_idx)
            ent = self._graph_entry(key, N, B, Tmax)
            st = ent.state
        else:
            st = _DecodeState(N, B, Tmax, dev)
        st.reset(prompt, self.pad_idx)

        # prefill [fs2 `_prefill`]: every prompt position but the last feeds the KV cache, and the log-prob of the NEXT prompt
        # token given the prefix seeds the hypothesis scores (a per-sentence constant that still matters once scores of
        # different lengths are normalised)
        for p in range(P - 1):
            probe = st.seqs[:, :, p + 1].reshape(R).contiguous()
            out = m.step(st.seqs[:, :, p].reshape(R).contiguous(), st.table, p, probe)
            st.cum.add_(out[3].view(N, B))
        st.tokens.copy_(st.seqs[:, :, P - 1].reshape(R))
        for g in range(max_gen):
            if ent is None:
                self._advance(st, g, P, min_gen, max_gen)
            else:
                graph = ent.graphs.get(g)
                if graph is None:  # record this step once (recording does not execute it), then replay
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, pool=ent.pool, stream=ent.stream):
                        self._advance(st, g, P, min_gen, max_gen)
                    ent.graphs[g] = graph
                graph.replay()
            if (g + 1) % self.sync_every == 0 and bool(st.done.all()):
                break

        m.check_inputs()
        CAP = st.CAP
        fin_score, fin_len, fin_seq = st.fin_score, st.fin_len, st.fin_seq
        # ---- best-first hypotheses (score desc, earlier-finished first on ties) ----
        order = torch.argsort(fin_score[:, :CAP], dim=1, descending=True, stable=True)[:, :B]
        s_sorted = torch.gather(fin_score[:, :CAP], 1, order).cpu()
        l_sorted = torch.gather(fin_len[:, :CAP], 1, order).cpu()
        q_sorted = torch.gather(fin_seq[:, :CAP], 1, order[:, :, None].expand(N, B, Tmax)).cpu()
        out: List[List[Hypothesis]] = []
        start = 0 if self.echo_prompt else P
        for i in range(N):
            hyps = []
            for j in range(B):
                sc = float(s_sorted[i, j])
                if sc == NEG_INF:
                    continue
                hyps.append(Hypothesis(seq=q_sorted[i, j, start : int(l_sorted[i, j])].clone(), score=sc))
            out.append(hyps)
        return Seq2SeqGeneratorOutput(out)


class SequenceToTextConverter:
    """fairseq2 ``SequenceToTextConverter`` [fs2] as used at ``text.py:322-333``: prompt = the tokenizer's target-mode
    prefix (``[</s>, __lang__]``), output = decoded best hypothesis per input."""

    def __init__(self, generator: BeamSearchSeq2SeqGenerator, tokenizer, task: str, target_lang: Optional[str] = None):
        self.generator = generator
        enc = tokenizer.create_encoder(task=task, lang=target_lang, mode="target", device=generator.model.device)
        prefix = getattr(enc, "prefix_indices", None)
        if prefix is None:
            raise ValueError("the tokenizer's target-mode encoder must expose `prefix_indices`")
        self.prompt = prefix.to(torch.int64)
        self.text_decoder = tokenizer.create_decoder()

    def batch_convert(self, source_seqs: Tensor, source_padding_mask=None):
        out = self.generator(source_seqs, source_padding_mask, self.prompt, None)
        texts = []
        for i, hyps in enumerate(out.hypotheses):
            if not hyps:
                raise RuntimeError(f"the generator returned no hypothesis at index {i}")
            texts.append(self.text_decoder(hyps[0].seq))
        return texts, out
