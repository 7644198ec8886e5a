"""CUDA decoder (sb_decoder_begin / sb_decoder_step through B200TextDecoderModel) against the fp32 CPU oracle
(oracle/text_decoder.py) on shared seeded synthetic weights -- BASELINE.json config 4 at sizes the oracle finishes
in seconds.  bf16 operands vs the fp32 oracle: log-probabilities agree to 2e-2 + 2e-3*|lprob| (bf16 operand rounding is
2^-9 relative on logits of magnitude ~10 with the peaky test weights; stated per check); the beam-search BOOKKEEPING is held to exact equality in tests/test_oracle_decoder.py (CPU)."""

import math

import pytest
import torch

from oracle.text_decoder import (BeamSearchConfig, OracleDecoderConfig, OracleTextDecoder, beam_search,
                                 make_synthetic_decoder_state_dict)

pytestmark = pytest.mark.gpu

VOCAB = 4096


@pytest.fixture(scope="module")
def small(native_lib, cuda_device):
    from sonar_b200 import B200TextDecoderModel, VocabularyInfo, sonar_text_decoder_config

    ocfg = OracleDecoderConfig(vocab_size=VOCAB, num_layers=2, max_seq_len=64)
    sd = make_synthetic_decoder_state_dict(ocfg, seed=2)
    sd["decoder_frontend.embed.weight"] *= 3.0  # peakier next-token distributions
    sd["final_proj.weight"] = sd["decoder_frontend.embed.weight"]
    cfg = sonar_text_decoder_config("basic", num_decoder_layers=2, max_seq_len=64,
                                    vocab_info=VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    return OracleTextDecoder(ocfg, sd), B200TextDecoderModel(cfg, sd, cuda_device)


def _emb(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n, 1024), generator=g) * 0.25 / math.sqrt(1024) * 32.0


@pytest.mark.parametrize("n,beam,steps", [(3, 2, 9), (26, 3, 5)])
def test_teacher_forced_steps_match_oracle(small, cuda_device, n, beam, steps):
    """6 hypothesis rows take the weight-streaming skinny GEMMs, 78 rows the wgmma tiles; both run the separate LayerNorm
    and add + LayerNorm kernels (the decoder folds no LayerNorm into a GEMM)."""
    oracle, model = small
    emb = _emb(n)
    g = torch.Generator().manual_seed(1)
    toks = torch.randint(4, VOCAB, (n * beam, steps), generator=g)
    model.begin(emb.to(cuda_device), beam, 16)
    r = n * beam
    table = torch.arange(r, dtype=torch.int32, device=cuda_device)[:, None].expand(r, 16).contiguous()
    enc_rows = emb[:, None, :].repeat_interleave(beam, 0)
    for t in range(steps):
        probe = toks[:, (t + 1) % steps].contiguous()  # log P of an arbitrary token per row (the generator's prompt scores)
        lp, tok, eos_lp, probe_lp = model.step(toks[:, t].contiguous().to(cuda_device), table, t, probe.to(cuda_device))
        ref = oracle.step_lprobs(toks[:, : t + 1], enc_rows)  # [R, V] fp32
        lp, tok, eos_lp = lp.cpu(), tok.cpu().long(), eos_lp.cpu()
        torch.testing.assert_close(probe_lp.cpu(), torch.gather(ref, 1, probe[:, None])[:, 0], rtol=2e-3, atol=2e-2)
        # the returned candidates carry the right log-probs ...
        torch.testing.assert_close(lp, torch.gather(ref, 1, tok), rtol=2e-3, atol=2e-2)
        torch.testing.assert_close(eos_lp, ref[:, 3], rtol=2e-3, atol=2e-2)
        # ... are sorted, normalised over the WHOLE vocabulary, and contain the oracle's arg-max
        assert bool((lp[:, :-1] >= lp[:, 1:]).all())
        assert bool((tok == ref.argmax(1, keepdim=True)).any(1).all())
        # the 16th-best oracle value bounds what may be missing from the candidate list
        kth = ref.topk(16, dim=1).values[:, -1:]
        assert bool((lp[:, -1:] >= kth - 0.25).all())


def test_out_of_range_token_is_reported(small, cuda_device):
    """A token id outside the vocabulary fed to one step makes check_inputs raise once: the check clears the flag.  Until
    then the flag survives the steps and a begin that follow."""
    _, model = small
    n, beam, max_len = 2, 2, 8
    r = n * beam
    emb = _emb(n, seed=3).to(cuda_device)
    table = torch.arange(r, dtype=torch.int32, device=cuda_device)[:, None].expand(r, max_len).contiguous()
    good = torch.full((r,), 5, dtype=torch.int64, device=cuda_device)
    bad = good.clone()
    bad[1] = VOCAB
    model.begin(emb, beam, max_len)
    model.check_inputs()  # no earlier test fed an out-of-range token
    model.step(bad, table, 0)
    model.step(good, table, 1)
    with pytest.raises(ValueError, match="vocab"):
        model.check_inputs()
    model.check_inputs()
    model.step(bad, table, 2)
    model.begin(emb, beam, max_len)
    model.step(good, table, 0)
    with pytest.raises(ValueError, match="vocab"):
        model.check_inputs()
    model.check_inputs()


def test_beam_reordering_through_the_ancestry_table(small, cuda_device):
    """Hypothesis r continues from a DIFFERENT physical row: results must equal decoding that token history directly."""
    oracle, model = small
    n, beam = 2, 3
    r = n * beam
    emb = _emb(n, seed=4)
    g = torch.Generator().manual_seed(2)
    hist = torch.randint(4, VOCAB, (r, 3), generator=g)
    model.begin(emb.to(cuda_device), beam, 8)
    table = torch.arange(r, dtype=torch.int32, device=cuda_device)[:, None].expand(r, 8).contiguous()
    for t in range(2):
        model.step(hist[:, t].contiguous().to(cuda_device), table, t)
    src = torch.tensor([1, 1, 0, 5, 3, 3])  # new row r descends from old row src[r] (within its sentence)
    table2 = table.index_select(0, src.to(cuda_device)).contiguous()
    table2[:, 1] = src.to(cuda_device).to(torch.int32)
    table2[:, 0] = src.to(cuda_device).to(torch.int32)
    new_tok = hist[:, 2]
    lp, tok, _ = model.step(new_tok.contiguous().to(cuda_device), table2, 2)
    seqs = torch.cat([hist[src, :2], new_tok[:, None]], 1)
    ref = oracle.step_lprobs(seqs, emb[:, None, :].repeat_interleave(beam, 0))
    torch.testing.assert_close(lp.cpu(), torch.gather(ref, 1, tok.cpu().long()), rtol=2e-3, atol=2e-2)


def test_reordering_at_every_step_to_position_60(small, cuda_device):
    """Teacher-forced steps to position 60 (four 16-key passes of the cached attention) with a new random within-sentence
    reordering of the ancestry table before every step, as beam search makes them: each hypothesis's results equal the
    oracle's on its own gathered token history."""
    oracle, model = small
    n, beam, steps = 2, 3, 61
    r = n * beam
    emb = _emb(n, seed=12)
    g = torch.Generator().manual_seed(13)
    model.begin(emb.to(cuda_device), beam, steps)
    table = torch.arange(r, dtype=torch.int32)[:, None].expand(r, steps).contiguous()
    hist = torch.zeros((r, 0), dtype=torch.int64)
    enc_rows = emb[:, None, :].repeat_interleave(beam, 0)
    sentence = torch.arange(r) // beam
    for t in range(steps):
        if t > 0:  # new hypothesis j continues old hypothesis src[j] of the same sentence
            src = sentence * beam + torch.randint(0, beam, (r,), generator=g)
            table = table[src].contiguous()
            table[:, t - 1] = src.to(torch.int32)  # src's position t - 1 was written to its own cache row
            hist = hist[src]
        tok_in = torch.randint(4, VOCAB, (r,), generator=g)
        probe = torch.randint(4, VOCAB, (r,), generator=g)
        hist = torch.cat([hist, tok_in[:, None]], 1)
        lp, tok, eos_lp, probe_lp = model.step(tok_in.to(cuda_device), table.to(cuda_device), t, probe.to(cuda_device))
        ref = oracle.step_lprobs(hist, enc_rows)
        lp, tok = lp.cpu(), tok.cpu().long()
        torch.testing.assert_close(lp, torch.gather(ref, 1, tok), rtol=2e-3, atol=2e-2)
        torch.testing.assert_close(eos_lp.cpu(), ref[:, 3], rtol=2e-3, atol=2e-2)
        torch.testing.assert_close(probe_lp.cpu(), torch.gather(ref, 1, probe[:, None])[:, 0], rtol=2e-3, atol=2e-2)
        assert bool((tok == ref.argmax(1, keepdim=True)).any(1).all()), t


def test_generation_is_near_optimal_and_scores_are_honest(small, cuda_device):
    from sonar_b200.generation import BeamSearchSeq2SeqGenerator

    oracle, model = small
    n, beam, max_gen = 6, 4, 8
    emb = _emb(n, seed=7)
    prompt = torch.tensor([3, 4000])
    gen = BeamSearchSeq2SeqGenerator(model, beam_size=beam, max_gen_len=(0, max_gen), pad_idx=0)
    out = gen(emb.to(cuda_device), None, prompt, None)
    enc1 = emb[:, None, :]
    ref = beam_search(lambda toks: oracle.step_lprobs(toks, enc1.repeat_interleave(beam, 0)), prompt, n,
                      BeamSearchConfig(beam_size=beam, max_gen_len=max_gen, pad_idx=0))
    exact = 0
    for i in range(n):
        hyps = out.hypotheses[i]
        assert len(hyps) >= 1 and int(hyps[0].seq[-1]) == 3  # ends with EOS
        for h in hyps:  # reported score == oracle score of that very sequence (teacher forced), within bf16 tolerance
            seq = torch.cat([prompt, h.seq])
            lps = torch.log_softmax(oracle.logits(seq[None, :-1], enc1[i : i + 1])[0].float(), -1)
            # fairseq2 scoring: prompt log-prob included, normalised by seq_len - 1 (prompt and EOS counted)
            s = sum(float(lps[p, seq[p + 1]]) for p in range(len(seq) - 1)) / (len(seq) - 1)
            assert abs(s - h.score) <= 2e-2 + 2e-3 * abs(s), (i, s, h.score)
        assert hyps[0].score >= ref[i][0][0] - (5e-2 + 4e-3 * abs(ref[i][0][0]))  # as good as the oracle's best hypothesis
        exact += int(hyps[0].seq.tolist() == ref[i][0][1])
    print("best-hypothesis exact matches vs fp32 oracle:", exact, "/", n)


def test_embedding_to_text_pipeline(small, cuda_device):
    from sonar_b200.inference_pipelines import EmbeddingToTextModelPipeline
    from sonar_b200.tokenizer import SyntheticTokenizer

    _, model = small
    pipe = EmbeddingToTextModelPipeline(model, SyntheticTokenizer(vocab_size=VOCAB), device=cuda_device)
    emb = _emb(7, seed=9)
    texts = pipe.predict(emb, target_lang="fra_Latn", batch_size=3, max_seq_len=12)
    assert len(texts) == 7 and all(isinstance(t, str) for t in texts)
    again = pipe.predict(emb, target_lang="fra_Latn", batch_size=7, max_seq_len=12)
    assert texts == again  # batch composition does not change the result
    with pytest.raises(ValueError):
        pipe.predict(emb, target_lang="fra_Latn", max_seq_len=2)  # no room after the 2-token prompt


def test_sampling_generator_on_the_cuda_decoder(small, cuda_device):
    """`predict(sampler=...)` (text.py:313-316): top-1 sampling is greedy search (= beam search with one beam); a seeded
    generator reproduces its draws; the sampled tokens' scores are the oracle's log-probs of those very tokens; a nucleus
    that needs more than the 16 returned candidates is refused."""
    from oracle.text_decoder import OracleTextDecoder  # noqa: F401  (fixture type)
    from sonar_b200.generation import BeamSearchSeq2SeqGenerator
    from sonar_b200.inference_pipelines import EmbeddingToTextModelPipeline
    from sonar_b200.sampling import SamplingSeq2SeqGenerator, TopKSampler, TopPSampler
    from sonar_b200.tokenizer import SyntheticTokenizer

    oracle, model = small
    emb = _emb(6, seed=4).to(cuda_device)
    prompt = torch.tensor([3, 77])
    greedy = BeamSearchSeq2SeqGenerator(model, beam_size=1, max_gen_len=(0, 12), pad_idx=0)(emb, None, prompt, None)
    top1 = SamplingSeq2SeqGenerator(model, TopKSampler(1), max_gen_len=(0, 12), pad_idx=0)(emb, None, prompt, None)
    for a, b in zip(greedy.hypotheses, top1.hypotheses):
        assert a[0].seq.tolist() == b[0].seq.tolist()

    # a random decoder with tied embeddings predicts its own input token with probability ~1 (the residual stream carries
    # that token's embedding straight into the output projection): shrink the embeddings so that 8 candidates leave something
    # to draw
    from sonar_b200 import B200TextDecoderModel, VocabularyInfo, sonar_text_decoder_config
    ocfg = OracleDecoderConfig(vocab_size=VOCAB, num_layers=2, max_seq_len=64)
    sd = make_synthetic_decoder_state_dict(ocfg, seed=3)
    sd["decoder_frontend.embed.weight"] *= 0.15
    sd["final_proj.weight"] = sd["decoder_frontend.embed.weight"]
    oracle = OracleTextDecoder(ocfg, sd)
    model = B200TextDecoderModel(sonar_text_decoder_config(
        "basic", num_decoder_layers=2, max_seq_len=64,
        vocab_info=VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1)), sd, cuda_device)

    def run(seed):
        gen = SamplingSeq2SeqGenerator(model, TopKSampler(8), num_gens=3, max_gen_len=(0, 10), compute_scores=True,
                                       normalize_scores=False, pad_idx=0,
                                       generator=torch.Generator(device=cuda_device).manual_seed(seed))
        return gen(emb, None, prompt, None)

    o1, o2, o3 = run(5), run(5), run(6)
    seqs = lambda o: [[h.seq.tolist() for h in hs] for hs in o.hypotheses]  # noqa: E731
    assert seqs(o1) == seqs(o2) and seqs(o1) != seqs(o3)
    assert all(len(hs) == 3 and hs[0].score >= hs[1].score >= hs[2].score for hs in o1.hypotheses)
    # raw score = sum of the fp32-oracle log-probs of the sampled tokens (teacher-forced), to the step's tolerance
    for i, hs in enumerate(o1.hypotheses):
        for h in hs:
            toks = torch.cat([prompt, h.seq])[None]
            want = 0.0
            for t in range(len(h.seq)):
                lp = oracle.step_lprobs(toks[:, : 2 + t], emb[i].cpu()[None, None, :])
                want += float(lp[0, int(h.seq[t])])
            assert abs(h.score - want) <= 2e-2 * len(h.seq) + 2e-3 * abs(want), (i, h.score, want)
    pipe = EmbeddingToTextModelPipeline(model, SyntheticTokenizer(vocab_size=VOCAB), device=cuda_device)
    texts = pipe.predict(emb, target_lang="fra_Latn", batch_size=4, sampler=TopKSampler(4), max_seq_len=12,
                         generator=torch.Generator(device=cuda_device).manual_seed(1))
    assert len(texts) == 6 and all(isinstance(t, str) for t in texts)
    with pytest.raises(ValueError, match="nucleus"):  # 4096 near-uniform tokens: 0.999 of the mass is not in 16 of them
        pipe.predict(emb, target_lang="fra_Latn", sampler=TopPSampler(0.999), max_seq_len=12)


def test_cuda_graph_replay_equals_eager_generation(small, cuda_device):
    """The per-step CUDA graphs (engine launches + beam bookkeeping, captured once per step index) reproduce the eager
    search token for token, also when the cached graphs are replayed for a second batch of the same shape."""
    from sonar_b200.generation import BeamSearchSeq2SeqGenerator

    _, model = small
    prompt = torch.tensor([2, 7])
    kw = dict(beam_size=3, max_seq_len=14, pad_idx=1)
    before = set(model.__dict__.get("_decode_graph_cache", {}))  # earlier tests of this module may have recorded graphs
    eager = BeamSearchSeq2SeqGenerator(model, cuda_graphs=False, **kw)
    graphed = BeamSearchSeq2SeqGenerator(model, cuda_graphs=True, **kw)
    for seed in (21, 22):  # second round replays the graphs recorded in the first
        emb = _emb(4, seed=seed).to(cuda_device)
        a = eager(emb, None, prompt, None)
        b = graphed(emb, None, prompt, None)
        assert len(a.hypotheses) == len(b.hypotheses) == 4
        for ha, hb in zip(a.hypotheses, b.hypotheses):
            assert len(ha) == len(hb)
            for x, y in zip(ha, hb):
                assert torch.equal(x.seq, y.seq) and x.score == y.score
    cache = model.__dict__["_decode_graph_cache"]
    mine = [k for k in cache if k not in before]
    assert len(mine) == 1 and len(cache[mine[0]].graphs) >= 1
    # a different batch size is a different graph set; the first one stays valid
    graphed(_emb(2, seed=5).to(cuda_device), None, prompt, None)
    assert len([k for k in cache if k not in before]) == 2 and mine[0] in cache
    c = graphed(_emb(4, seed=22).to(cuda_device), None, prompt, None)
    for ha, hc in zip(a.hypotheses, c.hypotheses):
        for x, y in zip(ha, hc):
            assert torch.equal(x.seq, y.seq) and x.score == y.score


@pytest.mark.parametrize("kw", [
    dict(beam_size=5, max_seq_len=20),
    dict(beam_size=3, max_seq_len=9, min_gen_len=3),
    dict(beam_size=1, max_seq_len=12),
    dict(beam_size=4, max_seq_len=16, unk_penalty=0.7, len_penalty=0.6),
    dict(beam_size=7, max_seq_len=10, normalize_scores=False),
])
def test_fused_beam_step_equals_the_torch_bookkeeping(native_lib, cuda_device, kw):
    """`sb_beam_step` (one launch per step) must make exactly the state transition of the vectorised torch ops in
    `generation.py::_advance` -- the version the CPU tests hold to the oracle.  A decoder whose EOS embedding is inflated
    finishes hypotheses at every step, so finalisation, the 2*beam cap, `done` and the forced EOS at the length limit are
    all exercised; hypotheses (tokens and scores) and the whole search state are compared bit for bit."""
    from sonar_b200 import B200TextDecoderModel, VocabularyInfo, sonar_text_decoder_config
    from sonar_b200 import generation as G

    ocfg = OracleDecoderConfig(vocab_size=VOCAB, num_layers=2, max_seq_len=64)
    sd = make_synthetic_decoder_state_dict(ocfg, seed=7)
    sd["decoder_frontend.embed.weight"] *= 3.0
    sd["decoder_frontend.embed.weight"][3] *= 2.5  # EOS (idx 3) competes at every step
    sd["decoder_frontend.embed.weight"][1] *= 2.0  # and so does UNK / PAD (idx 1): penalties and pad masking matter
    sd["final_proj.weight"] = sd["decoder_frontend.embed.weight"]
    cfg = sonar_text_decoder_config("basic", num_decoder_layers=2, max_seq_len=64,
                                    vocab_info=VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=0))
    model = B200TextDecoderModel(cfg, sd, cuda_device)
    prompt = torch.tensor([2, 9])
    emb = _emb(6, seed=31).to(cuda_device)
    states = {}
    orig_reset = G._DecodeState.reset

    outs = {}
    for fused in (False, True):
        gen = G.BeamSearchSeq2SeqGenerator(model, cuda_graphs=False, fused_beam_step=fused, pad_idx=0, **kw)
        captured = []

        def spy(self, prompt_, pad_, _c=captured):
            _c.append(self)
            return orig_reset(self, prompt_, pad_)

        G._DecodeState.reset = spy
        try:
            outs[fused] = gen(emb, None, prompt, None)
        finally:
            G._DecodeState.reset = orig_reset
        states[fused] = captured[0]
    a, b = outs[False], outs[True]
    n_finished = 0
    for ha, hb in zip(a.hypotheses, b.hypotheses):
        assert len(ha) == len(hb)
        n_finished += len(ha)
        for x, y in zip(ha, hb):
            assert torch.equal(x.seq, y.seq) and x.score == y.score
    assert n_finished > 0
    sa, sb_ = states[False], states[True]
    cap = sa.CAP
    for name in ("seqs", "table", "tokens", "cum", "alive", "done", "fin_count"):
        assert torch.equal(getattr(sa, name), getattr(sb_, name)), name
    assert torch.equal(sa.fin_score[:, :cap], sb_.fin_score[:, :cap])
    assert torch.equal(sa.fin_len[:, :cap], sb_.fin_len[:, :cap])
    assert torch.equal(sa.fin_seq[:, :cap], sb_.fin_seq[:, :cap])
