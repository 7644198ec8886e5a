"""CPU: the references of tests/test_gpu_decoder_kernels.py are the oracle's maths, and its tolerances can see the bugs
that matter in the decoder step's kernels."""

import math

import pytest
import torch

from oracle.text_decoder import OracleDecoderConfig, OracleTextDecoder, attention_core, make_synthetic_decoder_state_dict
from tests.decoder_kernel_cases import (BIG_VOCAB, EOS, HD, HEAD_EXACT_TOL, HEAD_REAL_TOL, LN_BEAMS, LN_DIMS, LN_ROWS, PASS,
                                        add_const_layernorm_reference, attention_reference, attn_violation, head_reference,
                                        ln_violation, make_attention_case, make_exact_head, make_ln_case, make_real_head,
                                        probe_tokens, tie_tokens, topk_lists, value_max)


# ---------------------------------------------------------------------------------------------------------------------
# KV-cache attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [0, 1, 16, 33])
def test_attention_reference_with_identity_table_is_causal_attention(t):
    """Identity table: hypothesis r's positions all live in row r; the last query row of the oracle's causal attention
    over the row's whole history is the reference."""
    case = make_attention_case(3, 4, t, table="identity", seed=t)
    d, n = case.dim, t + 1
    got = attention_reference(case)
    for r in range(3):
        qkv = case.qkv[r].double()
        k = torch.cat([case.kcache[r, :t].double(), qkv[None, d : 2 * d]])
        v = torch.cat([case.vcache[r, :t].double(), qkv[None, 2 * d :]])
        q = torch.cat([torch.randn((t, d), dtype=torch.float64), qkv[None, :d]])  # earlier queries do not matter
        causal = torch.full((n, n), -math.inf, dtype=torch.float64).triu(1)
        heads = lambda x: x.view(1, n, 4, HD).transpose(1, 2)  # noqa: E731
        want = attention_core(heads(q), heads(k), heads(v), causal)[0, -1]
        torch.testing.assert_close(got[r], want, rtol=1e-12, atol=1e-12)


def test_attention_reference_with_reordered_table_attends_over_the_gathered_history():
    """A table that points at other rows: the reference equals attention over the key / value history assembled row by
    row from the cache entries the table names."""
    t = 40
    case = make_attention_case(6, 8, t, seed=3)
    d = case.dim
    got = attention_reference(case)
    for r in range(6):
        hist_k = [case.kcache[int(case.table[r, p]), p] for p in range(t)] + [case.qkv[r, d : 2 * d]]
        hist_v = [case.vcache[int(case.table[r, p]), p] for p in range(t)] + [case.qkv[r, 2 * d :]]
        k = torch.stack(hist_k).double().view(1, t + 1, 8, HD).transpose(1, 2)
        v = torch.stack(hist_v).double().view(1, t + 1, 8, HD).transpose(1, 2)
        q = case.qkv[r, :d].double().view(1, 1, 8, HD).transpose(1, 2)
        assert bool(torch.isfinite(k).all())  # the NaN-poisoned cache holds values wherever the table points
        torch.testing.assert_close(got[r], attention_core(q, k, v, None)[0, 0], rtol=1e-12, atol=1e-12)


# (t, heads) on the inputs of the GPU test (R = 7, random table); every bug must miss the tolerance
ATTN_BUG_CASES = [(t, h) for t in (17, 33, 65, 129, 257, 511) for h in (4, 16)]


@pytest.mark.parametrize("t,heads", ATTN_BUG_CASES)
def test_attention_tolerance_catches_table_mask_and_pass_bugs(t, heads):
    case = make_attention_case(7, heads, t, seed=t * 31 + heads)
    ref = attention_reference(case)
    vmax = value_max(case)
    bugs = {"table shifted by one position": dict(table_shift=True), "last key dropped": dict(drop_last_key=True),
            "first 16-key pass dropped": dict(drop_pass=0), "last 16-key pass dropped": dict(drop_pass=t // PASS)}
    for bug, kw in bugs.items():
        v = attn_violation(attention_reference(case, **kw), ref, vmax)
        print(f"t={t} H={heads} {bug}: {v:.2f} x the tolerance")
        assert v > 2.0, (t, heads, bug, v)


# ---------------------------------------------------------------------------------------------------------------------
# vocabulary head
# ---------------------------------------------------------------------------------------------------------------------
def test_head_reference_is_log_softmax_of_the_oracle_logits():
    """On the oracle's own final states: the reference's values are log_softmax of OracleTextDecoder.logits at the returned
    tokens, the tokens are the 16 largest logits (value desc, token asc), EOS and probes are the same log_softmax."""
    v = 1000
    cfg = OracleDecoderConfig(model_dim=256, vocab_size=v, num_layers=1, num_heads=4, ffn_inner_dim=512, max_seq_len=16)
    sd = make_synthetic_decoder_state_dict(cfg, seed=5)
    oracle = OracleTextDecoder(cfg, sd, dtype=torch.float64)
    g = torch.Generator().manual_seed(0)
    toks = torch.randint(4, v, (5, 7), generator=g)
    enc = torch.randn((5, 1, 256), generator=g, dtype=torch.float64)
    hidden = oracle.hidden(toks, enc)[:, -1]
    want = torch.log_softmax(oracle.logits(toks, enc)[:, -1], -1)
    probes = probe_tokens(5, v)
    lp, tok, eos, probe = head_reference(hidden, oracle.sd["final_proj.weight"], EOS, probes)
    torch.testing.assert_close(lp, torch.gather(want, 1, tok), rtol=0, atol=1e-12)
    torch.testing.assert_close(eos, want[:, EOS], rtol=0, atol=1e-12)
    torch.testing.assert_close(probe, torch.gather(want, 1, probes.clamp(0, v - 1).masked_fill(probes >= v, 0)[:, None])[:, 0],
                               rtol=0, atol=1e-12)
    assert torch.equal(torch.sort(tok, 1).values, torch.sort(want.topk(16, 1).indices, 1).values)
    assert bool((lp[:, :-1] >= lp[:, 1:]).all())


def test_exact_head_operands_are_exact_in_fp32():
    """Every logit of the exact-operand inputs is the same number in fp32 and float64, so the top 16 and their order can be
    compared for equality; the tie row and the h = 0 row have the designed ties."""
    h, e, big = make_exact_head(5, 4196)
    l64 = h.double() @ e.double().T
    assert torch.equal(l64, (h.float() @ e.float().T).double())
    assert float(l64[0, -1]) == 2.0 and bool((l64[0, tie_tokens(4196)] == 1.0).all()) and len(tie_tokens(4196)) > 16
    assert bool((l64[1] == 0).all())
    assert float(l64[2, big]) - float(l64[2].index_fill(0, torch.tensor([big]), -1e9).max()) > 180
    lp, tok, _, _ = head_reference(h, e, EOS)
    assert tok[0].tolist() == [4195] + tie_tokens(4196)[:15] and tok[1].tolist() == list(range(16))
    assert abs(float(lp[1, 0]) + math.log(4196)) < 1e-12 and int(tok[2, 0]) == big and EOS not in tok[0].tolist()


@pytest.mark.parametrize("vocab,n_chunks", [(BIG_VOCAB, 63), (BIG_VOCAB, 2), (BIG_VOCAB, 1), (4196, 2), (32718, 128)])
def test_topk_lists_partition_the_vocabulary(vocab, n_chunks):
    lists = topk_lists(vocab, n_chunks)
    assert len(lists) == 2 * n_chunks
    assert torch.equal(torch.sort(torch.cat(lists)).values, torch.arange(vocab))


def test_head_tolerances_catch_merge_lse_and_tie_bugs():
    """On the exact-operand inputs of the GPU test at V = 256 206 (the step's split for 5 rows on 132 SMs: 63 chunks):
    the ragged tile's 206 columns left out of the log-sum-exp move every log-prob by more than the tolerance; a dropped
    candidate list, or ties broken by token descending, change the expected tokens."""
    h, e, _ = make_exact_head(5, BIG_VOCAB)
    ref = head_reference(h, e, EOS)
    last = (BIG_VOCAB - 1) // 256 * 256
    skip = head_reference(h, e, EOS, lse_skip=torch.arange(last, BIG_VOCAB))
    rows = [0, 1, 3, 4]  # row 2's lse is its 200-above-the-rest logit: nothing else reaches it in float64
    moved = float((skip[0] - ref[0])[rows].abs().min())
    assert moved > 4 * HEAD_EXACT_TOL, moved
    assert float((skip[2] - ref[2])[rows].abs().min()) > 4 * HEAD_EXACT_TOL
    for n_chunks in (63, 1, 2):
        lists = topk_lists(BIG_VOCAB, n_chunks)
        for row in range(5):  # the list holding the row's best token
            best = int(ref[1][row, 0])
            li = next(i for i, cols in enumerate(lists) if bool((cols == best).any()))
            drop = torch.zeros((5, BIG_VOCAB), dtype=torch.bool)
            drop[row, lists[li]] = True
            assert not torch.equal(head_reference(h, e, EOS, drop=drop)[1][row], ref[1][row]), (n_chunks, row)
    desc = head_reference(h, e, EOS, ties_descending=True)
    for row in (0, 1):  # the tie row and the all-equal row
        assert not torch.equal(desc[1][row], ref[1][row]), row


def test_real_scale_head_tolerance_sees_the_ragged_tile():
    """Gaussian h and E at the synthetic weights' scale: the 206 columns of the last tile carry about 8e-4 of the
    probability mass, eight times HEAD_REAL_TOL."""
    h, e = make_real_head(4, BIG_VOCAB, seed=1)
    ref = head_reference(h, e, EOS)
    last = (BIG_VOCAB - 1) // 256 * 256
    skip = head_reference(h, e, EOS, lse_skip=torch.arange(last, BIG_VOCAB))
    moved = float((skip[0] - ref[0]).abs().min())
    assert moved > 4 * HEAD_REAL_TOL, moved


# ---------------------------------------------------------------------------------------------------------------------
# add + LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", LN_DIMS)
@pytest.mark.parametrize("beam", [b for b in LN_BEAMS if b > 1])
def test_layernorm_tolerance_catches_the_sentence_index_bug(d, beam):
    """c indexed by the hypothesis row instead of its sentence (r instead of r // beam) misses the one-ulp bound by far."""
    x, c, gamma, beta = make_ln_case(LN_ROWS, beam, d, seed=d + beam)
    _, ref = add_const_layernorm_reference(x, c, beam, gamma, beta)
    _, bug = add_const_layernorm_reference(x, c, beam, gamma, beta, sentence_of_row_bug=True)
    v = ln_violation(bug.to(torch.bfloat16), ref)
    assert v > 64.0, v
    assert ln_violation(ref.to(torch.bfloat16), ref) <= 0.51  # round-to-nearest of the reference itself (via fp32)
