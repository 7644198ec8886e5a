"""Kernel-level parity of the decoder step's own kernels (through the C ABI, on the launch path sb_decoder_step uses)
against float64 references of the same operation on the same inputs: the KV-cache attention, the vocabulary head (the
top-16 / log-sum-exp sweep of the wgmma GEMM and the merge kernel), the embedding and the add + LayerNorm kernel.
Inputs, references and tolerances: tests/decoder_kernel_cases.py."""

import functools

import pytest
import torch

from tests.decoder_kernel_cases import (ATTN_HEADS, ATTN_POSITIONS, BIG_VOCAB, EOS, HEAD_EXACT_TOL, HEAD_REAL_TOL, LN_BEAMS,
                                        LN_DIMS, LN_EPS, LN_ROWS, add_const_layernorm_reference, attention_reference,
                                        attn_violation, head_reference, ln_violation, make_attention_case, make_exact_head,
                                        make_ln_case, make_real_head, probe_tokens, value_max)

pytestmark = pytest.mark.gpu

GUARD = 5            # rows of sentinel after every output
SENTINEL = -768.0    # exact in bf16 and fp32


@pytest.fixture(scope="module")
def ops(native_lib, cuda_device):
    from sonar_b200 import ops as _ops

    torch.cuda.set_device(cuda_device)
    return _ops


def _guarded(shape, dtype, device):
    return torch.full((shape[0] + GUARD,) + tuple(shape[1:]), SENTINEL, dtype=dtype, device=device)


def _check_guard(buf, what):
    tail = buf[-GUARD:]
    assert bool((tail == SENTINEL).all()), f"{what} wrote past its output rows"


def _bits(x):
    return x.view(torch.int16)


# ---------------------------------------------------------------------------------------------------------------------
# KV-cache attention
# ---------------------------------------------------------------------------------------------------------------------
def _attend(ops, case, device):
    """Runs the kernel on copies of the case's caches; checks the guard rows, the cache update and finiteness; returns
    the output (float64, on the device)."""
    r, d, t = case.rows, case.dim, case.t
    kc, vc = case.kcache.to(device), case.vcache.to(device)
    kc0, vc0 = kc.clone(), vc.clone()
    buf = _guarded((r, d), torch.bfloat16, device)
    out = ops.decoder_attention(case.qkv.to(device), kc, vc, case.table.to(device), t, case.heads, out=buf[:r])
    torch.cuda.synchronize()
    _check_guard(buf, "decoder_attention")
    # the caches change at (r, t) only, where they now hold this step's k and v bits
    qkv = case.qkv.to(device)
    kc0[torch.arange(r, device=device), t] = qkv[:, d : 2 * d]
    vc0[torch.arange(r, device=device), t] = qkv[:, 2 * d :]
    assert torch.equal(_bits(kc), _bits(kc0)) and torch.equal(_bits(vc), _bits(vc0)), "cache entries other than (r, t) changed"
    assert bool(torch.isfinite(out.float()).all()), "the kernel read a cache entry the table does not name"
    if t == 0:  # one key: softmax = 1, out = v bit for bit
        assert torch.equal(_bits(out), _bits(qkv[:, 2 * d :].contiguous()))
    return out


def _check_attention(ops, case, device, label):
    out = _attend(ops, case, device)
    ref = attention_reference(case).to(out.device)
    v = attn_violation(out, ref, value_max(case))
    err = (out.double() - ref).abs()
    print(f"{label}: max err {float(err.max()):.3e}, mean err {float(err.mean()):.3e}, {v:.3f} of the tolerance")
    assert v <= 1.0, (label, v)


@pytest.mark.parametrize("t", ATTN_POSITIONS)
@pytest.mark.parametrize("heads", ATTN_HEADS)
@pytest.mark.parametrize("rows,table", [(1, "random"), (7, "random"), (7, "identity")])
def test_decoder_attention_vs_float64_reference(ops, cuda_device, rows, table, heads, t):
    """Every position on a 16-key pass edge up to 511, tables that point at any row or at the row itself, key spreads
    up to about +-60 with the maximum late in the sweep; every cache entry the table does not name holds NaN.  The
    bounds and what they measured: ATTN_RTOL, ATTN_ATOL and ATTN_MEAN in tests/decoder_kernel_cases.py."""
    tmax = 512 if t == 511 else None
    case = make_attention_case(rows, heads, t, tmax=tmax, table=table, seed=1000 * heads + t + rows)
    _check_attention(ops, case, cuda_device, f"R={rows} {table} H={heads} t={t}")


@pytest.mark.parametrize("t", [0, 16, 17, 33, 129, 257, 511])
@pytest.mark.parametrize("heads", ATTN_HEADS)
def test_decoder_attention_2560_rows(ops, cuda_device, heads, t):
    """The benchmark's 512 sentences x beam 5, with a table that points anywhere (inputs made on the GPU)."""
    case = make_attention_case(2560, heads, t, tmax=512 if t == 511 else None, seed=7 * t + heads, device=cuda_device)
    _check_attention(ops, case, cuda_device, f"R=2560 H={heads} t={t}")


def test_decoder_attention_row_limit(ops, cuda_device):
    """65 535 rows (the grid's y limit) at a short history run; 65 536 rows, t outside [0, Tmax), Tmax > 512 and a model
    dim that is no multiple of 256 are refused with the step's messages."""
    case = make_attention_case(65535, 4, 3, tmax=4, seed=11, device=cuda_device)
    _check_attention(ops, case, cuda_device, "R=65535 H=4 t=3")
    dev = cuda_device

    def run(rows, heads, t, tmax):
        d = 64 * heads
        kc = torch.zeros((rows, tmax, d), dtype=torch.bfloat16, device=dev)
        ops.decoder_attention(torch.zeros((rows, 3 * d), dtype=torch.bfloat16, device=dev), kc, kc.clone(),
                              torch.zeros((rows, tmax), dtype=torch.int32, device=dev), t, heads)

    with pytest.raises(ValueError, match="too many rows"):
        run(65536, 4, 0, 1)
    with pytest.raises(ValueError, match="outside"):
        run(2, 4, 4, 4)
    with pytest.raises(ValueError, match="outside"):
        run(2, 4, -1, 4)
    with pytest.raises(ValueError, match="max_len 513"):
        run(2, 4, 3, 513)
    with pytest.raises(ValueError, match="multiple of 256"):
        run(2, 2, 0, 4)


# ---------------------------------------------------------------------------------------------------------------------
# vocabulary head
# ---------------------------------------------------------------------------------------------------------------------
def _head(ops, h, e, probes, n_chunks, device):
    r = h.shape[0]
    bufs = [_guarded((r, 16), torch.float32, device), _guarded((r, 16), torch.int32, device),
            _guarded((r,), torch.float32, device), None if probes is None else _guarded((r,), torch.float32, device)]
    out = ops.decoder_vocab_head(h, e, EOS, probes, n_chunks=n_chunks, out=tuple(None if b is None else b[:r] for b in bufs))
    torch.cuda.synchronize()
    for b, name in zip(bufs, ("lprob", "tok", "eos", "probe")):
        if b is not None:
            _check_guard(b, f"decoder_vocab_head {name}")
    return out


@functools.lru_cache(maxsize=8)
def _exact(rows, vocab, device):
    h, e, _ = make_exact_head(rows, vocab, seed=rows, device=device)
    probes = probe_tokens(rows, vocab, device)
    return h, e, probes, head_reference(h, e, EOS, probes)


@pytest.mark.parametrize("n_chunks", [0, 1, 2])
@pytest.mark.parametrize("rows", [1, 5, 255, 256, 257, 2560])
@pytest.mark.parametrize("vocab", [BIG_VOCAB, 4196, 20, 10])
def test_vocab_head_exact_operands(ops, cuda_device, vocab, rows, n_chunks):
    """Exact logits: the 16 tokens equal the float64 top 16 in order, ties included (V - 1 first, then the tied tokens
    spread over chunks, column halves and the ragged tile; all-zero logits give tokens 0..15); V < 16 pads with
    (-inf, -1).  log-probs, log P(EOS) and the probes (0, V - 1, and -1 / V scored as token 0) within HEAD_EXACT_TOL."""
    h, e, probes, (lp_ref, tok_ref, eos_ref, pr_ref) = _exact(rows, vocab, cuda_device)
    if n_chunks > (vocab + 255) // 256:
        with pytest.raises(ValueError, match="n_chunks"):
            _head(ops, h, e, probes, n_chunks, cuda_device)
        return
    lp, tok, eos, pr = _head(ops, h, e, probes, n_chunks, cuda_device)
    assert torch.equal(tok.long(), tok_ref), (vocab, rows, n_chunks)
    fin = torch.isfinite(lp_ref)
    assert torch.equal(torch.isfinite(lp), fin) and bool((lp[~fin] == float("-inf")).all())
    worst = max(float((lp.double()[fin] - lp_ref[fin]).abs().max()), float((eos.double() - eos_ref).abs().max()),
                float((pr.double() - pr_ref).abs().max()))
    print(f"V={vocab} R={rows} n_chunks={n_chunks}: max |lprob err| {worst:.3e}")
    assert worst <= HEAD_EXACT_TOL, worst


def test_vocab_head_256_lists(ops, cuda_device):
    """128 chunks of one tile at V = 32 718: 256 candidate lists, each lane's slice of the merge exactly 128 entries (its
    bitmap's capacity)."""
    h, e, _ = make_exact_head(257, 32718, seed=3, device=cuda_device)
    probes = probe_tokens(257, 32718, cuda_device)
    lp_ref, tok_ref, eos_ref, pr_ref = head_reference(h, e, EOS, probes)
    lp, tok, eos, pr = _head(ops, h, e, probes, 128, cuda_device)
    assert torch.equal(tok.long(), tok_ref)
    worst = max(float((lp.double() - lp_ref).abs().max()), float((eos.double() - eos_ref).abs().max()),
                float((pr.double() - pr_ref).abs().max()))
    assert worst <= HEAD_EXACT_TOL, worst


def test_vocab_head_refuses_more_than_256_lists(ops, cuda_device):
    h, e, _ = make_exact_head(4, BIG_VOCAB, device=cuda_device)
    with pytest.raises(ValueError, match="286 candidate lists"):
        _head(ops, h, e, None, 143, cuda_device)


def test_vocab_head_real_scale(ops, cuda_device):
    """Gaussian h (a LayerNorm output) and E at the synthetic weights' scale, D = 1024, V = 256 206, 2560 rows, the step's
    chunking: each value within HEAD_REAL_TOL of the float64 logit of its token minus the log-sum-exp; the token set is
    the float64 top 16 wherever the 16th and 17th float64 values are further apart than that."""
    h, e = make_real_head(2560, device=cuda_device)
    lp, tok, eos, _ = _head(ops, h, e, None, 0, cuda_device)
    worst, bad = 0.0, 0
    ef = e.double()
    for r0 in range(0, 2560, 256):
        logits = h[r0 : r0 + 256].double() @ ef.T
        lse = torch.logsumexp(logits, 1, keepdim=True)
        got = lp[r0 : r0 + 256].double()
        want = torch.gather(logits, 1, tok[r0 : r0 + 256].long()) - lse
        worst = max(worst, float((got - want).abs().max()), float((eos[r0 : r0 + 256].double() - (logits[:, EOS] - lse[:, 0])).abs().max()))
        top = logits.topk(17, 1)
        clear = (top.values[:, 15] - top.values[:, 16]) > HEAD_REAL_TOL
        same = torch.sort(tok[r0 : r0 + 256].long(), 1).values == torch.sort(top.indices[:, :16], 1).values
        bad += int((clear & ~same.all(1)).sum())
    print(f"real-scale head: max |lprob err| {worst:.3e}")
    assert worst <= HEAD_REAL_TOL and bad == 0, (worst, bad)


# ---------------------------------------------------------------------------------------------------------------------
# embedding and add + LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", LN_DIMS)
def test_decoder_embed(ops, cuda_device, d):
    """x = fp32 fma(E[token], scale, pos) within one fp32 ulp; ids -1 and V set the flag and embed row 0."""
    g = torch.Generator().manual_seed(d)
    v, r = 4196, LN_ROWS
    e = torch.randn((v, d), generator=g).to(torch.bfloat16)
    pos = torch.randn(d, generator=g)
    scale = float(d) ** 0.5
    tokens = torch.randint(0, v, (r,), generator=g)
    tokens[:3] = torch.tensor([0, v - 1, 5])
    buf = _guarded((r, d), torch.float32, cuda_device)
    x, flag = ops.decoder_embed(tokens.to(cuda_device), e.to(cuda_device), pos.to(cuda_device), scale, out=buf[:r])
    torch.cuda.synchronize()
    _check_guard(buf, "decoder_embed")
    assert not flag
    want = (e[tokens].double() * scale + pos.double()).float()
    ulp = torch.abs(torch.nextafter(want, torch.full_like(want, float("inf"))) - want)
    assert bool(((x.cpu() - want).abs() <= ulp).all())
    bad = tokens.clone()
    bad[1], bad[4] = -1, v
    x2, flag2 = ops.decoder_embed(bad.to(cuda_device), e.to(cuda_device), pos.to(cuda_device), scale)
    assert flag2
    x2, x = x2.cpu(), x.cpu()
    assert torch.equal(x2[1], x[0]) and torch.equal(x2[4], x[0])  # row 0 embedded (token 0 is row 0's id)
    assert torch.equal(x2[[0, 2, 3]], x[[0, 2, 3]])


@pytest.mark.parametrize("d", LN_DIMS)
@pytest.mark.parametrize("beam", LN_BEAMS)
def test_decoder_add_const_layernorm(ops, cuda_device, beam, d):
    """x = fp32 x + c[r // beam] bit for bit; h within one bf16 ulp of the float64 LayerNorm of that fp32 row (ulp taken
    at max(|h|, 1/8)); 37 rows (not a multiple of 8) about 1e3 away from zero."""
    x, c, gamma, beta = make_ln_case(LN_ROWS, beam, d, seed=d + beam)
    xn_ref, h_ref = add_const_layernorm_reference(x, c, beam, gamma, beta)
    xd = x.to(cuda_device)
    buf = _guarded((LN_ROWS, d), torch.bfloat16, cuda_device)
    h = ops.decoder_add_const_layernorm(xd, c.to(cuda_device), beam, gamma.to(cuda_device), beta.to(cuda_device), LN_EPS,
                                        out=buf[:LN_ROWS])
    torch.cuda.synchronize()
    _check_guard(buf, "decoder_add_const_layernorm")
    assert torch.equal(xd.cpu(), xn_ref)
    v = ln_violation(h.cpu(), h_ref)
    print(f"add+LN beam={beam} D={d}: {v:.3f} bf16 ulp")
    assert v <= 1.0, v
