"""Kernel-level parity of the text encoder's own kernels (through the C ABI, on the launch functions the encoder's
forward uses) against float64 references of the same operation on the same inputs: the packed self-attention, the
attention pooler's latent cross-attention, the embedding frontend and its LnFold outputs, both LayerNorm kernels and the
LayerNorm + pooling kernel.  Inputs, references and tolerances: tests/text_encoder_kernel_cases.py."""

import math

import pytest
import torch

from tests.text_encoder_kernel_cases import (ATTN_CASES, EMBED_DIMS, EMBED_VOCAB, HD, LA_DIMS, LA_HEADS, LN_DIMS,
                                             LN_EPS, LN_ROWS, POOL_LENS, POOL_LONG, POOL_MODES, attention_case,
                                             attention_reference, attn_violation, case_violation, embed_reference,
                                             embed_scale, latent_reference, latent_violation, ln_reference, ln_violation,
                                             make_embed_case, make_latent_case, make_latent_pointer_case, make_ln_case,
                                             make_pointer_case, make_pool_case, pointer_expected, pool_lens,
                                             pool_reference, pool_violation, starts_of, stats_violation)

pytestmark = pytest.mark.gpu

GUARD = 5            # rows of sentinel before and after every output
SENTINEL = -768.0    # exact in bf16 and fp32


@pytest.fixture(scope="module")
def ops(native_lib, cuda_device):
    from sonar_b200 import ops as _ops

    torch.cuda.set_device(cuda_device)
    return _ops


def _guarded(rows, cols, dtype, device):
    """(buffer with GUARD sentinel rows before and after, the [rows, cols] view between them)."""
    buf = torch.full((rows + 2 * GUARD, cols), SENTINEL, dtype=dtype, device=device)
    return buf, buf[GUARD : GUARD + rows]


def _check_guard(buf, what):
    assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all()), f"{what} wrote outside its rows"


def _bits(x):
    return x.contiguous().view(torch.int16 if x.element_size() == 2 else torch.int32)


def _cu(lens, device):
    from sonar_b200 import ops as _ops

    return _ops.cu_seqlens_of(lens).to(device)


# ---------------------------------------------------------------------------------------------------------------------
# packed self-attention
# ---------------------------------------------------------------------------------------------------------------------
def _attend(ops, qkv, lens, heads, device):
    t, d = qkv.shape[0], HD * heads
    buf, out = _guarded(t, d, torch.bfloat16, device)
    ops.attention(qkv, _cu(lens, device), heads, out=out)
    torch.cuda.synchronize()
    _check_guard(buf, "attention")
    return out


@pytest.mark.parametrize("name", list(ATTN_CASES))
def test_attention_vs_float64_reference(ops, cuda_device, name):
    """Every sentence of every case within ATTN_RTOL / ATTN_ATOL / ATTN_MEAN of the float64 reference (run on the GPU)."""
    case = attention_case(name, cuda_device)
    out = _attend(ops, case.qkv, case.lens, case.heads, cuda_device)
    ref = attention_reference(case)
    got = [None if r is None else out[s0 : s0 + n] for r, s0, n in zip(ref, case.starts, case.lens)]
    v = case_violation(got, ref, attn_violation)
    err = max(float((g.double() - r).abs().max()) for g, r in zip(got, ref) if r is not None)
    print(f"attention {name}: max err {err:.3e}, {v:.3f} of the tolerance")
    assert v <= 1.0, (name, v)


@pytest.mark.parametrize("heads", [16, 4])
def test_attention_pointer_operands_give_v_bit_for_bit(ops, cuda_device, heads):
    """Sign-vector queries and keys whose winner leads by > 160 in log2 units: every other probability underflows to 0
    (alpha of earlier tiles included) and row i is v[pi(i)] exactly; winners lie in earlier and later key tiles."""
    case, win = make_pointer_case([1, 2, 129, 5, 514, 3, 1031, 257, 64, 128, 385], heads, seed=heads)
    out = _attend(ops, case.qkv.to(cuda_device), case.lens, heads, cuda_device)
    assert torch.equal(_bits(out.cpu()), _bits(pointer_expected(case, win)))


def test_attention_pointer_ignores_a_stronger_key_in_the_next_sentence(ops, cuda_device):
    """The first row of every odd sentence holds a key twice as strong as a winner of the even sentence before it; the
    even sentences' rows are still v[pi(i)] bit for bit."""
    case, win = make_pointer_case([129, 7, 514, 3, 64, 2, 1, 5, 127, 1, 255, 9], 16, seed=5, plant_next=True)
    out = _attend(ops, case.qkv.to(cuda_device), case.lens, 16, cuda_device).cpu()
    want = pointer_expected(case, win)
    for b, (s0, n) in enumerate(zip(case.starts, case.lens)):
        if b % 2 == 0:
            assert torch.equal(_bits(out[s0 : s0 + n]), _bits(want[s0 : s0 + n])), b


@pytest.mark.parametrize("name", ["mixed", "empty", "d256"])
def test_attention_masked_keys_get_zero_probability(ops, cuda_device, name):
    """K and V rows of magnitude ~1e3 in the neighbouring sentences leave a sentence's output bits unchanged."""
    case = attention_case(name, cuda_device)
    d, lens = case.dim, case.lens
    base = _attend(ops, case.qkv, lens, case.heads, cuda_device)
    for parity in (0, 1):
        qkv = case.qkv.clone()
        for b, (s0, n) in enumerate(zip(case.starts, lens)):
            if b % 2 != parity:
                qkv[s0 : s0 + n, d:] = (1.0e3 * torch.sign(qkv[s0 : s0 + n, d:].float() + 0.5)).to(torch.bfloat16)
        out = _attend(ops, qkv, lens, case.heads, cuda_device)
        for b, (s0, n) in enumerate(zip(case.starts, lens)):
            if b % 2 == parity:
                assert torch.equal(_bits(out[s0 : s0 + n]), _bits(base[s0 : s0 + n])), (name, b)


@pytest.mark.parametrize("name", ["mixed", "empty", "d256"])
def test_attention_sentence_alone_equals_the_batch(ops, cuda_device, name):
    case = attention_case(name, cuda_device)
    base = _attend(ops, case.qkv, case.lens, case.heads, cuda_device)
    for s0, n in zip(case.starts, case.lens):
        if n > 0:
            solo = _attend(ops, case.qkv[s0 : s0 + n].contiguous(), [n], case.heads, cuda_device)
            assert torch.equal(_bits(solo), _bits(base[s0 : s0 + n])), (name, n)


# ---------------------------------------------------------------------------------------------------------------------
# latent cross-attention
# ---------------------------------------------------------------------------------------------------------------------
def _latent(ops, qt, mem, lens, device):
    b, hd, d = qt.shape
    buf, out = _guarded(b * hd, d, torch.bfloat16, device)
    u = ops.pool_latent_attention(qt.to(device), mem.to(device), _cu(lens, device), out=out.view(b, hd, d))
    torch.cuda.synchronize()
    _check_guard(buf, "pool_latent_attention")
    return u


@pytest.mark.parametrize("hd", LA_HEADS)
@pytest.mark.parametrize("d", LA_DIMS)
def test_latent_attention_vs_float64_reference(ops, cuda_device, d, hd):
    """Every sentence within LA_RTOL / LA_ATOL / LA_MEAN; empty sentences give exact zeros."""
    qt, mem, lens = make_latent_case(d, hd, seed=d + hd)
    u = _latent(ops, qt, mem, lens, cuda_device).cpu()
    ref = latent_reference(qt, mem, lens)
    full = [b for b, n in enumerate(lens) if n > 0]
    v = max(latent_violation(u[b], ref[b]) for b in full)
    print(f"latent D={d} Hd={hd}: max err {float((u.double() - ref).abs().max()):.3e}, {v:.3f} of the tolerance")
    assert v <= 1.0, v
    for b, n in enumerate(lens):
        if n == 0:
            assert torch.equal(_bits(u[b]), torch.zeros_like(_bits(u[b])))


@pytest.mark.parametrize("d", LA_DIMS)
def test_latent_pointer_operands_give_the_memory_row(ops, cuda_device, d):
    lens = [1, 15, 16, 17, 31, 32, 33, 0, 514, 1031, 2]
    qt, mem, win = make_latent_pointer_case(d, 7, lens, seed=d)
    u = _latent(ops, qt, mem, lens, cuda_device).cpu()
    for b, (s0, n) in enumerate(zip(starts_of(lens), lens)):
        want = mem[s0 + win[b]] if n > 0 else torch.zeros_like(u[b])
        assert torch.equal(_bits(u[b]), _bits(want)), (d, b)


# ---------------------------------------------------------------------------------------------------------------------
# embedding
# ---------------------------------------------------------------------------------------------------------------------
def _embed(ops, ids, table, pos, scale, lens, device, lnfold):
    t = sum(lens)
    buf, x = _guarded(t, table.shape[1], torch.float32, device)
    flag = torch.zeros(1, dtype=torch.int32, device=device)
    res = ops.embed(ids.to(device), _cu(lens, device), table.to(device), pos.to(device), scale, t, lnfold=lnfold, out=x,
                    flag=flag)
    torch.cuda.synchronize()
    _check_guard(buf, "embed")
    return res, bool(flag.item())


def _check_x(x, ref, d):
    want = ref.float()
    if d in (256, 1024):  # power-of-two scale: fmaf's single rounding of an exact sum
        assert torch.equal(_bits(x), _bits(want))
    else:
        ulp = (torch.nextafter(want, torch.full_like(want, math.inf)) - want).abs()
        assert bool(((x - want).abs() <= ulp).all())


@pytest.mark.parametrize("lnfold", [False, True])
@pytest.mark.parametrize("d", EMBED_DIMS)
def test_embed(ops, cuda_device, d, lnfold):
    """x = table[id] * scale + pos[t] (bit for bit at D = 256 / 1024); ids past each length are out of range and never
    read (flag clear); with the LnFold outputs h = bf16(x) bit for bit and (mean, M2) of every 128-column chunk within
    the bound of float64 ones of the stored x (rows 1e3 away from zero)."""
    ids, table, pos, lens = make_embed_case(d, seed=d)
    scale = embed_scale(d)
    res, flag = _embed(ops, ids, table, pos, scale, lens, cuda_device, lnfold)
    assert not flag
    x = res[0] if lnfold else res
    x = x.cpu()
    _check_x(x, embed_reference(ids, table, pos, scale, lens), d)
    if lnfold:
        h, stats = res[1].cpu(), res[2].cpu()
        assert torch.equal(_bits(h), _bits(x.to(torch.bfloat16)))
        v = stats_violation(stats, x)
        print(f"embed D={d}: stats at {v:.3f} of the bound")
        assert v <= 1.0, v


@pytest.mark.parametrize("d", [256, 768])
def test_embed_bad_ids_set_the_flag_and_embed_row_0(ops, cuda_device, d):
    ids, table, pos, lens = make_embed_case(d, seed=d + 1)
    ids[0, 3], ids[3, 8], ids[5, 0] = -1, EMBED_VOCAB, -1
    scale = embed_scale(d)
    (x, _, _), flag = _embed(ops, ids, table, pos, scale, lens, cuda_device, True)
    assert flag
    _check_x(x.cpu(), embed_reference(ids, table, pos, scale, lens), d)  # the reference embeds id 0 for them


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", LN_ROWS)
@pytest.mark.parametrize("d", LN_DIMS)
def test_layernorm_kernels(ops, cuda_device, d, t):
    """sb_layernorm (bf16) and sb_layernorm_dual (fp32 + bf16) within the derived bounds of the float64 LayerNorm;
    constant rows give beta exactly; the in-place run (out32 = x) gives the out-of-place bits; guard rows untouched."""
    x, gamma, beta = make_ln_case(t, d, seed=7 * d + t)
    ref = ln_reference(x, gamma, beta)
    xd, g, b = x.to(cuda_device), gamma.to(cuda_device), beta.to(cuda_device)
    y16 = ops.layernorm(xd, g, b, LN_EPS)
    buf32, o32 = _guarded(t, d, torch.float32, cuda_device)
    buf16, o16 = _guarded(t, d, torch.bfloat16, cuda_device)
    ops.layernorm_dual(xd, g, b, LN_EPS, out32=o32, out16=o16)
    xin = xd.clone()
    i32, i16 = ops.layernorm_dual(xin, g, b, LN_EPS, out32=xin)
    torch.cuda.synchronize()
    _check_guard(buf32, "layernorm_dual fp32")
    _check_guard(buf16, "layernorm_dual bf16")
    assert torch.equal(_bits(i32), _bits(o32)) and torch.equal(_bits(i16), _bits(o16))
    assert torch.equal(_bits(y16), _bits(o16))
    v32, v16 = ln_violation(o32.cpu(), x, gamma, beta, ref), ln_violation(o16.cpu(), x, gamma, beta, ref)
    print(f"layernorm D={d} T={t}: fp32 at {v32:.3f}, bf16 at {v16:.3f} of the bound")
    assert v32 <= 1.0 and v16 <= 1.0, (v32, v16)
    const = torch.arange(t) % 4 == 2
    if bool(const.any()):
        assert torch.equal(o32.cpu()[const], beta.expand(int(const.sum()), d))
        assert torch.equal(_bits(o16.cpu()[const]), _bits(beta.to(torch.bfloat16).expand(int(const.sum()), d)))


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm + pooling
# ---------------------------------------------------------------------------------------------------------------------
def _pool(ops, x, lens, mode, gamma, beta, device, s_padded=0):
    kw = dict(gamma=gamma.to(device), beta=beta.to(device)) if gamma is not None else {}
    res = ops.pool_packed(x, _cu(lens, device), mode, eps=LN_EPS, encoded_seq_len=s_padded, **kw)
    torch.cuda.synchronize()
    return res


@pytest.mark.parametrize("apply_ln", [0, 1])
@pytest.mark.parametrize("mode", POOL_MODES)
def test_pool_vs_static_pooling(ops, cuda_device, mode, apply_ln):
    """5000 sentences of every length 1..17 class and some of 514, all-negative values: within the bound of
    static_pooling of the float64 LayerNorm (MAX and LAST without LayerNorm exact); a second run and each length's
    sentence alone give the same bits."""
    lens = pool_lens()
    x, gamma, beta = make_pool_case(lens, 256, seed=11)
    g, b = (gamma, beta) if apply_ln else (None, None)
    xd = x.to(cuda_device)
    out = _pool(ops, xd, lens, mode, g, b, cuda_device)
    ref = pool_reference(x, lens, mode, g, b)
    if not apply_ln and mode != "mean":
        assert torch.equal(out.cpu().double(), ref)
    v = pool_violation(out, ref)
    print(f"pool {mode} apply_ln={apply_ln}: {v:.3f} of the bound")
    assert v <= 1.0, v
    assert torch.equal(_bits(_pool(ops, xd, lens, mode, g, b, cuda_device)), _bits(out))
    starts = starts_of(lens)
    for n in POOL_LENS + [POOL_LONG]:
        i = lens.index(n)
        solo = _pool(ops, xd[starts[i] : starts[i] + n].contiguous(), [n], mode, g, b, cuda_device)
        assert torch.equal(_bits(solo[0]), _bits(out[i])), (mode, n)


@pytest.mark.parametrize("extra", [0, 6])
@pytest.mark.parametrize("d", [256, 1024])
def test_pool_encoded_padded_and_empty_sentences(ops, cuda_device, d, extra):
    """encoded_padded with S_padded = the longest sentence and longer: the (normalised) rows of each sentence, then
    exactly +0.0.  Empty sentences: MEAN 0, MAX -inf, LAST 0 (static_pooling's LAST would read padded position 0)."""
    lens = [0] + [POOL_LENS[i % len(POOL_LENS)] for i in range(60)] + [POOL_LONG, 0, 3, 0]
    x, gamma, beta = make_pool_case(lens, d, seed=d + extra)
    s_pad = POOL_LONG + extra
    xd = x.to(cuda_device)
    rows = ln_reference(x, gamma, beta)
    for mode in POOL_MODES:
        out, enc = _pool(ops, xd, lens, mode, gamma, beta, cuda_device, s_pad)
        assert pool_violation(out, pool_reference(x, lens, mode, gamma, beta)) <= 1.0
        enc = enc.cpu()
        for bi, (s0, n) in enumerate(zip(starts_of(lens), lens)):
            err = (enc[bi, :n].double() - rows[s0 : s0 + n]).abs()
            assert bool((err <= 1e-4).all()), (mode, bi)
            assert torch.equal(_bits(enc[bi, n:]), torch.zeros_like(_bits(enc[bi, n:])))
            if n == 0:
                want = {"mean": 0.0, "max": -math.inf, "last": 0.0}[mode]
                assert bool((out[bi] == want).all()), (mode, bi)
