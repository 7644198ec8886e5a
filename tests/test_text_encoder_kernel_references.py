"""CPU checks of the text encoder kernel tests' references and tolerances (tests/text_encoder_kernel_cases.py): the
references are the oracle's maths, a float64 model of each kernel's own rounding passes its tolerance, and known bugs,
injected into the reference on the GPU test's own inputs, miss it (each printed in multiples of the tolerance)."""

import math

import pytest
import torch

from oracle.text_encoder import static_pooling
from tests.text_encoder_kernel_cases import (HD, LN_EPS, attention_case, attention_kernel_model, attention_reference,
                                             case_violation, chunk_stats, embed_reference, embed_scale,
                                             latent_kernel_model, latent_reference, latent_violation, ln_reference,
                                             ln_sum_of_squares_fp32, ln_violation, make_embed_case, make_latent_case,
                                             make_latent_pointer_case, make_ln_case, make_pointer_case, make_pool_case,
                                             pointer_expected, pool_reference, pool_violation, starts_of,
                                             stats_violation, sum_of_squares_stats, swap_fragment_rows)


def _miss(label, v):
    print(f"{label}: {v:.1f} x the tolerance")
    assert v > 1.0, (label, v)


# ---------------------------------------------------------------------------------------------------------------------
# self-attention
# ---------------------------------------------------------------------------------------------------------------------
def test_attention_reference_is_the_oracles_padded_attention():
    """Per-sentence, length-batched references equal the oracle's attention over the padded batch with its key-padding
    mask (the way OracleTextEncoder.forward calls it)."""
    from oracle.text_encoder import self_attention

    case = attention_case("mixed")
    ref = attention_reference(case)
    d, h, lens = case.dim, case.heads, case.lens
    s = max(lens)
    padded = torch.zeros((len(lens), s, 3 * d), dtype=torch.float64)
    for b, (s0, n) in enumerate(zip(case.starts, lens)):
        padded[b, :n] = case.qkv[s0 : s0 + n].double()
    q, k, v = (padded[:, :, j * d : (j + 1) * d].view(len(lens), s, h, HD).transpose(1, 2) for j in range(3))
    key_ok = torch.arange(s)[None, :] < torch.tensor(lens)[:, None]
    full = self_attention(q, k, v, key_ok).transpose(1, 2).reshape(len(lens), s, d)
    for b, n in enumerate(lens):
        torch.testing.assert_close(ref[b], full[b, :n], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", ["127-129", "513-514", "1031", "d256"])
def test_attention_kernel_rounding_model_passes(name):
    case = attention_case(name)
    v = case_violation(attention_kernel_model(case), attention_reference(case))
    print(f"{name}: the kernel's rounding model at {v:.3f} of the tolerance")
    assert v <= 0.6, v


def test_attention_faults_miss_the_tolerance():
    for name, n in (("127-129", 129), ("255-257", 257), ("513-514", 514)):
        case = attention_case(name)
        good, bad = attention_reference(case), attention_reference(case, drop_last_key_at=[n])
        _miss(f"last key dropped at {n}", case_violation(bad, good))
    case = attention_case("mixed")
    good = attention_reference(case)
    _miss("next sentence's first key attended", case_violation(attention_reference(case, next_first_key=True), good))
    _miss("scale 1/sqrt(D)", case_violation(attention_reference(case, scale=1.0 / math.sqrt(case.dim)), good))
    _miss("head h reads head h+1's K", case_violation(attention_reference(case, k_head_shift=True), good))
    _miss("head h reads head h+1's V", case_violation(attention_reference(case, v_head_shift=True), good))
    _miss("rows r and r + 8 of a fragment swapped", case_violation([None if r is None else swap_fragment_rows(r) for r in good], good))
    _miss("output scaled by 1.02", case_violation([None if r is None else 1.02 * r for r in good], good))
    case = attention_case("255-257")
    _miss("second key tile read from the first",
          case_violation(attention_reference(case, second_tile_from_first=True), attention_reference(case)))
    case = attention_case("513-514")
    _miss("online-softmax rescale omitted",
          case_violation(attention_kernel_model(case, skip_rescale=True), attention_reference(case)))


def test_pointer_cases_are_exact():
    """The float64 reference of a pointer case is v[pi(i)] to far below a bf16 ulp, also with the planted neighbour
    keys, which the next-key bug would pick up instead."""
    case, win = make_pointer_case([1, 2, 129, 5, 514, 3], 4, seed=3)
    want = pointer_expected(case, win).double()
    for b, (r, s0, n) in enumerate(zip(attention_reference(case), case.starts, case.lens)):
        assert float((r - want[s0 : s0 + n]).abs().max()) < 1e-30
    case, win = make_pointer_case([129, 7, 514, 3, 64, 2], 4, seed=4, plant_next=True)
    want = pointer_expected(case, win).double()
    bad = attention_reference(case, next_first_key=True)
    for b, (r, s0, n) in enumerate(zip(attention_reference(case), case.starts, case.lens)):
        if b % 2 == 0:
            assert float((r - want[s0 : s0 + n]).abs().max()) < 1e-30
            assert float((bad[b] - want[s0 : s0 + n]).abs().max()) > 0.1


# ---------------------------------------------------------------------------------------------------------------------
# latent cross-attention
# ---------------------------------------------------------------------------------------------------------------------
def test_latent_reference_is_softmax_attention_and_model_passes():
    qt, mem, lens = make_latent_case(256, 7, seed=1)
    ref = latent_reference(qt, mem, lens)
    for b, (s0, n) in enumerate(zip(starts_of(lens), lens)):
        if n == 0:
            assert bool((ref[b] == 0).all())
            continue
        m = mem[s0 : s0 + n].double()
        want = torch.nn.functional.scaled_dot_product_attention(qt[b].double()[None], m[None], m[None], scale=0.125)[0]
        torch.testing.assert_close(ref[b], want, rtol=1e-12, atol=1e-12)
    v = latent_violation(latent_kernel_model(qt, mem, lens), ref)
    print(f"latent: the kernel's rounding model at {v:.3f} of the tolerance")
    assert v <= 0.6, v


def test_latent_faults_miss_the_tolerance():
    d = 256
    qt, mem, lens = make_latent_case(d, 7, seed=1)
    good = latent_reference(qt, mem, lens)
    _miss("last key dropped at 17", latent_violation(latent_reference(qt, mem, lens, drop_last_key_at=[17]), good))
    _miss("last key dropped at 33", latent_violation(latent_reference(qt, mem, lens, drop_last_key_at=[33]), good))
    _miss("one key past len", latent_violation(latent_reference(qt, mem, lens, one_past=True), good))
    _miss("second tile from the first stage", latent_violation(latent_reference(qt, mem, lens, second_tile_from_first=True), good))
    _miss("scale 1/sqrt(D)", latent_violation(latent_reference(qt, mem, lens, scale=1.0 / math.sqrt(d)), good))
    _miss("query row Hd leaks", latent_violation(latent_reference(qt, mem, lens, row_hd_leak=True), good))


def test_latent_pointer_case_is_exact():
    lens = [1, 15, 17, 33, 514, 1031]
    qt, mem, win = make_latent_pointer_case(256, 7, lens, seed=2)
    ref = latent_reference(qt, mem, lens)
    for b, s0 in enumerate(starts_of(lens)):
        assert float((ref[b] - mem[s0 + win[b]].double()).abs().max()) < 1e-30


# ---------------------------------------------------------------------------------------------------------------------
# embedding, LayerNorm, pooling
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [256, 1024])
def test_embed_reference_is_exact_at_power_of_two_scales(d):
    """At scale 16 / 32 a bf16 value times the scale has 8 significant bits and the float64 sum with an fp32 position
    value is exact (it gives both terms back bit for bit), so its fp32 rounding is what fmaf gives."""
    ids, table, pos, lens = make_embed_case(d)
    scale = embed_scale(d)
    ref = embed_reference(ids, table, pos, scale, lens)
    s0 = 0
    for b, n in enumerate(lens):
        i = ids[b, :n].clamp(0, table.shape[0] - 1)
        assert torch.equal(ref[s0 : s0 + n] - pos[:n].double(), table[i].double() * scale)
        s0 += n


def test_lnfold_stats_bound():
    """A two-pass fp32 (mean, M2) passes; the sum-of-squares M2 of rows 1e3 away from zero misses."""
    ids, table, pos, lens = make_embed_case(1024)
    x = embed_reference(ids, table, pos, embed_scale(1024), lens).float()
    c = x.view(x.shape[0], -1, 128)
    mean = c.sum(-1) / 128.0
    two_pass = torch.stack([mean, ((c - mean[..., None]) ** 2).sum(-1)], -1)
    v = stats_violation(two_pass, x)
    print(f"two-pass fp32 stats at {v:.3f} of the bound")
    assert v <= 0.5
    _miss("sum-of-squares M2", stats_violation(sum_of_squares_stats(x), x))
    assert torch.allclose(chunk_stats(x)[..., 0], x.double().view(x.shape[0], -1, 128).mean(-1))


@pytest.mark.parametrize("d", [128, 768, 1024])
def test_layernorm_bound(d):
    """An fp32 two-pass LayerNorm passes the fp32 and bf16 bounds; an fp32 sum-of-squares variance and a variance
    divided by D - 1 miss the fp32 bound; constant rows give beta."""
    x, gamma, beta = make_ln_case(4099, d, seed=d)
    ref = ln_reference(x, gamma, beta)
    assert torch.equal(ref[2::4], beta.double().expand_as(ref[2::4]))
    mean = x.mean(1, keepdim=True)
    var = ((x - mean) ** 2).mean(1, keepdim=True)
    y32 = (x - mean) / torch.sqrt(var + LN_EPS) * gamma + beta
    v32, v16 = ln_violation(y32, x, gamma, beta, ref), ln_violation(y32.to(torch.bfloat16), x, gamma, beta, ref)
    print(f"D={d}: fp32 two-pass LayerNorm at {v32:.3f} (fp32) / {v16:.3f} (bf16) of the bound")
    assert v32 <= 0.5 and v16 <= 1.0
    _miss(f"D={d} sum-of-squares variance", ln_violation(ln_sum_of_squares_fp32(x, gamma, beta).float(), x, gamma, beta, ref))
    _miss(f"D={d} variance over D - 1", ln_violation(ln_reference(x, gamma, beta, unbiased=True).float(), x, gamma, beta, ref))


def test_pool_reference_is_static_pooling_of_the_padded_batch():
    lens = [1, 7, 8, 9, 0, 17, 3]
    x, gamma, beta = make_pool_case(lens, 128, seed=5)
    s = max(lens)
    padded = torch.full((len(lens), s, 128), 1.0e6, dtype=torch.float64)  # padding that must not leak
    ln = ln_reference(x, gamma, beta)
    for b, (s0, n) in enumerate(zip(starts_of(lens), lens)):
        padded[b, :n] = ln[s0 : s0 + n]
    for mode in ("mean", "max", "last"):
        ref = pool_reference(x, lens, mode, gamma, beta)
        full = static_pooling(padded, torch.tensor(lens), mode)
        for b, n in enumerate(lens):
            if n > 0:
                torch.testing.assert_close(ref[b], full[b], rtol=1e-12, atol=1e-12)
        # an empty sentence: MEAN 0 and MAX -inf as the kernel gives them; the reference's LAST reads padded position 0
        # where the kernel writes zeros
        empty = full[4]
        want = {"mean": torch.zeros(128, dtype=torch.float64), "max": torch.full((128,), -math.inf, dtype=torch.float64),
                "last": padded[4, 0]}[mode]
        assert torch.equal(empty, want), mode


def test_pool_faults_miss_the_tolerance():
    lens = [1, 7, 8, 9, 15, 16, 17, 514]
    x, gamma, beta = make_pool_case(lens, 256, seed=6)
    for ln in (False, True):
        g, b = (gamma, beta) if ln else (None, None)
        _miss(f"MAX from 0 (apply_ln={int(ln)})",
              pool_violation(pool_reference(x, lens, "max", g, b, max_zero_init=True), pool_reference(x, lens, "max", g, b)))
        _miss(f"LAST takes the first row (apply_ln={int(ln)})",
              pool_violation(pool_reference(x, lens, "last", g, b, last_first_row=True), pool_reference(x, lens, "last", g, b)))
