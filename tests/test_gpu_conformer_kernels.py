"""Kernel-level parity of the speech encoder's own kernels (through the C ABI, on the launch path the encoder's forward
uses) against float64 references of the same operation on the same bf16 inputs: both relative-position attention kernels,
the conv module's GLU / depthwise conv / BatchNorm / SiLU kernel and the frontend's frame stacking + LayerNorm.  Inputs,
references and tolerances: tests/conformer_kernel_cases.py."""

import functools

import pytest
import torch

from tests.conformer_kernel_cases import (ATTN_CASES, CONV_DIMS, attn_violation, conv_reference, conv_violation,
                                          make_conv_case, make_relpos_case, relpos_reference)

pytestmark = pytest.mark.gpu

IMPLS = ["wgmma", "mma_sync"]
GUARD = 7           # rows of sentinel before and after every output
SENTINEL = -768.0   # exact in bf16
MULTI = [n for n, (lens, _) in ATTN_CASES.items() if len(lens) > 1]


@pytest.fixture(scope="module")
def ops(native_lib, cuda_device):
    from sonar_b200 import ops as _ops

    torch.cuda.set_device(cuda_device)
    return _ops


@functools.lru_cache(maxsize=None)
def _case(name):
    lens, heads = ATTN_CASES[name]
    return make_relpos_case(lens, heads)


def _guarded(rows, cols, device):
    return torch.full((rows + 2 * GUARD, cols), SENTINEL, dtype=torch.bfloat16, device=device)


def _check_guards(buf, what):
    guard = torch.full((GUARD, buf.shape[1]), SENTINEL, dtype=torch.bfloat16, device=buf.device)
    assert torch.equal(buf[:GUARD], guard) and torch.equal(buf[-GUARD:], guard), f"{what} wrote outside its output rows"


def _attend(ops, case, impl, device, qkv=None, lens=None, p=None):
    """The kernel's output rows (cpu bf16) for the packed qkv rows of `lens`; checks the guard rows around the output."""
    lens = case.lens if lens is None else lens
    qkv = case.qkv if qkv is None else qkv
    p = case.p(max(lens)) if p is None else p
    t, d = sum(lens), case.dim
    buf = _guarded(t, d, device)
    out = ops.attention_relpos(qkv.to(device), p.to(device), case.u_bias.to(device), case.v_bias.to(device),
                               ops.cu_seqlens_of(lens).to(device), case.heads, impl=impl, out=buf[GUARD : GUARD + t])
    torch.cuda.synchronize()
    assert out.data_ptr() == buf[GUARD].data_ptr()
    _check_guards(buf, f"attention_relpos[{impl}]")
    return out.cpu()


@pytest.mark.parametrize("name", list(ATTN_CASES))
@pytest.mark.parametrize("impl", IMPLS)
def test_relpos_attention_vs_float64_reference(ops, cuda_device, impl, name):
    case = _case(name)
    out = _attend(ops, case, impl, cuda_device)
    assert bool(torch.isfinite(out.float()).all())
    c = max(case.lens)
    worst = max((attn_violation(out[s : s + n], relpos_reference(case, b, c), impl), b)
                for b, (s, n) in enumerate(zip(case.starts, case.lens)))
    print(f"{impl} {name}: worst utterance {worst[1]} at {worst[0]:.3f} of the tolerance")
    assert worst[0] <= 1.0, (impl, name, worst)


def _perturbed_neighbours(case, keep_parity):
    """qkv with the K and V rows of every utterance b with b % 2 != keep_parity replaced by values of magnitude ~1e3."""
    g = torch.Generator().manual_seed(99)
    qkv, d = case.qkv.clone(), case.dim
    for b, (s, n) in enumerate(zip(case.starts, case.lens)):
        if b % 2 != keep_parity:
            qkv[s : s + n, d:] = (torch.randn((n, 2 * d), generator=g) * 1e3).to(torch.bfloat16)
    return qkv


@pytest.mark.parametrize("name", MULTI)
@pytest.mark.parametrize("impl", IMPLS)
def test_relpos_attention_masked_keys_get_zero_probability(ops, cuda_device, impl, name):
    """Keys past an utterance's end (the next utterance's rows, read by the last key block / tile) must get probability
    exactly 0: huge K and V there leave the utterance's output bits unchanged."""
    case = _case(name)
    base = _attend(ops, case, impl, cuda_device)
    for parity in (0, 1):
        out = _attend(ops, case, impl, cuda_device, qkv=_perturbed_neighbours(case, parity))
        for b, (s, n) in enumerate(zip(case.starts, case.lens)):
            if b % 2 == parity:
                assert torch.equal(out[s : s + n], base[s : s + n]), (impl, name, b)


@pytest.mark.parametrize("name", MULTI)
@pytest.mark.parametrize("impl", IMPLS)
def test_relpos_attention_utterance_alone_gives_the_same_bits(ops, cuda_device, impl, name):
    """Attended alone (its own S_center and Npad, so another window of p and other p rows per tile), an utterance gets the
    bits it gets in the mixed batch: the rows of a relative position of p hold the same bits for any S_center, and both
    kernels align their key blocks to the utterance, not to the batch."""
    case = _case(name)
    base = _attend(ops, case, impl, cuda_device)
    for b, (s, n) in enumerate(zip(case.starts, case.lens)):
        alone = _attend(ops, case, impl, cuda_device, qkv=case.qkv[s : s + n], lens=[n])
        assert torch.equal(alone, base[s : s + n]), (impl, name, b, n)


BIG_PATTERN = [1, 2, 3, 17, 64, 65, 129, 31]


def _big_case(batch):
    return make_relpos_case([BIG_PATTERN[i % len(BIG_PATTERN)] for i in range(batch)], 4, seed=5)


def _check_all(case, out, impl):
    c = max(case.lens)
    for b, (s, n) in enumerate(zip(case.starts, case.lens)):
        v = attn_violation(out[s : s + n], relpos_reference(case, b, c), impl)
        assert v <= 1.0, (impl, b, n, v)


def test_relpos_attention_wgmma_at_its_batch_capacity(ops, cuda_device):
    """2047 utterances: the wgmma kernel stages cu_seqlens and the query-tile prefix in shared memory at their capacity, and
    there are far more (utterance, tile, head) items than CTAs."""
    case = _big_case(2047)
    _check_all(case, _attend(ops, case, "wgmma", cuda_device), "wgmma")


def test_relpos_attention_2048_utterances_take_mma_sync(ops, cuda_device):
    """2048 utterances: beyond the wgmma kernel's capacity (refused), the mma.sync kernel the encoder falls back to."""
    case = _big_case(2048)
    _check_all(case, _attend(ops, case, "mma_sync", cuda_device), "mma_sync")
    with pytest.raises(ValueError, match="2047"):
        _attend(ops, case, "wgmma", cuda_device)


# ---------------------------------------------------------------------------------------------------------------------
# conv module
# ---------------------------------------------------------------------------------------------------------------------
def _conv(ops, case, device, g=None):
    g = case.g if g is None else g
    t, d = g.shape[0], g.shape[1] // 2
    buf = _guarded(t, d, device)
    out = ops.conformer_conv(g.to(device), ops.cu_seqlens_of(case.lens).to(device), case.dw.to(device),
                             case.bn_scale.to(device), case.bn_shift.to(device), out=buf[GUARD : GUARD + t])
    torch.cuda.synchronize()
    _check_guards(buf, "conformer_conv")
    return out.cpu()


@pytest.mark.parametrize("d", CONV_DIMS)
def test_conformer_conv_vs_float64_reference(ops, cuda_device, d):
    case = make_conv_case(d, seed=d)
    out = _conv(ops, case, cuda_device)
    worst = max((conv_violation(out[s : s + n], conv_reference(case, b)), n)
                for b, (s, n) in enumerate(zip(case.starts, case.lens)))
    print(f"conv D={d}: worst length {worst[1]} at {worst[0]:.3f} of the tolerance")
    assert worst[0] <= 1.0, worst


@pytest.mark.parametrize("d", CONV_DIMS)
def test_conformer_conv_halo_reads_zeros_past_utterance_ends(ops, cuda_device, d):
    case = make_conv_case(d, seed=d)
    base = _conv(ops, case, cuda_device)
    gen = torch.Generator().manual_seed(98)
    for parity in (0, 1):
        g = case.g.clone()
        for b, (s, n) in enumerate(zip(case.starts, case.lens)):
            if b % 2 != parity:
                g[s : s + n] = (torch.randn((n, 2 * d), generator=gen) * 1e3).to(torch.bfloat16)
        out = _conv(ops, case, cuda_device, g)
        for b, (s, n) in enumerate(zip(case.starts, case.lens)):
            if b % 2 == parity:
                assert torch.equal(out[s : s + n], base[s : s + n]), (d, b, n)


# ---------------------------------------------------------------------------------------------------------------------
# frontend
# ---------------------------------------------------------------------------------------------------------------------
def test_speech_frontend_vs_layer_norm(ops, cuda_device):
    """Odd frame counts drop the trailing frame (positions = frames // 2); padded_frames exceeds twice every length, and
    every frame the kernel must not read holds 1e3."""
    frames = [3, 2, 17, 129, 998, 1001, 64]
    lens = [f // 2 for f in frames]
    padded = 2 * max(lens) + 6
    g = torch.Generator().manual_seed(21)
    fb = torch.full((len(frames), padded, 80), 1e3)
    for b, n in enumerate(lens):
        fb[b, : 2 * n] = torch.randn((2 * n, 80), generator=g) * 3.0 + 0.7
    gamma = 1.0 + torch.randn(160, generator=g) * 0.1
    beta = torch.randn(160, generator=g) * 0.1
    t = sum(lens)
    buf = _guarded(t, 192, cuda_device)
    out = ops.speech_frontend(fb.to(cuda_device), ops.cu_seqlens_of(lens).to(cuda_device), gamma.to(cuda_device),
                              beta.to(cuda_device), 1e-5, out=buf[GUARD : GUARD + t])
    torch.cuda.synchronize()
    _check_guards(buf, "speech_frontend")
    out = out.cpu()
    assert not bool(out[:, 160:].float().any())  # the projection's zero K padding
    s = 0
    for b, n in enumerate(lens):
        ref = torch.nn.functional.layer_norm(fb[b, : 2 * n].reshape(n, 160), (160,), gamma, beta, 1e-5)
        got = out[s : s + n, :160].float()
        # bf16 output rounding, as test_layernorm
        assert bool(((got - ref).abs() <= ref.abs() * 2 ** -8 + 1e-5).all()), (b, float((got - ref).abs().max()))
        s += n
