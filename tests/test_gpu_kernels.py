"""Kernel-level parity tests (through the C ABI) against plain fp32 torch references of the
same op on the same bf16-rounded inputs.  Tolerances are written next to each check."""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops(native_lib, cuda_device):
    from sonar_b200 import ops as _ops

    torch.cuda.set_device(cuda_device)
    return _ops


def _rand(shape, scale, seed, device, dtype=torch.float32):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(device=device, dtype=dtype)


GEMM_SHAPES = [
    (128, 256, 64),      # one tile, one k-block
    (256, 256, 128),     # one paired tile
    (300, 512, 192),     # M tail inside a tile
    (1000, 1024, 1024),  # out-proj shape, ragged M
    (2048, 3072, 1024),  # QKV shape
    (777, 1024, 8192),   # FFN2 shape (long K), odd M
    (4096, 8192, 1024),  # FFN1 shape: more tiles than SMs -> persistent loop, smem ring wraps
    (1, 256, 64),        # single row
]


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("m,n,k", GEMM_SHAPES)
def test_gemm_bias_bf16(ops, cuda_device, cta_group, m, n, k):
    a = _rand((m, k), 1.0, 1, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 2, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 3, cuda_device)
    out = ops.gemm_bf16(a, w, bias, epilogue="bias", cta_group=cta_group)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().T + bias
    # fp32 accumulate; output rounded to bf16 (rel 2^-9) -> allow 1.5 bf16 ulps of |ref| + small abs
    err = (out.float() - ref).abs()
    tol = ref.abs() * (1.5 * 2 ** -8) + 2e-2
    assert bool((err <= tol).all()), f"max err {err.max().item()} at {err.argmax().item()}"


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gemm_relu_bf16(ops, cuda_device, cta_group):
    m, n, k = 1536, 2048, 1024
    a = _rand((m, k), 1.0, 4, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 5, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 6, cuda_device)
    out = ops.gemm_bf16(a, w, bias, epilogue="relu", cta_group=cta_group)
    ref = torch.relu(a.float() @ w.float().T + bias)
    err = (out.float() - ref).abs()
    assert bool((err <= ref.abs() * (1.5 * 2 ** -8) + 2e-2).all()), err.max().item()
    assert float(out.float().min()) >= 0.0


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("m,n,k", [(515, 1024, 1024), (2000, 1024, 8192)])
def test_gemm_residual_fp32_inplace(ops, cuda_device, cta_group, m, n, k):
    a = _rand((m, k), 1.0, 7, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 8, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 9, cuda_device)
    x = _rand((m, n), 2.0, 10, cuda_device)
    ref = x + a.float() @ w.float().T + bias
    out = ops.gemm_bf16(a, w, bias, epilogue="residual", residual=x, out=x, cta_group=cta_group)  # x += ...
    assert out.data_ptr() == x.data_ptr()
    # fp32 output: only accumulation-order differences remain
    torch.testing.assert_close(x, ref, rtol=1e-4, atol=2e-3)


SKINNY_SHAPES = [(1, 1024, 1024), (7, 3072, 1024), (16, 1024, 8192), (25, 8192, 1024), (25, 1024, 8192), (33, 1024, 1024),
                 (64, 3072, 1024), (5, 8, 256)]


@pytest.mark.parametrize("m,n,k", SKINNY_SHAPES)
@pytest.mark.parametrize("epilogue", ["bias", "relu", "silu"])
def test_gemm_skinny_rows(ops, cuda_device, m, n, k, epilogue):
    """M <= 64 goes down the weight-streaming mma.sync path (gemm_skinny.cu): the decoder's small-batch beam step and the
    speech pooler.  Same contract and tolerances as the wgmma path."""
    a = _rand((m, k), 1.0, 31, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 32, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 33, cuda_device)
    out = ops.gemm_bf16(a, w, bias, epilogue=epilogue, cta_group=0)  # 0 = automatic dispatch
    ref = a.float() @ w.float().T + bias
    if epilogue == "relu":
        ref = torch.relu(ref)
    elif epilogue == "silu":
        ref = torch.nn.functional.silu(ref)
    err = (out.float() - ref).abs()
    assert bool((err <= ref.abs() * (1.5 * 2 ** -8) + 2e-2).all()), f"max err {err.max().item()}"
    out32 = ops.gemm_bf16(a, w, bias, epilogue=epilogue, out_dtype=torch.float32, cta_group=0)
    tol = dict(rtol=1e-4, atol=2e-3) if epilogue != "silu" else dict(rtol=2e-3, atol=2e-3)  # tanh.approx in the SiLU
    torch.testing.assert_close(out32, ref, **tol)


@pytest.mark.parametrize("m,n,k", [(25, 1024, 8192), (40, 1024, 1024)])
def test_gemm_skinny_residual_inplace_and_reproducible(ops, cuda_device, m, n, k):
    a = _rand((m, k), 1.0, 34, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 35, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 36, cuda_device)
    x0 = _rand((m, n), 2.0, 37, cuda_device)
    ref = x0 + a.float() @ w.float().T + bias
    x = x0.clone()
    out = ops.gemm_bf16(a, w, bias, epilogue="residual", residual=x, out=x, cta_group=0)
    assert out.data_ptr() == x.data_ptr()
    torch.testing.assert_close(x, ref, rtol=1e-4, atol=2e-3)
    y = x0.clone()
    ops.gemm_bf16(a, w, bias, epilogue="residual", residual=y, out=y, cta_group=0)
    assert torch.equal(x, y)  # fixed reduction order across the K-split warps
    # rows are independent of the batch they sit in (beam search relies on it): row 3 alone == row 3 of the batch
    z = x0[3:4].clone()
    ops.gemm_bf16(a[3:4].contiguous(), w, bias, epilogue="residual", residual=z, out=z, cta_group=0)
    assert torch.equal(z[0], x[3])


def test_gemm_rejects_bad_shapes(ops, cuda_device):
    a = torch.zeros((8, 64), dtype=torch.bfloat16, device=cuda_device)
    w = torch.zeros((100, 64), dtype=torch.bfloat16, device=cuda_device)
    with pytest.raises(ValueError):
        ops.gemm_bf16(a, w, torch.zeros(100, device=cuda_device))


@pytest.mark.parametrize("t,d", [(1, 1024), (37, 1024), (4096, 1024), (100, 256)])
def test_layernorm(ops, cuda_device, t, d):
    x = _rand((t, d), 3.0, 11, cuda_device) + 0.7
    g = 1.0 + _rand((d,), 0.1, 12, cuda_device)
    b = _rand((d,), 0.1, 13, cuda_device)
    y = ops.layernorm(x, g, b, 1e-5)
    ref = torch.nn.functional.layer_norm(x, (d,), g, b, 1e-5)
    # bf16 output rounding: half ulp = 2^-9 relative
    assert bool(((y.float() - ref).abs() <= ref.abs() * 2 ** -8 + 1e-5).all())


ATTN_CASES = [[128] * 4, [1, 2, 17, 64, 65, 128], [200, 129, 514], [33], [128, 90, 3, 300, 514],
              [128] * 700 + [5, 77, 128, 31] * 20,  # > 2 x 132 CTAs worth of items: persistent loop
              # multi-tile sentences (online softmax across 128-key tiles) mixed with short ones, uneven item costs per CTA
              [514, 1, 256, 257, 128, 129, 383, 16, 512, 300] * 4,
              [130] * 40 + [7] * 5,
              [0, 37, 0, 0, 200, 0],  # empty sentences have no units
              [1, 3] * 4100]  # >= 8192 sentences: cu_seqlens is read from global memory instead of shared memory


@pytest.mark.parametrize("lens", ATTN_CASES)
def test_attention_vs_sdpa(ops, cuda_device, lens):
    h, hd = 16, 64
    d = h * hd
    t = sum(lens)
    qkv = _rand((t, 3 * d), 1.0, 14, cuda_device, torch.bfloat16)
    cu = ops.cu_seqlens_of(lens).to(cuda_device)
    out = ops.attention(qkv, cu, h)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out.float()).all())
    start = 0
    for i, n in enumerate(lens):
        if n == 0 or (i >= 12 and i % 97 != 0):  # an empty sentence has no rows; spot-check the long cases
            start += n
            continue
        blk = qkv[start : start + n].float()
        q, k, v = (blk[:, j * d : (j + 1) * d].view(n, h, hd).transpose(0, 1) for j in range(3))
        ref = torch.nn.functional.scaled_dot_product_attention(q[None], k[None], v[None])[0]
        ref = ref.transpose(0, 1).reshape(n, d)
        got = out[start : start + n].float()
        # P is rounded to bf16 before P.V and the output to bf16: ~2^-8 relative of |v|-scale values
        torch.testing.assert_close(got, ref, rtol=2e-2, atol=2e-2)
        start += n


def test_attention_sentence_alone_equals_its_rows_in_the_batch(ops, cuda_device):
    h, d = 16, 1024
    lens = [128, 90, 3, 300, 514]
    qkv = _rand((sum(lens), 3 * d), 1.0, 21, cuda_device, torch.bfloat16)
    cu = ops.cu_seqlens_of(lens).to(cuda_device)
    a = ops.attention(qkv, cu, h).float()
    # each sentence's rows depend on that sentence only: bitwise equal when it is attended on its own
    solo = ops.attention(qkv[128:218].contiguous(), ops.cu_seqlens_of([90]).to(cuda_device), h).float()
    assert torch.equal(solo, a[128:218])


def test_embed(ops, cuda_device):
    v, d, s = 1000, 1024, 20
    lens = [20, 3, 11]
    table = _rand((v, d), d ** -0.5, 15, cuda_device, torch.bfloat16)
    pos = _rand((s + 2, d), 1.0, 16, cuda_device)
    g = torch.Generator().manual_seed(17)
    ids = torch.randint(0, v, (len(lens), s), generator=g).to(cuda_device)
    cu = ops.cu_seqlens_of(lens).to(cuda_device)
    x = ops.embed(ids, cu, table, pos, 32.0, sum(lens))
    start = 0
    for b, n in enumerate(lens):
        ref = table[ids[b, :n]].float() * 32.0 + pos[:n]
        torch.testing.assert_close(x[start : start + n], ref, rtol=1e-6, atol=1e-6)
        start += n
    bad = ids.clone()
    bad[0, 0] = v
    with pytest.raises(ValueError):
        ops.embed(bad, cu, table, pos, 32.0, sum(lens))


# ---- reference pooling KATs (tests/unit_tests/test_sonar_pooling.py:16-68) on the GPU kernel;
#      the 2 feature columns are embedded in the first columns of a D=128 row ----
def _kat(seqs, device):
    n, s, f = seqs.shape
    full = torch.zeros((n, s, 128), device=device)
    full[:, :, :f] = seqs.to(device)
    return full


@pytest.mark.parametrize("mode,expected", [
    ("MAX", [[7.0, 4.0], [-1.0, -2.0]]),
    ("MEAN", [[5.0, 3.0], [-1.0, -2.0]]),
    ("LAST", [[3.0, 4.0], [-1.0, -2.0]]),
])
def test_pooling_kat_with_mask(native_lib, cuda_device, mode, expected):
    from sonar_b200 import B200TextEncoderModel, PaddingMask, Pooling

    seqs = torch.tensor([[[7, 2], [3, 4], [10, 20]], [[-1, -2], [100, 1000], [-10, -20]]], dtype=torch.float32)
    pm = PaddingMask(torch.tensor([2, 1]), batch_seq_len=3)
    out = B200TextEncoderModel.static_pooling(_kat(seqs, cuda_device), pm, getattr(Pooling, mode))
    torch.testing.assert_close(out[:, :2].cpu(), torch.tensor(expected))


def test_pooling_kat_no_mask(native_lib, cuda_device):
    from sonar_b200 import B200TextEncoderModel, Pooling

    seqs = torch.tensor([[[7, 2], [3, 2], [2, 20]], [[-1, -3], [-4, 2], [-7, -2]]], dtype=torch.float32)
    x = _kat(seqs, cuda_device)
    pool = B200TextEncoderModel.static_pooling
    torch.testing.assert_close(pool(x, None, Pooling.LAST)[:, :2].cpu(), torch.tensor([[2.0, 20], [-7, -2]]))
    torch.testing.assert_close(pool(x, None, Pooling.MAX)[:, :2].cpu(), torch.tensor([[7.0, 20], [-1, 2]]))
    torch.testing.assert_close(pool(x, None, Pooling.MEAN)[:, :2].cpu(), torch.tensor([[4.0, 8], [-4, -1]]))


def test_ln_pool_matches_torch(ops, cuda_device):
    d = 1024
    lens = [5, 128, 1, 77]
    x = _rand((sum(lens), d), 2.0, 18, cuda_device)
    g = 1.0 + _rand((d,), 0.1, 19, cuda_device)
    b = _rand((d,), 0.1, 20, cuda_device)
    cu = ops.cu_seqlens_of(lens).to(cuda_device)
    out, enc = ops.pool_packed(x, cu, "mean", gamma=g, beta=b, encoded_seq_len=128)
    y = torch.nn.functional.layer_norm(x, (d,), g, b, 1e-5)
    start = 0
    for i, n in enumerate(lens):
        ref = y[start : start + n].sum(0) * (1.0 / (torch.tensor(float(n)) + 1e-7)).item()
        torch.testing.assert_close(out[i], ref, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(enc[i, :n], y[start : start + n], rtol=1e-5, atol=1e-5)
        assert float(enc[i, n:].abs().max()) == 0.0 if n < 128 else True
        start += n


# ------------------------------------------------------------------------------------------------
# LayerNorm folded into the GEMMs (LnFold): residual GEMM that emits statistics, consumer GEMM that applies them
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,k", [(1000, 1024), (4096, 8192), (300, 256), (77, 1024)])
def test_gemm_residual_stats(ops, cuda_device, m, k):
    """x += a.W^T + b (fp32, in place) with the bf16 copy and the (mean, M2) partials of the NEW rows: partial 2t + g covers
    column half g (128 columns) of 256-column tile t.
    The rows get a large common offset (mean >> std) so a sum-of-squares style variance would visibly cancel."""
    n = 1024
    a = _rand((m, k), 1.0, 31, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 32, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 33, cuda_device)
    x0 = _rand((m, n), 1.0, 34, cuda_device) + 40.0
    x = x0.clone()
    h, stats = ops.gemm_residual_stats(a, w, bias, x)
    torch.cuda.synchronize()
    ref = x0.double() + a.double() @ w.double().T + bias.double()
    torch.testing.assert_close(x.double(), ref, rtol=1e-5, atol=2e-3)  # fp32 accumulate over K products + fp32 add
    assert torch.equal(h, x.to(torch.bfloat16))                       # the bf16 copy is the rounding of what was stored
    xc = x.double().view(m, n // 128, 128)  # [row, 2t + g, 128]
    torch.testing.assert_close(stats[..., 0].double(), xc.mean(-1), rtol=1e-6, atol=1e-5)
    m2 = ((xc - xc.mean(-1, keepdim=True)) ** 2).sum(-1)
    torch.testing.assert_close(stats[..., 1].double(), m2, rtol=2e-5, atol=1e-4)


# ------------------------------------------------------------------------------------------------
# ordered split-K of the accumulate epilogue (the decoder's residual GEMMs at 2 560 hypothesis rows)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,n,k", [(2560, 1024, 8192),   # config 4: 40 tile pairs -> 3 K slices
                                   (2560, 1024, 1024),   # too little K per slice: not split
                                   (2500, 512, 4096),    # ragged last row tile, 20 tile pairs
                                   (700, 256, 2048),     # 3 tile pairs -> 4 slices
                                   (40000, 1024, 8192)])  # plenty of tiles: plain accumulate epilogue
def test_gemm_residual_splitk(ops, cuda_device, m, n, k):
    """x += a.W^T + b through the split-K path: right value, the SAME bits on every run (the slices add in a fixed order),
    hand-over counters back at zero, and x rows beyond M untouched."""
    a = _rand((m, k), 1.0, 51, cuda_device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 52, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 53, cuda_device)
    x0 = _rand((m + 3, n), 1.0, 54, cuda_device)
    counters = torch.zeros(4 * ((m + 255) // 256) * (n // 256) + 8, dtype=torch.int32, device=cuda_device)
    ref = x0[:m].double() + a.double() @ w.double().T + bias.double()
    runs = []
    for _ in range(4):
        x = x0.clone()
        ops.gemm_residual_splitk(a, w, bias, x[:m], counters)
        torch.cuda.synchronize()
        assert int(counters.abs().sum()) == 0
        assert torch.equal(x[m:], x0[m:])
        torch.testing.assert_close(x[:m].double(), ref, rtol=1e-5, atol=2e-3)
        runs.append(x)
    assert all(torch.equal(runs[0], r) for r in runs[1:])
    # against the unsplit accumulate epilogue: same products, another summation order
    y = x0[:m].clone()
    ops.gemm_bf16(a, w, bias, epilogue="residual", residual=y, out=y)
    torch.testing.assert_close(runs[0][:m], y, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("m,n,k", [(1000, 3072, 1024), (2048, 8192, 1024), (130, 512, 512)])
def test_gemm_ln_consumer_equals_layernorm_then_linear(ops, cuda_device, relu, m, n, k):
    """rstd * (bf16(x).Wf^T - mean * colsum) + bias_f  ==  LN(x; gamma, beta).W^T + b  (fp32 reference), with gamma/beta far
    from (1, 0) and rows whose mean is comparable to their spread."""
    x = _rand((m, k), 2.0, 41, cuda_device) + _rand((m, 1), 1.5, 42, cuda_device)
    gamma = 1.0 + _rand((k,), 0.5, 43, cuda_device)
    beta = _rand((k,), 0.5, 44, cuda_device)
    w = _rand((n, k), 1.0 / math.sqrt(k), 45, cuda_device, torch.bfloat16)
    bias = _rand((n,), 0.5, 46, cuda_device)
    wf, colsum, bias_f = ops.fold_layernorm(w, bias, gamma, beta)
    torch.testing.assert_close(wf.float(), (w.float() * gamma).to(torch.bfloat16).float(), rtol=0, atol=0)
    torch.testing.assert_close(colsum, wf.float().sum(1), rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(bias_f, bias + w.float() @ beta, rtol=1e-5, atol=1e-4)
    # statistics as a producer would emit them: (mean, M2) of 128-column subsets (any partition merges to the same result)
    xc = x.double().view(m, k // 128, 128)
    stats = torch.stack([xc.mean(-1), ((xc - xc.mean(-1, keepdim=True)) ** 2).sum(-1)], -1).float().contiguous()
    out = ops.gemm_ln_consumer(x.to(torch.bfloat16), wf, bias_f, colsum, stats, 1e-5, relu=relu)
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x, (k,), gamma, beta, 1e-5) @ w.float().T + bias
    if relu:
        ref = torch.relu(ref)
    # bf16 rounding of x (instead of LN(x)) and of W*gamma: same 2^-9 relative operand error as the unfused path, summed over
    # K products of magnitude ~ |LN(x)| |W| -> a few 1e-2 absolute on outputs of magnitude ~1.5
    err = (out.float() - ref).abs()
    tol = ref.abs() * (1.5 * 2 ** -8) + 4e-2
    assert bool((err <= tol).all()), f"max err {err.max().item()}"
    assert float(err.mean()) < 6e-3
