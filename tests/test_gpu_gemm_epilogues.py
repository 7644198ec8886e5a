"""The wgmma GEMM's column-wise epilogues (bias, ReLU, SiLU, residual, in-place accumulate) in both output types.

Every epilogue of one (A, W) pair runs the same main loop, so its accumulators are the same bits: the fp32 bias output
is fl(acc + bias) itself, and the others must be exactly what that value turns into -- rounded to bf16, clamped by the
ReLU, or added to the residual.  Any element written to the wrong place or rounded twice shows up as a mismatch."""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu

# (M tail inside a tile) and (more tiles than clusters: the persistent loop and the staging buffers wrap across tiles)
SHAPES = [(1000, 1024, 1024), (4096, 2048, 256)]


@pytest.fixture(scope="module")
def ops(native_lib, cuda_device):
    from sonar_b200 import ops as _ops

    torch.cuda.set_device(cuda_device)
    return _ops


def _rand(shape, scale, seed, device, dtype=torch.float32):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(device=device, dtype=dtype)


def _operands(m, n, k, device):
    a = _rand((m, k), 1.0, 41, device, torch.bfloat16)
    w = _rand((n, k), 1.0 / math.sqrt(k), 42, device, torch.bfloat16)
    bias = _rand((n,), 0.5, 43, device)
    return a, w, bias


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("m,n,k", SHAPES)
def test_gemm_epilogues_agree_bitwise(ops, cuda_device, cta_group, m, n, k):
    a, w, bias = _operands(m, n, k, cuda_device)
    y = ops.gemm_bf16(a, w, bias, epilogue="bias", out_dtype=torch.float32, cta_group=cta_group)  # fl(acc + bias)
    ref = a.float() @ w.float().T + bias
    torch.testing.assert_close(y, ref, rtol=1e-4, atol=2e-3)
    assert torch.equal(ops.gemm_bf16(a, w, bias, epilogue="bias", cta_group=cta_group), y.to(torch.bfloat16))
    assert torch.equal(ops.gemm_bf16(a, w, bias, epilogue="relu", cta_group=cta_group), torch.relu(y).to(torch.bfloat16))
    assert torch.equal(ops.gemm_bf16(a, w, bias, epilogue="relu", out_dtype=torch.float32, cta_group=cta_group),
                       torch.relu(y))
    # residual, not aliased: fp32 and bf16 (the bf16 residual is added in fp32, then rounded)
    r32 = _rand((m, n), 2.0, 44, cuda_device)
    out = ops.gemm_bf16(a, w, bias, epilogue="residual", residual=r32, out_dtype=torch.float32, cta_group=cta_group)
    assert torch.equal(out, y + r32)
    r16 = r32.to(torch.bfloat16)
    out = ops.gemm_bf16(a, w, bias, epilogue="residual", residual=r16, cta_group=cta_group)
    assert torch.equal(out, (y + r16.float()).to(torch.bfloat16))
    # x += a w^T + b in place: the add happens in L2, fl32(x + fl32(acc + bias))
    x = r32.clone()
    ops.gemm_bf16(a, w, bias, epilogue="residual", residual=x, out=x, cta_group=cta_group)
    assert torch.equal(x, r32 + y)


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("m,n,k", SHAPES)
def test_gemm_silu(ops, cuda_device, cta_group, m, n, k):
    a, w, bias = _operands(m, n, k, cuda_device)
    ref = torch.nn.functional.silu(a.float() @ w.float().T + bias)
    out = ops.gemm_bf16(a, w, bias, epilogue="silu", cta_group=cta_group)
    err = (out.float() - ref).abs()
    assert bool((err <= ref.abs() * (1.5 * 2 ** -8) + 2e-2).all()), f"max err {err.max().item()}"
    out32 = ops.gemm_bf16(a, w, bias, epilogue="silu", out_dtype=torch.float32, cta_group=cta_group)
    torch.testing.assert_close(out32, ref, rtol=2e-3, atol=2e-3)  # tanh.approx in the SiLU
    assert torch.equal(out, out32.to(torch.bfloat16))
