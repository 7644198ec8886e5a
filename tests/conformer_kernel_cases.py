"""Inputs, float64 references and tolerances of the Conformer kernel tests.

``tests/test_gpu_conformer_kernels.py`` compares the relative-position attention kernels and the conv-module kernel with
these references; ``tests/test_conformer_kernel_references.py`` checks on the same inputs, without a GPU, that known
position, bias, mask and halo bugs miss these tolerances by far.
The references are the pinned oracle's own functions (``oracle.speech_encoder.relpos_attention`` / ``conv_module_middle``)
run in float64 on the packed bf16 inputs, so the kernel contract "row S_center - 1 - i + j of p is relative position
i - j" is checked against the convention the oracle shares with HuggingFace.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from oracle.speech_encoder import conv_module_middle, relpos_attention
from sonar_b200.speech_encoder import relative_position_table, relpos_rows

HD = 64  # head dim of both attention kernels
CONV_TAPS = 31

# ---------------------------------------------------------------------------------------------------------------------
# relative-position attention
# ---------------------------------------------------------------------------------------------------------------------
# Batches (one list = one call) on the tile edges of both kernels: 64-key blocks (mma.sync), 128-query and 128-key tiles
# (wgmma), and the windows of p they read; mixed batches whose S_center is set by a longer neighbour; one utterance of
# > 1000 positions (the mma.sync 256-row ring of p wraps many times and the wgmma window starts before row 0 and ends past
# Npad).  (lens, heads)
ATTN_CASES = {
    "1": ([1], 16),
    "2": ([2], 16),
    "63-65": ([63, 64, 65], 16),
    "127-129": ([127, 128, 129], 16),
    "255-257": ([255, 256, 257], 16),
    "499": ([499], 16),
    "1031": ([1031], 16),
    "mixed": ([17, 300, 1, 129, 64, 2, 191], 16),
    "mixed-long": ([5, 1031, 130, 63, 256], 16),
    "d256": ([63, 64, 65, 200, 1, 129], 4),
}

# Element-wise |got - ref| <= ATTN_RTOL |ref| + atol and mean |got - ref| <= mean bound, per kernel.  ATTN_RTOL covers the
# bf16 rounding of the output (half an ulp: up to 2^-8 relative).  The absolute terms cover the bf16 rounding of the
# unnormalised probabilities before P.V (both kernels) and, for wgmma, of q + u and q + v before the two products: with
# q, k, v ~ N(0, 1) and position and content terms of equal spread, |out| stays below about 1.5.
ATTN_RTOL = 2.0 ** -8
ATTN_TOL = {"mma_sync": (1.0e-2, 2.5e-3), "wgmma": (1.5e-2, 3.0e-3)}  # (atol, mean bound)


@dataclass
class RelposCase:
    lens: List[int]
    heads: int
    qkv: torch.Tensor     # bf16 [T, 3D]  q | k | v, packed rows
    u_bias: torch.Tensor  # fp32 [D]
    v_bias: torch.Tensor  # fp32 [D]
    table: torch.Tensor   # bf16 [2 Smax - 1, D]: row k = r_proj of relative position Smax - 1 - k

    @property
    def dim(self) -> int:
        return HD * self.heads

    @property
    def starts(self) -> List[int]:
        out, s = [], 0
        for n in self.lens:
            out.append(s)
            s += n
        return out

    def p(self, s_center: int) -> torch.Tensor:
        """bf16 [relpos_rows(s_center), D]: the table of a batch whose longest utterance has s_center positions; the rows of
        a relative position hold the same bits whatever s_center is."""
        smax = max(self.lens)
        out = torch.zeros((relpos_rows(s_center), self.dim), dtype=torch.bfloat16)
        out[: 2 * s_center - 1] = self.table[smax - s_center : smax + s_center - 1]
        return out


def make_relpos_case(lens: List[int], heads: int, seed: int = 0) -> RelposCase:
    """q, k, v ~ N(0, 1) and u, v ~ N(0, 0.5) in bf16 / fp32; p = bf16 of the float64 product of the relative-position
    table with an r_proj scaled so that p has unit spread, like k: the position term (q + v).p then varies as much as the
    content term (q + u).k, so a wrong offset, sign or bias moves the scores by as much as the content does."""
    g = torch.Generator().manual_seed(seed)
    d, smax = HD * heads, max(lens)
    qkv = torch.randn((sum(lens), 3 * d), generator=g).to(torch.bfloat16)
    u = torch.randn(d, generator=g) * 0.5
    v = torch.randn(d, generator=g) * 0.5
    wr = torch.randn((d, d), generator=g, dtype=torch.float64)
    rel = relative_position_table(smax, d, 2 * smax - 1).double() @ wr.T
    return RelposCase(list(lens), heads, qkv, u, v, (rel / rel.std()).to(torch.bfloat16))


def relpos_reference(case: RelposCase, b: int, s_center: int, *, row_shift: int = 0, flip: bool = False,
                     drop_u: bool = False, drop_v: bool = False, drop_position: bool = False,
                     mask_last_key: bool = False) -> torch.Tensor:
    """float64 [n, D] attention output of utterance b as the kernels see it (p of a batch with S_center = s_center).  The
    keyword arguments inject the bugs the tests must be able to see: read p `row_shift` rows off (an off-by-one
    Transformer-XL shift or S_center), relative position i - j read as j - i, a bias or the whole position term
    dropped, the utterance's last key masked."""
    n, d, h = case.lens[b], case.dim, case.heads
    rows = case.qkv[case.starts[b] : case.starts[b] + n].double()
    q, k, v = (rows[:, j * d : (j + 1) * d].view(1, n, h, HD) for j in range(3))
    p = case.p(s_center).double()
    # the oracle's r row m (relative position n - 1 - m) is row m + s_center - n of p; rows outside p read as zero
    idx = torch.arange(2 * n - 1) + (s_center - n + row_shift)
    inside = (idx >= 0) & (idx < p.shape[0])
    r = torch.zeros((2 * n - 1, d), dtype=torch.float64)
    r[inside] = p[idx[inside]]
    if flip:
        r = r.flip(0)
    if drop_position:
        r.zero_()
    u = torch.zeros(d, dtype=torch.float64) if drop_u else case.u_bias.double()
    vb = torch.zeros(d, dtype=torch.float64) if drop_v else case.v_bias.double()
    key_ok = torch.ones((1, n), dtype=torch.bool)
    if mask_last_key:
        key_ok[0, -1] = False
    return relpos_attention(q, k, v, r.view(2 * n - 1, h, HD), u.view(h, HD), vb.view(h, HD), key_ok)[0]


def attn_violation(got: torch.Tensor, ref: torch.Tensor, impl: str) -> float:
    """How far `got` is from `ref` in units of the tolerance of `impl` (<= 1 passes)."""
    atol, mean_bound = ATTN_TOL[impl]
    err = (got.double() - ref.double()).abs()
    return max(float((err / (ATTN_RTOL * ref.double().abs() + atol)).max()), float(err.mean()) / mean_bound)


# ---------------------------------------------------------------------------------------------------------------------
# conv module: GLU -> depthwise conv (31 taps) -> BatchNorm scale / shift -> SiLU
# ---------------------------------------------------------------------------------------------------------------------
# Lengths on the 15-position halo at the 64-position tile edges and at both ends of an utterance, packed in one batch.
CONV_LENS = [1, 2, 15, 16, 17, 31, 63, 64, 65, 79, 80, 128, 499, 1000]
CONV_DIMS = [256, 1024]
# bf16 rounding of the output (half an ulp: up to 2^-8 relative) + the tanh.approx sigmoid of the GLU and of the SiLU (absolute
# error ~ 2^-11 of values of order 1, summed over 31 taps of std 0.2)
CONV_RTOL, CONV_ATOL, CONV_MEAN = 2.0 ** -8, 4.0e-3, 1.5e-3


@dataclass
class ConvCase:
    lens: List[int]
    g: torch.Tensor         # bf16 [T, 2D]  value | gate
    dw: torch.Tensor        # fp32 [D, 31]
    bn_scale: torch.Tensor  # fp32 [D]
    bn_shift: torch.Tensor  # fp32 [D]

    @property
    def starts(self) -> List[int]:
        out, s = [], 0
        for n in self.lens:
            out.append(s)
            s += n
        return out


def make_conv_case(d: int, lens: Optional[List[int]] = None, seed: int = 0) -> ConvCase:
    g = torch.Generator().manual_seed(seed)
    lens = list(lens or CONV_LENS)
    x = torch.randn((sum(lens), 2 * d), generator=g).to(torch.bfloat16)
    dw = torch.randn((d, CONV_TAPS), generator=g) * 0.2  # no symmetry: reversed taps give another result
    scale = 1.0 + torch.randn(d, generator=g) * 0.3
    shift = torch.randn(d, generator=g) * 0.5
    return ConvCase(lens, x, dw, scale, shift)


def conv_rows_reference(case: ConvCase, g_rows: torch.Tensor, dw: Optional[torch.Tensor] = None) -> torch.Tensor:
    """float64 [n, D] conv module middle of the rows g_rows (bf16 [n, 2D]) as one utterance, zero outside it.  BatchNorm
    with mean 0 and variance 1 - eps (+ eps = 1 exactly in float64) is exactly the folded scale / shift."""
    dw = case.dw if dw is None else dw
    d, eps = dw.shape[0], 2.0 ** -30
    zeros, var = torch.zeros(d, dtype=torch.float64), torch.full((d,), 1.0 - eps, dtype=torch.float64)
    y = conv_module_middle(g_rows.double().T[None], dw.double()[:, None, :], zeros, var, case.bn_scale.double(),
                           case.bn_shift.double(), eps)
    return y[0].T


def conv_reference(case: ConvCase, b: int, *, reverse_taps: bool = False, tile_halo_cut: bool = False,
                   neighbour_halo: bool = False) -> torch.Tensor:
    """float64 [n, D] for utterance b, with optional bugs: taps reversed; positions of each 64-position tile convolved
    without the halo from the neighbouring tiles; the halo reading the neighbouring packed utterances instead of zeros."""
    n, s = case.lens[b], case.starts[b]
    dw = case.dw.flip(1) if reverse_taps else None
    if tile_halo_cut:
        return torch.cat([conv_rows_reference(case, case.g[s + t : s + min(t + 64, n)], dw) for t in range(0, n, 64)])
    if neighbour_halo:
        h = CONV_TAPS // 2
        lo, hi = max(0, s - h), min(case.g.shape[0], s + n + h)
        return conv_rows_reference(case, case.g[lo:hi], dw)[s - lo : s - lo + n]
    return conv_rows_reference(case, case.g[s : s + n], dw)


def conv_violation(got: torch.Tensor, ref: torch.Tensor) -> float:
    err = (got.double() - ref.double()).abs()
    return max(float((err / (CONV_RTOL * ref.double().abs() + CONV_ATOL)).max()), float(err.mean()) / CONV_MEAN)
