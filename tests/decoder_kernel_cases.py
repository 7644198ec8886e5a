"""Inputs, float64 references and tolerances of the decoder step's kernel tests.

``tests/test_gpu_decoder_kernels.py`` compares the KV-cache attention, the vocabulary head (top-16 / log-sum-exp sweep
and merge), the embedding and the add + LayerNorm kernels with these references; ``tests/test_decoder_kernel_references.py``
checks without a GPU that the references are the oracle's maths and that known indexing, masking, merge and tie bugs
miss these tolerances.  Every reference runs in float64 on the same bf16 / fp32 inputs the kernel gets, on whatever
device those inputs live.
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional

import torch

from oracle.text_decoder import attention_core

HD = 64      # head dim of the decoder
PASS = 16    # keys per pass of decode_attention_kernel (four 8-lane groups x 4)
TOPK = 16
BIG_VOCAB = 256206  # SONAR's vocabulary: 1001 tiles of 256 columns, the last one 206 wide

# ---------------------------------------------------------------------------------------------------------------------
# KV-cache attention
# ---------------------------------------------------------------------------------------------------------------------
# Positions on the pass edges (16 keys per pass, 4 per 8-lane group) and the longest the step accepts.
ATTN_POSITIONS = [0, 1, 3, 4, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511]
ATTN_HEADS = [4, 8, 16]
# Per head h % 4: score spread at position 0 and its growth to position t.  q ~ N(0, 1) and k scaled by s(p) give scores
# q.k/8 of spread s(p): a near-uniform head, a flat one, and two whose largest scores sit late in the sweep (the last
# one reaches about +-60), so the maximum falls in whichever 8-lane group owns one of the last keys.
HEAD_SCALES = [(1.0, 0.0), (0.3, 0.0), (1.0, 3.0), (4.0, 3.0)]

# |got - ref| <= ATTN_RTOL |ref| + ATTN_ATOL * max|v| element-wise, and
# mean |got - ref| <= ATTN_RTOL / 2 * mean |ref| + ATTN_MEAN * max|v|.
# ATTN_RTOL is the bf16 rounding of the output (half an ulp: up to 2^-8 relative, about half that on average); the fp32
# online softmax and the exp2f of the kernel stay far below the absolute terms.  Measured on an H100 80GB HBM3 (700 W)
# over the 202 cases of the GPU test: at most 0.71 of this tolerance (R = 2560, H = 4, t = 511), max |err| 1.6e-2 on
# outputs of up to about 4, mean |err| at most 1.1e-3.
ATTN_RTOL, ATTN_ATOL, ATTN_MEAN = 2.0 ** -8, 1.0e-3, 2.5e-4


@dataclass
class AttnCase:
    heads: int
    t: int
    qkv: torch.Tensor     # bf16 [R, 3D]  q | k | v of position t
    kcache: torch.Tensor  # bf16 [R, Tmax, D]; NaN wherever the reference reads nothing
    vcache: torch.Tensor
    table: torch.Tensor   # int32 [R, Tmax]

    @property
    def dim(self) -> int:
        return HD * self.heads

    @property
    def rows(self) -> int:
        return self.qkv.shape[0]


def _head_scale(heads: int, positions: torch.Tensor, t: int) -> torch.Tensor:
    """fp32 [len(positions), D] factor of k at each position, per head (HEAD_SCALES)."""
    base = torch.tensor([HEAD_SCALES[h % 4][0] for h in range(heads)])
    ramp = torch.tensor([HEAD_SCALES[h % 4][1] for h in range(heads)])
    s = base[None, :] * (1.0 + ramp[None, :] * positions.float()[:, None].cpu() / max(t, 1))
    return s.repeat_interleave(HD, 1).to(positions.device)


def make_attention_case(rows: int, heads: int, t: int, *, tmax: Optional[int] = None, table: str = "random",
                        seed: int = 0, device="cpu") -> AttnCase:
    """Random q, k, v (k scaled per HEAD_SCALES) and an ancestry table that points at any row ("random") or at the row
    itself ("identity").  Only the cache entries (table[r, t'], t') with t' < t hold values; every other entry is NaN, so
    a kernel that reads one of them returns NaN.  tmax defaults to t + 2 (a NaN position past t)."""
    g = torch.Generator(device=device).manual_seed(seed)
    d = HD * heads
    tmax = t + 2 if tmax is None else tmax
    qkv = torch.randn((rows, 3 * d), generator=g, device=device)
    qkv[:, d : 2 * d] *= _head_scale(heads, torch.tensor([t], device=device), t)
    qkv = qkv.to(torch.bfloat16)
    if table == "identity":
        tab = torch.arange(rows, dtype=torch.int32, device=device)[:, None].expand(rows, tmax).contiguous()
    else:
        tab = torch.randint(0, rows, (rows, tmax), generator=g, device=device, dtype=torch.int32)
    kc = torch.full((rows, tmax, d), float("nan"), dtype=torch.bfloat16, device=device)
    vc = torch.full_like(kc, float("nan"))
    if t > 0:
        pos = torch.arange(t, device=device)
        src = tab[:, :t].long()
        k = torch.randn((rows, t, d), generator=g, device=device) * _head_scale(heads, pos, t)[None]
        v = torch.randn((rows, t, d), generator=g, device=device)
        kc[src, pos[None, :].expand(rows, t)] = k.to(torch.bfloat16)
        vc[src, pos[None, :].expand(rows, t)] = v.to(torch.bfloat16)
    return AttnCase(heads, t, qkv, kc, vc, tab)


def attention_reference(case: AttnCase, *, table_shift: bool = False, drop_last_key: bool = False,
                        drop_pass: Optional[int] = None, chunk: int = 128) -> torch.Tensor:
    """float64 [R, D]: softmax(q . k / 8) . v over positions 0..t of each hypothesis, position t' < t read from cache row
    table[r, t'], position t from qkv.  The keywords inject the bugs the tests must see: the table read one position
    late (position t' from the row of t' - 1), the current key left out, the keys of one 16-key pass left out."""
    t, d, h = case.t, case.dim, case.heads
    out = []
    for r0 in range(0, case.rows, chunk):
        qkv = case.qkv[r0 : r0 + chunk].double()
        n = qkv.shape[0]
        pos = torch.arange(t, device=qkv.device)
        col = (pos - 1).clamp(min=0) if table_shift else pos
        src = case.table[r0 : r0 + chunk][:, col].long()
        kk = torch.cat([case.kcache[src, pos[None, :].expand(n, t)].double(), qkv[:, None, d : 2 * d]], 1)
        vv = torch.cat([case.vcache[src, pos[None, :].expand(n, t)].double(), qkv[:, None, 2 * d :]], 1)
        keep = torch.ones(t + 1, dtype=torch.bool, device=qkv.device)
        if drop_last_key:
            keep[t] = False
        if drop_pass is not None:
            keep[PASS * drop_pass : PASS * (drop_pass + 1)] = False
        mask = torch.zeros((1, t + 1), dtype=torch.float64, device=qkv.device).masked_fill(~keep, -math.inf)
        q = qkv[:, :d].view(n, h, 1, HD)
        k = kk.view(n, t + 1, h, HD).transpose(1, 2)
        v = vv.view(n, t + 1, h, HD).transpose(1, 2)
        out.append(attention_core(q, k, v, mask)[:, 0])
    return torch.cat(out)


def attn_violation(got: torch.Tensor, ref: torch.Tensor, vmax: float) -> float:
    """How far `got` is from `ref` in units of the tolerance (<= 1 passes); vmax = the largest |v| of the case.  A NaN
    (a read of a cache entry the table does not name) is infinitely far."""
    if not bool(torch.isfinite(got).all()):
        return math.inf
    err = (got.double() - ref.double()).abs()
    mag = ref.double().abs()
    return max(float((err / (ATTN_RTOL * mag + ATTN_ATOL * vmax)).max()),
               float(err.mean()) / (0.5 * ATTN_RTOL * float(mag.mean()) + ATTN_MEAN * vmax))


def value_max(case: AttnCase) -> float:
    v = case.vcache.float()
    return max(float(v[torch.isfinite(v)].abs().max()) if case.t > 0 else 0.0,
               float(case.qkv[:, 2 * case.dim :].float().abs().max()))


# ---------------------------------------------------------------------------------------------------------------------
# vocabulary head
# ---------------------------------------------------------------------------------------------------------------------
HEAD_DIM = 256         # D of the exact-operand cases (a multiple of 64 = the GEMM's k-block)
EOS = 3
# |lprob - ref| of the exact-operand cases: the logits are exact in fp32, what is left is the fp32 log-sum-exp (__expf of
# each column, fp32 sums per list and across lists, logf) and the fp32 subtraction.  Measured on an H100 80GB HBM3
# (700 W) over all 60 cases the GPU test runs: at most 3.5e-6.
HEAD_EXACT_TOL = 1.0e-5
# Gaussian h at LayerNorm scale, E at the synthetic weights' scale, D = 1024: the bf16 products summed in fp32 as well.
# Measured (same card, 2560 rows, V = 256 206): at most 8.2e-6.
HEAD_REAL_TOL = 3.0e-5


def probe_tokens(rows: int, vocab: int, device="cpu") -> torch.Tensor:
    """0, V - 1, and the out-of-range ids -1 and V (scored as token 0) in turn."""
    return torch.tensor([0, vocab - 1, -1, vocab], dtype=torch.int64, device=device).repeat((rows + 3) // 4)[:rows]


def tie_tokens(vocab: int) -> List[int]:
    """Tokens that share one value in the tie row: spread over the first and last chunks, both column halves of a tile
    and the ragged last tile (its full piece, its partial piece); V - 1 holds that row's unique maximum."""
    last = (vocab - 1) // 256 * 256
    cand = [1, 2, 130, 255, 256, 300, 4000, 4100, vocab // 3, vocab // 2, vocab // 2 + 129, vocab - 300,
            last - 1, last, last + 1, last + 77, last + 127, last + 128, last + 130, last + 150, last + 191, last + 192,
            last + 200, vocab - 2]
    return sorted({c for c in cand if 0 <= c < vocab - 1 and c != EOS})


def make_exact_head(rows: int, vocab: int, seed: int = 0, device="cpu"):
    """(h bf16 [rows, D], E bf16 [vocab, D], big_token): integers times 2^-2 (h) and 2^-3 (E), so every partial sum of a
    logit is exact in fp32 and the expected top-16 is exact, ties included.
      row 0: the tie row -- logits = column D - 2 of E: 2 at V - 1, 1 at tie_tokens(V), at most 3/8 elsewhere;
      row 1: h = 0 -- all V logits equal (expect tokens 0..15, log-prob -log V);
      row 2: random, plus the single logit 200 above the rest (column D - 1 of E, zero except at big_token);
      rows 3..: random (column D - 1 of h zero)."""
    g = torch.Generator(device=device).manual_seed(seed)
    d = HEAD_DIM
    h = torch.randint(-3, 4, (rows, d), generator=g, device=device).float() * 0.25
    e = torch.randint(-3, 4, (vocab, d), generator=g, device=device).float() * 0.125
    big = vocab // 3 + 1
    e[:, d - 1] = 0.0
    e[big, d - 1] = 200.0
    e[torch.tensor(tie_tokens(vocab), device=device, dtype=torch.long), d - 2] = 1.0
    e[vocab - 1, d - 2] = 2.0
    if EOS < vocab - 1:
        e[EOS, d - 2] = -1.0  # EOS outside the tie row's top 16
    h[:, d - 1] = 0.0
    h[0] = 0.0
    h[0, d - 2] = 1.0
    if rows > 1:
        h[1] = 0.0
    if rows > 2:
        h[2, d - 1] = 1.0
    return h.to(torch.bfloat16), e.to(torch.bfloat16), big


def make_real_head(rows: int, vocab: int = BIG_VOCAB, d: int = 1024, seed: int = 0, device="cpu"):
    """h ~ N(0, 1) (a LayerNorm output), E ~ N(0, 1/d) (the synthetic decoder weights), both bf16."""
    g = torch.Generator(device=device).manual_seed(seed)
    h = torch.randn((rows, d), generator=g, device=device).to(torch.bfloat16)
    e = (torch.randn((vocab, d), generator=g, device=device) / math.sqrt(d)).to(torch.bfloat16)
    return h, e


def topk_lists(vocab: int, n_chunks: int) -> List[torch.Tensor]:
    """The columns of each candidate list of gemm_bf16_topk: list 2c + g = column half g of the tiles of n-chunk c."""
    tiles = (vocab + 255) // 256
    tpc = (tiles + n_chunks - 1) // n_chunks
    out = []
    for c in range(n_chunks):
        for g in range(2):
            cols = [torch.arange(256 * tt + 128 * g, min(256 * tt + 128 * (g + 1), vocab))
                    for tt in range(c * tpc, min((c + 1) * tpc, tiles)) if 256 * tt + 128 * g < vocab]
            out.append(torch.cat(cols) if cols else torch.zeros(0, dtype=torch.long))
    return out


def head_reference(h: torch.Tensor, e: torch.Tensor, eos: int, probes: Optional[torch.Tensor] = None, *,
                   lse_skip: Optional[torch.Tensor] = None, drop: Optional[torch.Tensor] = None,
                   ties_descending: bool = False, chunk: int = 256):
    """float64 (lprob [R, 16], tok int64 [R, 16], eos [R], probe [R] or None, logits-minus-lse of every token [R, V] is not
    kept).  Top 16 by (value desc, token asc); fewer than 16 tokens pad with (-inf, -1); an out-of-range probe scores
    token 0.  Bugs: lse_skip = columns left out of the log-sum-exp, drop = bool [R, V] of columns that are no candidates
    (a dropped list), ties broken by token descending."""
    v = e.shape[0]
    k = min(TOPK, v)
    lps, toks, eoss, prs = [], [], [], []
    ef = e.double()
    for r0 in range(0, h.shape[0], chunk):
        logits = h[r0 : r0 + chunk].double() @ ef.T
        n = logits.shape[0]
        kept = logits if lse_skip is None else logits.index_fill(1, lse_skip.to(logits.device), -math.inf)
        lse = torch.logsumexp(kept, 1, keepdim=True)
        cand = logits if drop is None else logits.masked_fill(drop[r0 : r0 + chunk].to(logits.device), -math.inf)
        if ties_descending:
            order = v - 1 - torch.sort(-cand.flip(1), dim=1, stable=True).indices[:, :k]
        else:
            order = torch.sort(-cand, dim=1, stable=True).indices[:, :k]
        lp = torch.gather(logits, 1, order) - lse
        if k < TOPK:
            pad = TOPK - k
            lp = torch.cat([lp, torch.full((n, pad), -math.inf, dtype=lp.dtype, device=lp.device)], 1)
            order = torch.cat([order, torch.full((n, pad), -1, dtype=order.dtype, device=order.device)], 1)
        lps.append(lp)
        toks.append(order)
        eoss.append(logits[:, eos] - lse[:, 0])
        if probes is not None:
            p = probes[r0 : r0 + chunk].to(logits.device)
            p = torch.where((p < 0) | (p >= v), torch.zeros_like(p), p)
            prs.append(torch.gather(logits, 1, p[:, None])[:, 0] - lse[:, 0])
    return torch.cat(lps), torch.cat(toks), torch.cat(eoss), (torch.cat(prs) if probes is not None else None)


# ---------------------------------------------------------------------------------------------------------------------
# embedding and add + LayerNorm
# ---------------------------------------------------------------------------------------------------------------------
LN_DIMS = [256, 1024]
LN_BEAMS = [1, 3, 5]
LN_ROWS = 37            # not a multiple of the kernel's 8 rows per CTA
LN_OFFSET = 1.0e3       # every row of x sits about 1e3 away from zero: the mean must be taken out before the variance
LN_EPS = 1.0e-5


def make_ln_case(rows: int, beam: int, d: int, seed: int = 0, device="cpu"):
    """(x fp32 [rows, D], c fp32 [ceil(rows / beam), D], gamma, beta)."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn((rows, d), generator=g, device=device) + LN_OFFSET * (1.0 + torch.rand((rows, 1), generator=g, device=device))
    c = torch.randn(((rows + beam - 1) // beam, d), generator=g, device=device)
    gamma = 1.0 + 0.2 * torch.randn(d, generator=g, device=device)
    beta = 0.2 * torch.randn(d, generator=g, device=device)
    return x, c, gamma, beta


def add_const_layernorm_reference(x: torch.Tensor, c: torch.Tensor, beam: int, gamma: torch.Tensor, beta: torch.Tensor,
                                  eps: float = LN_EPS, *, sentence_of_row_bug: bool = False):
    """(x_new fp32 = fp32 x + c[r // beam], h float64 = LayerNorm(x_new) of the fp32 row); the bug indexes c by r."""
    idx = torch.arange(x.shape[0], device=x.device)
    idx = idx.clamp(max=c.shape[0] - 1) if sentence_of_row_bug else idx // beam
    xn = x + c[idx]
    y = xn.double()
    mean = y.mean(1, keepdim=True)
    var = ((y - mean) ** 2).mean(1, keepdim=True)
    return xn, (y - mean) / torch.sqrt(var + eps) * gamma.double() + beta.double()


def bf16_ulp(ref: torch.Tensor) -> torch.Tensor:
    """The spacing of bf16 numbers at |ref| (8 significant bits)."""
    a = ref.double().abs().clamp(min=2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


# h within one bf16 ulp of the reference, the ulp taken at max(|ref|, LN_ULP_FLOOR): the fp32 row statistics of rows
# 1e3 away from zero carry an absolute error of a few 1e-4 in (x - mean) * rstd, more than an ulp of the smallest outputs.
# Measured on an H100 80GB HBM3 (700 W): at most 0.61 ulp.
LN_ULP_FLOOR = 2.0 ** -3


def ln_violation(h: torch.Tensor, ref: torch.Tensor) -> float:
    """max |h - ref| in bf16 ulps of max(|ref|, LN_ULP_FLOOR) (<= 1 passes)."""
    return float(((h.double() - ref).abs() / bf16_ulp(ref.abs().clamp(min=LN_ULP_FLOOR))).max())
