"""Inputs, float64 references and tolerances of the text encoder's kernel tests.

``tests/test_gpu_text_encoder_kernels.py`` compares the packed self-attention, the attention pooler's latent
cross-attention, the embedding frontend (with its LnFold outputs), both LayerNorm kernels and the LayerNorm + pooling
kernel with these references; ``tests/test_text_encoder_kernel_references.py`` checks without a GPU that the references
are the oracle's maths, that a float64 model of each kernel's own rounding passes its tolerance, and that known
indexing, masking, scaling and reduction bugs miss it.  The references are ``oracle.text_encoder.self_attention`` and
``oracle.text_encoder.static_pooling`` run in float64 on the very bf16 / fp32 operands the kernels get, on whatever
device those operands live.
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from oracle.text_encoder import self_attention, static_pooling

HD = 64            # head dim of the text encoder
TILE = 128         # query / key tile of the wgmma attention kernel
LA_KEYS = 16       # keys per shared-memory tile of the latent cross-attention kernel
LOG2E = 1.4426950408889634
SCALE_LOG2 = 0.125 * LOG2E  # the kernels' 1/8 * log2(e)
UNDERFLOW_LOG2 = 160.0      # 2^-160 is below the smallest fp32 denormal (2^-149): such a probability is exactly 0


def starts_of(lens: List[int]) -> List[int]:
    out, s = [], 0
    for n in lens:
        out.append(s)
        s += n
    return out


def bf16_round(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(x.dtype)


# ---------------------------------------------------------------------------------------------------------------------
# packed self-attention (sb_attention)
# ---------------------------------------------------------------------------------------------------------------------
# Batches (one list = one call) on the 128-query / 128-key tile edges, empty sentences first / in the middle / last,
# H = 16 and H = 4 (D = 256), far more (sentence, head) items than SMs (persistent loop), and > 8191 sentences (cu_seqlens
# read from global memory instead of shared memory).  (lens, heads)
ATTN_CASES: Dict[str, tuple] = {
    "1-2": ([1, 2], 16),
    "63-65": ([63, 64, 65], 16),
    "127-129": ([127, 128, 129], 16),
    "255-257": ([255, 256, 257], 16),
    "383-385": ([383, 384, 385], 16),
    "513-514": ([513, 514], 16),
    "1031": ([1031], 16),
    "mixed": ([17, 300, 1, 129, 64, 2, 191, 514, 128, 385], 16),
    "empty": ([0, 5, 130, 0, 0, 64, 257, 0], 16),
    "d256": ([63, 64, 65, 200, 1, 129, 0, 514, 257], 4),
    "many-items": ([128] * 300 + [5, 77, 129, 31] * 20, 16),
    "8200": ([1, 3] * 4100, 16),
}
# q ~ N(0, 1), k ~ 2 N(0, 1), v ~ N(0, 1): scores q.k / 8 of spread 2 make each row's softmax peaked (a handful of keys
# carry most of the weight), so a key dropped, added or misplaced moves some outputs by a good part of |v|.
ATTN_K_SCALE = 2.0

# Element-wise |got - ref| <= ATTN_RTOL |ref| + ATTN_ATOL and mean |got - ref| <= ATTN_RTOL mean |ref| + ATTN_MEAN.
# The rounding model (``attention_kernel_model``): the bf16 output adds half an ulp (<= 2^-8 |out|, about 0.75 x 2^-9
# |out| on average) -- the ATTN_RTOL terms; the numerators P are rounded to bf16 before P.V (relative error <= 2^-9
# each), at most 2^-9 sum_j w_j |v_j| <= 2^-9 max|v|, which short sentences (a few keys of comparable weight) come close
# to: ATTN_ATOL = 2^-9 x 5 covers that worst case for |v| <= 5 (N(0, 1) values); ex2.approx (2^-22 relative) and the fp32
# sums stay far below both.  An output 2 % off misses by about 5x, a dropped or misplaced key by 40x or more.
# Measured on an H100 80GB HBM3 (700 W power limit) over the 12 cases of the GPU test, every sentence: max |err| 1.6e-2
# (the 8200-sentence case, on outputs up to about 4), at most 0.63 of this tolerance.
ATTN_RTOL, ATTN_ATOL, ATTN_MEAN = 2.0 ** -8, 5 * 2.0 ** -9, 1.0e-4


@dataclass
class AttnCase:
    lens: List[int]
    heads: int
    qkv: torch.Tensor  # bf16 [T, 3D]  q | k | v, packed rows

    @property
    def dim(self) -> int:
        return HD * self.heads

    @property
    def starts(self) -> List[int]:
        return starts_of(self.lens)


def attention_case(name: str, device="cpu") -> "AttnCase":
    """The inputs of ATTN_CASES[name], the same on the CPU and the GPU."""
    lens, heads = ATTN_CASES[name]
    case = make_attention_case(lens, heads, seed=list(ATTN_CASES).index(name))
    return AttnCase(case.lens, case.heads, case.qkv.to(device))


def make_attention_case(lens: List[int], heads: int, seed: int = 0) -> AttnCase:
    g = torch.Generator().manual_seed(seed)
    d = HD * heads
    qkv = torch.randn((sum(lens), 3 * d), generator=g)
    qkv[:, d : 2 * d] *= ATTN_K_SCALE
    return AttnCase(list(lens), heads, qkv.to(torch.bfloat16))


def _heads(rows: torch.Tensor, d: int, h: int, which: int) -> torch.Tensor:
    """[G, n, 3D] -> [G, H, n, 64] of q (0), k (1) or v (2)."""
    g, n = rows.shape[:2]
    return rows[:, :, which * d : (which + 1) * d].reshape(g, n, h, HD).transpose(1, 2)


def attention_reference(case: AttnCase, *, drop_last_key_at: Optional[List[int]] = None, next_first_key: bool = False,
                        second_tile_from_first: bool = False, scale: Optional[float] = None, k_head_shift: bool = False,
                        v_head_shift: bool = False, chunk: int = 64) -> List[Optional[torch.Tensor]]:
    """float64 [n, D] of every sentence (None for an empty one): ``self_attention`` over the sentence's own rows, the
    float64 reference batched over sentences of equal length.  The keywords inject the bugs the tests must see: the last
    key masked in sentences of the listed lengths; the next sentence's first row attended as one more key; the keys and
    values of tile 1 (keys 128..255) read from tile 0; softmax scale `scale` instead of 1/8; head h reading head h+1's K
    or V."""
    d, h, lens = case.dim, case.heads, case.lens
    out: List[Optional[torch.Tensor]] = [None] * len(lens)
    starts = case.starts
    total = case.qkv.shape[0]
    by_len: Dict[int, List[int]] = {}
    for b, n in enumerate(lens):
        if n > 0:
            by_len.setdefault(n, []).append(b)
    for n, group in by_len.items():
        extra = 1 if next_first_key else 0
        for c0 in range(0, len(group), chunk):
            bs = group[c0 : c0 + chunk]
            idx = torch.tensor([[starts[b] + j for j in range(n + extra)] for b in bs], device=case.qkv.device)
            ok = idx < total
            rows = case.qkv[idx.clamp(max=total - 1)].double()  # [G, n (+1), 3D]
            q = _heads(rows, d, h, 0)[:, :, :n]
            k, v = _heads(rows, d, h, 1), _heads(rows, d, h, 2)
            if k_head_shift:
                k = k.roll(-1, 1)
            if v_head_shift:
                v = v.roll(-1, 1)
            if second_tile_from_first and n > TILE:
                hi = min(n, 2 * TILE)
                k, v = k.clone(), v.clone()
                k[:, :, TILE:hi] = k[:, :, : hi - TILE]
                v[:, :, TILE:hi] = v[:, :, : hi - TILE]
            key_ok = ok.clone()
            if drop_last_key_at is not None and n in drop_last_key_at:
                key_ok[:, n - 1] = False
            if scale is not None:
                q = q * (scale * 8.0)
            o = self_attention(q, k, v, key_ok)  # [G, H, n, 64]
            o = o.transpose(1, 2).reshape(len(bs), n, d)
            for i, b in enumerate(bs):
                out[b] = o[i]
    return out


def attention_kernel_model(case: AttnCase, *, skip_rescale: bool = False, chunk: int = 64) -> List[Optional[torch.Tensor]]:
    """float64 model of the kernel's arithmetic: per 128-key tile the running maximum m, numerators
    p = 2^((s - m) log2(e) / 8) rounded to bf16 before P.V, O and l rescaled by 2^((m_old - m_new) log2(e) / 8) between
    tiles (l from the unrounded p), the output rounded to bf16.  ``skip_rescale``: the bug of never rescaling O and l
    of the earlier tiles."""
    d, h = case.dim, case.heads
    out: List[Optional[torch.Tensor]] = [None] * len(case.lens)
    by_len: Dict[int, List[int]] = {}
    for b, n in enumerate(case.lens):
        if n > 0:
            by_len.setdefault(n, []).append(b)
    for n, group in by_len.items():
        for c0 in range(0, len(group), chunk):
            bs = group[c0 : c0 + chunk]
            idx = torch.tensor([[case.starts[b] + j for j in range(n)] for b in bs], device=case.qkv.device)
            rows = case.qkv[idx].double()
            q, k, v = (_heads(rows, d, h, j) for j in range(3))
            s = (q @ k.transpose(-1, -2)) * SCALE_LOG2  # log2 units
            m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=s.dtype, device=s.device)
            o = torch.zeros(q.shape, dtype=s.dtype, device=s.device)
            l = torch.zeros(m.shape, dtype=s.dtype, device=s.device)
            for t0 in range(0, n, TILE):
                st = s[..., t0 : t0 + TILE]
                m_new = torch.maximum(m, st.amax(-1, keepdim=True))
                alpha = torch.ones_like(m) if skip_rescale else torch.exp2(m - m_new)
                p = torch.exp2(st - m_new)
                o = o * alpha + bf16_round(p) @ v[..., t0 : t0 + TILE, :]
                l = l * alpha + p.sum(-1, keepdim=True)
                m = m_new
            res = bf16_round(o / l).transpose(1, 2).reshape(len(bs), n, d)
            for i, b in enumerate(bs):
                out[b] = res[i]
    return out


def swap_fragment_rows(x: torch.Tensor) -> torch.Tensor:
    """The bug of storing rows r and r + 8 of each 16-row accumulator fragment in each other's place."""
    n = x.shape[0]
    idx = torch.arange(n, device=x.device)
    r = idx % 16
    sw = torch.where(r < 8, idx + 8, idx - 8)
    sw = torch.where(sw < n, sw, idx)
    return x[sw]


def attn_violation(got: torch.Tensor, ref: torch.Tensor) -> float:
    """How far `got` [n, D] is from `ref` in units of the tolerance (<= 1 passes)."""
    if not bool(torch.isfinite(got).all()):
        return math.inf
    err, mag = (got.double() - ref.double()).abs(), ref.double().abs()
    return max(float((err / (ATTN_RTOL * mag + ATTN_ATOL)).max()),
               float(err.mean()) / (ATTN_RTOL * float(mag.mean()) + ATTN_MEAN))


def case_violation(got: List[Optional[torch.Tensor]], ref: List[Optional[torch.Tensor]], violation=attn_violation) -> float:
    """The worst violation over the sentences of a case (empty sentences have no rows)."""
    return max([violation(a, b) for a, b in zip(got, ref) if b is not None], default=0.0)


# ---- exact-operand "pointer" cases ----
# k_j = 8 s_j and q_i = 8 s_pi(i) for random +-1 sign vectors s (exact in bf16): q_i . k_j = 64 (64 - 2 hamming(s_pi(i),
# s_j)), so after the kernel's scale the winner pi(i) leads every other key by 64 x 2 hamming x log2(e) / 8 = 23.1 hamming
# in log2 units.  Past UNDERFLOW_LOG2 (hamming >= 7) every other numerator, and the alpha of every earlier tile the winner
# beats, is exactly 0, the winner's numerator rounds to 1 and row i is v[pi(i)] bit for bit.
POINTER_AMP = 8.0
POINTER_STRONG = 16.0  # the planted neighbour key: twice the winner's score


def _pointer_gap(q: torch.Tensor, k: torch.Tensor, win: torch.Tensor) -> float:
    """min over rows of (winner score - best other score) in log2 units; q [.., n, 64], k [.., m, 64], win [.., n]."""
    s = (q.double() @ k.double().transpose(-1, -2)) * SCALE_LOG2
    best = s.gather(-1, win[..., None]).squeeze(-1)
    other = s.scatter(-1, win[..., None], -math.inf).amax(-1)
    return float((best - other).min()) if other.numel() else math.inf


def make_pointer_case(lens: List[int], heads: int, seed: int = 0, *, plant_next: bool = False):
    """(AttnCase, win int64 [T, H]: the key (row within the sentence) each query must copy).  With ``plant_next``, the
    first row of every sentence b + 1 holds, in head h, a stronger copy (POINTER_STRONG) of the key that query h mod n_b
    of sentence b points at; only the even-indexed sentences are then checked (the odd ones are the planted
    neighbours).  The builder redraws the signs until every checked row's gap exceeds UNDERFLOW_LOG2, and checks that
    winners lie both in earlier and in later key tiles than their queries."""
    g = torch.Generator().manual_seed(seed)
    d, total = HD * heads, sum(lens)
    starts = starts_of(lens)
    for _ in range(20):
        qkv = torch.zeros((total, 3 * d))
        win = torch.zeros((total, heads), dtype=torch.int64)
        signs = torch.randint(0, 2, (total, heads, HD), generator=g).double() * 2 - 1
        qkv[:, d : 2 * d] = (POINTER_AMP * signs).reshape(total, d).float()
        qkv[:, 2 * d :] = torch.randn((total, d), generator=g)
        ok = True
        for b, n in enumerate(lens):
            if n == 0:
                continue
            s0 = starts[b]
            perm = torch.stack([torch.randperm(n, generator=g) for _ in range(heads)], 1)  # [n, H]
            win[s0 : s0 + n] = perm
            qs = POINTER_AMP * signs[s0 + perm, torch.arange(heads)[None, :]]  # [n, H, 64]
            qkv[s0 : s0 + n, :d] = qs.reshape(n, d).float()
        if plant_next:
            for b in range(0, len(lens) - 1, 2):
                n, nxt = lens[b], starts[b] + lens[b]
                if n == 0 or lens[b + 1] == 0:
                    continue
                for hh in range(heads):
                    w = int(win[starts[b] + hh % n, hh])
                    qkv[nxt, d + hh * HD : d + (hh + 1) * HD] = (POINTER_STRONG * signs[starts[b] + w, hh]).float()
        for b, n in enumerate(lens):
            if n == 0 or (plant_next and b % 2 == 1):
                continue
            s0 = starts[b]
            if n > 2 * TILE:  # some winners lie in earlier, some in later key tiles than their queries
                qtile, wtile = torch.arange(n)[:, None] // TILE, win[s0 : s0 + n] // TILE
                assert bool((wtile < qtile).any()) and bool((wtile > qtile).any())
            q = qkv[s0 : s0 + n, :d].reshape(n, heads, HD).transpose(0, 1)
            k = qkv[s0 : s0 + n, d : 2 * d].reshape(n, heads, HD).transpose(0, 1)
            if n > 1 and _pointer_gap(q, k, win[s0 : s0 + n].T) <= UNDERFLOW_LOG2:
                ok = False
                break
        if ok:
            return AttnCase(list(lens), heads, qkv.to(torch.bfloat16)), win
    raise AssertionError("could not draw sign vectors with a clear winner for every query")


def pointer_expected(case: AttnCase, win: torch.Tensor) -> torch.Tensor:
    """bf16 [T, D]: row i of head h = v[start + win[i, h]] of head h."""
    d, h = case.dim, case.heads
    out = torch.empty((case.qkv.shape[0], d), dtype=torch.bfloat16)
    for b, n in enumerate(case.lens):
        s0 = case.starts[b]
        for hh in range(h):
            src = s0 + win[s0 : s0 + n, hh]
            out[s0 : s0 + n, hh * HD : (hh + 1) * HD] = case.qkv[src, 2 * d + hh * HD : 2 * d + (hh + 1) * HD]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# latent cross-attention of the attention pooler (sb_pool_latent_attention)
# ---------------------------------------------------------------------------------------------------------------------
LA_DIMS = [256, 512, 768, 1024]
LA_HEADS = [1, 4, 7, 16]
# on the 16-key tiles and the double-buffer stage wrap (tiles 0, 1, 2 = stages 0, 1, 0), empty sentences first, in the
# middle and last
LA_LENS = [0, 1, 15, 16, 17, 31, 32, 33, 0, 514, 1031, 2, 0]
# memory rows ~ N(0, 1) (final-LayerNorm outputs), qt ~ N(0, (16 / sqrt(D))^2): scores qt.m / 8 of spread 2, as peaked as
# the self-attention cases.  Same rounding model (bf16 P before P.M, exp2f, bf16 output) and so the same constants.
# Measured (same card, 16 shapes, every sentence): max |err| 9.8e-3, at most 0.53 of the tolerance.
LA_Q_SPREAD = 16.0
LA_RTOL, LA_ATOL, LA_MEAN = ATTN_RTOL, ATTN_ATOL, ATTN_MEAN


def make_latent_case(d: int, hd: int, lens: Optional[List[int]] = None, seed: int = 0, device="cpu"):
    """(qt bf16 [B, Hd, D], mem bf16 [T, D], lens)."""
    g = torch.Generator(device=device).manual_seed(seed)
    lens = list(LA_LENS if lens is None else lens)
    mem = torch.randn((sum(lens), d), generator=g, device=device).to(torch.bfloat16)
    qt = (torch.randn((len(lens), hd, d), generator=g, device=device) * (LA_Q_SPREAD / math.sqrt(d))).to(torch.bfloat16)
    return qt, mem, lens


def latent_reference(qt: torch.Tensor, mem: torch.Tensor, lens: List[int], *, drop_last_key_at: Optional[List[int]] = None,
                     one_past: bool = False, second_tile_from_first: bool = False, scale: float = 0.125,
                     row_hd_leak: bool = False) -> torch.Tensor:
    """float64 [B, Hd, D] = softmax(qt . m / 8) . m over each sentence's rows (zeros for an empty one).  Bugs: the last
    key masked in sentences of the listed lengths; one key past len attended; the keys of tile 1 (16..31) read from tile
    0's stage; scale `scale`; the zero query row Hd (the plain mean of the memory rows) stored over row 0 of the next
    sentence."""
    b_, hd, d = qt.shape
    out = torch.zeros((b_, hd, d), dtype=torch.float64, device=qt.device)
    total = mem.shape[0]
    for b, (s0, n) in enumerate(zip(starts_of(lens), lens)):
        if n == 0:
            continue
        m_rows = n + 1 if (one_past and s0 + n < total) else n
        m = mem[s0 : s0 + m_rows].double()
        if second_tile_from_first and n > LA_KEYS:
            m = m.clone()
            hi = min(n, 2 * LA_KEYS)
            m[LA_KEYS:hi] = m[: hi - LA_KEYS]
        s = qt[b].double() @ m.T * scale
        if drop_last_key_at is not None and n in drop_last_key_at:
            s[:, n - 1] = -math.inf
        out[b] = torch.softmax(s, -1) @ m
    if row_hd_leak:
        leak = out.clone()
        for b, (s0, n) in enumerate(zip(starts_of(lens), lens)):
            if b + 1 < b_ and n > 0:
                leak[b + 1, 0] = mem[s0 : s0 + n].double().mean(0)
        return leak
    return out


def latent_kernel_model(qt: torch.Tensor, mem: torch.Tensor, lens: List[int]) -> torch.Tensor:
    """float64 model of the kernel's rounding: numerators relative to the running maximum of each 16-key tile rounded to
    bf16 before P.M, l from the unrounded numerators, output rounded to bf16."""
    b_, hd, d = qt.shape
    out = torch.zeros((b_, hd, d), dtype=torch.float64, device=qt.device)
    for b, (s0, n) in enumerate(zip(starts_of(lens), lens)):
        if n == 0:
            continue
        m = mem[s0 : s0 + n].double()
        s = qt[b].double() @ m.T * SCALE_LOG2
        mx = torch.full((hd, 1), -math.inf, dtype=torch.float64, device=qt.device)
        o = torch.zeros((hd, d), dtype=torch.float64, device=qt.device)
        l = torch.zeros((hd, 1), dtype=torch.float64, device=qt.device)
        for t0 in range(0, n, LA_KEYS):
            st = s[:, t0 : t0 + LA_KEYS]
            mn = torch.maximum(mx, st.amax(-1, keepdim=True))
            corr = torch.exp2(mx - mn)
            p = torch.exp2(st - mn)
            o = o * corr + bf16_round(p) @ m[t0 : t0 + LA_KEYS]
            l = l * corr + p.sum(-1, keepdim=True)
            mx = mn
        out[b] = bf16_round(o / l)
    return out


def latent_violation(got: torch.Tensor, ref: torch.Tensor) -> float:
    if not bool(torch.isfinite(got).all()):
        return math.inf
    err, mag = (got.double() - ref.double()).abs(), ref.double().abs()
    return max(float((err / (LA_RTOL * mag + LA_ATOL)).max()),
               float(err.mean()) / (LA_RTOL * float(mag.mean()) + LA_MEAN))


# pointer case: memory rows of +-1 signs and qt[b, h] = LA_POINTER_AMP m_pi(b, h): the winner scores
# LA_POINTER_AMP D / 8 and another row 2 LA_POINTER_AMP hamming / 8 less, 0.36 LA_POINTER_AMP hamming in log2 units; at
# D = 256 a random pair differs in about 128 +- 8 signs, so 8 clears UNDERFLOW_LOG2 from hamming 56 on.
LA_POINTER_AMP = 8.0


def make_latent_pointer_case(d: int, hd: int, lens: List[int], seed: int = 0):
    """(qt, mem, win int64 [B, Hd] = the row within its sentence that u[b, h] must equal bit for bit)."""
    g = torch.Generator().manual_seed(seed)
    for _ in range(20):
        mem = torch.randint(0, 2, (sum(lens), d), generator=g).float() * 2 - 1
        qt = torch.zeros((len(lens), hd, d))
        win = torch.zeros((len(lens), hd), dtype=torch.int64)
        ok = True
        for b, (s0, n) in enumerate(zip(starts_of(lens), lens)):
            if n == 0:
                continue
            w = torch.randint(0, n, (hd,), generator=g)
            win[b] = w
            qt[b] = LA_POINTER_AMP * mem[s0 + w]
            if n > 1:
                s = (qt[b].double() @ mem[s0 : s0 + n].double().T) * SCALE_LOG2
                best = s.gather(1, w[:, None])[:, 0]
                other = s.scatter(1, w[:, None], -math.inf).amax(1)
                if float((best - other).min()) <= UNDERFLOW_LOG2:
                    ok = False
                    break
        if ok:
            return qt.to(torch.bfloat16), mem.to(torch.bfloat16), win
    raise AssertionError("could not draw memory rows with a clear winner for every query")


# ---------------------------------------------------------------------------------------------------------------------
# embedding frontend (sb_embed) and its LnFold outputs
# ---------------------------------------------------------------------------------------------------------------------
EMBED_DIMS = [256, 512, 768, 1024]
EMBED_S = 37                       # > 8 and no multiple of 8: the kernel's blockIdx.y covers 8 positions
EMBED_LENS = [37, 1, 0, 9, 8, 20, 36]
EMBED_VOCAB = 3000
EMBED_OFFSET = 1.0e3               # common offset of every row (through the position table): a sum-of-squares M2 cancels


def embed_scale(d: int) -> float:
    """sqrt(D) in fp32, as the encoder's config gives it: 16 and 32 at D = 256 and 1024 (powers of two)."""
    return float(torch.tensor(math.sqrt(d), dtype=torch.float32))


def make_embed_case(d: int, seed: int = 0):
    """(ids int64 [B, S] with out-of-range ids past each length, table bf16 [V, D] ~ N(0, 1/D), pos fp32 [S, D] =
    EMBED_OFFSET + sinusoid-like values, lens)."""
    g = torch.Generator().manual_seed(seed)
    lens = EMBED_LENS
    ids = torch.randint(0, EMBED_VOCAB, (len(lens), EMBED_S), generator=g)
    for b, n in enumerate(lens):
        ids[b, n:] = torch.where(torch.arange(EMBED_S - n) % 2 == 0, -7, EMBED_VOCAB + 5)
    ids[0, :2] = torch.tensor([0, EMBED_VOCAB - 1])
    table = (torch.randn((EMBED_VOCAB, d), generator=g) / math.sqrt(d)).to(torch.bfloat16)
    pos = EMBED_OFFSET + torch.sin(torch.randn((EMBED_S, d), generator=g) * 3.0)
    return ids, table, pos.float(), list(lens)


def embed_reference(ids: torch.Tensor, table: torch.Tensor, pos: torch.Tensor, scale: float, lens: List[int]) -> torch.Tensor:
    """float64 [T, D]: table[id] * scale + pos[t] (id 0 for an out-of-range id), rows packed."""
    rows = []
    for b, n in enumerate(lens):
        i = ids[b, :n].clone()
        i[(i < 0) | (i >= table.shape[0])] = 0
        rows.append(table[i].double() * scale + pos[:n].double())
    return torch.cat(rows)


def chunk_stats(x: torch.Tensor) -> torch.Tensor:
    """float64 [T, D/128, 2]: (mean, M2) of each 128-column chunk of the rows of x."""
    c = x.double().view(x.shape[0], -1, 128)
    mean = c.mean(-1)
    return torch.stack([mean, ((c - mean[..., None]) ** 2).sum(-1)], -1)


def sum_of_squares_stats(x: torch.Tensor) -> torch.Tensor:
    """The bug of an fp32 M2 taken as sum(x^2) - 128 mean^2."""
    c = x.float().view(x.shape[0], -1, 128)
    mean = c.sum(-1) / 128.0
    return torch.stack([mean, (c * c).sum(-1) - 128.0 * mean * mean], -1).double()


# |mean - ref| <= STATS_MEAN_ULPS * 2^-24 * max|x| of the chunk: eight fp32 adds per lane and four shuffle levels, each
# at most half an ulp of a partial sum <= 128 max|x|, divided by 128.  |M2 - ref| <= STATS_M2_RTOL * ref +
# 128 (mean error)^2: the deviations from an fp32 mean that is off by e add 128 e^2; the fp32 squares and sums add at
# most ~12 half-ulps relative.  Measured (same card, D = 256 ... 1024): at most 0.09 of the bound.
STATS_MEAN_ULPS, STATS_M2_RTOL = 16.0, 2.0 ** -18


def stats_violation(got: torch.Tensor, x: torch.Tensor) -> float:
    """How far the (mean, M2) partials `got` [T, D/128, 2] are from float64 ones of x in units of the bound."""
    ref = chunk_stats(x)
    amax = x.double().abs().view(x.shape[0], -1, 128).amax(-1)
    mean_bound = STATS_MEAN_ULPS * 2.0 ** -24 * amax
    em = (got[..., 0].double() - ref[..., 0]).abs()
    m2_bound = STATS_M2_RTOL * ref[..., 1] + 128.0 * mean_bound ** 2 + 1e-30
    e2 = (got[..., 1].double() - ref[..., 1]).abs()
    return max(float((em / mean_bound).max()), float((e2 / m2_bound).max()))


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm (sb_layernorm, sb_layernorm_dual)
# ---------------------------------------------------------------------------------------------------------------------
LN_DIMS = [128, 256, 512, 768, 1024]
LN_ROWS = [1, 7, 8, 9, 4099]
LN_EPS = 1.0e-5
LN_OFFSET = 1.0e3
LN_CONSTANTS = [3.5, -0.75, 96.0, 0.0, -1.5e3]  # few mantissa bits: D copies sum exactly, the mean is exact


def make_ln_case(t: int, d: int, seed: int = 0, device="cpu"):
    """(x fp32 [T, D], gamma, beta).  Row r % 4: 0 = N(0, 1); 1 = N(0, 1) + LN_OFFSET x (1 + U(0, 1)) (|mean| ~ 1e3 to 2e3
    standard deviations); 2 = a constant from LN_CONSTANTS (the output is exactly beta); 3 = N(5, 16)."""
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn((t, d), generator=g, device=device)
    r = torch.arange(t, device=device)
    off = LN_OFFSET * (1.0 + torch.rand((t, 1), generator=g, device=device))
    x = torch.where((r % 4 == 1)[:, None], x + off, x)
    x = torch.where((r % 4 == 3)[:, None], 4.0 * x + 5.0, x)
    consts = torch.tensor(LN_CONSTANTS, device=device)[(r // 4) % len(LN_CONSTANTS)]
    x = torch.where((r % 4 == 2)[:, None], consts[:, None].expand(t, d), x)
    gamma = 1.0 + 0.3 * torch.randn(d, generator=g, device=device)
    beta = 0.3 * torch.randn(d, generator=g, device=device)
    return x.contiguous(), gamma, beta


def ln_reference(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = LN_EPS, *,
                 unbiased: bool = False) -> torch.Tensor:
    """float64 LayerNorm of the fp32 rows (``unbiased``: the bug of dividing the variance by D - 1)."""
    y = x.double()
    mean = y.mean(1, keepdim=True)
    var = ((y - mean) ** 2).sum(1, keepdim=True) / (y.shape[1] - (1 if unbiased else 0))
    return (y - mean) / torch.sqrt(var + eps) * gamma.double() + beta.double()


def ln_sum_of_squares_fp32(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = LN_EPS) -> torch.Tensor:
    """The bug of an fp32 variance taken as mean(x^2) - mean^2."""
    mean = x.float().mean(1, keepdim=True)
    var = (x.float() * x.float()).mean(1, keepdim=True) - mean * mean
    return ((x.float() - mean) / torch.sqrt(var.clamp(min=0) + eps) * gamma + beta).double()


# fp32 output: |y - ref| <= LN_MEAN_ULPS 2^-24 (1 + |mean| / std) |gamma| + 2^-21 (|ref| + |beta|).  The first term is the
# fp32 mean's error (per-lane sums of up to 32 values then five shuffle levels: at most ~37 half-ulps of the sum of |x|,
# i.e. of D (|mean| + std)) seen through rstd; the second covers rstd (sqrtf, a division) and the final products.  bf16
# output: that plus half a bf16 ulp (<= 2^-8 |ref|), i.e. a check that the bf16 value is the rounding of an accurate
# fp32 one; over thousands of rows some value always lies near a rounding midpoint, so that check reaches about 0.99 of
# its bound by construction.  Measured (same card, 25 shapes): the fp32 output at most 0.17 of its bound.
LN_MEAN_ULPS = 48.0


def ln_bound(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, ref: torch.Tensor, bf16: bool) -> torch.Tensor:
    y = x.double()
    mean = y.mean(1, keepdim=True)
    std = y.std(1, unbiased=False, keepdim=True)
    ratio = torch.where(std > 0, mean.abs() / std.clamp(min=1e-300), torch.zeros_like(std))
    b = LN_MEAN_ULPS * 2.0 ** -24 * (1.0 + ratio) * gamma.double().abs() + 2.0 ** -21 * (ref.abs() + beta.double().abs())
    return b + 2.0 ** -8 * ref.abs() if bf16 else b


def ln_violation(got: torch.Tensor, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, ref: torch.Tensor) -> float:
    bf16 = got.dtype == torch.bfloat16
    err = (got.double() - ref).abs()
    return float((err / ln_bound(x, gamma, beta, ref, bf16)).max())


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm + pooling (sb_pool)
# ---------------------------------------------------------------------------------------------------------------------
POOL_MODES = ["mean", "max", "last"]
POOL_LENS = [1, 7, 8, 9, 15, 16, 17]      # every warp-count remainder of the kernel's 8-warp striding
POOL_LONG = 514
POOL_BATCH = 5000
POOL_SHIFT = -4.0                          # rows ~ N(-4, 1): every raw value negative (a MAX started at 0 would show)
POOL_BETA = -6.0                           # LayerNorm outputs z gamma + beta with gamma ~ 0.5: all negative as well


def pool_lens(batch: int = POOL_BATCH, long_every: int = 700) -> List[int]:
    """POOL_LENS in turn, a POOL_LONG sentence every `long_every` sentences."""
    return [POOL_LONG if i % long_every == long_every // 2 else POOL_LENS[i % len(POOL_LENS)] for i in range(batch)]


def make_pool_case(lens: List[int], d: int, seed: int = 0, device="cpu"):
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn((sum(lens), d), generator=g, device=device) + POOL_SHIFT
    gamma = 0.5 + 0.1 * torch.randn(d, generator=g, device=device)
    beta = POOL_BETA + 0.2 * torch.randn(d, generator=g, device=device)
    return x, gamma, beta


def pool_reference(x: torch.Tensor, lens: List[int], mode: str, gamma: Optional[torch.Tensor] = None,
                   beta: Optional[torch.Tensor] = None, eps: float = LN_EPS, *, max_zero_init: bool = False,
                   last_first_row: bool = False) -> torch.Tensor:
    """float64 [B, D]: ``static_pooling`` of each sentence's (float64-LayerNormed) rows, batched over sentences of equal
    length, on the CPU.  Empty sentences are left NaN (the kernel's own values for them are pinned separately).  Bugs:
    MAX started from 0 instead of -inf; LAST taking the sentence's first row."""
    d = x.shape[1]
    xs = x.double().cpu()
    if gamma is not None:
        xs = ln_reference(xs, gamma.cpu(), beta.cpu(), eps)
    out = torch.full((len(lens), d), math.nan, dtype=torch.float64)
    starts = starts_of(lens)
    by_len: Dict[int, List[int]] = {}
    for b, n in enumerate(lens):
        if n > 0:
            by_len.setdefault(n, []).append(b)
    for n, group in by_len.items():
        idx = torch.tensor([starts[b] for b in group])[:, None] + torch.arange(n)[None, :]
        seqs = xs[idx]  # [G, n, D]
        if last_first_row and mode == "last":
            seqs = seqs[:, :1]
        r = static_pooling(seqs, torch.full((len(group),), seqs.shape[1], dtype=torch.int64), mode)
        if max_zero_init and mode == "max":
            r = r.clamp(min=0.0)
        out[torch.tensor(group)] = r
    return out


# |got - ref| <= POOL_RTOL |ref| + POOL_ATOL: the fp32 LayerNorm (ln_bound: ~1e-5 on these rows) and, for MEAN, the fp32
# sums over up to 514 rows (at most ~(514 / 8 + 8) half-ulps of sums of values ~8) and the fp32 1 / len.  With
# apply_ln = 0, MAX and LAST select fp32 values and must be exact; MEAN keeps the bound.
# Measured (same card, every mode, 5000 sentences): at most 0.02 of the bound.
POOL_RTOL, POOL_ATOL = 2.0 ** -20, 1.0e-4


def pool_violation(got: torch.Tensor, ref: torch.Tensor) -> float:
    keep = ~torch.isnan(ref)
    err = (got.double().cpu() - ref)[keep].abs()
    return float((err / (POOL_RTOL * ref[keep].abs() + POOL_ATOL)).max()) if err.numel() else 0.0
