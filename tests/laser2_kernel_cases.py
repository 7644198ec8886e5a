"""Inputs, float64 references and tolerances of the LASER2 kernel tests.

``tests/test_gpu_laser2_kernels.py`` compares the cluster-resident LSTM recurrence (``sb_lstm_recurrent``), the embedding
gather (``sb_laser2_embed``) and the gate-order repack of ``sb_laser2_create`` with these references;
``tests/test_laser2_kernel_references.py`` checks without a GPU that the references are the oracle's maths, that a model of
the kernel's rounding stays within half of each tolerance, and that known indexing, routing and masking bugs miss them.

The recurrence reference runs in float64 on the kernel's own operands: the bf16 G (already in gate order), the bf16 W_hh
and h rounded to bf16 before each matmul, as the kernel's wgmma reads it.  y is compared with the float64 h (the kernel
stores bf16(h)); the pool with the max of the unrounded h (the kernel keeps it in fp32).  It runs on whatever device holds
its inputs, so that long cases run in float64 on the GPU.
"""

from __future__ import annotations

import math
from dataclasses import dataclass, replace
from typing import List, Optional, Sequence

import torch

H = 512      # hidden size of the recurrent kernel
CTAS = 16    # CTAs per cluster; CTA c owns hidden units [32 c, 32 c + 32) of all four gates
UNITS = H // CTAS
TILE = 64    # sequences per tile (the wgmma M)
K16 = 16     # h columns per wgmma k-step

# Lengths on the step edges: one step, the prefetch of step 1, the accumulator k-steps and tile-sized counts, up to the
# 2048 steps of the longest case.
EDGE_LENGTHS = [1, 2, 3, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 1023, 1024, 1025, 2047, 2048]
WEIGHT_BOUNDS = [0.1, 1.0 / math.sqrt(H)]  # the synthetic engine tests' bound and torch's default U(-1/sqrt(H), 1/sqrt(H))


def gate_rows(dirs: int = 1) -> torch.Tensor:
    """int64 [dirs * 4H]: the row of torch.nn.LSTM's stacked [i | f | g | o] matrices that row n of the kernel's gate order
    holds, written from the kernel's definition: row 128 c + 32 gate + u is gate `gate` of hidden unit 32 c + u."""
    n = torch.arange(4 * H)
    cta, gate, u = n // (4 * UNITS), (n % (4 * UNITS)) // UNITS, n % UNITS
    one = gate * H + cta * UNITS + u
    return torch.cat([one + d * 4 * H for d in range(dirs)])


def split_gates(z: torch.Tensor):
    """z [n, 4H] in gate order -> (i, f, g, o), each [n, H] over hidden units 0..H-1."""
    q = z.view(z.shape[0], CTAS, 4, UNITS)
    return tuple(q[:, :, k].reshape(z.shape[0], H) for k in range(4))


def cta_block(p: int) -> slice:
    return slice(UNITS * p, UNITS * (p + 1))


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class LstmCase:
    dirs: int
    G: torch.Tensor          # bf16 [T, >= dirs * 4H], gate order (may be a column view of a wider buffer)
    w_hh: torch.Tensor       # bf16 [dirs * 4H, H], gate order
    lens: List[int]
    tile_seqs: torch.Tensor  # int32 [tiles * 64], -1 = empty row
    pad: Optional[torch.Tensor] = None   # uint8 [T]
    tail: Optional[torch.Tensor] = None  # uint8 [B]
    pad_value: float = 0.0
    label: str = ""

    @property
    def cu(self) -> torch.Tensor:
        cu = torch.zeros(len(self.lens) + 1, dtype=torch.int32)
        cu[1:] = torch.cumsum(torch.tensor(self.lens, dtype=torch.int64), 0).to(torch.int32)
        return cu

    @property
    def tokens(self) -> int:
        return sum(self.lens)

    def tiled(self) -> List[int]:
        """The sequences named in tile_seqs (the ones the kernel runs)."""
        return sorted(int(s) for s in self.tile_seqs.tolist() if s >= 0)

    def to(self, device) -> "LstmCase":
        mv = lambda t: None if t is None else t.to(device)  # noqa: E731
        return replace(self, G=mv(self.G), w_hh=mv(self.w_hh), tile_seqs=mv(self.tile_seqs), pad=mv(self.pad),
                       tail=mv(self.tail))


def tile_layout(order: Sequence[int], holes: Sequence[int] = (), empty_tiles: int = 0) -> torch.Tensor:
    """int32 tile_seqs: the sequences of `order` fill the rows in turn, skipping the tile rows listed in `holes` (-1
    there), the last tile is padded with -1 and `empty_tiles` all -1 tiles follow."""
    rows, it, r = [], iter(order), 0
    pending = list(order)
    while pending:
        if r in holes:
            rows.append(-1)
        else:
            rows.append(next(it))
            pending.pop()
        r += 1
    rows += [-1] * ((-len(rows)) % TILE + TILE * empty_tiles)
    return torch.tensor(rows, dtype=torch.int32)


def random_weights(dirs: int, bound: float, g: torch.Generator, device="cpu") -> torch.Tensor:
    return ((torch.rand((dirs * 4 * H, H), generator=g, device=device) * 2 - 1) * bound).to(torch.bfloat16)


def poisoned_g(T: int, dirs: int, extra_cols: int, device="cpu") -> torch.Tensor:
    """A NaN-filled bf16 [T, dirs * 4H + extra_cols] buffer; the case writes its G into the first dirs * 4H columns."""
    return torch.full((T, dirs * 4 * H + extra_cols), float("nan"), dtype=torch.bfloat16, device=device)


def make_random_case(dirs: int, lens: Sequence[int], *, bound: float = 0.1, g_std: float = 1.0, seed: int = 0,
                     holes: Sequence[int] = (), empty_tiles: int = 0, orphans: Sequence[int] = (), extra_cols: int = 0,
                     order: Optional[Sequence[int]] = None, device="cpu", draw_on_device: bool = False,
                     label: str = "") -> LstmCase:
    """G ~ N(0, g_std) and W_hh ~ U(-bound, bound), both bf16, drawn on the CPU (the same numbers on any device) unless
    draw_on_device.  Sequences in `orphans` are left out of tile_seqs and their G rows hold NaN, as do the `extra_cols`
    columns past the G every row has (G is then a column view)."""
    gen = device if draw_on_device else "cpu"
    g = torch.Generator(device=gen).manual_seed(seed)
    lens = list(lens)
    T = sum(lens)
    buf = poisoned_g(T, dirs, extra_cols, device)
    G = buf[:, : dirs * 4 * H]
    G.copy_((torch.randn((T, dirs * 4 * H), generator=g, device=gen) * g_std).to(torch.bfloat16))
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    for b in orphans:
        G[cu[b] : cu[b + 1]] = float("nan")
    w = random_weights(dirs, bound, g, gen).to(device)
    if order is None:
        order = [b for b in torch.randperm(len(lens), generator=torch.Generator().manual_seed(seed)).tolist()
                 if b not in set(orphans)]
    return LstmCase(dirs, G, w, lens, tile_layout(order, holes, empty_tiles).to(device), label=label)


def permutation_weights(dirs: int, device="cpu") -> torch.Tensor:
    """W_hh with one nonzero per gate row, +-2^-1 or +-1: row 128 c + 32 gate + j (unit 32 c + j) reads unit
    32 ((c + j + gate) % 16) + (7 j + 5 gate + 3 c + d) % 32.  Over j the source CTA (c + j + gate) % 16 runs through all
    16 CTAs, CTA c itself included, so every CTA's 128 rows read every slice of h: its own through shared memory, the 15
    others as delivered by their owners.  The wgmma sum of a row is then one exact product."""
    w = torch.zeros((dirs * 4 * H, H))
    vals = [0.5, -1.0, -0.5, 1.0]
    for d in range(dirs):
        for n in range(4 * H):
            c, gate, j = n // 128, (n % 128) // 32, n % 32
            col = UNITS * ((c + j + gate) % CTAS) + (7 * j + 5 * gate + 3 * c + d) % UNITS
            w[d * 4 * H + n, col] = vals[(j + gate + d) % 4]
    return w.to(torch.bfloat16).to(device)


def make_exact_case(dirs: int, lens: Sequence[int], kind: str, *, seed: int = 0, device="cpu") -> LstmCase:
    """Exact-operand inputs: the matmul of each gate row is exact in fp32, so the kernel and the float64 reference differ
    only by the SFU functions, fp32 c and the bf16 rounding of h.
      "zero":        W_hh = 0, G ~ N(0, 1): z = G isolates the token mapping (position, base, prefetch, c carried over).
      "permutation": permutation_weights, G ~ N(0, 1).
      "saturated":   per hidden unit u one regime, by u % 4, of G values:
                     0: f = +90, i = +100, g = 0.5 + |N(0, 1)|, o = +-90 / +-100 at random: c grows by tanh(g) every
                        step to ~1.5e3 at 2048 steps, h = 0 or tanh(c) = 1;
                     1: f = -100, i = -90: c = 0 after every step, so h = 0 (+-1e-40 in float64);
                     2: f = +100, i = +100, g = +-90, o = +100: c walks over the integers, h = tanh(c), with __expf(-100)
                        underflowing and __expf(90) overflowing inside the sigmoid (it must come out exactly 1 or 0);
                     3: random N(0, 3) gates (the unsaturated neighbours).
                     The W_hh rows of regimes 0 and 2 are zero, so their c integrates G alone; regimes 1 and 3 keep
                     permutation_weights, and read the saturated h = 0 / +-1 through them."""
    g = torch.Generator().manual_seed(seed)
    lens = list(lens)
    T = sum(lens)
    z = torch.randn((T, dirs * 4 * H), generator=g)
    w = torch.zeros((dirs * 4 * H, H), dtype=torch.bfloat16) if kind == "zero" else permutation_weights(dirs)
    if kind == "saturated":
        z = z.view(T, dirs, CTAS, 4, UNITS)
        regime = (torch.arange(H) % 4).view(CTAS, UNITS)
        r0, r1, r2 = [(regime == k)[None, None] for k in range(3)]
        rnd = lambda: torch.rand(z[..., 0, :].shape, generator=g) < 0.5  # noqa: E731
        sign, mag = torch.where(rnd(), -1.0, 1.0), torch.where(rnd(), 90.0, 100.0)
        full = lambda v: torch.full_like(z[..., 0, :], v)  # noqa: E731
        zi, zf, zg, zo = (z[..., k, :].clone() * 3 for k in range(4))
        zi = torch.where(r0 | r2, full(100.0), torch.where(r1, full(-90.0), zi))
        zf = torch.where(r0, full(90.0), torch.where(r1, full(-100.0), torch.where(r2, full(100.0), zf)))
        zg = torch.where(r0, 0.5 + z[..., 2, :].abs(), torch.where(r2, sign * 90.0, zg))
        zo = torch.where(r0, sign * mag, torch.where(r2, full(100.0), zo))
        z = torch.stack([zi, zf, zg, zo], 3).reshape(T, dirs * 4 * H)
        rows = (regime.view(1, CTAS, 1, UNITS).expand(dirs, CTAS, 4, UNITS).reshape(-1)) % 2 == 0
        w[rows] = 0
    G = z.to(torch.bfloat16).to(device)
    order = torch.randperm(len(lens), generator=torch.Generator().manual_seed(seed)).tolist()
    return LstmCase(dirs, G, w.to(device), lens, tile_layout(order, holes=(5, 40)).to(device), label=kind)


def with_pool(case: LstmCase, *, pad_rate: float = 0.15, all_pad: Sequence[int] = (), tail_rate: float = 0.5,
              pad_value: float = 0.25, seed: int = 0) -> LstmCase:
    """Random pad flags (sequences in `all_pad` are pad at every token) and tail flags."""
    g = torch.Generator().manual_seed(seed)
    pad = (torch.rand(case.tokens, generator=g) < pad_rate).to(torch.uint8)
    cu = case.cu
    for b in all_pad:
        pad[int(cu[b]) : int(cu[b + 1])] = 1
    tail = (torch.rand(len(case.lens), generator=g) < tail_rate).to(torch.uint8)
    dev = case.G.device
    return replace(case, pad=pad.to(dev), tail=tail.to(dev), pad_value=pad_value)


# ---------------------------------------------------------------------------------------------------------------------
# the recurrence reference, the rounding model and the fault injections
# ---------------------------------------------------------------------------------------------------------------------
FAULTS = {
    "reverse direction reads position s": "reverse_reads_s",
    "i and f gates swapped": "swap_if",
    "g and o gates swapped": "swap_go",
    "G prefetched one step ahead": "prefetch_ahead",
    "peer slice 5 stale by one step": "stale_peer",
    "slice of CTA 3 delivered to CTA 4's slot": "misroute",
    "k16 block 7 of h ignored": "skip_k16",
    "tile rows 3 and 11 swapped": "swap_rows",
    "finished row keeps updating its max": "finished_max",
    "pad token included in the max": "pad_in_max",
    "tail flag ignored": "tail_ignored",
    "tail applied with min": "tail_min",
    "output scaled by 1.01": "scale",
}


class _SfuModel:
    """The kernel's fp32 gate maths with each SFU result off by a random amount within its documented bound (CUDA C
    Programming Guide, intrinsic and single-precision function accuracy): __expf 2 + floor(|1.173 x|) ulp, __fdividef
    2 ulp, tanhf 2 ulp; one ulp taken as 2^-23 of the value (the coarse end of a binade)."""

    def __init__(self, device, seed: int) -> None:
        self.g = torch.Generator(device=device).manual_seed(seed)

    def _wiggle(self, v: torch.Tensor, ulps: torch.Tensor) -> torch.Tensor:
        u = torch.rand(v.shape, generator=self.g, device=v.device, dtype=torch.float32) * 2 - 1
        return v * (1 + u * ulps * 2.0 ** -23)

    def sigmoid(self, x: torch.Tensor) -> torch.Tensor:
        e = self._wiggle(torch.exp(-x), 2 + torch.floor((1.173 * x).abs()))
        return self._wiggle(1.0 / (1.0 + e), torch.full_like(x, 2.0))

    def tanh(self, x: torch.Tensor) -> torch.Tensor:
        return self._wiggle(torch.tanh(x), torch.full_like(x, 2.0))


def lstm_reference(case: LstmCase, *, round_h: bool = True, model_seed: Optional[int] = None, fault: Optional[str] = None,
                   seqs: Optional[Sequence[int]] = None):
    """(y float64 [T, dirs * H], pool float64 [B, dirs * H]) of the sequences the kernel runs (those in tile_seqs, or
    `seqs`); rows of other tokens and sequences are NaN.  y is h (the kernel stores bf16(h)); the pool is the max of h over
    the sequence's tokens without pad flag, then the max with pad_value where the tail flag is set (-inf if nothing).

    round_h=False feeds the matmul the unrounded h (the LSTM's own maths, for the oracle comparison).  model_seed runs the
    rounding model instead: fp32 arithmetic with the SFU errors of _SfuModel, y = bf16(h).  `fault` injects one of the
    FAULTS bugs."""
    dev = case.G.device
    dirs = case.dirs
    dt = torch.float32 if model_seed is not None else torch.float64
    sfu = _SfuModel(dev, model_seed) if model_seed is not None else None
    sig = sfu.sigmoid if sfu else torch.sigmoid
    tanh = sfu.tanh if sfu else torch.tanh
    cu = case.cu.to(dev).long()
    lens = cu[1:] - cu[:-1]
    B, T = lens.numel(), case.G.shape[0]
    run = torch.tensor(sorted(seqs) if seqs is not None else case.tiled(), dtype=torch.long, device=dev)
    n = run.numel()
    L, base = lens[run], cu[run]
    steps = L.clone()
    src = torch.arange(n, device=dev)  # whose h row each row's matmul reads
    tiles = case.tile_seqs.to(dev).long().view(-1, TILE)
    if fault in ("swap_rows", "finished_max"):
        pos_of = {int(s): i for i, s in enumerate(run.tolist())}
        if fault == "swap_rows":
            a, b = pos_of[int(tiles[0, 3])], pos_of[int(tiles[0, 11])]
            src[a], src[b] = b, a
        else:
            for row in tiles:
                live = row[row >= 0]
                if live.numel():
                    m = lens[live].max()
                    for s in live.tolist():
                        if s in pos_of:
                            steps[pos_of[s]] = m
    y = torch.full((T, dirs * H), math.nan, dtype=torch.float64, device=dev)
    pool = torch.full((B, dirs * H), math.nan, dtype=torch.float64, device=dev)
    bf = (lambda t: t.to(torch.bfloat16).to(dt)) if round_h else (lambda t: t)  # noqa: E731
    pad = case.pad.to(dev).bool() if case.pad is not None else None
    for d in range(dirs):
        W = case.w_hh[d * 4 * H : (d + 1) * 4 * H].to(dt)
        Gd = case.G[:, d * 4 * H : (d + 1) * 4 * H]
        h = torch.zeros((n, H), dtype=dt, device=dev)
        h2, c = torch.zeros_like(h), torch.zeros_like(h)
        hmax = torch.full((n, H), -math.inf, dtype=dt, device=dev)
        for s in range(int(steps.max()) if n else 0):
            a = (steps > s).nonzero()[:, 0]
            la, ba = L[a], base[a]
            live = la > s
            pos = (la - 1 - s) if d else torch.full_like(la, s)
            tok = ba + pos.clamp(min=0)
            if fault == "reverse_reads_s" and d:
                rpos = torch.full_like(la, s)
            elif fault == "prefetch_ahead":
                rpos = (la - 2 - s) if d else torch.full_like(la, s + 1)
                live_read = la > s + 1
            else:
                rpos = pos
            rlive = live_read if fault == "prefetch_ahead" else live
            gz = Gd[(ba + rpos.clamp(min=0, max=None)).clamp(max=T - 1)].to(dt)
            gz = torch.where(rlive[:, None], gz, torch.zeros_like(gz))
            hin = bf(h[src[a]])
            if fault == "skip_k16":
                hin[:, K16 * 7 : K16 * 8] = 0
            if fault == "stale_peer":
                hin[:, cta_block(5)] = bf(h2[src[a]])[:, cta_block(5)]
            if fault == "misroute":  # every CTA but 3 and 4 finds slice 3 in slot 4 and nothing (zeros) in slot 3
                wrong = hin.clone()
                wrong[:, cta_block(4)] = hin[:, cta_block(3)]
                wrong[:, cta_block(3)] = 0
                z = torch.cat([(hin if p in (3, 4) else wrong) @ W[128 * p : 128 * (p + 1)].T for p in range(CTAS)], 1)
            else:
                z = hin @ W.T
            z = gz + z
            zi, zf, zg, zo = split_gates(z)
            if fault == "swap_if":
                zi, zf = zf, zi
            if fault == "swap_go":
                zg, zo = zo, zg
            cn = sig(zf) * c[a] + sig(zi) * tanh(zg)
            hn = sig(zo) * tanh(cn)
            yv = hn.to(torch.bfloat16).double() if sfu else hn.double()
            y[tok[live], d * H : (d + 1) * H] = yv[live]
            take = live.clone()
            if pad is not None and fault != "pad_in_max":
                take[live] &= ~pad[tok[live]]
            if fault == "finished_max":
                take |= ~live
            hmax[a] = torch.where(take[:, None], torch.maximum(hmax[a], hn), hmax[a])
            c[a], h2[a], h[a] = cn, h[a], hn
        hm = hmax.double()
        if case.tail is not None and fault != "tail_ignored":
            t = case.tail.to(dev).bool()[run][:, None]
            pv = torch.tensor(case.pad_value, dtype=torch.float64, device=dev)
            hm = torch.where(t, torch.minimum(hm, pv) if fault == "tail_min" else torch.maximum(hm, pv), hm)
        pool[run, d * H : (d + 1) * H] = hm
    if fault == "scale":
        y, pool = y * 1.01, pool * 1.01
    return y, pool


def subset(case: LstmCase, seqs: Sequence[int]):
    """(the case restricted to `seqs`, token index into the full case): their G rows packed in order, one tile layout."""
    cu = case.cu
    idx = torch.cat([torch.arange(int(cu[b]), int(cu[b + 1])) for b in seqs])
    dev = case.G.device
    sub = LstmCase(case.dirs, case.G[idx.to(dev)], case.w_hh, [case.lens[b] for b in seqs],
                   tile_layout(list(range(len(seqs)))).to(dev),
                   pad=None if case.pad is None else case.pad[idx.to(dev)],
                   tail=None if case.tail is None else case.tail[torch.tensor(list(seqs), device=dev)],
                   pad_value=case.pad_value, label=case.label)
    return sub, idx


# ---------------------------------------------------------------------------------------------------------------------
# tolerances
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Tol:
    """|err| <= atol + rtol |ref| element-wise, mean |err| <= mean * mean |ref|, and the error's projection on the
    reference |sum(err * ref)| / sum(ref^2) <= bias: a scale error of the whole output shows up there whatever its sign,
    while rounding errors of either sign cancel."""

    atol: float
    rtol: float
    mean: float
    bias: float


# The output's own rounding: y = bf16(h) is within half a bf16 ulp of h, at most 2^-8 |h| (half of 2^-7 at the bottom of a
# binade), and on average a quarter ulp, about 2^-10 |h|.  Every rtol and mean term below starts from these.
#
# Random weights (the recurrence family).  Each step rounds h to bf16 for the matmul.  Where the kernel's fp32 h and the
# float64 h straddle a bf16 rounding boundary, the two matmuls read inputs one ulp apart, and the difference travels
# through W_hh into later steps, where it moves more h values across boundaries; the carried error is absolute, not
# relative to h.  The rounding model (fp32 z and c, the SFU results off by up to their documented ulp bounds, bf16 h into
# the matmul and out) reaches a carried error of 2.3e-3 (bound 0.1) and 1.9e-3 (1/sqrt(512)) over the CPU cases; atol is
# four times that, rtol one output rounding.  The mean term, here and below, is 2^-8 of mean |ref|, twice the mean output
# rounding and about 1.4x the model's mean error; the bias term is 2e-3: a 1 % scale error moves the bias by 1e-2.
# Measured on an H100 80GB HBM3 (700 W power limit) over the GPU test's random-weight cases: y at most 0.375 of this
# tolerance (2048 steps, dirs = 1, bound 0.1; 11.6 % of the outputs not bit-equal to bf16 of the reference), the pool at
# most 0.054, the 32 768-sequence sample 0.360 (y) / 0.029 (pool).
RANDOM_TOL = Tol(atol=1.0e-2, rtol=2.0 ** -8, mean=2.0 ** -8, bias=2.0e-3)
# W_hh = 0: nothing is carried through the matmul, c is carried in fp32 (relative error ~ steps * 2^-24 at most).  The
# output rounding alone reaches 2^-8 |ref| at the bottom of a binade, and fp32 h landing on the other side of a rounding
# boundary adds its own (tiny) error to that; rtol = 2.5 output roundings keeps the rounding at 0.4 of the element term.
# Measured (same card): y 0.398 of this tolerance, 0.007 % of the outputs not bit-equal; pool 0.001.
ZERO_TOL = Tol(atol=1.0e-5, rtol=5 * 2.0 ** -9, mean=2.0 ** -8, bias=1.0e-3)
# Permutation and saturated W_hh: every matmul is one exact product, but a bf16 flip of the h it reads (one ulp, at most
# 2^-8 for |h| < 1, times a weight of at most 1) is carried into the next step: 2^-8 absolute on top of ZERO_TOL.  A
# stale, misrouted or skipped slice moves z by a whole product, O(0.1), which is 25x this atol.
# Measured (same card): permutation y 0.360 (0.009 % not bit-equal), saturated y 0.222 (0.001 %); pools at most 0.023.
EXACT_TOL = Tol(atol=2.0 ** -8, rtol=5 * 2.0 ** -9, mean=2.0 ** -8, bias=1.0e-3)


# The input GEMM's G = x . W_ih^T + b at LASER's shapes (K = 320, 1024; N = 4096): the bf16 output rounding (up to
# 2^-8 |ref|, kept at 0.4 of rtol as for ZERO_TOL), the fp32 accumulation over K <= 1024 products (well under atol near
# zero), the mean output rounding doubled, and the bias term at 1e-3: a 0.5 % scale error moves it by 5e-3.
# Measured (same card) over the five layers of the `laser2` shape at T = 7369: at most 0.388 of this tolerance.
GEMM_TOL = Tol(atol=1.0e-3, rtol=5 * 2.0 ** -9, mean=2.0 ** -8, bias=1.0e-3)


def violation(got: torch.Tensor, ref: torch.Tensor, tol: Tol) -> float:
    """How far `got` is from `ref` in units of the tolerance (<= 1 passes), over the elements where `ref` is not NaN.
    Infinite entries must agree exactly; a NaN in `got` where `ref` has a value is infinitely far."""
    keep = ~torch.isnan(ref)
    got, ref = got.double()[keep], ref.double()[keep]
    if bool(torch.isnan(got).any()):
        return math.inf
    inf = torch.isinf(ref) | torch.isinf(got)
    if not torch.equal(got[inf], ref[inf]):
        return math.inf
    got, ref = got[~inf], ref[~inf]
    if got.numel() == 0:
        return 0.0
    err = got - ref
    elem = float((err.abs() / (tol.atol + tol.rtol * ref.abs())).max())
    mag = float(ref.abs().mean())
    mean = float(err.abs().mean()) / (tol.mean * mag) if mag > 0 else 0.0
    denom = float((ref * ref).sum())
    bias = abs(float((err * ref).sum())) / denom / tol.bias if denom > 0 else 0.0
    return max(elem, mean, bias)


def not_bit_equal(y: torch.Tensor, ref: torch.Tensor) -> float:
    """Share of the bf16 outputs that differ from bf16(ref), over the elements where ref is not NaN.  References below
    the smallest normal fp32 count as zero: the kernel's sigmoid of -90 is exactly 0 (__expf(90) overflows), float64's
    is 8e-40."""
    keep = ~torch.isnan(ref)
    r = ref[keep].double()
    r = torch.where(r.abs() < 2.0 ** -126, torch.zeros_like(r), r)
    return float((y[keep].view(torch.int16) != r.to(torch.bfloat16).view(torch.int16)).double().mean())


# ---------------------------------------------------------------------------------------------------------------------
# the embedding gather and the repack
# ---------------------------------------------------------------------------------------------------------------------
def embed_reference(ids: torch.Tensor, lens: Sequence[int], S: int, table: torch.Tensor, pad_idx: int):
    """(x bf16 [T, D], pad uint8 [T], tail uint8 [B], bad): row cu[b] + t = table[ids[b, t]] (zeros for an id outside
    [0, V)), pad = id == pad_idx, tail[b] = some ids[b, t] != pad_idx for len_b <= t < S, bad = any id outside [0, V)."""
    V = table.shape[0]
    rows = [ids[b, :n] for b, n in enumerate(lens)]
    tok = torch.cat(rows) if rows else ids.new_zeros(0)
    ok = (tok >= 0) & (tok < V)
    x = torch.where(ok[:, None], table[tok.clamp(0, V - 1)], torch.zeros((), dtype=table.dtype, device=table.device))
    pad = (tok == pad_idx).to(torch.uint8)
    tail = torch.tensor([bool((ids[b, n:S] != pad_idx).any()) for b, n in enumerate(lens)], dtype=torch.uint8)
    return x, pad, tail.to(ids.device), bool((~ok).any())


def repack_reference(w_nat: torch.Tensor, b_ih: torch.Tensor, b_hh: torch.Tensor, dirs: int):
    """(rows of the stacked natural-order weights in gate order, fp32 b_ih + b_hh in gate order) for `dirs` directions
    stacked along dim 0."""
    rows = gate_rows(dirs).to(w_nat.device)
    return w_nat[rows], (b_ih.float() + b_hh.float())[rows]


# ---------------------------------------------------------------------------------------------------------------------
# the GPU test's recurrence inputs
# ---------------------------------------------------------------------------------------------------------------------
G_STD = {WEIGHT_BOUNDS[0]: 1.0, WEIGHT_BOUNDS[1]: 0.5}  # about the spread of x . W_ih^T + b at the same bound, D = 320
EXACT_LENGTHS = [1, 2, 3, 17, 64, 65, 129, 300, 2048] + list(range(4, 80, 3))


def mixed_case(dirs: int, bound: float, device="cpu") -> LstmCase:
    """72 sequences of 1..129 tokens and one of 300 (the long neighbour), in two tiles: -1 holes at rows 5 and 37 of the
    first, at row 70 in the middle of the second (partly filled) one and -1 rows at its end; then a tile with no
    sequence.  Sequences 9 and 50 are in no tile (NaN G rows); G is a column view whose 64 extra columns hold NaN.  Pad
    flags at 15 %, sequence 20 all pad, tail flags at 50 %, padding value 0.25."""
    g = torch.Generator().manual_seed(17 * dirs)
    lens = torch.randint(1, 130, (73,), generator=g).tolist()
    lens[3], lens[40], lens[60] = 1, 300, 2
    case = make_random_case(dirs, lens, bound=bound, g_std=G_STD[bound], seed=dirs, holes=(5, 37, 70), empty_tiles=1,
                            orphans=(9, 50), extra_cols=64, device=device, label=f"mixed dirs={dirs} bound={bound:.3f}")
    return with_pool(case, all_pad=(20,), seed=dirs)


def edge_case(dirs: int, bound: float, device="cpu") -> LstmCase:
    """EDGE_LENGTHS and 30 sequences of 1..40 tokens, shuffled over one tile with a hole at row 30."""
    g = torch.Generator().manual_seed(5 + dirs)
    lens = EDGE_LENGTHS + torch.randint(1, 41, (30,), generator=g).tolist()
    return make_random_case(dirs, lens, bound=bound, g_std=G_STD[bound], seed=100 + dirs, holes=(30,), device=device,
                            label=f"edges dirs={dirs} bound={bound:.3f}")
