"""Kernel-level parity of the LASER2 encoder's own kernels (through the C ABI, on the launch paths sb_laser2_forward uses)
against float64 references of the same operation on the same inputs: the cluster-resident LSTM recurrence, the embedding
gather and the gate-order repack; then the whole encoder against the chain of those parts, bit for bit.
Inputs, references and tolerances: tests/laser2_kernel_cases.py."""

import pytest
import torch

from tests.laser2_kernel_cases import (EDGE_LENGTHS, EXACT_LENGTHS, EXACT_TOL, GEMM_TOL, H, RANDOM_TOL, WEIGHT_BOUNDS,
                                       ZERO_TOL, LstmCase, edge_case, embed_reference, lstm_reference, make_exact_case,
                                       make_random_case, mixed_case, not_bit_equal, repack_reference, subset, tile_layout,
                                       violation, with_pool)

pytestmark = pytest.mark.gpu

GUARD = 3            # guard rows after every output, and GUARD_COLS columns past its data
GUARD_COLS = 16      # even: the leading dimension stays even
SENTINEL = -768.0    # exact in bf16 and fp32


@pytest.fixture(scope="module")
def ops(native_lib, cuda_device):
    from sonar_b200 import ops as _ops

    torch.cuda.set_device(cuda_device)
    return _ops


def _bits(x):
    return x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32)


def _run(ops, case: LstmCase, pool: bool, *, null_masks: bool = False):
    """The kernel on `case` into a guarded buffer (rows and columns of SENTINEL around the output); checks the guards and
    that rows the kernel must not write (tokens and sequences of no tile) still hold SENTINEL.  -> the output view."""
    dev = case.G.device
    rows = len(case.lens) if pool else case.tokens
    width = case.dirs * H
    dtype = torch.float32 if pool else torch.bfloat16
    buf = torch.full((rows + GUARD, width + GUARD_COLS), SENTINEL, dtype=dtype, device=dev)
    out = buf[:rows, :width]
    cu = case.cu.to(dev)
    ops.lstm_recurrent(case.G, case.w_hh, cu, case.tile_seqs, case.dirs, pool=pool,
                       pad_mask=None if null_masks else case.pad, tail_keep=None if null_masks else case.tail,
                       padding_value=case.pad_value, out=out)
    torch.cuda.synchronize()
    assert bool((buf[rows:] == SENTINEL).all()) and bool((buf[:, width:] == SENTINEL).all()), "wrote past its output"
    tiled = set(case.tiled())
    missing = [b for b in range(len(case.lens)) if b not in tiled]
    if missing:
        idx = torch.tensor(missing) if pool else torch.cat([torch.arange(int(case.cu[b]), int(case.cu[b + 1])) for b in missing])
        assert bool((out[idx.to(dev)] == SENTINEL).all()), "wrote rows of a sequence in no tile"
    return out


def _report(label, v, extra=""):
    print(f"{label}: {v:.3f} of the tolerance{extra}")
    assert v <= 1.0, (label, v)


# ---------------------------------------------------------------------------------------------------------------------
# recurrence against the float64 reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bound", WEIGHT_BOUNDS)
@pytest.mark.parametrize("dirs", [1, 2])
def test_recurrence_mixed_tiles_vs_float64(ops, cuda_device, dirs, bound):
    """Two tiles with -1 holes in the middle and at the end, a tile with no sequence, two sequences in no tile whose G
    rows are NaN, G a column view whose other columns are NaN; y and the pool (pad flags, an all-pad sequence, tail
    flags) within RANDOM_TOL, guards and untiled rows untouched."""
    case = mixed_case(dirs, bound, device=cuda_device)
    y_ref, p_ref = lstm_reference(case)
    y = _run(ops, case, pool=False)
    p = _run(ops, case, pool=True)
    _report(f"{case.label} y", violation(y, y_ref, RANDOM_TOL), f", {not_bit_equal(y, y_ref):.4f} not bit-equal")
    _report(f"{case.label} pool", violation(p, p_ref, RANDOM_TOL))


@pytest.mark.parametrize("bound", WEIGHT_BOUNDS)
@pytest.mark.parametrize("dirs", [1, 2])
def test_recurrence_step_edges_to_2048_vs_float64(ops, cuda_device, dirs, bound):
    case = edge_case(dirs, bound, device=cuda_device)
    assert max(case.lens) == max(EDGE_LENGTHS)
    y_ref, _ = lstm_reference(case)
    y = _run(ops, case, pool=False)
    _report(f"{case.label} y", violation(y, y_ref, RANDOM_TOL), f", {not_bit_equal(y, y_ref):.4f} not bit-equal")


def test_recurrence_32768_sequences_vs_float64_sample(ops, cuda_device):
    """512 tiles x 2 directions: many waves of clusters.  Sequences of 1..6 tokens; the reference runs on 256 of them
    spread over all tiles (a row's result does not depend on its neighbours)."""
    g = torch.Generator().manual_seed(9)
    B = 32768
    lens = torch.randint(1, 7, (B,), generator=g).tolist()
    case = make_random_case(2, lens, bound=WEIGHT_BOUNDS[0], seed=9, order=list(range(B)), device=cuda_device,
                            draw_on_device=True)
    case = with_pool(case, seed=9, pad_value=-0.0625)
    y = _run(ops, case, pool=False)
    p = _run(ops, case, pool=True)
    sample = sorted(set(torch.randint(0, B, (256,), generator=g).tolist()) | {0, 63, 64, B - 1})
    sub, idx = subset(case, sample)
    y_ref, p_ref = lstm_reference(sub)
    _report("B=32768 sample y", violation(y[idx.to(cuda_device)], y_ref, RANDOM_TOL))
    _report("B=32768 sample pool", violation(p[torch.tensor(sample, device=cuda_device)], p_ref, RANDOM_TOL))


# ---------------------------------------------------------------------------------------------------------------------
# exact operands
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["zero", "permutation", "saturated"])
def test_recurrence_exact_operands(ops, cuda_device, kind):
    case = with_pool(make_exact_case(2, EXACT_LENGTHS, kind, seed=3, device=cuda_device), seed=3)
    tol = ZERO_TOL if kind == "zero" else EXACT_TOL
    y_ref, p_ref = lstm_reference(case)
    y = _run(ops, case, pool=False)
    p = _run(ops, case, pool=True)
    _report(f"{kind} y", violation(y, y_ref, tol), f", {not_bit_equal(y, y_ref):.5f} not bit-equal")
    _report(f"{kind} pool", violation(p, p_ref, tol))
    if kind == "saturated":  # sigma(+-90), sigma(+-100) exactly 0 or 1: the units of regimes 1 (h = 0) and 2 (tanh(integer))
        units = torch.arange(2 * H, device=cuda_device) % H % 4
        assert bool((y[:, units == 1] == 0).all())
        r2 = y[:, units == 2].float()
        steps = torch.tanh(torch.arange(-64, 65, device=cuda_device, dtype=torch.float64)).to(torch.bfloat16).float()
        assert bool(torch.isin(r2, steps).all()), "h = tanh(c) of an integer c"


# ---------------------------------------------------------------------------------------------------------------------
# bitwise structure
# ---------------------------------------------------------------------------------------------------------------------
def test_a_sequence_gives_the_same_bits_in_any_row_tile_and_neighbourhood(ops, cuda_device):
    """Sequence 0 (57 tokens) in tile row 0, in row 63, in the second tile, and amid neighbours of up to 700 tokens whose
    G is 20x larger: the same y and pool bits every time."""
    g = torch.Generator().manual_seed(21)
    lens = [57] + torch.randint(1, 701, (70,), generator=g).tolist()
    base = make_random_case(2, lens, bound=0.1, seed=21, device=cuda_device)
    base.G[57:] *= 20
    base = with_pool(base, seed=21)
    others = list(range(1, 71))
    layouts = {"row 0": [0] + others, "row 63": others[:63] + [0] + others[63:],
               "second tile": others[:64] + [0] + others[64:], "alone": [0]}
    outs = {}
    for name, order in layouts.items():
        case = LstmCase(2, base.G, base.w_hh, lens, tile_layout(order).to(cuda_device), base.pad, base.tail, base.pad_value)
        outs[name] = (_run(ops, case, pool=False)[:57].clone(), _run(ops, case, pool=True)[0].clone())
    for name, (y, p) in outs.items():
        assert torch.equal(_bits(y), _bits(outs["alone"][0])) and torch.equal(_bits(p), _bits(outs["alone"][1])), name


def test_directions_are_independent_and_reverse_is_time_reversed_forward(ops, cuda_device):
    """The forward half of a dirs = 2 run is a dirs = 1 run on the forward weights; the reverse half is a forward run on
    each sequence's time-reversed G, reversed back; bit for bit, y and pool."""
    g = torch.Generator().manual_seed(23)
    lens = torch.randint(1, 200, (80,), generator=g).tolist()
    both = with_pool(make_random_case(2, lens, bound=0.1, seed=23, device=cuda_device), seed=23)
    y2, p2 = _run(ops, both, pool=False), _run(ops, both, pool=True)
    fwd = LstmCase(1, both.G[:, : 4 * H], both.w_hh[: 4 * H].contiguous(), lens, both.tile_seqs, both.pad, both.tail,
                   both.pad_value)
    assert torch.equal(_bits(_run(ops, fwd, pool=False)), _bits(y2[:, :H].contiguous()))
    assert torch.equal(_bits(_run(ops, fwd, pool=True)), _bits(p2[:, :H].contiguous()))
    cu = both.cu
    rev = torch.cat([torch.arange(int(cu[b + 1]) - 1, int(cu[b]) - 1, -1) for b in range(len(lens))]).to(cuda_device)
    back = LstmCase(1, both.G[rev, 4 * H :].contiguous(), both.w_hh[4 * H :].contiguous(), lens, both.tile_seqs,
                    both.pad[rev], both.tail, both.pad_value)
    yb = _run(ops, back, pool=False)
    assert torch.equal(_bits(yb[rev]), _bits(y2[:, H:].contiguous()))
    assert torch.equal(_bits(_run(ops, back, pool=True)), _bits(p2[:, H:].contiguous()))


# ---------------------------------------------------------------------------------------------------------------------
# pool
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pad_value,null_masks", [(-0.0625, False), (0.25, True)])
def test_pool_masks_tail_and_null_masks(ops, cuda_device, pad_value, null_masks):
    """Pad flags at 30 % with three all-pad sequences (-inf unless their tail is set), tail flags with a negative
    padding value; or pad_mask and tail_keep passed as NULL (every token counts, no tail)."""
    g = torch.Generator().manual_seed(29)
    lens = torch.randint(1, 60, (100,), generator=g).tolist()
    lens[7] = 1
    case = with_pool(make_random_case(2, lens, bound=0.1, seed=29, device=cuda_device), pad_rate=0.3, all_pad=(7, 30, 31),
                     pad_value=pad_value, seed=29)
    case.tail[30] = 0
    case.tail[31] = 1
    if null_masks:
        case = LstmCase(2, case.G, case.w_hh, lens, case.tile_seqs, label="null masks")
    p_ref = lstm_reference(case)[1]
    p = _run(ops, case, pool=True, null_masks=null_masks)
    if not null_masks:
        assert bool(torch.isinf(p[30]).all()) and bool((p[31] == pad_value).all())
    _report(f"pool pad_value={pad_value} null_masks={null_masks}", violation(p, p_ref, RANDOM_TOL))


# ---------------------------------------------------------------------------------------------------------------------
# embedding gather
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 320, 1024])
def test_embed_gather_flags_and_bad_ids(ops, cuda_device, D):
    """Bit-exact rows; pad flags including a pad id inside a sentence; tail flags read only positions < S although the
    ids rows are wider; ids -1 and V gather zeros and set the flag; an all-valid batch leaves it clear."""
    V, pad_idx, S, stride = 1000, 1, 24, 40
    g = torch.Generator().manual_seed(D)
    table = torch.randn((V, D), generator=g).to(torch.bfloat16).to(cuda_device)
    lens = torch.randint(1, S + 1, (50,), generator=g).tolist()
    lens[0], lens[1], lens[2] = S, 3, 5
    ids = torch.randint(3, V, (50, stride), generator=g)
    for b, n in enumerate(lens):
        ids[b, n:S] = pad_idx
    ids[1, 1] = pad_idx            # inside the sentence
    ids[2, S + 3] = 7              # past S: not a tail
    ids[3, lens[3]:S] = 0 if lens[3] < S else ids[3, lens[3]:S]  # padded with id 0: a tail when there is room
    ids = ids.to(cuda_device)
    cu = torch.zeros(51, dtype=torch.int32)
    cu[1:] = torch.cumsum(torch.tensor(lens), 0)
    cu = cu.to(cuda_device)
    T = int(cu[-1])
    x_buf = torch.full((T + GUARD, D), SENTINEL, dtype=torch.bfloat16, device=cuda_device)
    pad, tail = torch.full((T + GUARD,), 7, dtype=torch.uint8, device=cuda_device), torch.full((53,), 7, dtype=torch.uint8,
                                                                                                device=cuda_device)
    x, pad_o, tail_o, flag = ops.laser_embed(ids, cu, table, pad_idx, seq_len=S, out=(x_buf[:T], pad, tail))
    torch.cuda.synchronize()
    want = embed_reference(ids, lens, S, table, pad_idx)
    assert torch.equal(_bits(x), _bits(want[0])) and not want[3] and int(flag) == 0
    assert torch.equal(pad_o[:T], want[1]) and torch.equal(tail_o[:50], want[2])
    assert bool((x_buf[T:] == SENTINEL).all()) and bool((pad[T:] == 7).all()) and bool((tail[50:] == 7).all())
    assert int(tail_o[1]) == 0 and int(pad_o[int(cu[1]) + 1]) == 1
    bad = ids.clone()
    bad[0, 0], bad[4, 0] = -1, V
    x, _, _, flag = ops.laser_embed(bad, cu, table, pad_idx, seq_len=S)
    want = embed_reference(bad, lens, S, table, pad_idx)
    assert int(flag) == 1 and want[3] and torch.equal(_bits(x), _bits(want[0]))
    assert bool((x[0] == 0).all()) and bool((x[int(cu[4])] == 0).all())


def test_embed_32768_sequences(ops, cuda_device):
    V, D, S = 50004, 320, 12
    g = torch.Generator(device=cuda_device).manual_seed(3)
    table = torch.randn((V, D), generator=g, device=cuda_device).to(torch.bfloat16)
    lens = torch.randint(1, S + 1, (32768,), generator=g, device=cuda_device)
    ids = torch.randint(0, V, (32768, S), generator=g, device=cuda_device)
    cu = torch.zeros(32769, dtype=torch.int32, device=cuda_device)
    cu[1:] = torch.cumsum(lens, 0)
    x, pad, tail, flag = ops.laser_embed(ids, cu, table, 1)
    pos = torch.arange(S, device=cuda_device)[None, :]
    live = pos < lens[:, None]
    assert torch.equal(_bits(x), _bits(table[ids[live]])) and int(flag) == 0
    assert torch.equal(pad.bool(), ids[live] == 1)
    assert torch.equal(tail.bool(), ((ids != 1) & ~live).any(1))


# ---------------------------------------------------------------------------------------------------------------------
# repack and the engine as the chain of its parts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def laser2(ops, cuda_device):
    from oracle.laser_lstm import OracleLaser2Config, make_synthetic_laser2_state_dict
    from sonar_b200 import B200LaserLstmEncoder, Laser2Config

    cfg = OracleLaser2Config()  # the `laser2` shape: vocab 50004, 320 -> 5 x bidirectional 512
    sd = make_synthetic_laser2_state_dict(cfg, seed=5, weight_bound=0.1)
    lcfg = Laser2Config(vocabulary_size=cfg.vocabulary_size, pad_idx=cfg.pad_idx, model_dim=cfg.model_dim,
                        hidden_size=cfg.hidden_size, num_layers=cfg.num_layers, bidirectional=cfg.bidirectional,
                        padding_value=cfg.padding_value)
    return cfg, sd, B200LaserLstmEncoder(lcfg, sd, cuda_device)


def test_repack_is_gate_order_bit_for_bit(ops, laser2):
    cfg, sd, model = laser2
    for layer in range(cfg.num_layers):
        w_ih, bias, w_hh = ops.laser2_layer_weights(model, layer)
        sfx = ["", "_reverse"]
        cat = lambda k: torch.cat([sd[f"lstm.{k}_l{layer}{s}"] for s in sfx]).to(model.device)  # noqa: E731
        want_ih, want_b = repack_reference(cat("weight_ih").to(torch.bfloat16), cat("bias_ih"), cat("bias_hh"), 2)
        want_hh, _ = repack_reference(cat("weight_hh").to(torch.bfloat16), cat("bias_ih"), cat("bias_hh"), 2)
        assert torch.equal(_bits(w_ih), _bits(want_ih)), layer
        assert torch.equal(_bits(w_hh), _bits(want_hh)), layer
        assert torch.equal(_bits(bias), _bits(want_b)), layer


def test_engine_is_the_chain_of_its_parts(ops, laser2, cuda_device):
    """sb_laser2_forward = laser_embed -> gemm_bf16 (the handle's w_ih and bias) -> lstm_recurrent x 5 -> the pooling
    recurrence, bit for bit, on mixed lengths with the masking quirks; G of every layer against float64 x . W_ih^T + b."""
    cfg, sd, model = laser2
    g = torch.Generator().manual_seed(31)
    lens = torch.randint(1, 90, (150,), generator=g).tolist()
    lens[5], lens[77] = 700, 1
    S = max(lens) + 3
    ids = torch.full((150, S), cfg.pad_idx, dtype=torch.int64)
    for b, n in enumerate(lens):
        ids[b, :n] = torch.randint(3, cfg.vocabulary_size, (n,), generator=g)
    ids[0, 2] = cfg.pad_idx      # inside a sentence
    ids[1, lens[1]:] = 0         # padded with id 0: a tail
    ids[2, : lens[2]] = cfg.pad_idx  # all pad
    ids = ids.to(cuda_device)
    want = model(ids, torch.tensor(lens))
    torch.cuda.synchronize()
    model.check_inputs()
    cu = ops.cu_seqlens_of(lens).to(cuda_device)
    order = sorted(range(150), key=lambda b: -lens[b])  # the engine's tiles: longest first, ties in input order
    tiles = tile_layout(order).to(cuda_device)
    table = sd["embed_tokens.weight"].to(torch.bfloat16).to(cuda_device)
    x, pad, tail, flag = ops.laser_embed(ids, cu, table, cfg.pad_idx)
    assert int(flag) == 0
    worst = 0.0
    for layer in range(cfg.num_layers):
        w_ih, bias, w_hh = ops.laser2_layer_weights(model, layer)
        G = ops.gemm_bf16(x, w_ih, bias)
        v = violation(G, x.double() @ w_ih.double().T + bias.double(), GEMM_TOL)
        worst = max(worst, v)
        assert v <= 1.0, (layer, v)
        last = layer == cfg.num_layers - 1
        x = ops.lstm_recurrent(G, w_hh, cu, tiles, 2, pool=last, pad_mask=pad if last else None,
                               tail_keep=tail if last else None, padding_value=cfg.padding_value)
    torch.cuda.synchronize()
    print(f"G vs float64 x . W_ih^T + b: {worst:.3f} of the tolerance (K = 320, 1024; N = 4096; T = {sum(lens)})")
    assert torch.equal(_bits(x), _bits(want))
    assert bool(torch.isinf(want[2]).all()) and bool((want[1] >= 0).all())
