"""CPU: the references of tests/test_gpu_laser2_kernels.py are the oracle's maths, a model of the recurrent kernel's rounding
stays within half of each tolerance, and the tolerances can see the indexing, routing and masking bugs that matter in the
LASER2 kernels.  The argument checks of the kernel-level entry points run here too: they refuse before touching a device."""

import ctypes as C

import pytest
import torch

from oracle.laser_lstm import OracleLaser2, OracleLaser2Config, make_synthetic_laser2_state_dict
from tests.laser2_kernel_cases import (EDGE_LENGTHS, EXACT_LENGTHS, EXACT_TOL, FAULTS, H, RANDOM_TOL, WEIGHT_BOUNDS,
                                       ZERO_TOL, LstmCase, edge_case, embed_reference, gate_rows, lstm_reference,
                                       make_exact_case, mixed_case, permutation_weights, repack_reference, tile_layout,
                                       violation)


@pytest.fixture(autouse=True, scope="module")
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(max(n, 4))
    yield
    torch.set_num_threads(n)


# ---------------------------------------------------------------------------------------------------------------------
# the references are the oracle's maths
# ---------------------------------------------------------------------------------------------------------------------
def test_gate_rows_match_torch_lstm_layout_and_ops():
    """Running torch.nn.LSTM on natural-order weights equals the reference on the same weights taken in gate order, and
    gate_rows is the ops wrapper's lstm_gate_rows."""
    from sonar_b200.ops import lstm_gate_rows

    for dirs in (1, 2):
        assert torch.equal(gate_rows(dirs), lstm_gate_rows(H, dirs))
    rows = gate_rows(2)
    assert torch.equal(torch.sort(rows).values, torch.arange(2 * 4 * H))
    g = torch.Generator().manual_seed(0)
    lstm = torch.nn.LSTM(8, H, bidirectional=True).double()
    x = torch.randn((5, 1, 8), generator=g, dtype=torch.float64)
    with torch.no_grad():
        want, _ = lstm(x)
        w_ih = torch.cat([lstm.weight_ih_l0, lstm.weight_ih_l0_reverse])
        w_hh = torch.cat([lstm.weight_hh_l0, lstm.weight_hh_l0_reverse])
        b = torch.cat([lstm.bias_ih_l0 + lstm.bias_hh_l0, lstm.bias_ih_l0_reverse + lstm.bias_hh_l0_reverse])
        G = x[:, 0] @ w_ih[rows].T + b[rows]
        case = LstmCase(2, G, w_hh[rows], [5], tile_layout([0]))
        y, _ = lstm_reference(case, round_h=False)
    torch.testing.assert_close(y, want[:, 0], rtol=0, atol=1e-12)


def test_repack_reference_is_gate_order_and_fp32_bias_sum():
    g = torch.Generator().manual_seed(1)
    w = torch.randn((2 * 4 * H, 24), generator=g).to(torch.bfloat16)
    b_ih, b_hh = torch.randn(2 * 4 * H, generator=g), torch.randn(2 * 4 * H, generator=g)
    wr, br = repack_reference(w, b_ih, b_hh, 2)
    for n in (0, 31, 32, 127, 128, 1000, 2047, 2048, 4095):  # row 128 c + 32 gate + u of direction d
        d, m = divmod(n, 4 * H)
        c, gate, u = m // 128, (m % 128) // 32, m % 32
        src = d * 4 * H + gate * H + 32 * c + u
        assert torch.equal(wr[n], w[src]) and float(br[n]) == float(b_ih[src].float() + b_hh[src].float())


@pytest.mark.parametrize("bidirectional", [False, True])
def test_reference_chained_over_layers_is_the_oracle(bidirectional):
    """Embedding gather, then per layer G = x . W_ih^T + b in float64 and the recurrence reference without rounding, then
    the max with the oracle's masking (pad ids -inf, positions past the length padding_value): OracleLaser2 exactly."""
    cfg = OracleLaser2Config(vocabulary_size=40, model_dim=64, num_layers=2, bidirectional=bidirectional, padding_value=0.5)
    sd = make_synthetic_laser2_state_dict(cfg, seed=4, weight_bound=0.1)
    dirs = 2 if bidirectional else 1
    lens = [5, 1, 7, 3]
    S = 8
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(3, cfg.vocabulary_size, (4, S), generator=g)
    ids[0, 2] = cfg.pad_idx             # a pad id inside a sentence
    ids[1, 1:] = cfg.pad_idx            # padded with pad ids: no tail
    ids[3, :] = cfg.pad_idx             # all pad: -inf, no tail
    ids[2, 7] = cfg.pad_idx             # the one position past length 7 is a pad id: no tail
    x, pad, tail, bad = embed_reference(ids, lens, S, sd["embed_tokens.weight"].double(), cfg.pad_idx)
    assert not bad and tail.tolist() == [1, 0, 0, 0]
    rows = gate_rows(dirs)
    for layer in range(cfg.num_layers):
        sfx = ["", "_reverse"][:dirs]
        w_ih = torch.cat([sd[f"lstm.weight_ih_l{layer}{s}"] for s in sfx]).double()
        w_hh = torch.cat([sd[f"lstm.weight_hh_l{layer}{s}"] for s in sfx]).double()
        b = torch.cat([sd[f"lstm.bias_ih_l{layer}{s}"].double() + sd[f"lstm.bias_hh_l{layer}{s}"].double() for s in sfx])
        case = LstmCase(dirs, x @ w_ih[rows].T + b[rows], w_hh[rows], lens, tile_layout(range(4)), pad=pad, tail=tail,
                        pad_value=cfg.padding_value)
        x, pool = lstm_reference(case, round_h=False)
    want = OracleLaser2(cfg, sd)(ids, torch.tensor(lens))
    assert torch.equal(torch.isinf(pool), torch.isinf(want)) and bool(torch.isinf(pool[3]).all())
    fin = torch.isfinite(want)
    torch.testing.assert_close(pool[fin], want[fin], rtol=0, atol=1e-12)


def test_embed_reference_flags():
    table = torch.arange(12, dtype=torch.float32).view(4, 3).to(torch.bfloat16)
    ids = torch.tensor([[2, 1, 3, 9, 1], [-1, 4, 1, 1, 7]])
    x, pad, tail, bad = embed_reference(ids, [3, 2], 4, table, pad_idx=1)
    assert bad and pad.tolist() == [0, 1, 0, 0, 0] and tail.tolist() == [1, 0]  # position 4 (>= S) does not count
    assert torch.equal(x[0], table[2]) and bool((x[3] == 0).all()) and bool((x[4] == 0).all())


def test_permutation_weights_read_every_slice_in_every_cta():
    w = permutation_weights(2).float()
    assert bool(((w != 0).sum(1) == 1).all()) and set(w[w != 0].abs().tolist()) == {0.5, 1.0}
    for d in range(2):
        for c in range(16):
            src = w[d * 4 * H + 128 * c : d * 4 * H + 128 * (c + 1)].nonzero()[:, 1] // 32
            assert sorted(set(src.tolist())) == list(range(16)), (d, c)


# ---------------------------------------------------------------------------------------------------------------------
# the rounding model stays within half of each tolerance
# ---------------------------------------------------------------------------------------------------------------------
def _model_fraction(case, tol):
    y, pool = lstm_reference(case)
    ym, pm = lstm_reference(case, model_seed=7)
    return violation(ym, y, tol), violation(pm, pool, tol)


@pytest.mark.parametrize("bound", WEIGHT_BOUNDS)
@pytest.mark.parametrize("dirs", [1, 2])
def test_rounding_model_within_half_the_random_tolerance(dirs, bound):
    vy, vp = _model_fraction(mixed_case(dirs, bound), RANDOM_TOL)
    print(f"mixed dirs={dirs} bound={bound:.3f}: rounding model at {vy:.3f} (y) / {vp:.3f} (pool) of the tolerance")
    assert vy <= 0.5 and vp <= 0.5


@pytest.mark.parametrize("bound", WEIGHT_BOUNDS)
@pytest.mark.parametrize("dirs", [1, 2])
def test_rounding_model_within_half_the_random_tolerance_at_2048_steps(dirs, bound):
    case = edge_case(dirs, bound)
    assert max(case.lens) == max(EDGE_LENGTHS) == 2048
    vy, vp = _model_fraction(case, RANDOM_TOL)
    print(f"edges dirs={dirs} bound={bound:.3f}: rounding model at {vy:.3f} (y) / {vp:.3f} (pool) of the tolerance")
    assert vy <= 0.5 and vp <= 0.5


@pytest.mark.parametrize("kind", ["zero", "permutation", "saturated"])
def test_rounding_model_within_half_the_exact_tolerance(kind):
    vy, vp = _model_fraction(make_exact_case(2, EXACT_LENGTHS, kind, seed=3), ZERO_TOL if kind == "zero" else EXACT_TOL)
    print(f"{kind}: rounding model at {vy:.3f} (y) / {vp:.3f} (pool) of the tolerance")
    assert vy <= 0.5 and vp <= 0.5


def test_saturated_case_saturates():
    """The saturated inputs reach the sigmoid's ends exactly in fp32 (sigma(+-90), sigma(+-100) = 1 or 0), and c grows
    past 1e3 over 2048 steps."""
    case = make_exact_case(1, [2048], "saturated", seed=3)
    z = case.G[:, : 4 * H].float()
    assert set(z.abs().unique().tolist()) >= {90.0, 100.0}
    sig = 1.0 / (1.0 + torch.exp(-torch.tensor([90.0, 100.0, -90.0, -100.0])))
    assert sig.tolist() == [1.0, 1.0, 0.0, 0.0]
    y, _ = lstm_reference(case)
    assert bool((y.abs() <= 1).all()) and float((y == 1.0).double().mean()) > 0.05


# ---------------------------------------------------------------------------------------------------------------------
# every fault misses its tolerance on the GPU test's own inputs
# ---------------------------------------------------------------------------------------------------------------------
POOL_ONLY = {"finished_max", "pad_in_max", "tail_ignored", "tail_min"}


@pytest.mark.parametrize("bound", WEIGHT_BOUNDS)
def test_faults_miss_the_random_tolerance(bound):
    case = mixed_case(2, bound)
    y, pool = lstm_reference(case)
    for name, f in FAULTS.items():
        yf, pf = lstm_reference(case, fault=f)
        v = violation(pf, pool, RANDOM_TOL) if f in POOL_ONLY else min(violation(yf, y, RANDOM_TOL),
                                                                        violation(pf, pool, RANDOM_TOL))
        print(f"mixed bound={bound:.3f}, {name}: {v:.2f} x the tolerance")
        assert v > 1.0, (name, v)


@pytest.mark.parametrize("kind", ["zero", "permutation", "saturated"])
def test_faults_miss_the_exact_tolerance(kind):
    """The W_hh = 0 case carries nothing between units, so only the token-mapping and scale faults apply to it; on the
    permutation and saturated cases every routing fault moves y by a whole product."""
    case = make_exact_case(2, EXACT_LENGTHS, kind, seed=3)
    tol = ZERO_TOL if kind == "zero" else EXACT_TOL
    y, _ = lstm_reference(case)
    routing = {"stale_peer", "misroute", "skip_k16", "swap_rows"}
    for name, f in FAULTS.items():
        if f in POOL_ONLY or (kind == "zero" and f in routing):
            continue
        v = violation(lstm_reference(case, fault=f)[0], y, tol)
        print(f"{kind}, {name}: {v:.2f} x the tolerance")
        assert v > 1.0, (name, v)


# ---------------------------------------------------------------------------------------------------------------------
# argument checks: refused before any launch (fake device addresses; nothing is dereferenced)
# ---------------------------------------------------------------------------------------------------------------------
A = 1 << 20  # a 1 MB-aligned fake device address


def _lstm_rc(lib, *, G=A, ldg=2 * 4 * H, w=A, y=A, ldy=2 * H, pool=None, ldp=0, dirs=2):
    return lib.sb_lstm_recurrent(G, ldg, w, A, A, 1, dirs, y, ldy, pool, ldp, None, None, 0.0, None)


def test_lstm_recurrent_refuses_bad_leading_dimensions_and_alignment(native_lib):
    from sonar_b200 import _lib

    bad = {"ldg < dirs * 4H": dict(ldg=2 * 4 * H - 2), "odd ldg": dict(ldg=2 * 4 * H + 1),
           "ldy < dirs * H": dict(ldy=2 * H - 2), "odd ldy": dict(ldy=2 * H + 1),
           "ldp < dirs * H": dict(y=None, pool=A, ldp=H), "odd ldp": dict(y=None, pool=A, ldp=2 * H + 1),
           "ldg for one direction with two": dict(ldg=4 * H),
           "G 2-byte aligned": dict(G=A + 2), "y 2-byte aligned": dict(y=A + 2), "pool 4-byte aligned": dict(y=None, pool=A + 4, ldp=2 * H),
           "w_hh 8-byte aligned": dict(w=A + 8), "three directions": dict(dirs=3)}
    for what, kw in bad.items():
        assert _lstm_rc(native_lib, **kw) == _lib.SB_ERR_INVALID, what
        assert "sb_lstm_recurrent" in _lib.last_error(), what


def test_laser2_embed_and_create_refuse_misaligned_tables(native_lib):
    from sonar_b200 import _lib

    def embed(table=A, x=A, D=320, stride=8, S=8):
        return native_lib.sb_laser2_embed(A, stride, A, 2, S, table, 100, D, 1, x, A, A, A, None)

    for what, kw in {"table 8-byte aligned": dict(table=A + 8), "x 2-byte aligned": dict(x=A + 2), "D = 12": dict(D=12),
                     "stride < S": dict(stride=7)}.items():
        assert embed(**kw) == _lib.SB_ERR_INVALID, what
        assert "sb_laser2_embed" in _lib.last_error()
    cfg = _lib.SbLaser2Config(vocab_size=100, pad_idx=1, embed_dim=64, hidden_size=512, num_layers=1, bidirectional=0,
                              padding_value=0.0, num_sms=0)
    layers = (_lib.SbLstmLayerWeights * 1)(_lib.SbLstmLayerWeights(A, A, A, A))
    w = _lib.SbLaser2Weights(embed=A + 8, layers=layers)
    out = C.c_void_p()
    assert native_lib.sb_laser2_create(C.byref(cfg), C.byref(w), C.byref(out)) == _lib.SB_ERR_INVALID
    assert "16-byte aligned" in _lib.last_error() and not out.value
