"""CPU: the references and tolerances of tests/test_gpu_conformer_kernels.py can see the bugs that matter, and the engine's
relative-position table is the oracle's."""

import pytest
import torch

from oracle.speech_encoder import rel_pos_table
from sonar_b200.speech_encoder import relative_position_table, relpos_rows
from tests.conformer_kernel_cases import (ATTN_CASES, ATTN_TOL, CONV_DIMS, attn_violation, conv_reference, conv_violation,
                                          make_conv_case, make_relpos_case, relpos_reference)


@pytest.mark.parametrize("s", [1, 2, 64, 129, 499, 1031])
@pytest.mark.parametrize("d", [256, 1024])
def test_engine_relpos_table_is_the_oracle_table(s, d):
    t = relative_position_table(s, d, relpos_rows(s))
    assert t.shape == (relpos_rows(s), d) and relpos_rows(s) % 256 == 0 and relpos_rows(s) >= 2 * s - 1
    assert torch.equal(t[: 2 * s - 1], rel_pos_table(s, d))
    assert not bool(t[2 * s - 1 :].any())


# Reading p one row off is what an off-by-one Transformer-XL shift does, and what an S_center one off does in either
# kernel (both only use it as the row of relative position 0); a table built for S_center - 1 reads the neighbouring
# relative position with real values instead of zero rows at the ends.
ATTN_BUGS = {
    "shift +1": dict(row_shift=1),
    "shift -1": dict(row_shift=-1),
    "relative position sign flipped": dict(flip=True),
    "u_bias dropped": dict(drop_u=True),
    "v_bias dropped": dict(drop_v=True),
    "position term dropped": dict(drop_position=True),
    "last key masked": dict(mask_last_key=True),
    "table built for S_center - 1": dict(center=-1, row_shift=1),
}


@pytest.mark.parametrize("name", [n for n in ATTN_CASES if max(ATTN_CASES[n][0]) > 1])  # one key: every score bug is invisible
def test_relpos_tolerances_catch_position_and_mask_bugs(name):
    """On the inputs of the GPU test, each bug moves the reference by at least 4x the tolerance of either kernel."""
    lens, heads = ATTN_CASES[name]
    case = make_relpos_case(lens, heads)
    c = max(lens)
    ref = torch.cat([relpos_reference(case, b, c) for b in range(len(lens))])
    for bug, kw in ATTN_BUGS.items():
        kw = dict(kw)
        center = c + kw.pop("center", 0)
        got = torch.cat([relpos_reference(case, b, center, **kw) if not (bug == "last key masked" and n < 2)
                         else relpos_reference(case, b, c) for b, n in enumerate(lens)])
        for impl in ATTN_TOL:
            v = attn_violation(got, ref, impl)
            assert v >= 4.0, (name, bug, impl, v)


@pytest.mark.parametrize("d", CONV_DIMS)
def test_conv_tolerances_catch_tap_and_halo_bugs(d):
    case = make_conv_case(d, seed=d)
    ref = torch.cat([conv_reference(case, b) for b in range(len(case.lens))])
    for bug in ("reverse_taps", "tile_halo_cut", "neighbour_halo"):
        got = torch.cat([conv_reference(case, b, **{bug: True}) for b in range(len(case.lens))])
        v = conv_violation(got, ref)
        assert v >= 4.0, (bug, v)
