"""Env-gated real-weight goldens of BLASER 2.0.  Nothing here runs offline -- the checkpoints cannot be downloaded in this
environment -- but with

    SONAR_B200_CHECKPOINT_DIR=<dir>   holding   blaser_2_0_ref.pt   (the `blaser_2_0_ref` card's checkpoint)
                                                blaser_2_0_qe.pt    (the `blaser_2_0_qe` card's checkpoint)

this reproduces the reference's own check (tests/integration_tests/test_blaser.py:13-39): the five scores of a constant
embedding (every component 1/32) against itself and its negation.  The reference asserts torch's default fp32 tolerance on
an fp32 CPU model.  The engine computes the features and the first hidden layer in bf16 (relative rounding 2^-9) and the
tanh with MUFU.TANH (relative error 2^-11); on synthetic weights with a score spread of 0.76 that moves a score by up to
about 0.014, so it is held to 5e-2 absolute here."""

import os
from pathlib import Path

import pytest
import torch

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.environ.get("SONAR_B200_CHECKPOINT_DIR"), reason="real BLASER checkpoints not available")]

# (card, mt sign, ref sign, expected score); src = emb
GOLDEN = [("blaser_2_0_ref", 1, 1, 5.255207538604736), ("blaser_2_0_ref", 1, -1, 2.309619665145874),
          ("blaser_2_0_ref", -1, 1, -2.178907632827759), ("blaser_2_0_qe", 1, None, 4.981893062591553),
          ("blaser_2_0_qe", -1, None, -0.8291061520576477)]


@pytest.mark.parametrize("card", ["blaser_2_0_ref", "blaser_2_0_qe"])
def test_blaser2_scalar_goldens(native_lib, cuda_device, card):
    from sonar_b200 import load_blaser_model

    if not (Path(os.environ["SONAR_B200_CHECKPOINT_DIR"]) / f"{card}.pt").exists():
        pytest.skip(f"{card}.pt not found")
    model = load_blaser_model(card, device=cuda_device)
    emb = torch.zeros([1, 1024]) + 1 / 32
    for name, mt_sign, ref_sign, want in GOLDEN:
        if name != card:
            continue
        ref = None if ref_sign is None else ref_sign * emb
        pred = model(src=emb, mt=mt_sign * emb, ref=ref).item()
        assert abs(pred - want) <= 5e-2, (card, mt_sign, ref_sign, pred, want)
