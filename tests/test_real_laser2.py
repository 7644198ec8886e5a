"""Env-gated real-weight golden of the LASER2 text encoder.  Nothing here runs offline -- the checkpoint and the
SentencePiece model cannot be downloaded in this environment -- but with

    SONAR_B200_CHECKPOINT_DIR=<dir>   holding   laser2.pt   (the `laser2_text_encoder` card's checkpoint)
                                                laser2.spm  (its SentencePiece model)

this reproduces the reference's own check (tests/integration_tests/test_laser2_text.py): the 4 x 4 cosine-similarity matrix
of four sentences, tokenized, right-padded with id 1 and encoded by the model, stored in tests/golden/laser2_cosine_golden.json.
The reference asserts 1e-4 on an fp32 CPU model; the bf16 engine is held to 2e-3 absolute on the cosines, the allowance of
the SONAR text golden."""

import json
import os
from pathlib import Path

import pytest
import torch

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.environ.get("SONAR_B200_CHECKPOINT_DIR"), reason="real LASER2 checkpoint not available")]

GOLDEN = Path(__file__).resolve().parent / "golden" / "laser2_cosine_golden.json"


def test_laser2_cosine_golden(native_lib, cuda_device):
    from sonar_b200 import B200LaserLstmEncoder
    from sonar_b200.batching import collate
    from sonar_b200.tokenizer import Laser2Tokenizer

    d = Path(os.environ["SONAR_B200_CHECKPOINT_DIR"])
    ckpt, spm = d / "laser2.pt", d / "laser2.spm"
    if not ckpt.exists() or not spm.exists():
        pytest.skip(f"{ckpt} or {spm} not found")
    golden = json.loads(GOLDEN.read_text())
    tok = Laser2Tokenizer(str(spm))
    enc = tok.create_encoder()
    ids, lens, _ = collate([enc(s) for s in golden["sentences"]], tok.vocab_info.pad_idx)
    model = B200LaserLstmEncoder.from_checkpoint(ckpt, device=cuda_device)
    emb = torch.nn.functional.normalize(model(ids.to(cuda_device), torch.tensor(lens)), dim=-1)
    model.check_inputs()
    sim = (emb @ emb.T).cpu()
    torch.testing.assert_close(sim, torch.tensor(golden["cosine"]), rtol=0, atol=2e-3)
