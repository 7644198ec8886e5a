"""Env-gated harness for the reference's REAL-WEIGHT goldens (VERDICT r1 item 6.v).  Nothing here runs offline -- the
checkpoints and the SentencePiece model cannot be downloaded in this environment -- but the moment

    SONAR_B200_CHECKPOINT_DIR=<dir>   holding   text_sonar_basic_encoder.pt, text_sonar_basic_decoder.pt
                                                (fairseq2 state dicts under the key "model"),
                                                sentencepiece.source.256000.model  (the NLLB SPM model of the SONAR card)
                                                and nllb_langs.txt (one FLORES-200 code per line, NLLB dictionary order)

is set, these tests run the reference's own assertions (/root/reference/tests/integration_tests/test_text_sonar.py) against the
CUDA engine: the cosine-similarity golden of test_text_encoder_sonar_basic (:46-53) and the exact translations of
test_encoder_decoder_translate / test_vec2text_decode (:107-118).  Tolerance for the cosine matrix: the reference asserts
1e-4 on an fp32 CPU model; the bf16 engine is held to 2e-3 absolute on the cosines (BASELINE.json north_star: embeddings within
1e-3 cosine of the fp32 path)."""

import os
from pathlib import Path

import pytest
import torch

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.environ.get("SONAR_B200_CHECKPOINT_DIR"), reason="real SONAR checkpoints not available")]

# the reference test's own sentence pairs (test_text_sonar.py:20-21)
ENG = ["Hello, my name is Paul", "I'm working as a teacher"]
FRA = ["Bonjour, mon nom est Paul", "Je travaille comme professeur."]


def _dir() -> Path:
    return Path(os.environ["SONAR_B200_CHECKPOINT_DIR"])


def _sentences():
    return ENG, FRA


@pytest.fixture(scope="module")
def tokenizer():
    from sonar_b200.tokenizer import NllbTokenizer

    d = _dir()
    spm, langs = d / "sentencepiece.source.256000.model", d / "nllb_langs.txt"
    if not spm.exists() or not langs.exists():
        pytest.skip("tokenizer files missing")
    return NllbTokenizer(str(spm), [l.strip() for l in langs.read_text().splitlines() if l.strip()])


@pytest.fixture(scope="module")
def text2vec(native_lib, cuda_device, tokenizer):
    from sonar_b200 import B200TextEncoderModel
    from sonar_b200.inference_pipelines import TextToEmbeddingModelPipeline

    ckpt = _dir() / "text_sonar_basic_encoder.pt"
    if not ckpt.exists():
        pytest.skip(f"{ckpt} not found")
    return TextToEmbeddingModelPipeline(B200TextEncoderModel.from_checkpoint(ckpt, device=cuda_device), tokenizer,
                                        device=cuda_device)


def test_text_encoder_cosine_golden(text2vec):
    eng, fr = _sentences()
    e = torch.nn.functional.normalize(text2vec.predict(eng, source_lang="eng_Latn"), dim=-1)
    f = torch.nn.functional.normalize(text2vec.predict(fr, source_lang="fra_Latn"), dim=-1)
    sim = (e @ f.T).cpu()
    torch.testing.assert_close(sim, torch.tensor([[0.9367, 0.3658], [0.3787, 0.8596]]), rtol=0, atol=2e-3)


def test_vec2text_reproduces_the_reference_translations(text2vec, tokenizer, cuda_device):
    from sonar_b200 import B200TextDecoderModel
    from sonar_b200.inference_pipelines import EmbeddingToTextModelPipeline

    ckpt = _dir() / "text_sonar_basic_decoder.pt"
    if not ckpt.exists():
        pytest.skip(f"{ckpt} not found")
    eng, fr = _sentences()
    vec2text = EmbeddingToTextModelPipeline(B200TextDecoderModel.from_checkpoint(ckpt, device=cuda_device), tokenizer,
                                            device=cuda_device)
    emb = text2vec.predict(eng, source_lang="eng_Latn")
    assert vec2text.predict(emb, target_lang="fra_Latn", max_seq_len=512) == fr
