"""End-to-end parity of the CUDA text encoder (through sb_encoder_forward) against the fp32
CPU oracle on shared seeded synthetic weights and ids (SURVEY §8(d) configs 1/2 at sizes the
oracle finishes in seconds), plus the reference's behavioural properties of the pipeline
(order preservation, batch-composition invariance, truncation warning:
/root/reference/tests/integration_tests/test_text_sonar.py:56-59,120-161).

Tolerances (BASELINE.json north_star + SURVEY §8(d)): per sentence 1 - cos <= 1e-3; and because
that alone is a weak discriminator on random weights: mean-centred cosine >= 0.999 and relative
L2 <= 1e-2."""

import warnings

import pytest
import torch

from oracle.text_encoder import OracleEncoderConfig, OracleTextEncoder, make_synthetic_state_dict
from tests.helpers import parity_metrics

pytestmark = pytest.mark.gpu

VOCAB = 4096


def _build(num_layers, device, seed=1, weight_std=0.02):
    from sonar_b200 import B200TextEncoderModel, VocabularyInfo, sonar_text_encoder_config

    ocfg = OracleEncoderConfig(vocab_size=VOCAB, num_layers=num_layers)
    sd = make_synthetic_state_dict(ocfg, seed=seed, weight_std=weight_std)
    cfg = sonar_text_encoder_config(
        "basic", num_encoder_layers=num_layers,
        vocab_info=VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    return OracleTextEncoder(ocfg, sd), B200TextEncoderModel(cfg, sd, device)


def _batch(lens, s, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros((len(lens), s), dtype=torch.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(4, VOCAB, (n,), generator=g)
    return ids


def _check(m, what):
    print(what, m)
    assert m["one_minus_cos_max"] <= 1e-3, (what, m)
    assert m["centred_cos_min"] >= 0.999, (what, m)
    assert m["rel_l2_max"] <= 1e-2, (what, m)


@pytest.fixture(scope="module")
def two_layer(native_lib, cuda_device):
    return _build(2, cuda_device)


def test_two_layers_ragged_vs_oracle(two_layer, cuda_device):
    from sonar_b200 import PaddingMask, SequenceBatch

    oracle, model = two_layer
    lens = [64, 1, 2, 17, 33, 64, 48, 5, 63, 31, 16, 8]
    ids = _batch(lens, 64)
    ref, ref_states = oracle(ids, torch.tensor(lens))
    model.return_encoded_seqs = True
    out = model(SequenceBatch(ids.to(cuda_device), PaddingMask(torch.tensor(lens), 64, lens)))
    model.return_encoded_seqs = False
    torch.cuda.synchronize()
    _check(parity_metrics(out.sentence_embeddings, ref), "2-layer ragged")
    for i, n in enumerate(lens):  # encoded_seqs parity at real positions
        got, exp = out.encoded_seqs[i, :n].cpu(), ref_states[i, :n]
        assert float((got - exp).norm() / exp.norm()) <= 1e-2


def test_two_layers_dense_no_mask(two_layer, cuda_device):
    from sonar_b200 import SequenceBatch

    oracle, model = two_layer
    ids = _batch([128] * 6, 128, seed=3)
    ref, _ = oracle(ids, None)
    out = model(SequenceBatch(ids.to(cuda_device), None)).sentence_embeddings
    _check(parity_metrics(out, ref), "2-layer dense S=128")


def test_long_sequences_up_to_model_max(two_layer, cuda_device):
    from sonar_b200 import PaddingMask, SequenceBatch

    oracle, model = two_layer
    lens = [514, 300, 129, 257]
    ids = _batch(lens, 514, seed=4)
    ref, _ = oracle(ids, torch.tensor(lens))
    out = model(SequenceBatch(ids.to(cuda_device), PaddingMask(torch.tensor(lens), 514, lens))).sentence_embeddings
    _check(parity_metrics(out, ref), "2-layer long")
    with pytest.raises(ValueError):  # longer than the position table
        model(SequenceBatch(torch.zeros((1, 515), dtype=torch.int64, device=cuda_device), None))


def test_full_depth_24_layers_vs_oracle(native_lib, cuda_device):
    """BASELINE.json config 1 shape: 32 sentences, lengths U{8..64} (seed 0), full 24 layers."""
    from sonar_b200 import PaddingMask, SequenceBatch

    oracle, model = _build(24, cuda_device)
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(8, 65, (32,), generator=g).tolist()
    ids = _batch(lens, 64, seed=5)
    ref, _ = oracle(ids, torch.tensor(lens))
    out = model(SequenceBatch(ids.to(cuda_device), PaddingMask(torch.tensor(lens), 64, lens))).sentence_embeddings
    _check(parity_metrics(out, ref), "24-layer config-1")


def test_batch_composition_invariance_bitwise(two_layer, cuda_device):
    """Each sentence's embedding must not depend on its batch neighbours (the reference test allows
    fp32 default tolerances; the packed engine is bitwise invariant)."""
    from sonar_b200 import PaddingMask, SequenceBatch

    _, model = two_layer
    lens = [40, 7, 64, 23, 64]
    ids = _batch(lens, 64, seed=6).to(cuda_device)
    full = model(SequenceBatch(ids, PaddingMask(torch.tensor(lens), 64, lens))).sentence_embeddings
    for i, n in enumerate(lens):
        one = model(SequenceBatch(ids[i : i + 1, :n].contiguous(), None)).sentence_embeddings
        assert torch.equal(one[0], full[i]), i
    pair = model(SequenceBatch(ids[1:3], PaddingMask(torch.tensor(lens[1:3]), 64, lens[1:3]))).sentence_embeddings
    assert torch.equal(pair, full[1:3])


def test_out_of_range_token_is_reported(two_layer, cuda_device):
    from sonar_b200 import SequenceBatch

    _, model = two_layer
    ids = torch.full((2, 8), VOCAB, dtype=torch.int64, device=cuda_device)
    model(SequenceBatch(ids, None))
    with pytest.raises(ValueError):
        model.check_inputs()
    model(SequenceBatch(torch.full((2, 8), 5, dtype=torch.int64, device=cuda_device), None))
    model.check_inputs()


# ---------------------------------------------------------------- pipeline behaviour
@pytest.fixture(scope="module")
def pipeline(two_layer, cuda_device):
    from sonar_b200.inference_pipelines import TextToEmbeddingModelPipeline
    from sonar_b200.tokenizer import SyntheticTokenizer

    _, model = two_layer
    return TextToEmbeddingModelPipeline(model, SyntheticTokenizer(vocab_size=VOCAB), device=cuda_device)


SENTS = ["the quick brown fox", "a", "jumps over the lazy dog again and again", "hello world",
         "one two three four five six seven eight nine ten", "b c", "sonar embeds sentences"]


def test_pipeline_matches_oracle_and_preserves_order(pipeline, two_layer):
    oracle, _ = two_layer
    emb = pipeline.predict(SENTS, source_lang="eng_Latn", batch_size=3)
    assert emb.shape == (len(SENTS), 1024) and emb.dtype == torch.float32
    enc = pipeline.tokenizer.create_encoder(lang="eng_Latn")
    for i, s in enumerate(SENTS):
        ids = enc(s)[None]
        ref, _ = oracle(ids, None)
        m = parity_metrics(emb[i : i + 1], ref)
        assert m["one_minus_cos_max"] <= 1e-3 and m["rel_l2_max"] <= 1e-2, (i, m)


def test_pipeline_batch_args_invariance(pipeline):
    """test_text_sonar.py:120-161: batch_size 2 vs 1 vs batch_max_tokens 5 / 30 vs one-by-one."""
    a = pipeline.predict(SENTS, "eng_Latn", batch_size=2)
    for kw in (dict(batch_size=1), dict(batch_size=None, batch_max_tokens=5),
               dict(batch_size=None, batch_max_tokens=30), dict(batch_size=20, batch_max_tokens=30)):
        b = pipeline.predict(SENTS, "eng_Latn", **kw)
        torch.testing.assert_close(a, b, rtol=1.3e-6, atol=1e-5)
    one = torch.cat([pipeline.predict([s], "eng_Latn") for s in SENTS])
    torch.testing.assert_close(a, one, rtol=1.3e-6, atol=1e-5)


def test_pipeline_truncation_warns(pipeline):
    """test_text_sonar.py:56-59."""
    long_text = " ".join(["word%d" % i for i in range(600)])
    with pytest.warns(UserWarning, match="truncated to 514"):
        emb = pipeline.predict([long_text, "short"], "eng_Latn")
    assert emb.shape == (2, 1024) and bool(torch.isfinite(emb).all())
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        pipeline.predict(["short one"], "eng_Latn", max_seq_len=16)


def test_pipeline_file_input_and_target_device(pipeline, tmp_path):
    p = tmp_path / "in.txt"
    p.write_text("\n".join(SENTS) + "\n")
    a = pipeline.predict(p, "eng_Latn", batch_size=4, target_device="cpu")
    b = pipeline.predict(SENTS, "eng_Latn", batch_size=4)
    assert a.device.type == "cpu"
    torch.testing.assert_close(a, b.cpu(), rtol=1.3e-6, atol=1e-5)


@pytest.mark.parametrize("lens_kind", ["dense", "ragged_tail"])
def test_layernorm_folded_into_the_gemms_matches_the_separate_kernels(native_lib, cuda_device, lens_kind):
    """The default schedule folds every encoder-layer LayerNorm into the GEMMs around it (`ln_fold`): the residual GEMMs'
    epilogues emit per-row statistics + the bf16 copy of the stream, the QKV / FFN1 GEMMs apply (mean, rstd) to weights
    pre-multiplied by gamma.  It must agree with the classic schedule (separate LayerNorm kernels) to bf16-rounding level
    and with the fp32 oracle to the engine's tolerances; sizes: many more tiles than CTAs, a row count that is not a multiple
    of the 256-row tile, LayerNorm gains / biases far from (1, 0) so a wrong fold cannot hide, repeated runs bitwise equal."""
    from sonar_b200 import B200TextEncoderModel, PaddingMask, SequenceBatch, VocabularyInfo, sonar_text_encoder_config

    ocfg = OracleEncoderConfig(vocab_size=VOCAB, num_layers=3)
    sd = make_synthetic_state_dict(ocfg, seed=5)
    g = torch.Generator().manual_seed(9)
    for k in list(sd):  # exaggerate gamma / beta: the fold moves them into W', c and b'
        if "layer_norm.weight" in k:
            sd[k] = 1.0 + 0.5 * torch.randn(sd[k].shape, generator=g)
        elif "layer_norm.bias" in k:
            sd[k] = 0.5 * torch.randn(sd[k].shape, generator=g)
    cfg = sonar_text_encoder_config("basic", num_encoder_layers=3,
                                    vocab_info=VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    folded = B200TextEncoderModel(cfg, sd, cuda_device, ln_fold=1)       # both LayerNorms of a layer folded
    folded1 = B200TextEncoderModel(cfg, sd, cuda_device, ln_fold=2)      # only the attention-block LayerNorm
    classic = B200TextEncoderModel(cfg, sd, cuda_device, ln_fold=0)
    if lens_kind == "dense":
        lens = [128] * 320  # 40 960 rows = 160 pair tiles x 4 n-tiles
    else:
        lens = [int(v) for v in torch.randint(1, 129, (333,), generator=g)]
        lens[-1] = 77
    ids = _batch(lens, 128, seed=4)
    mask = PaddingMask(torch.tensor(lens), 128, lens)
    got = folded(SequenceBatch(ids.to(cuda_device), mask)).sentence_embeddings.clone()
    want = classic(SequenceBatch(ids.to(cuda_device), mask)).sentence_embeddings
    m = parity_metrics(got, want.cpu())
    print("folded vs separate LayerNorm:", m)
    assert m["one_minus_cos_max"] <= 1e-5 and m["rel_l2_max"] <= 5e-3, m
    for _ in range(2):  # deterministic
        assert torch.equal(folded(SequenceBatch(ids.to(cuda_device), mask)).sentence_embeddings, got)
    m1 = parity_metrics(folded1(SequenceBatch(ids.to(cuda_device), mask)).sentence_embeddings, want.cpu())
    assert m1["one_minus_cos_max"] <= 1e-5 and m1["rel_l2_max"] <= 5e-3, m1
    rows = list(range(0, len(lens), 23))
    ref, _ = OracleTextEncoder(ocfg, sd)(ids[rows], torch.tensor([lens[i] for i in rows]))
    _check(parity_metrics(got[rows], ref), "3-layer folded LayerNorm vs oracle")
