"""GPU parity of the speech path against the CPU oracle (BASELINE.json config 3)."""

import os

import pytest
import torch

from oracle.speech_frontend import collate_fbank, waveform_to_fbank

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "fbank_golden.pt")


def test_fbank_kernel_matches_oracle_and_golden(native_lib, cuda_device):
    from sonar_b200.speech_frontend import WaveformToFbank

    conv = WaveformToFbank(cuda_device)
    g = torch.load(GOLDEN, weights_only=True)
    gen = torch.Generator().manual_seed(3)
    waves = list(g["waveforms"]) + [(torch.randn(160000, generator=gen) * 0.05).clamp(-1, 1),   # config-3 shape: 10 s
                                    (torch.randn(16000 * 3 + 77, generator=gen) * 0.3).clamp(-1, 1),
                                    (torch.sin(torch.arange(400 + 160 * 5) * 0.05) * 0.5 + 0.02 * torch.randn(400 + 160 * 5, generator=gen))]  # tone + noise floor
    out, frames = conv([w.to(cuda_device) for w in waves])
    torch.cuda.synchronize()
    ref, ref_lens = collate_fbank([waveform_to_fbank(w) for w in waves])
    assert frames == ref_lens and out.shape == ref.shape
    # standardised log-mel, fp32 FFT/mel round-off on both sides (the oracle itself sits 1e-4 from torchaudio)
    torch.testing.assert_close(out.cpu(), ref, rtol=0, atol=2e-3)
    for i, std in enumerate(g["fbank_standardized"]):  # and against the torchaudio golden directly
        torch.testing.assert_close(out[i, : std.shape[0]].cpu(), std, rtol=0, atol=2e-3)
    assert frames[2] == 998


def test_fbank_rejects_bad_input(native_lib, cuda_device):
    from sonar_b200.speech_frontend import WaveformToFbank

    conv = WaveformToFbank(cuda_device)
    with pytest.raises(ValueError):
        conv([torch.zeros(100, device=cuda_device)])
    with pytest.raises(ValueError):
        conv([torch.zeros((2, 1000), device=cuda_device)])
    with pytest.raises(RuntimeError):
        WaveformToFbank("cpu")


# ---------------------------------------------------------------- Conformer encoder + pooler vs the oracle
def _speech_models(pooler_layers, device):
    from oracle.speech_encoder import OracleSpeechConfig, OracleSpeechEncoder, make_synthetic_speech_state_dict
    from sonar_b200 import B200SpeechEncoderModel, sonar_speech_encoder_config

    ocfg = OracleSpeechConfig(num_layers=2, pooler_layers=pooler_layers)
    sd = make_synthetic_speech_state_dict(ocfg, seed=3)
    cfg = sonar_speech_encoder_config("english", num_encoder_layers=2, num_decoder_layers=pooler_layers)
    return OracleSpeechEncoder(ocfg, sd), B200SpeechEncoderModel(cfg, sd, device)  # default attention kernel (mma.sync)


@pytest.fixture(scope="module")
def speech_small(native_lib, cuda_device):
    return _speech_models(2, cuda_device)


def _speech_check(m, what):
    print(what, m)
    assert m["one_minus_cos_max"] <= 1e-3 and m["rel_l2_max"] <= 2e-2, (what, m)


def test_speech_encoder_vs_oracle(speech_small, cuda_device):
    from sonar_b200 import PaddingMask, SequenceBatch
    from tests.helpers import parity_metrics

    g = torch.Generator().manual_seed(5)
    frames = [300, 131, 64, 257, 2]
    tmax = 300
    fb = torch.zeros((len(frames), tmax, 80))
    for i, n in enumerate(frames):
        fb[i, :n] = torch.randn((n, 80), generator=g)
    for pooler_layers in (2, 6):  # the fixture's pooler, and the `non_english` pooler depth
        oracle, model = speech_small if pooler_layers == 2 else _speech_models(pooler_layers, cuda_device)
        ref, ref_enc, lens = oracle(fb, frames)
        model.return_encoded_seqs = True
        out = model(SequenceBatch(fb.to(cuda_device), PaddingMask(torch.tensor(frames), tmax, frames)))
        model.return_encoded_seqs = False
        torch.cuda.synchronize()
        # encoder states (after model.layer_norm) at the real positions, packed order
        start = 0
        for i, n in enumerate(lens):
            got, exp = out.encoded_seqs[start : start + n].cpu(), ref_enc[i, :n]
            rel = float((got - exp).norm() / exp.norm())
            assert rel <= 2e-2, (pooler_layers, i, rel)
            start += n
        _speech_check(parity_metrics(out.sentence_embeddings, ref), f"speech 2+{pooler_layers} layers ragged")


def test_speech_batch_invariance_and_long_utterance(speech_small, cuda_device):
    from sonar_b200 import PaddingMask, SequenceBatch
    from tests.helpers import parity_metrics

    oracle, model = speech_small
    g = torch.Generator().manual_seed(6)
    frames = [998, 400]  # config-3 shape: 10 s -> 998 frames -> 499 positions
    fb = torch.zeros((2, 998, 80))
    for i, n in enumerate(frames):
        fb[i, :n] = torch.randn((n, 80), generator=g)
    both = model(SequenceBatch(fb.to(cuda_device), PaddingMask(torch.tensor(frames), 998, frames))).sentence_embeddings
    alone = model(SequenceBatch(fb[1:, :400].contiguous().to(cuda_device), None)).sentence_embeddings
    assert torch.equal(both[1], alone[0])  # an utterance gets the same bits whatever batch (and batch maximum) it is in
    ref, _, _ = oracle(fb, frames)
    _speech_check(parity_metrics(both, ref), "speech 998-frame utterance")


def test_speech_pipeline_end_to_end(speech_small, cuda_device, tmp_path):
    import wave

    from oracle.speech_frontend import collate_fbank, waveform_to_fbank
    from sonar_b200.inference_pipelines import SpeechToEmbeddingModelPipeline
    from tests.helpers import parity_metrics

    oracle, model = speech_small
    pipe = SpeechToEmbeddingModelPipeline(model, device=cuda_device)
    g = torch.Generator().manual_seed(8)
    waves = [(torch.randn(16000 + 123 * i, generator=g) * 0.1).clamp(-1, 1) for i in range(4)]
    emb = pipe.predict([w[None, :] for w in waves], batch_size=3)
    assert emb.shape == (4, 1024)
    feats = [waveform_to_fbank(w) for w in waves]
    refs = []
    for grp in (feats[:3], feats[3:]):  # same bucketing as batch_size=3
        fb, fl = collate_fbank(grp)
        refs.append(oracle(fb, fl)[0])
    _speech_check(parity_metrics(emb, torch.cat(refs)), "speech pipeline")
    # a PCM-16 wav file gives the same embedding as its tensor (test_sonar_speech_pipeline_models.py:28-40 analogue)
    pcm = (waves[0] * 32767).round().clamp(-32768, 32767).to(torch.int16)
    path = tmp_path / "a.wav"
    with wave.open(str(path), "wb") as f:
        f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes(pcm.numpy().tobytes())
    e_file = pipe.predict([str(path)])
    e_tensor = pipe.predict([(pcm.float() / 32768.0)[None, :]])
    torch.testing.assert_close(e_file, e_tensor, rtol=1e-5, atol=1e-5)


def test_speech_to_text_pipeline_composes_encoder_and_decoder(speech_small, cuda_device):
    """``SpeechToTextModelPipeline`` (speech.py:311-400) = speech encoder -> one-position encoder output -> beam
    search: its texts equal EmbeddingToText over SpeechToEmbedding's vectors with the same bucketing."""
    from oracle.text_decoder import OracleDecoderConfig, make_synthetic_decoder_state_dict
    from sonar_b200 import B200TextDecoderModel, VocabularyInfo, sonar_text_decoder_config
    from sonar_b200.inference_pipelines import (EmbeddingToTextModelPipeline, SpeechToEmbeddingModelPipeline,
                                                SpeechToTextModelPipeline)
    from sonar_b200.tokenizer import SyntheticTokenizer

    _, enc = speech_small
    vocab = 4096
    ocfg = OracleDecoderConfig(vocab_size=vocab, num_layers=2, max_seq_len=64)
    sd = make_synthetic_decoder_state_dict(ocfg, seed=4)
    cfg = sonar_text_decoder_config("basic", num_decoder_layers=2, max_seq_len=64,
                                    vocab_info=VocabularyInfo(size=vocab, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    dec = B200TextDecoderModel(cfg, sd, cuda_device)
    tok = SyntheticTokenizer(vocab_size=vocab)
    g = torch.Generator().manual_seed(11)
    waves = [(torch.randn(12000 + 777 * i, generator=g) * 0.1).clamp(-1, 1)[None, :] for i in range(4)]
    s2t = SpeechToTextModelPipeline(enc, dec, tok, device=cuda_device)
    texts = s2t.predict(waves, target_lang="fra_Latn", batch_size=2, max_seq_len=10)
    assert len(texts) == 4 and all(isinstance(t, str) for t in texts)
    emb = SpeechToEmbeddingModelPipeline(enc, device=cuda_device).predict(waves, batch_size=2)
    want = EmbeddingToTextModelPipeline(dec, tok, device=cuda_device).predict(emb, target_lang="fra_Latn", batch_size=2,
                                                                              max_seq_len=10)
    assert texts == want


def test_tsv_pipelines_match_the_model_pipelines(speech_small, cuda_device, tmp_path):
    """`SpeechToEmbeddingPipeline` / `SpeechToTextPipeline` (reference speech.py:150-274): a TSV manifest naming WAV files
    under a root directory gives, bucket by bucket, what the tensor-driven pipelines give for the same waveforms."""
    import wave

    from oracle.text_decoder import OracleDecoderConfig, make_synthetic_decoder_state_dict
    from sonar_b200 import B200TextDecoderModel, VocabularyInfo, sonar_text_decoder_config
    from sonar_b200.inference_pipelines import (SpeechInferenceParams, SpeechToEmbeddingModelPipeline,
                                                SpeechToEmbeddingPipeline, SpeechToTextModelPipeline, SpeechToTextPipeline)
    from sonar_b200.tokenizer import SyntheticTokenizer

    _, enc = speech_small
    g = torch.Generator().manual_seed(13)
    (tmp_path / "clips").mkdir()
    lines, waves = ["id\taudio\tnote"], []
    for i in range(5):
        pcm = ((torch.randn(9000 + 640 * i, generator=g) * 0.1).clamp(-1, 1) * 32767).round().to(torch.int16)
        with wave.open(str(tmp_path / "clips" / f"u{i}.wav"), "wb") as f:
            f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes(pcm.numpy().tobytes())
        lines.append(f"{i}\tclips/u{i}.wav\tx")
        waves.append((pcm.float() / 32768.0)[None, :])
    manifest = tmp_path / "test.tsv"
    manifest.write_text("\n".join(lines) + "\n")
    ctx = SpeechInferenceParams(data_file=manifest, audio_root_dir=tmp_path, audio_path_index=1, batch_size=2,
                                device=cuda_device, target_lang="fra_Latn")
    outs = list(SpeechToEmbeddingPipeline(enc).build_pipeline(ctx))
    assert [o.sentence_embeddings.shape[0] for o in outs] == [2, 2, 1]
    want = SpeechToEmbeddingModelPipeline(enc, device=cuda_device).predict(waves, batch_size=2)
    assert torch.equal(torch.cat([o.sentence_embeddings for o in outs]), want)

    vocab = 4096
    sd = make_synthetic_decoder_state_dict(OracleDecoderConfig(vocab_size=vocab, num_layers=2, max_seq_len=64), seed=4)
    cfg = sonar_text_decoder_config("basic", num_decoder_layers=2, max_seq_len=64,
                                    vocab_info=VocabularyInfo(size=vocab, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    dec = B200TextDecoderModel(cfg, sd, cuda_device)
    tok = SyntheticTokenizer(vocab_size=vocab)
    texts = [t for bucket_texts in SpeechToTextPipeline(enc, dec, tok).build_pipeline(ctx, max_seq_len=10) for t in bucket_texts]
    assert texts == SpeechToTextModelPipeline(enc, dec, tok, device=cuda_device).predict(waves, target_lang="fra_Latn",
                                                                                       batch_size=2, max_seq_len=10)


def test_relpos_attention_tcgen05_agrees_with_mma_sync_and_is_batch_invariant(native_lib, cuda_device):
    """The relative-position attention has two implementations: the wgmma kernel (attention_relpos_tc.cu: S and the band
    product on the tensor cores (wgmma), the Transformer-XL shift through a skewed shared-memory buffer, P in registers) and the
    mma.sync kernel.  Same model, both kernels, utterances whose position counts sit on and around the 128-row tile
    edges; both must agree with each other and with the oracle, and the wgmma path must give an utterance the same bits
    whatever batch it is in (the band window it reads depends on the utterance, not on the batch maximum)."""
    from oracle.speech_encoder import OracleSpeechConfig, OracleSpeechEncoder, make_synthetic_speech_state_dict
    from sonar_b200 import B200SpeechEncoderModel, PaddingMask, SequenceBatch, sonar_speech_encoder_config
    from tests.helpers import parity_metrics

    ocfg = OracleSpeechConfig(num_layers=2, pooler_layers=2)
    sd = make_synthetic_speech_state_dict(ocfg, seed=11)
    cfg = sonar_speech_encoder_config("english", num_encoder_layers=2, num_decoder_layers=2)
    tc = B200SpeechEncoderModel(cfg, sd, cuda_device, attn_impl="tcgen05")
    ms = B200SpeechEncoderModel(cfg, sd, cuda_device, attn_impl="mma_sync")
    g = torch.Generator().manual_seed(12)
    frames = [998, 258, 256, 2, 514, 770, 254, 600]  # positions 499, 129, 128, 1, 257, 385, 127, 300
    tmax = 998
    fb = torch.zeros((len(frames), tmax, 80))
    for i, n in enumerate(frames):
        fb[i, :n] = torch.randn((n, 80), generator=g)
    batch = SequenceBatch(fb.to(cuda_device), PaddingMask(torch.tensor(frames), tmax, frames))
    a = tc(batch).sentence_embeddings
    b = ms(batch).sentence_embeddings
    m = parity_metrics(a, b.cpu())
    print("wgmma vs mma.sync rel-pos attention:", m)
    assert m["one_minus_cos_max"] <= 1e-5 and m["rel_l2_max"] <= 5e-3, m
    ref, _, _ = OracleSpeechEncoder(ocfg, sd)(fb, frames)
    _speech_check(parity_metrics(a, ref), "speech wgmma attention vs oracle")
    assert torch.equal(tc(batch).sentence_embeddings, a)  # deterministic
    for i in (1, 4, 7):  # alone in a batch of one: a different batch maximum, the same bits
        n = frames[i]
        alone = tc(SequenceBatch(fb[i : i + 1, :n].contiguous().to(cuda_device), None)).sentence_embeddings
        assert torch.equal(alone[0], a[i]), i
