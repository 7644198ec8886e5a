"""The engines' host side: every C-ABI entry point that carves the caller's workspace rejects one that is too small
(SB_ERR_INVALID, a message that names the entry point) instead of writing past its end, the Python wrappers keep the
weights the engines point into out of reach of ``nn.Module`` conversions, and the pinned ring through which the text
encoder, the speech encoder and LASER2 stage their host lengths is not rewritten while a copy still reads it.  Engines are
the small configurations of the other GPU tests."""

import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

VOCAB = 4096


@pytest.fixture(scope="module")
def engines(native_lib, cuda_device):
    from oracle.speech_encoder import OracleSpeechConfig, make_synthetic_speech_state_dict
    from oracle.text_decoder import OracleDecoderConfig, make_synthetic_decoder_state_dict
    from oracle.text_encoder import OracleEncoderConfig, make_synthetic_state_dict
    from sonar_b200 import (B200SpeechEncoderModel, B200TextDecoderModel, B200TextEncoderModel, VocabularyInfo,
                            sonar_speech_encoder_config, sonar_text_decoder_config, sonar_text_encoder_config)

    vocab = VocabularyInfo(size=VOCAB, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1)
    enc_sd = make_synthetic_state_dict(OracleEncoderConfig(vocab_size=VOCAB, num_layers=2), seed=1)
    encoder = B200TextEncoderModel(sonar_text_encoder_config("basic", num_encoder_layers=2, vocab_info=vocab), enc_sd,
                                   cuda_device)
    dec_sd = make_synthetic_decoder_state_dict(OracleDecoderConfig(vocab_size=VOCAB, num_layers=2, max_seq_len=64), seed=2)
    decoder = B200TextDecoderModel(sonar_text_decoder_config("basic", num_decoder_layers=2, max_seq_len=64,
                                                             vocab_info=vocab), dec_sd, cuda_device)
    sp_sd = make_synthetic_speech_state_dict(OracleSpeechConfig(num_layers=2, pooler_layers=2), seed=3)
    speech = B200SpeechEncoderModel(sonar_speech_encoder_config("english", num_encoder_layers=2, num_decoder_layers=2),
                                    sp_sd, cuda_device)
    return encoder, decoder, speech


def test_too_small_workspace_is_rejected_with_host_lengths(engines, cuda_device):
    """Every entry point that carves a workspace refuses a 1-byte one; the speech forward takes its lengths on the host
    only, and the decoder's begin and step are refused although its layout no longer starts with an input flag."""
    from sonar_b200 import _lib

    encoder, decoder, speech = engines
    lib = encoder._lib
    dev = cuda_device
    bufs = []

    def t(*shape, dtype=torch.float32):
        bufs.append(torch.zeros(shape, dtype=dtype, device=dev))
        return bufs[-1].data_ptr()

    w, stream = t(1, dtype=torch.uint8), torch.cuda.current_stream(dev).cuda_stream
    B, S, D = 4, 16, 1024                 # text / speech batch
    n, beam, max_len = 3, 2, 16           # decoder: sentences x beam hypotheses
    R = n * beam
    lens = (C.c_int32 * B)(*[8] * B)      # 8 speech positions per utterance (16 fbank frames)
    rows = 256                            # relative-position table rows for 8 positions: roundup(2 * 8 - 1, 256)
    x, y = t(256, 64), t(512, 64)         # xsim: 256 x 512 rows of dimension 64
    calls = {
        "sb_encoder_forward": lambda: lib.sb_encoder_forward(
            encoder._handle, t(B, S, dtype=torch.int64), S, None, B, S, t(B, D), None, w, 1, stream),
        "sb_decoder_begin": lambda: lib.sb_decoder_begin(decoder._handle, t(n, D), n, beam, max_len, w, 1, stream),
        "sb_decoder_step": lambda: lib.sb_decoder_step(
            decoder._handle, t(R, dtype=torch.int64), t(R, max_len, dtype=torch.int32), 0, n, beam, max_len, t(R, 16),
            t(R, 16, dtype=torch.int32), t(R), None, None, w, 1, stream),
        "sb_speech_encoder_forward": lambda: lib.sb_speech_encoder_forward(
            speech._handle, t(B, 2 * 8, 80), 2 * 8, lens, B, t(rows, D, dtype=torch.bfloat16), rows, t(B, D), None, w, 1,
            stream),
        "sb_xsim_knn": lambda: lib.sb_xsim_knn(
            x, y, 256, 512, 64, 4, t(256, 4, dtype=torch.float64), t(256, 4, dtype=torch.int32), w, 1, stream),
        "sb_xsim_knn_bidir": lambda: lib.sb_xsim_knn_bidir(
            x, y, 256, 512, 64, 4, t(256, 4, dtype=torch.float64), t(256, 4, dtype=torch.int32),
            t(512, 4, dtype=torch.float64), t(512, 4, dtype=torch.int32), t(1, dtype=torch.int32), w, 1, stream),
    }
    for name, call in calls.items():
        with torch.cuda.device(dev):
            rc = call()
        msg = _lib.last_error()
        assert rc == _lib.SB_ERR_INVALID, (name, rc, msg)
        assert msg.startswith(f"{name}: workspace too small"), (name, msg)
    torch.cuda.synchronize(dev)


def test_module_conversions_leave_the_engines_alone(engines, cuda_device):
    """No engine weight is a buffer or a parameter, so ``.half()``, ``.to(dtype)`` and ``.to(device)`` have nothing to
    replace (or free while the engine still reads it): the outputs afterwards are bitwise those from before.  The inputs
    start on the CPU, so each wrapper also moves them to its device."""
    from sonar_b200 import PaddingMask, SequenceBatch

    encoder, decoder, speech = engines
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(4, VOCAB, (3, 16), generator=g)
    fb = torch.randn((2, 40, 80), generator=g)
    emb = torch.randn((3, 1024), generator=g) * 0.25
    beam, max_len = 2, 8
    tokens = torch.full((3 * beam,), 2, dtype=torch.int64, device=cuda_device)
    table = torch.arange(3 * beam, dtype=torch.int32, device=cuda_device)[:, None].expand(3 * beam, max_len).contiguous()

    def decode():
        decoder.begin(emb, beam, max_len)
        return decoder.step(tokens, table, 0)

    runs = [
        (encoder, lambda: [encoder(SequenceBatch(ids, PaddingMask(torch.tensor([16, 9, 1]), 16, [16, 9, 1])))
                           .sentence_embeddings]),
        (decoder, decode),
        (speech, lambda: [speech(SequenceBatch(fb, PaddingMask(torch.tensor([40, 23]), 40, [40, 23])))
                          .sentence_embeddings]),
    ]
    for model, run in runs:
        name = type(model).__name__
        assert list(model.buffers()) == [] and list(model.parameters()) == [], name
        before = [t.clone() for t in run()]
        model.half()
        model.to(torch.bfloat16)
        model.to(cuda_device)
        after = run()
        torch.cuda.synchronize(cuda_device)
        assert all(torch.equal(a, b) for a, b in zip(before, after)), name


@pytest.fixture(scope="module")
def laser2(native_lib, cuda_device):
    from oracle.laser_lstm import OracleLaser2Config, make_synthetic_laser2_state_dict
    from sonar_b200 import B200LaserLstmEncoder, Laser2Config

    cfg = OracleLaser2Config(vocabulary_size=VOCAB, model_dim=128, num_layers=2, bidirectional=True)
    sd = make_synthetic_laser2_state_dict(cfg, seed=4, weight_bound=0.1)
    return B200LaserLstmEncoder(Laser2Config(vocabulary_size=VOCAB, pad_idx=cfg.pad_idx, model_dim=cfg.model_dim,
                                             num_layers=cfg.num_layers, bidirectional=cfg.bidirectional), sd, cuda_device)


@pytest.mark.parametrize("engine", ["text_encoder", "laser2", "speech"])
def test_a_burst_that_laps_the_staging_ring(engines, laser2, cuda_device, engine):
    """17 forwards, more than twice the ring's 8 slots, enqueued on one stream behind a sleeping kernel.  An event recorded
    right after the sleep is still pending once the first 8 are enqueued, so none of them synchronised with the stream.
    The ninth reuses the first one's slot, so it must wait until that forward's copy has run: the host laps the ring only
    as fast as the stream frees its slots.  Every output is bitwise that of the same batch run on its own.  For the token
    engines, one out-of-range id in a middle forward makes check_inputs raise once; that check clears it.  The speech
    batches are ragged but each has one utterance of the longest length, so the relative-position table is built once,
    during the warm-up."""
    from sonar_b200 import PaddingMask, SequenceBatch

    burst, slots, max_batch, S = 17, 8, 48, 40
    dev = cuda_device
    g = torch.Generator().manual_seed(17)
    if engine == "speech":
        model = engines[2]

        def make(lens):
            return torch.randn((len(lens), 2 * S, 80), generator=g)

        def run(fb, lens):
            frames = [2 * n for n in lens]
            return model(SequenceBatch(fb, PaddingMask(torch.tensor(frames), 2 * S, frames))).sentence_embeddings
    else:
        def make(lens):
            ids = torch.ones((len(lens), S), dtype=torch.int64)  # pad_idx 1
            for i, n in enumerate(lens):
                ids[i, :n] = torch.randint(4, VOCAB, (n,), generator=g)
            return ids

        if engine == "text_encoder":
            model = engines[0]

            def run(ids, lens):
                return model(SequenceBatch(ids, PaddingMask(torch.tensor(lens), S, lens))).sentence_embeddings
        else:
            model = laser2

            def run(ids, lens):
                return model(ids, torch.tensor(lens))

    batches = []
    for _ in range(burst):
        lens = torch.randint(1, S + 1, (int(torch.randint(1, max_batch + 1, (1,), generator=g)),), generator=g).tolist()
        if engine == "speech":
            lens[int(torch.randint(0, len(lens), (1,), generator=g))] = S
        batches.append((make(lens).to(dev), lens))  # on the device already: the wrappers make no blocking copy
    assert len({tuple(lens) for _, lens in batches}) == burst
    if engine != "speech":
        batches[burst // 2][0][0, 0] = VOCAB

    run(make([S] * max_batch).to(dev), [S] * max_batch)  # grows the workspace once
    torch.cuda.synchronize(dev)
    if engine != "speech":
        model.check_inputs()
    stream = torch.cuda.current_stream(dev)
    torch.cuda._sleep(50_000_000)  # tens of milliseconds: the stream is busy while the host enqueues the burst
    slept = torch.cuda.Event()
    slept.record(stream)
    outs = [run(x, lens) for x, lens in batches[:slots]]
    assert not slept.query(), f"{engine}: a forward of the burst waited for the stream"
    outs += [run(x, lens) for x, lens in batches[slots:]]
    torch.cuda.synchronize(dev)
    if engine != "speech":
        with pytest.raises(ValueError, match="vocab"):
            model.check_inputs()
        model.check_inputs()
    for i, (x, lens) in enumerate(batches):
        alone = run(x, lens)
        torch.cuda.synchronize(dev)
        assert torch.equal(outs[i], alone), f"{engine}: forward {i} of the burst"
    if engine != "speech":
        with pytest.raises(ValueError, match="vocab"):  # set again by the out-of-range batch on its own
            model.check_inputs()
