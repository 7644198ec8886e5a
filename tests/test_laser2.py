"""CPU tests of the LASER2 text encoder: the float64 oracle (oracle/laser_lstm.py) against torch.nn.LSTM on packed
sequences with the reference's masking and max pooling, the LASER2 tokenizer on a SentencePiece model trained here, the
config envelope, the ctypes struct layouts, and the library build."""

import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle.laser_lstm import OracleLaser2, OracleLaser2Config, make_synthetic_laser2_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _packed_lstm_reference(cfg: OracleLaser2Config, sd, seqs: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
    """torch.nn.Embedding + torch.nn.LSTM over pack_padded_sequence, pad_packed_sequence(padding_value), positions whose
    id is pad_idx set to -inf, max over time: the computation the reference model runs, in float64."""
    emb = torch.nn.Embedding(cfg.vocabulary_size, cfg.model_dim, padding_idx=cfg.pad_idx).double()
    lstm = torch.nn.LSTM(cfg.model_dim, cfg.hidden_size, num_layers=cfg.num_layers, bidirectional=cfg.bidirectional).double()
    emb.load_state_dict({"weight": sd["embed_tokens.weight"]})
    lstm.load_state_dict({k[len("lstm."):]: v for k, v in sd.items() if k.startswith("lstm.")})
    order = torch.argsort(-lens, stable=True)
    x = emb(seqs[order]).transpose(0, 1)  # [S, B, E]
    packed = torch.nn.utils.rnn.pack_padded_sequence(x, lens[order])
    with torch.no_grad():
        out, _ = lstm(packed)
    y, _ = torch.nn.utils.rnn.pad_packed_sequence(out, padding_value=cfg.padding_value)  # [max_len, B, dirs * H]
    y = y.masked_fill(seqs[order].eq(cfg.pad_idx).t().unsqueeze(-1), float("-inf"))
    return y.max(dim=0).values[torch.argsort(order)]


def _small_cfg(**kw) -> OracleLaser2Config:
    return OracleLaser2Config(**{**dict(vocabulary_size=60, pad_idx=1, model_dim=24, hidden_size=16, num_layers=5,
                                        bidirectional=True, padding_value=0.0), **kw})


def _ragged_batch(lens, pad_value, vocab, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((len(lens), max(lens)), pad_value, dtype=torch.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = torch.randint(3, vocab, (n,), generator=g)
    return ids, torch.tensor(lens)


@pytest.mark.parametrize("num_layers,bidirectional", [(1, False), (1, True), (5, False), (5, True)])
def test_oracle_matches_packed_torch_lstm(num_layers, bidirectional):
    cfg = _small_cfg(num_layers=num_layers, bidirectional=bidirectional)
    sd = make_synthetic_laser2_state_dict(cfg, seed=3, weight_bound=0.5)
    ids, lens = _ragged_batch([7, 3, 1, 9, 5, 9], cfg.pad_idx, cfg.vocabulary_size)
    ids[0, 2] = cfg.pad_idx  # a pad id inside a sentence: masked like padding
    got = OracleLaser2(cfg, sd)(ids, lens)
    want = _packed_lstm_reference(cfg, sd, ids, lens)
    assert got.shape == (6, cfg.hidden_size * (2 if bidirectional else 1)) and got.dtype == torch.float64
    torch.testing.assert_close(got, want, rtol=0, atol=1e-10)


def test_oracle_padding_value_joins_the_max_when_the_pad_id_differs():
    """Batches padded with an id other than pad_idx: pad_packed_sequence's padding_value takes part in the max."""
    for padding_value in (0.0, 0.75):
        cfg = _small_cfg(num_layers=2, padding_value=padding_value)
        sd = make_synthetic_laser2_state_dict(cfg, seed=4, weight_bound=0.5)
        ids, lens = _ragged_batch([6, 2, 4], 0, cfg.vocabulary_size, seed=1)  # padded with id 0 != pad_idx 1
        got = OracleLaser2(cfg, sd)(ids, lens)
        torch.testing.assert_close(got, _packed_lstm_reference(cfg, sd, ids, lens), rtol=0, atol=1e-10)
        assert bool((got[1] >= padding_value).all())  # the short rows saw padding_value
        # the same batch padded with pad_idx leaves padding out
        ids_p = ids.clone()
        ids_p[ids == 0] = cfg.pad_idx
        got_p = OracleLaser2(cfg, sd)(ids_p, lens)
        torch.testing.assert_close(got_p, _packed_lstm_reference(cfg, sd, ids_p, lens), rtol=0, atol=1e-10)


def test_oracle_dense_batch_and_length_one():
    cfg = _small_cfg(num_layers=3)
    sd = make_synthetic_laser2_state_dict(cfg, seed=5, weight_bound=0.5)
    ids, lens = _ragged_batch([8, 8, 8], cfg.pad_idx, cfg.vocabulary_size, seed=2)
    torch.testing.assert_close(OracleLaser2(cfg, sd)(ids, lens), _packed_lstm_reference(cfg, sd, ids, lens), rtol=0, atol=1e-10)
    ids, lens = _ragged_batch([1], cfg.pad_idx, cfg.vocabulary_size, seed=3)
    torch.testing.assert_close(OracleLaser2(cfg, sd)(ids, lens), _packed_lstm_reference(cfg, sd, ids, lens), rtol=0, atol=1e-10)


def test_oracle_refuses_a_zero_length():
    cfg = _small_cfg(num_layers=1)
    sd = make_synthetic_laser2_state_dict(cfg, seed=6)
    ids, _ = _ragged_batch([3, 2], cfg.pad_idx, cfg.vocabulary_size)
    with pytest.raises(ValueError):
        OracleLaser2(cfg, sd)(ids, torch.tensor([3, 0]))
    with pytest.raises(RuntimeError):  # what the reference's packing does with it
        _packed_lstm_reference(cfg, sd, ids, torch.tensor([3, 0]))


def test_lstm_gate_rows_definition():
    from sonar_b200.ops import lstm_gate_rows

    rows = lstm_gate_rows(512, 2)
    assert rows.shape == (4096,) and sorted(rows.tolist()) == list(range(4096))
    for n in (0, 31, 32, 127, 128, 1000, 2047):
        c, gate, u = n // 128, (n % 128) // 32, n % 32
        assert int(rows[n]) == gate * 512 + 32 * c + u and int(rows[2048 + n]) == 2048 + gate * 512 + 32 * c + u


def test_laser2_config_and_envelope():
    from sonar_b200.laser2 import _check_supported, laser2_config

    cfg = laser2_config("laser2")
    assert (cfg.vocabulary_size, cfg.pad_idx, cfg.model_dim, cfg.hidden_size, cfg.num_layers, cfg.bidirectional,
            cfg.padding_value) == (50004, 1, 320, 512, 5, True, 0.0)
    for ok in (dict(), dict(num_layers=1), dict(bidirectional=False), dict(model_dim=1024), dict(vocabulary_size=7)):
        _check_supported(laser2_config("laser2", **ok))
    for bad in (dict(hidden_size=256), dict(hidden_size=1024), dict(model_dim=300), dict(model_dim=0), dict(num_layers=0)):
        with pytest.raises(NotImplementedError, match="does not support"):
            _check_supported(laser2_config("laser2", **bad))
    with pytest.raises(ValueError):
        laser2_config("laser3")


def test_laser2_tokenizer_ids(tmp_path):
    spm = pytest.importorskip("sentencepiece")
    from sonar_b200.tokenizer import Laser2Tokenizer

    words = ["to", "be", "or", "not", "want", "go", "biking", "faire", "du", "vélo", "être", "ou", "ne", "pas", "je", "veux"]
    g = torch.Generator().manual_seed(0)
    lines = [" ".join(words[int(i)] for i in torch.randint(0, len(words), (int(torch.randint(3, 10, (1,), generator=g)),),
                                                            generator=g)) for _ in range(2000)]
    corpus = tmp_path / "corpus.txt"
    corpus.write_text("\n".join(lines) + "\n")
    prefix = str(tmp_path / "toy")
    spm.SentencePieceTrainer.train(input=str(corpus), model_prefix=prefix, vocab_size=120, model_type="bpe",
                                   character_coverage=1.0, hard_vocab_limit=False, minloglevel=2)
    sp = spm.SentencePieceProcessor(model_file=prefix + ".model")
    assert (sp.unk_id(), sp.bos_id(), sp.eos_id()) == (0, 1, 2)

    tok = Laser2Tokenizer(prefix + ".model")
    vi = tok.vocab_info
    assert (vi.pad_idx, vi.unk_idx, vi.eos_idx, vi.size) == (1, 0, 2, sp.get_piece_size() + 4)
    enc = tok.create_encoder()
    text = "to be or not to be 日"  # the last character is outside the training corpus: <unk>
    ids = enc(text)
    raw = sp.encode(text)
    assert 0 in raw
    assert ids.dtype == torch.int64 and ids.tolist() == [i + 4 if i >= 3 else i for i in raw] + [2]
    assert int(ids[-1]) == 2 and 1 not in ids.tolist() and enc.suffix_indices.tolist() == [2]
    assert int(ids[ids != 0][:-1].min()) >= 7  # pieces start at SentencePiece id 3, shifted by 4
    assert tok.create_encoder(lang="eng_Latn")(text).tolist() == ids.tolist()  # no language


def _header_fields(header, name):
    body = re.search(r"typedef struct " + name + r" \{(.*?)\} " + name + ";", header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return re.findall(r"(\w+)\s*;", body)


@pytest.mark.parametrize("name", ["SbLaser2Config", "SbLaser2Weights", "SbLstmLayerWeights"])
def test_laser2_ctypes_structs_match_the_header(name, tmp_path):
    from sonar_b200 import _lib

    header = open(os.path.join(ROOT, "include", "sonar_b200.h")).read()
    struct = getattr(_lib, name)
    fields = [f for f, _ in struct._fields_]
    assert fields == _header_fields(header, name)
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to measure the C layout")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sonar_b200.h"\nint main(void) {\n'
                   f'  printf("%zu\\n", sizeof({name}));\n' +
                   "".join(f'  printf("%zu\\n", offsetof({name}, {f}));\n' for f in fields) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(struct)] + [getattr(struct, f).offset for f in fields]


def test_lstm_kernel_builds_for_sm90a_without_spills(native_lib):
    """The recurrent kernel is in the library, issues wgmma, and ptxas reports no spills and no function call for it."""
    from sonar_b200 import _lib, build

    assert "lstm.cu" in build.SOURCES and native_lib.sb_version() >= 107
    for name in ("sb_laser2_create", "sb_laser2_forward", "sb_lstm_recurrent"):
        assert hasattr(native_lib, name)
    log = (build.LIB_DIR / "build.log").read_text()
    blocks = re.findall(r"Function properties for \S*lstm_recurrent_kernel\S*\n(.*?)\n.*?Used (\d+) registers", log)
    assert len(blocks) == 2, blocks  # the layer and the pooling variant
    for spills, regs in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in spills and int(regs) <= 255
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.lib_path())], capture_output=True, text=True).stdout
    kernels = [f for f in sass.split("Function : ")[1:] if f.split("\n", 1)[0].find("lstm_recurrent_kernel") >= 0]
    assert len(kernels) == 2
    for k in kernels:
        assert "HGMMA" in k and "CALL" not in k
