"""CPU tests of the host logic: batcher semantics (SURVEY App. A.1), tokenizer layout,
pipeline argument validation, and that the C-ABI library loads and exports every symbol
include/sonar_b200.h declares (no compute calls without a GPU)."""

import os
import re

import pytest
import torch

from sonar_b200.batching import bucket, collate, dynamic_bucket, prefetch, to_sequence_batch
from sonar_b200.sequence import PaddingMask
from sonar_b200.tokenizer import SyntheticTokenizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dynamic_bucket_max_examples():
    out = list(dynamic_bucket(range(7), 2**31, lambda x: 1, max_num_examples=3))
    assert out == [[0, 1, 2], [3, 4, 5], [6]]


def test_dynamic_bucket_threshold_includes_crossing_example():
    # lengths 3,3,3 with threshold 5: the 2nd example crosses -> bucket of 2, then the rest
    out = list(dynamic_bucket([3, 3, 3], 5, lambda x: x, max_num_examples=20000))
    assert out == [[3, 3], [3]]
    # a single example longer than the threshold still makes progress (test_text_sonar.py:139-144)
    out = list(dynamic_bucket([9, 9], 5, lambda x: x, max_num_examples=20000))
    assert out == [[9], [9]]


def test_dynamic_bucket_drop_remainder_and_min():
    out = list(dynamic_bucket([1, 1, 1, 1, 1], 2, lambda x: x, min_num_examples=3, max_num_examples=10,
                              drop_remainder=True))
    assert out == [[1, 1, 1]]


def test_bucket():
    assert list(bucket(range(5), 2)) == [[0, 1], [2, 3], [4]]


def test_collate_ragged_and_dense():
    ids, lens, ragged = collate([torch.tensor([5, 6, 7]), torch.tensor([8])], pad_value=0)
    assert ids.tolist() == [[5, 6, 7], [8, 0, 0]] and lens == [3, 1] and ragged
    ids, lens, ragged = collate([torch.tensor([5, 6]), torch.tensor([8, 9])], pad_value=0)
    assert not ragged
    b = to_sequence_batch(ids, lens, ragged, "cpu")
    assert b.padding_mask is None  # utils.py:18-21: no mask when not ragged


def test_padding_mask_materialize():
    pm = PaddingMask(torch.tensor([2, 1]), 3)
    assert pm.materialize().tolist() == [[True, True, False], [True, False, False]]
    assert pm.seq_lens_host == [2, 1]


def test_prefetch_order_and_errors():
    assert list(prefetch(iter(range(10)), 2)) == list(range(10))

    def boom():
        yield 1
        raise KeyError("x")

    with pytest.raises(KeyError):
        list(prefetch(boom(), 2))


def test_synthetic_tokenizer_layout():
    tok = SyntheticTokenizer()
    enc = tok.create_encoder(lang="eng_Latn")
    ids = enc("a b c")
    assert ids.dtype == torch.int64 and ids.shape[0] == 5
    assert ids[-1].item() == 3 and ids[0].item() >= 256206 - 205  # [lang, pieces..., </s>]
    assert tok.vocab_info.pad_idx == 0
    assert torch.equal(ids, enc("a b c"))


def test_library_exports_every_declared_symbol(native_lib):
    header = open(os.path.join(ROOT, "include", "sonar_b200.h")).read()
    declared = set(re.findall(r"\b(sb_[a-z0-9_]+)\s*\(", header))
    from sonar_b200 import _lib

    assert declared == set(_lib._SIGNATURES), declared ^ set(_lib._SIGNATURES)
    for name in declared:
        assert hasattr(native_lib, name), name
    assert native_lib.sb_version() >= 100


def test_library_contains_hopper_sass(native_lib):
    """wgmma / TMA must be what the hot GEMM compiles to."""
    import shutil
    import subprocess

    from sonar_b200 import _lib

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.lib_path())], capture_output=True, text=True).stdout
    assert "HGMMA" in sass and "UTMALDG" in sass and "UTMASTG" in sass


def test_wgmma_pipeline_is_not_serialized(native_lib):
    """ptxas says so in the build log when it has to wait for every wgmma right after issuing it (a function call such as
    printf in the kernel, a wgmma under a branch, too few registers): the kernels must keep their groups in flight."""
    from sonar_b200 import build

    log = (build.LIB_DIR / "build.log").read_text()
    assert "wgmma.mma_async" in log or "gemm_wgmma" in log  # the log is the one of this library
    assert "wgmma.mma_async instructions are serialized" not in log


def test_pipeline_argument_validation():
    from sonar_b200.inference_pipelines.text import TextToEmbeddingModelPipeline

    class FakeEncoder(torch.nn.Module):
        class _F:
            class pos_encoder:
                max_seq_len = 514

        encoder_frontend = _F()
        dtype = torch.float32

    pipe = TextToEmbeddingModelPipeline(FakeEncoder(), SyntheticTokenizer(), device="cpu")
    with pytest.raises(ValueError, match="at least one of"):
        pipe.predict(["a"], "eng_Latn", batch_size=None, batch_max_tokens=None)
    with pytest.raises(ValueError, match="batch_max_tokens"):
        pipe.predict(["a"], "eng_Latn", batch_max_tokens=0)
    with pytest.raises(ValueError, match="batch_size"):
        pipe.predict(["a"], "eng_Latn", batch_size=0)
    with pytest.raises(ValueError, match="max_seq_len cannot be larger"):
        pipe.predict(["a"], "eng_Latn", max_seq_len=515)


def test_no_cpu_fallback_in_product():
    """The product package must not import the oracle nor offer a CPU compute path."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "sonar_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f
    from sonar_b200 import (B200SpeechEncoderModel, B200TextDecoderModel, B200TextEncoderModel,
                            sonar_speech_encoder_config, sonar_text_decoder_config, sonar_text_encoder_config)

    # the device is checked before the (empty) state dict is read
    for cls, config in ((B200TextEncoderModel, sonar_text_encoder_config()),
                        (B200TextDecoderModel, sonar_text_decoder_config()),
                        (B200SpeechEncoderModel, sonar_speech_encoder_config())):
        with pytest.raises(RuntimeError, match="CUDA"):
            cls(config, {}, device="cpu")


def test_annotations_resolve():
    """Every annotation in the package names something importable (``from __future__ import annotations`` defers them,
    so an unimported name only shows when a caller such as ``dataclasses`` tooling asks for ``get_type_hints``)."""
    import importlib
    import inspect
    import pkgutil
    import typing

    import sonar_b200

    for info in pkgutil.walk_packages(sonar_b200.__path__, "sonar_b200."):
        mod = importlib.import_module(info.name)
        for obj in vars(mod).values():
            if getattr(obj, "__module__", None) != mod.__name__:
                continue
            if inspect.isclass(obj):
                targets = [obj] + [f for f in vars(obj).values() if inspect.isfunction(f)]
            elif inspect.isfunction(obj):
                targets = [obj]
            else:
                continue
            for t in targets:
                typing.get_type_hints(t)  # NameError on an annotation that names nothing


def test_tsv_manifest_reader(tmp_path):
    """`read_tsv_audio_paths`: skip the header, right-trim, take one column (reference speech.py:103-109)."""
    from sonar_b200.inference_pipelines import SpeechInferenceParams, read_tsv_audio_paths

    f = tmp_path / "m.tsv"
    f.write_text("id\ttext\taudio\n1\thello\ta.wav  \n2\tworld\tsub/b.wav\n\n")
    assert list(read_tsv_audio_paths(f, 2)) == ["a.wav", "sub/b.wav"]
    assert list(read_tsv_audio_paths(f, 0)) == ["1", "2"]
    with pytest.raises(ValueError):
        list(read_tsv_audio_paths(f, 5))
    ctx = SpeechInferenceParams(data_file=f, audio_root_dir=tmp_path, audio_path_index=2, batch_size=4)
    assert ctx.pad_idx == 0 and ctx.n_parallel == 4 and ctx.n_prefetched_batches == 4 and ctx.target_lang is None


def test_bench_reference_arm_prints_one_contract_line():
    """`bench.py --impl reference` (the CPU restatement timed on host cores) needs no GPU: exactly one JSON line on stdout
    carrying the driver's keys."""
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    # reduced depth / vocabulary: the contract line is what is under test, not the 24-layer timing (ADVICE r1: the full
    # model took > 600 s on an 8-core CI box)
    p = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--layers", "2", "--vocab", "4096"],
                       capture_output=True, text=True, timeout=600, cwd=root)
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "sentences/sec->1024-d" and d["unit"] == "sentences/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["steps"] == 1
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_clock_sampler_parses_power_and_reasons():
    import bench

    class _P:
        def terminate(self):
            pass

    c = bench.ClockSampler(0)
    c.proc = _P()
    c.rows = ["0, 1290, 1965, 987.5, Not Active, Not Active, Not Active, Active, 1000.00",
              "0, 1305, 1965, 991.2, Not Active, Not Active, Not Active, Active, 1000.00", "garbage"]
    out = c.stop()
    assert out["sm_max_mhz"] == 1965.0 and out["reasons"] == ["sw_power_cap"] and out["samples"] == 2
    assert out["power_w"] == 991.2 and out["power_limit_w"] == 1000.0
    c.rows = ["0, 1290, 1965, [N/A], Not Active, Active, Not Active, Not Active"]
    out = c.stop()
    assert out["reasons"] == ["hw_thermal_slowdown"] and out["power_w"] is None


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_bench_product_arm_refuses_to_run_without_a_gpu():
    """No CPU fallback: without a CUDA device the product arm exits with an error instead of timing anything."""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--steps", "1"], capture_output=True, text=True,
                       timeout=300, cwd=root)
    assert p.returncode != 0
    assert "no CUDA device" in (p.stderr + p.stdout)
    assert not [l for l in p.stdout.splitlines() if l.startswith("{")]
