"""Drop-in mirrors of ``sonar.inference_pipelines.speech.SpeechToEmbeddingModelPipeline``
(``/root/reference/sonar/inference_pipelines/speech.py:402-474``) and ``SpeechToTextModelPipeline``
(``speech.py:311-400``): same constructor / ``predict`` signature; the
fairseq2n operators are replaced by the GPU fbank frontend (``sonar_b200.speech_frontend``) and the model stage by
``B200SpeechEncoderModel``.  Inputs are ``[C, T]`` waveform tensors at 16 kHz (``_decode_audio`` transposes to
``[T, C]``, ``speech.py:298-304``) or paths to PCM-16 mono ``.wav`` files (the reference decodes any libsndfile
format; only plain WAV is read here, with the standard library).
"""

from __future__ import annotations

import wave
from pathlib import Path
from typing import Iterable, List, Sequence, Union

import torch
from torch import Tensor

from ..batching import bucket, prefetch
from ..generation import BeamSearchSeq2SeqGenerator, SequenceToTextConverter
from ..sequence import PaddingMask, SequenceBatch
from ..speech_encoder import B200SpeechEncoderModel
from ..speech_frontend import SAMPLE_RATE, WaveformToFbank
from ..text_decoder import B200TextDecoderModel
from .utils import add_progress_bar

Device = Union[str, torch.device]
CPU_DEVICE = torch.device("cpu")


def _read_wav(path: Union[str, Path]) -> Tensor:
    with wave.open(str(path), "rb") as f:
        if f.getsampwidth() != 2 or f.getnchannels() != 1:
            raise ValueError(f"{path}: only 16-bit mono PCM WAV is supported")
        if f.getframerate() != SAMPLE_RATE:
            raise ValueError(f"{path}: sample rate must be {SAMPLE_RATE} Hz")
        pcm = torch.frombuffer(bytearray(f.readframes(f.getnframes())), dtype=torch.int16)
    return (pcm.float() / 32768.0)[None, :]  # [C=1, T] like a decoded file handed to the pipeline as a tensor


class SpeechToEmbeddingModelPipeline(torch.nn.Module):
    model: B200SpeechEncoderModel

    def __init__(self, encoder: Union[str, B200SpeechEncoderModel], device: Device = CPU_DEVICE,
                 fbank_dtype: torch.dtype = torch.float32) -> None:
        super().__init__()
        if isinstance(encoder, str):
            raise FileNotFoundError(f"speech encoder card {encoder!r} cannot be resolved offline; pass a "
                                    "B200SpeechEncoderModel object")
        if fbank_dtype != torch.float32:
            raise NotImplementedError("the CUDA frontend produces fp32 features; the encoder computes in bf16/fp32")
        self.device = torch.device(device)
        self.model = encoder.eval()
        self.convert_to_fbank = WaveformToFbank(self.model.device)

    def _decode_audio(self, inp: Union[str, Path, Tensor]) -> Tensor:
        if isinstance(inp, Tensor):
            if inp.dim() != 2:
                raise ValueError("waveform tensors must be [channels, samples]")
            return inp
        return _read_wav(inp)

    @torch.inference_mode()
    def predict(self, input: Union[Sequence[str], Sequence[Tensor]], batch_size: int = 3, n_parallel: int = 1,
                pad_idx: int = 0, n_prefetched_batches: int = 2, progress_bar: bool = False) -> Tensor:
        if pad_idx != 0:
            raise NotImplementedError("fbank batches are zero padded (the reference default)")

        def batches():
            for group in bucket((self._decode_audio(x) for x in input), batch_size):
                yield group

        def run(group: List[Tensor]) -> Tensor:
            fb, frames = self.convert_to_fbank(group)
            mask = PaddingMask(torch.tensor(frames), fb.shape[1], seq_lens_host=frames)
            return self.model(SequenceBatch(fb, mask)).sentence_embeddings

        pipeline: Iterable = (run(g) for g in prefetch(batches(), n_prefetched_batches))
        if progress_bar:
            pipeline = add_progress_bar(pipeline, inputs=input, batch_size=batch_size)
        results = list(iter(pipeline))
        return torch.cat(results, dim=0)


class SpeechToTextModelPipeline(SpeechToEmbeddingModelPipeline):
    """Speech -> text (``speech.py:311-400``).  The reference wraps encoder and decoder as
    ``SonarEncoderDecoderModel`` whose ``encode`` hands the decoder the pooled sentence embedding as a one-position
    encoder output (``sonar/models/sonar_translation/model.py:48-53``); here the speech engine produces that
    embedding and the decoder engine's beam search consumes it, both on the device, per bucket of utterances."""

    decoder: B200TextDecoderModel

    def __init__(self, encoder: Union[str, B200SpeechEncoderModel], decoder: Union[str, B200TextDecoderModel], tokenizer,
                 device: Device = CPU_DEVICE, fbank_dtype: torch.dtype = torch.float32) -> None:
        super().__init__(encoder, device=device, fbank_dtype=fbank_dtype)
        if isinstance(decoder, str):
            raise FileNotFoundError(f"decoder card {decoder!r} cannot be resolved offline; pass a B200TextDecoderModel object")
        if isinstance(tokenizer, str):
            raise FileNotFoundError(f"tokenizer card {tokenizer!r} cannot be resolved offline; pass a tokenizer object")
        self.decoder = decoder.eval()  # type: ignore
        self.tokenizer = tokenizer

    @torch.inference_mode()
    def predict(self, input: Union[Sequence[str], Sequence[Tensor]], target_lang: str, batch_size: int = 3,  # type: ignore
                n_parallel: int = 1, pad_idx: int = 0, n_prefetched_batches: int = 2, progress_bar: bool = False,
                **generator_kwargs) -> List[str]:
        if pad_idx != 0:
            raise NotImplementedError("fbank batches are zero padded (the reference default)")
        generator_kwargs.setdefault("pad_idx", self.tokenizer.vocab_info.pad_idx)
        generator = BeamSearchSeq2SeqGenerator(self.decoder, **generator_kwargs)
        converter = SequenceToTextConverter(generator, self.tokenizer, task="translation", target_lang=target_lang)

        def run(group: List[Tensor]) -> List[str]:
            fb, frames = self.convert_to_fbank(group)
            mask = PaddingMask(torch.tensor(frames), fb.shape[1], seq_lens_host=frames)
            emb = self.model(SequenceBatch(fb, mask)).sentence_embeddings
            texts, _ = converter.batch_convert(emb, None)
            return texts

        groups = bucket((self._decode_audio(x) for x in input), batch_size)
        pipeline: Iterable = (run(g) for g in prefetch(groups, n_prefetched_batches))
        if progress_bar:
            pipeline = add_progress_bar(pipeline, inputs=input, batch_size=batch_size)
        results: List[List[str]] = list(iter(pipeline))
        return [x for y in results for x in y]


# ---------------------------------------------------------------------------------------------------------------------
# TSV-driven pipelines (reference ``speech.py:42-274``): a manifest whose column ``audio_path_index`` names audio files
# under ``audio_root_dir``; the first line is a header.  ``build_pipeline(context)`` returns an iterable with one item per
# bucket of ``batch_size`` lines -- the model output the reference's ``DataPipeline`` yields under ``audio.data``.
# ---------------------------------------------------------------------------------------------------------------------
from dataclasses import dataclass  # noqa: E402
from typing import Iterator, Optional  # noqa: E402


@dataclass
class SpeechInferenceParams:
    """Same fields and defaults as the reference dataclass (``speech.py:42-77``)."""

    data_file: Path
    audio_root_dir: Path
    audio_path_index: int
    batch_size: int
    fbank_dtype: torch.dtype = torch.float32
    target_lang: Optional[str] = None
    pad_idx: int = 0
    device: Device = CPU_DEVICE
    n_parallel: int = 4
    n_prefetched_batches: int = 4


def read_tsv_audio_paths(data_file: Union[str, Path], audio_path_index: int) -> Iterator[str]:
    """``read_text(rtrim=True).skip(1).map(StrSplitter(indices=[audio_path_index]))`` (``speech.py:103-109``)."""
    with open(data_file, "r", encoding="utf-8") as f:
        for lineno, line in enumerate(f):
            if lineno == 0:
                continue  # header
            line = line.rstrip()
            if not line:
                continue
            fields = line.split("\t")
            if audio_path_index >= len(fields):
                raise ValueError(f"{data_file}:{lineno + 1}: no column {audio_path_index}")
            yield fields[audio_path_index]


class AudioToFbankDataPipelineBuilder:
    """Manifest -> buckets of waveforms -> (fbank ``SequenceBatch``) per bucket (``speech.py:94-147``); the fbank runs on the
    device of ``context``."""

    def build_pipeline(self, context: SpeechInferenceParams) -> Iterator[SequenceBatch]:
        if context.pad_idx != 0:
            raise NotImplementedError("fbank batches are zero padded (the reference default)")
        if context.fbank_dtype != torch.float32:
            raise NotImplementedError("the CUDA frontend produces fp32 features")
        frontend = WaveformToFbank(torch.device(context.device))
        root = Path(context.audio_root_dir)
        waves = (_read_wav(root / p) for p in read_tsv_audio_paths(context.data_file, context.audio_path_index))

        def batches():  # file decoding runs ahead on the prefetch thread; the fbank kernels stay on the caller's thread
            for group in prefetch(bucket(waves, context.batch_size), context.n_prefetched_batches):
                fb, frames = frontend(group)
                yield SequenceBatch(fb, PaddingMask(torch.tensor(frames), fb.shape[1], seq_lens_host=frames))

        return batches()


class SpeechToEmbeddingPipeline:
    """``SpeechToEmbeddingPipeline`` (``speech.py:150-201``): yields the encoder output of every bucket."""

    def __init__(self, model: B200SpeechEncoderModel) -> None:
        self.model = model.eval()
        self.audio_to_fbank_dp_builder = AudioToFbankDataPipelineBuilder()

    @classmethod
    def load_model_from_name(cls, encoder_name: str) -> "SpeechToEmbeddingPipeline":
        raise FileNotFoundError(f"speech encoder card {encoder_name!r} cannot be resolved offline; construct with a model object")

    def build_pipeline(self, context: SpeechInferenceParams):
        @torch.inference_mode()
        def run():
            for batch in self.audio_to_fbank_dp_builder.build_pipeline(context):
                yield self.model(batch)

        return run()


class SpeechToTextPipeline:
    """``SpeechToTextPipeline`` (``speech.py:204-274``): yields the translated texts of every bucket."""

    def __init__(self, encoder: B200SpeechEncoderModel, decoder: B200TextDecoderModel, tokenizer) -> None:
        self.encoder = encoder.eval()
        self.decoder = decoder.eval()  # type: ignore
        self.tokenizer = tokenizer
        self.audio_to_fbank_dp_builder = AudioToFbankDataPipelineBuilder()

    def build_pipeline(self, context: SpeechInferenceParams, **generator_kwargs):
        assert context.target_lang is not None
        generator_kwargs.setdefault("pad_idx", self.tokenizer.vocab_info.pad_idx)
        generator = BeamSearchSeq2SeqGenerator(self.decoder, **generator_kwargs)
        converter = SequenceToTextConverter(generator, self.tokenizer, task="translation", target_lang=context.target_lang)

        @torch.inference_mode()
        def run():
            for batch in self.audio_to_fbank_dp_builder.build_pipeline(context):
                texts, _ = converter.batch_convert(self.encoder(batch).sentence_embeddings, None)
                yield texts

        return run()
