"""Drop-in mirror of ``sonar.inference_pipelines.text.TextToEmbeddingModelPipeline``
(``/root/reference/sonar/inference_pipelines/text.py:140-269``): same constructor and
``predict`` signature, same argument validation, truncation warning, length-sorted
dynamic bucketing and output-order restoration -- with the model stage running on the
CUDA engine (``sonar_b200.text_encoder.B200TextEncoderModel``).
"""

from __future__ import annotations

import contextlib
import os
import warnings
from pathlib import Path
from typing import Dict, Iterable, Iterator, List, Optional, Sequence, Union, cast

import torch
from torch import Tensor

from ..batching import collate, dynamic_bucket, prefetch, to_sequence_batch
from ..batching import bucket
from ..generation import BeamSearchSeq2SeqGenerator, SequenceToTextConverter
from ..sampling import SamplingSeq2SeqGenerator
from ..text_decoder import B200TextDecoderModel, sonar_text_decoder_config
from ..text_encoder import B200TextEncoderModel, sonar_text_encoder_config
from .utils import add_progress_bar

Device = Union[str, torch.device]
CPU = torch.device("cpu")


_MATMUL_PRECISION = {torch.bfloat16: "medium", torch.float16: "medium", torch.float32: "high", torch.float64: "highest"}


@contextlib.contextmanager
def precision_context(dtype: torch.dtype):
    """What the reference wraps every pipeline run in (``text.py:36-54``): torch's float32 matmul precision follows the model
    dtype for the duration of the call and is put back afterwards.  The sm_90a kernels are not affected by that switch
    (bf16 operands, fp32 accumulate, always); it is honoured so that torch code a caller runs inside the same ``with`` block
    behaves as it would around the reference."""
    before = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision(_MATMUL_PRECISION.get(dtype, "high"))
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(before)


def _load_encoder_card(name: str, device: Device) -> B200TextEncoderModel:
    """Resolve a reference card name (e.g. ``text_sonar_basic_encoder``,
    ``sonar/cards/text_sonar_basic_encoder.yaml``) to a local fairseq2-layout checkpoint
    ``$SONAR_B200_CHECKPOINT_DIR/<name>.pt``.  There is no downloader (no network)."""
    root = os.environ.get("SONAR_B200_CHECKPOINT_DIR")
    if not root or not (Path(root) / f"{name}.pt").exists():
        raise FileNotFoundError(
            f"encoder card {name!r}: set SONAR_B200_CHECKPOINT_DIR to a directory holding {name}.pt "
            "(fairseq2 state dict under the key 'model'), or pass a B200TextEncoderModel object")
    arch = "basic"
    return B200TextEncoderModel.from_checkpoint(Path(root) / f"{name}.pt", sonar_text_encoder_config(arch), device)


def _read_text(path: Path) -> Iterator[str]:
    """``fairseq2.data.text.read_text`` default behaviour: one example per line, line
    terminators stripped."""
    with open(path, "r", encoding="utf-8") as f:
        for line in f:
            yield line.rstrip("\r\n")


class TextToEmbeddingModelPipeline(torch.nn.Module):
    model: B200TextEncoderModel

    def __init__(
        self,
        encoder: Union[str, B200TextEncoderModel],
        tokenizer,
        device: Device = CPU,
        dtype: Optional[torch.dtype] = None,
    ) -> None:
        """
        Args:
            encoder: card name or model object exposing the reference encoder seam
                (``.eval()``, ``.dtype``, ``.encoder_frontend.pos_encoder.max_seq_len``,
                ``__call__(SequenceBatch) -> .sentence_embeddings``)
            tokenizer: tokenizer object (``create_encoder(lang=, device=)``, ``vocab_info.pad_idx``)
            device: device the token batches are sent to.  The engine itself is CUDA-only: with the
                reference's default (CPU) the batches are staged on the host and the model moves them.
            dtype: dtype of the returned embeddings (default: float32)
        """
        super().__init__()
        if isinstance(encoder, str):
            encoder = _load_encoder_card(encoder, device if torch.device(device).type == "cuda" else "cuda")
        if isinstance(tokenizer, str):
            raise FileNotFoundError(
                f"tokenizer card {tokenizer!r} cannot be resolved offline; pass a tokenizer object "
                "(sonar_b200.tokenizer.NllbTokenizer / SyntheticTokenizer)")
        self.tokenizer = tokenizer
        self.model = encoder.eval()  # type: ignore
        self.device = torch.device(device)
        self.dtype = dtype

    @torch.inference_mode()
    def predict(
        self,
        input: Union[Path, Sequence[str]],
        source_lang: str,
        batch_size: Optional[int] = 5,
        batch_max_tokens: Optional[int] = None,
        max_seq_len: Optional[int] = None,
        progress_bar: bool = False,
        target_device: Optional[Device] = None,
    ) -> Tensor:
        """
        Transform the input texts (from a list of strings or from a text file) into a matrix of their embeddings.
        The texts are truncated to `max_seq_len` tokens,
        or, if it is not specified, to the maximum that the model supports.
        """
        if batch_max_tokens is None and batch_size is None:
            raise ValueError("at least one of `batch_size` or `batch_max_tokens` should be provided")
        if batch_max_tokens is not None and batch_max_tokens <= 0:
            raise ValueError("`batch_max_tokens` should be strictly positive")
        if batch_size is not None and batch_size <= 0:
            raise ValueError("`batch_size` should be strictly positive")

        tokenizer_encoder = self.tokenizer.create_encoder(lang=source_lang, device=self.device)
        model_max_len = cast(Optional[int], self.model.encoder_frontend.pos_encoder.max_seq_len)
        if max_seq_len is None:
            max_seq_len = model_max_len
        if max_seq_len is not None and model_max_len is not None:
            if max_seq_len > model_max_len:
                raise ValueError(
                    f"max_seq_len cannot be larger than max_seq_len of the encoder model: {model_max_len}")

        n_truncated = 0

        def truncate(x: Tensor) -> Tensor:
            if max_seq_len is None:
                return x
            if x.shape[0] > max_seq_len:
                nonlocal n_truncated
                n_truncated += 1
            return x[:max_seq_len]

        if isinstance(input, (str, Path)):
            source: Iterable[str] = _read_text(Path(input))
            sorting_index = None
        else:
            # a list of sentences: encode in order of character length, restore the order at the end
            sorting_index = torch.argsort(torch.tensor(list(map(len, input))))
            source = (input[int(i)] for i in sorting_index.tolist())

        pad_idx = self.tokenizer.vocab_info.pad_idx
        on_cuda = self.device.type == "cuda"

        def batches():
            tokens = (truncate(tokenizer_encoder(s)) for s in source)
            for group in dynamic_bucket(tokens, batch_max_tokens or 2**31, len, min_num_examples=1,
                                        max_num_examples=batch_size or 20_000, drop_remainder=False):
                ids, lens, ragged = collate(group, pad_idx, pin_memory=True)
                yield to_sequence_batch(ids, lens, ragged, self.device if on_cuda else CPU)

        out_device = torch.device(target_device) if target_device is not None else self.device

        n_known = None if isinstance(input, (str, Path)) else len(input)
        sink = _HostSink(self, n_known) if (on_cuda and out_device.type == "cpu") else None

        def run_model() -> Iterable[Tensor]:
            # One batch of lag between launching a batch and collecting its embeddings: batch k+1 is already queued on the
            # GPU when the host blocks on the device->host copy of batch k, so the GPU never idles between batches (the
            # reference's `.map(self.model)` + `.to(target_device)` per batch leaves that gap).
            pending = None
            for b in prefetch(batches(), 2):
                emb = self.model(b).sentence_embeddings
                cur = sink.push(emb) if sink is not None and emb.is_cuda else _Ready(emb.to(out_device, non_blocking=True))
                if pending is not None:
                    yield pending.get()
                pending = cur
            if pending is not None:
                yield pending.get()

        pipeline: Iterable = run_model()
        if progress_bar:
            pipeline = add_progress_bar(pipeline, inputs=input,
                                        batch_size=batch_size if batch_max_tokens is None else None)

        with precision_context(self.model.dtype):
            results: List[Tensor] = list(iter(pipeline))
        # the reference's F.embedding raises on an id outside the table; the engine records it in a device flag --
        # surface it once per call (one 4-byte D2H) so a tokenizer / vocabulary mismatch cannot pass silently
        check = getattr(self.model, "check_inputs", None)
        if check is not None:
            check()

        if n_truncated:
            warnings.warn(
                f"For {n_truncated} input tensors for SONAR text encoder, "
                f"the length was truncated to {max_seq_len} elements.")

        whole = sink.result(results) if sink is not None else None
        sentence_embeddings = whole if whole is not None else torch.cat(results, dim=0)
        if self.dtype is not None:
            sentence_embeddings = sentence_embeddings.to(self.dtype)

        if sorting_index is not None:
            reversed_index = torch.argsort(sorting_index)
            sentence_embeddings = sentence_embeddings[reversed_index.to(sentence_embeddings.device)]
        return sentence_embeddings


class _Ready:
    def __init__(self, t: Tensor) -> None:
        self._t = t

    def get(self) -> Tensor:
        return self._t


class _HostSink:
    """Device -> host path of `predict(target_device="cpu")`.  Every batch is copied (asynchronously, on the launching
    stream, right behind its kernels) into one of TWO pinned staging buffers that live as long as the pipeline -- no pinned
    allocation per batch (`cudaHostAlloc` takes milliseconds to hundreds of milliseconds depending on the host's memory
    state) -- and from there into its slice of ONE result tensor allocated up front when the number of sentences is known,
    so there is no final `torch.cat` either.  With one batch of lag (see `predict`) slot k % 2 is free again when batch k + 2
    arrives."""

    def __init__(self, owner, n_total: Optional[int]) -> None:
        self._owner = owner
        self._n_total = n_total
        self._out: Optional[Tensor] = None
        self._pos = 0
        self._k = 0

    def push(self, emb: Tensor) -> "_HostSink._Slot":
        n, d = emb.shape
        ring = getattr(self._owner, "_d2h_ring", None)
        if ring is None or ring[0].shape[0] < n or ring[0].shape[1] != d or ring[0].dtype != emb.dtype:
            ring = [torch.empty((n, d), dtype=emb.dtype, pin_memory=True) for _ in range(2)]
            self._owner._d2h_ring = ring
        stage = ring[self._k % 2][:n]
        self._k += 1
        stage.copy_(emb, non_blocking=True)
        event = torch.cuda.Event()
        event.record(torch.cuda.current_stream(emb.device))
        if self._n_total is not None and self._out is None:
            self._out = torch.empty((self._n_total, d), dtype=emb.dtype)
        dst = None
        if self._out is not None and self._pos + n <= self._out.shape[0]:
            dst = self._out[self._pos:self._pos + n]
            self._pos += n
        return _HostSink._Slot(stage, event, dst)

    def result(self, parts: List[Tensor]) -> Optional[Tensor]:
        """The preallocated result when every batch landed in it, else None (the caller concatenates)."""
        if self._out is not None and self._pos == self._out.shape[0] and sum(p.shape[0] for p in parts) == self._pos:
            return self._out
        return None

    class _Slot:
        def __init__(self, stage: Tensor, event, dst: Optional[Tensor]) -> None:
            self._stage, self._event, self._dst = stage, event, dst

        def get(self) -> Tensor:
            self._event.synchronize()
            if self._dst is None:
                return self._stage.clone()
            self._dst.copy_(self._stage)
            return self._dst


def _load_decoder_card(name: str, device: Device) -> B200TextDecoderModel:
    root = os.environ.get("SONAR_B200_CHECKPOINT_DIR")
    if not root or not (Path(root) / f"{name}.pt").exists():
        raise FileNotFoundError(
            f"decoder card {name!r}: set SONAR_B200_CHECKPOINT_DIR to a directory holding {name}.pt "
            "(fairseq2 state dict under the key 'model'), or pass a B200TextDecoderModel object")
    return B200TextDecoderModel.from_checkpoint(Path(root) / f"{name}.pt", sonar_text_decoder_config("basic"), device)


class EmbeddingToTextModelPipeline(torch.nn.Module):
    """Mirror of ``sonar.inference_pipelines.text.EmbeddingToTextModelPipeline`` (``text.py:272-346``): sentence
    embeddings -> text with beam search.  ``self.model`` is the CUDA decoder itself: the reference wraps it as
    ``SonarEncoderDecoderModel(DummyEncoderModel, decoder)`` whose ``encode`` only un-squeezes the embedding to
    ``[N,1,D]`` (``sonar/models/sonar_translation/model.py:48-53,81-95``); the generator here does that reshape."""

    model: B200TextDecoderModel

    def __init__(self, decoder: Union[str, B200TextDecoderModel], tokenizer, device: Device = CPU,
                 dtype: Optional[torch.dtype] = None) -> None:
        super().__init__()
        if isinstance(decoder, str):
            decoder = _load_decoder_card(decoder, device if torch.device(device).type == "cuda" else "cuda")
        if isinstance(tokenizer, str):
            raise FileNotFoundError(f"tokenizer card {tokenizer!r} cannot be resolved offline; pass a tokenizer object")
        self.device = torch.device(device)
        self.tokenizer = tokenizer
        self.model = decoder.eval()  # type: ignore

    @torch.inference_mode()
    def predict(self, inputs: Tensor, target_lang: str, batch_size: int = 5, progress_bar: bool = False,
                sampler=None, **generator_kwargs) -> List[str]:
        generator_kwargs.setdefault("pad_idx", self.tokenizer.vocab_info.pad_idx)
        if sampler is not None:  # text.py:313-316
            generator = SamplingSeq2SeqGenerator(self.model, sampler, **generator_kwargs)
        else:
            generator = BeamSearchSeq2SeqGenerator(self.model, **generator_kwargs)
        converter = SequenceToTextConverter(generator, self.tokenizer, task="translation", target_lang=target_lang)

        def _do_translate(src_tensors: List[Tensor]) -> List[str]:
            texts, _ = converter.batch_convert(torch.stack(src_tensors).to(self.model.device), None)
            return texts

        pipeline: Iterable = (_do_translate(b) for b in bucket(list(inputs), batch_size))
        if progress_bar:
            pipeline = add_progress_bar(pipeline, inputs=inputs, batch_size=batch_size)
        with precision_context(self.model.dtype):
            results: List[List[str]] = list(iter(pipeline))
        return [x for y in results for x in y]


class TextToTextModelPipeline(torch.nn.Module):
    """Mirror of ``TextToTextModelPipeline`` (``text.py:57-137``): encode with the CUDA encoder, decode with the CUDA
    decoder.  ``max_seq_len`` is clamped to the decoder's position table like the reference (``:102-107``)."""

    def __init__(self, encoder: Union[str, B200TextEncoderModel], decoder: Union[str, B200TextDecoderModel], tokenizer,
                 device: Device = CPU, dtype: Optional[torch.dtype] = None) -> None:
        super().__init__()
        self.t2vec = TextToEmbeddingModelPipeline(encoder, tokenizer, device=device, dtype=None)
        self.vec2text = EmbeddingToTextModelPipeline(decoder, tokenizer, device=device, dtype=None)
        self.tokenizer = tokenizer

    @torch.inference_mode()
    def predict(self, input: Union[Path, Sequence[str]], source_lang: str, target_lang: str, batch_size: int = 5,
                progress_bar: bool = False, **generator_kwargs) -> List[str]:
        generator_kwargs = generator_kwargs or {}
        model_max_seq_len = self.vec2text.model.decoder_frontend.pos_encoder.max_seq_len
        generator_kwargs["max_seq_len"] = min(model_max_seq_len, generator_kwargs.get("max_seq_len", model_max_seq_len))
        emb = self.t2vec.predict(input, source_lang=source_lang, batch_size=batch_size, progress_bar=progress_bar)
        return self.vec2text.predict(emb, target_lang=target_lang, batch_size=batch_size, progress_bar=progress_bar,
                                     **generator_kwargs)
