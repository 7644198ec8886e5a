"""Tokenizers with the surface the pipelines use (``sonar/inference_pipelines/text.py:199-201,241``):
``tokenizer.create_encoder(lang=..., device=...) -> callable(str) -> int64[len]`` and
``tokenizer.vocab_info.pad_idx``.

* ``NllbTokenizer`` wraps a SentencePiece model in the NLLB layout the SONAR cards use
  (``tokenizer_family: nllb``; ids pad=0 unk=1 bos=2 eos=3, then pieces, then the
  ``__lang__`` control symbols; source encoding ``[__lang__] + pieces + [</s>]``;
  SURVEY App. F1).  Needs the ``sentencepiece.bpe.model`` file, which is not available
  offline; the class exists so real checkpoints work wherever the files do.
* ``Laser2Tokenizer`` wraps the LASER2 SentencePiece model (``laser2.spm``; tokenizer family ``lstm``).
* ``SyntheticTokenizer`` is a dependency-free stand-in (hashes whitespace words into the
  piece id range) for tests and benchmarks: same control-token layout, deterministic.
"""

from __future__ import annotations

import zlib
from typing import Callable, List, Optional, Sequence

import torch
from torch import Tensor

from .text_encoder import VocabularyInfo

# FLORES-200 language codes in NLLB dictionary order are only needed with a real SPM
# model; the synthetic tokenizer derives a stable id for any code.
_NUM_LANG_SLOTS = 202


class _TokenEncoder:
    """``prefix_indices`` / ``suffix_indices`` mirror fairseq2's text encoders: in NLLB *target* mode the prefix is
    ``[</s>, __lang__]`` -- the decoder prompt ``SequenceToTextConverter`` feeds the generator (SURVEY App. C / F1)."""

    def __init__(self, fn: Callable[[str], List[int]], prefix: Optional[List[int]] = None,
                 suffix: Optional[List[int]] = None) -> None:
        self._fn = fn
        self.prefix_indices = torch.tensor(prefix, dtype=torch.int64) if prefix is not None else None
        self.suffix_indices = torch.tensor(suffix, dtype=torch.int64) if suffix is not None else None

    def __call__(self, text: str) -> Tensor:
        return torch.tensor(self._fn(text), dtype=torch.int64)


class _TokenDecoder:
    def __init__(self, fn: Callable[[List[int]], str]) -> None:
        self._fn = fn

    def __call__(self, ids: Tensor) -> str:
        return self._fn([int(i) for i in ids.tolist()])


class SyntheticTokenizer:
    """Deterministic word-hash tokenizer with the NLLB id layout (test/bench utility)."""

    def __init__(self, vocab_size: int = 256206, pieces_per_word: int = 1) -> None:
        if vocab_size < 4 + _NUM_LANG_SLOTS + 8:
            raise ValueError("vocab too small for the NLLB control-token layout")
        self.vocab_info = VocabularyInfo(size=vocab_size, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=0)
        self._lang_base = vocab_size - _NUM_LANG_SLOTS - 3
        self._num_pieces = self._lang_base - 4
        self._ppw = pieces_per_word

    def lang_id(self, lang: str) -> int:
        return self._lang_base + zlib.crc32(lang.encode("utf-8")) % _NUM_LANG_SLOTS

    def _encode(self, text: str, lang: str) -> List[int]:
        ids = [self.lang_id(lang)]
        for w in text.split():
            for k in range(self._ppw):
                ids.append(4 + zlib.crc32(f"{k}:{w}".encode("utf-8")) % self._num_pieces)
        ids.append(self.vocab_info.eos_idx)
        return ids

    def create_encoder(self, *, task: Optional[str] = None, lang: Optional[str] = None, mode: Optional[str] = None,
                       device=None, pin_memory: bool = False) -> _TokenEncoder:
        if lang is None:
            raise ValueError("`lang` is required")
        eos = self.vocab_info.eos_idx
        if mode == "target":  # [</s>, __lang__] pieces... </s>
            return _TokenEncoder(lambda text: [eos] + self._encode(text, lang), prefix=[eos, self.lang_id(lang)],
                                 suffix=[eos])
        return _TokenEncoder(lambda text: self._encode(text, lang), prefix=[self.lang_id(lang)], suffix=[eos])

    def create_decoder(self) -> "_TokenDecoder":
        """ids -> text; control symbols are dropped, every piece id prints as ``t<id>`` (the hash is one-way)."""
        lo, hi = 4, self._lang_base

        def dec(ids: List[int]) -> str:
            return " ".join(f"t{i}" for i in ids if lo <= i < hi)

        return _TokenDecoder(dec)


class NllbTokenizer:
    """SentencePiece-backed NLLB tokenizer (source mode), ids as in fairseq2's NLLB family."""

    def __init__(self, spm_path: str, langs: Sequence[str], extra_control: Sequence[str] = ("<MINED_DATA>", "<MMT_BT_DATA>", "<SMT_BT_DATA>")) -> None:
        import sentencepiece as spm  # local import: optional dependency

        self._sp = spm.SentencePieceProcessor(model_file=str(spm_path))
        n = self._sp.get_piece_size()
        # fairseq2 appends the control symbols after the SPM pieces (and remaps pad/unk/bos/eos to 0..3)
        self._lang_ids = {f"__{l}__": n + 1 + i for i, l in enumerate(langs)}
        size = n + 1 + len(langs) + len(extra_control)
        self.vocab_info = VocabularyInfo(size=size, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=0)

    def create_encoder(self, *, task: Optional[str] = None, lang: Optional[str] = None, mode: Optional[str] = None,
                       device=None, pin_memory: bool = False) -> _TokenEncoder:
        if lang is None or f"__{lang}__" not in self._lang_ids:
            raise ValueError(f"`lang` must be one of the tokenizer's languages, got {lang!r}")
        lang_id = self._lang_ids[f"__{lang}__"]
        sp = self._sp

        def enc(text: str) -> List[int]:
            # SPM ids: <unk>=0,<s>=1,</s>=2 then pieces; NLLB/fairseq2 ids: pad0 unk1 bos2 eos3 then pieces (+1)
            return [lang_id] + [i + 1 for i in sp.encode(text)] + [3]

        if mode == "target":
            return _TokenEncoder(lambda text: [3] + enc(text), prefix=[3, lang_id], suffix=[3])
        return _TokenEncoder(enc, prefix=[lang_id], suffix=[3])

    def create_decoder(self) -> "_TokenDecoder":
        sp = self._sp
        n = sp.get_piece_size()

        def dec(ids: List[int]) -> str:
            return sp.decode([i - 1 for i in ids if 4 <= i <= n])

        return _TokenDecoder(dec)


class Laser2Tokenizer:
    """The LASER2 tokenizer (``sonar/models/laser2_text/tokenizer.py:27-87``): SentencePiece ids with a ``</s>`` suffix,
    then ``id + 4`` for every id >= 3, so ids 0 (``<unk>``) and 2 (``</s>``) are unchanged and 1 is never produced.
    Batches are padded with ``vocab_info.pad_idx`` = 1, the id the ``laser2`` config masks (``config.py:33``).

    The reference builds its vocabulary information through fairseq2's ``SentencePieceModel(path, ["<pad>"])`` and
    ``vocab_info_from_sentencepiece`` [fs2]; which id fairseq2 gives the added ``<pad>`` control symbol is not pinned
    here.  ``pad_idx`` = 1 is what the model and the reference's own test (``Collater(pad_value=1)``) use."""

    def __init__(self, spm_path: str) -> None:
        import sentencepiece as spm  # local import: optional dependency

        self._sp = spm.SentencePieceProcessor(model_file=str(spm_path))
        # shifted piece ids reach piece_size + 3
        self.vocab_info = VocabularyInfo(size=self._sp.get_piece_size() + 4, unk_idx=0, bos_idx=None, eos_idx=2, pad_idx=1)

    def create_encoder(self, *, task: Optional[str] = None, lang: Optional[str] = None, mode: Optional[str] = None,
                       device=None, pin_memory: bool = False) -> _TokenEncoder:
        """No language: LASER2 is language-agnostic.  ``task`` / ``lang`` / ``mode`` are accepted and ignored, as in the
        reference."""
        sp = self._sp
        eos = sp.eos_id()

        def enc(text: str) -> List[int]:
            return [i + 4 if i >= 3 else i for i in sp.encode(text) + [eos]]

        return _TokenEncoder(enc, suffix=[eos])
