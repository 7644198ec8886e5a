"""Host-side mirror of the reference text encoder model, backed by the CUDA engine.

``B200TextEncoderModel`` is what a user passes as ``encoder=`` to
``TextToEmbeddingModelPipeline`` in place of fairseq2's
``SonarTextTransformerEncoderModel`` (``sonar/models/sonar_text/model.py:30-143``).
It exposes exactly the seam the pipeline touches (SURVEY §8b):

* ``.eval()``, ``.dtype`` (``sonar/models/encoder_model.py:56-58``)
* ``.encoder_frontend.pos_encoder.max_seq_len`` (``sonar/inference_pipelines/text.py:202``)
* ``__call__(SequenceBatch) -> SonarEncoderOutput`` (``text.py:244-245``)

All arithmetic happens in ``libsonar_b200.so`` (``sb_encoder_forward``); this file
only repacks weights (bf16, fused QKV) and owns device buffers.
"""

from __future__ import annotations

import ctypes as C
import dataclasses
import math
from dataclasses import dataclass, field
from enum import Enum
from typing import Dict, List, Optional, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib, ops
from ._engine import EngineModel
from .sequence import PaddingMask, SequenceBatch, SonarEncoderOutput


class Pooling(Enum):
    """Same members/values as the reference enum (``model.py:23-27``)."""

    MAX = 1
    MEAN = 2
    LAST = 3
    ATTENTION = 4


@dataclass
class VocabularyInfo:
    size: int
    unk_idx: Optional[int] = None
    bos_idx: Optional[int] = None
    eos_idx: Optional[int] = None
    pad_idx: Optional[int] = None


@dataclass
class SonarTextEncoderConfig:
    """Field-for-field mirror of the reference dataclass
    (``sonar/models/sonar_text/config.py:14-84``); defaults = arch ``basic`` (``:92-116``)."""

    model_dim: int = 1024
    max_seq_len: int = 512
    vocab_info: VocabularyInfo = field(
        default_factory=lambda: VocabularyInfo(size=256206, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    num_encoder_layers: int = 24
    num_decoder_layers: int = 24
    num_encoder_attn_heads: int = 16
    num_decoder_attn_heads: int = 16
    ffn_inner_dim: int = 1024 * 8
    pooling: str = "mean"
    embedding_dim: Optional[int] = None
    decoder_ffn_inner_dim: Optional[int] = None
    activation_fn: str = "ReLU"
    layernorm_embedding: bool = False
    no_scale_embedding: bool = False
    no_token_positional_embeddings: bool = False
    learned_pos: bool = False
    emb_dropout_p: float = 0.1
    attention_dropout_p: float = 0.1
    activation_dropout_p: float = 0.1
    normalize_before: bool = False
    _from_fairseq: bool = True


def sonar_text_encoder_config(arch: str = "basic", **overrides) -> SonarTextEncoderConfig:
    """Named archs of ``register_sonar_text_encoder_configs`` (``config.py:87-127``)."""
    if arch == "basic":
        cfg = SonarTextEncoderConfig()
    elif arch == "small":  # config.py:118-127
        cfg = SonarTextEncoderConfig(
            vocab_info=VocabularyInfo(size=32005, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1),
            num_encoder_layers=6, num_decoder_layers=6, ffn_inner_dim=1024 * 4)
    else:
        raise ValueError(f"unknown sonar text encoder arch {arch!r}")
    return dataclasses.replace(cfg, **overrides)


def sinusoidal_position_table(num_pos: int, dim: int, legacy_pad_idx: int) -> Tensor:
    """fp32 table whose row t encodes position ``t + legacy_pad_idx + 1``: fairseq2
    ``SinusoidalPositionEncoder(_legacy_pad_idx=pad_idx)`` as built at ``factory.py:88-92``
    ([sin | cos] halves, frequencies ``exp(-j ln(1e4) / (dim/2 - 1))``)."""
    half = dim // 2
    start = legacy_pad_idx + 1
    steps = torch.arange(start, start + num_pos, dtype=torch.float32)
    freq = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000.0) / (half - 1)))
    ang = steps[:, None] * freq[None, :]
    return torch.cat([torch.sin(ang), torch.cos(ang)], dim=1).contiguous()


class _PosEncoderInfo:
    def __init__(self, max_seq_len: int) -> None:
        self.max_seq_len = max_seq_len


class _FrontendInfo:
    """Carries ``encoder_frontend.pos_encoder.max_seq_len`` / ``decoder_frontend.pos_encoder.max_seq_len`` (read at
    ``text.py:202`` and ``text.py:102``)."""

    def __init__(self, max_seq_len: int, model_dim: int) -> None:
        self.pos_encoder = _PosEncoderInfo(max_seq_len)
        self.model_dim = model_dim


def _embedding_dim(cfg: SonarTextEncoderConfig) -> int:
    """Width of the sentence embeddings (``SonarTextEncoderFactory.embedding_dim``, ``factory.py:66-69``)."""
    return cfg.embedding_dim or cfg.model_dim


def _pooler_ffn_inner_dim(cfg: SonarTextEncoderConfig) -> int:
    """Inner width of the attention pooler's FFNs (``create_ffn(inner_dim=decoder_ffn_inner_dim)``, ``factory.py:143-148``)."""
    return cfg.decoder_ffn_inner_dim or cfg.ffn_inner_dim


def _check_supported(cfg: SonarTextEncoderConfig) -> None:
    bad = []
    pooling = cfg.pooling.lower()
    if pooling not in ("mean", "max", "last", "attention"):
        bad.append(f"pooling={cfg.pooling!r}")
    if cfg.activation_fn != "ReLU":
        bad.append(f"activation_fn={cfg.activation_fn!r}")
    if cfg.layernorm_embedding or cfg.no_token_positional_embeddings or cfg.learned_pos:
        bad.append("layernorm_embedding / no_token_positional_embeddings / learned_pos")
    if cfg.model_dim != 64 * cfg.num_encoder_attn_heads:
        bad.append("head_dim != 64")
    e = _embedding_dim(cfg)
    if pooling != "attention":
        if e != cfg.model_dim:
            bad.append("embedding_dim != model_dim without attention pooling")
    else:
        if e % 256 != 0 or e > 1024 or e != 64 * cfg.num_decoder_attn_heads:
            bad.append(f"attention pooling with embedding_dim={e}, num_decoder_attn_heads={cfg.num_decoder_attn_heads} "
                       "(needs a multiple of 256, <= 1024, head_dim 64)")
        if _pooler_ffn_inner_dim(cfg) % 256 != 0:
            bad.append(f"attention pooling with a pooler FFN width of {_pooler_ffn_inner_dim(cfg)} (needs a multiple of 256)")
        if cfg.num_decoder_layers < 1:
            bad.append("attention pooling with num_decoder_layers < 1")
        if cfg.normalize_before:
            bad.append("attention pooling with normalize_before=True (a PRE-LN pooler)")
    if bad:
        raise NotImplementedError("sonar_b200 text encoder does not support: " + "; ".join(bad))


class B200TextEncoderModel(EngineModel):
    """SONAR text encoder (24-layer pre-LN Transformer + final LN + pooling) on sm_90a kernels.

    ``pooling="attention"`` runs the reference's trainable pooler (``factory.py:155-226``): one BOS query through
    ``num_decoder_layers`` POST-LN decoder layers cross-attending the final-LayerNormed token states, then
    ``projection_out``; the sentence embeddings are ``embedding_dim`` wide."""

    _abi = "encoder"
    _default_config = staticmethod(sonar_text_encoder_config)

    def __init__(self, config: SonarTextEncoderConfig, state_dict: Dict[str, Tensor],
                 device: Union[str, torch.device] = "cuda", *, cta_group: int = 2,
                 ln_fold: Union[bool, int] = False) -> None:
        """``ln_fold=True``: the engine folds every encoder-layer LayerNorm into the GEMMs around it (see
        ``SbEncoderConfig.ln_fold`` in ``include/sonar_b200.h``); the default runs the separate LayerNorm kernels
        (``bench.py`` A/Bs the schedules in every run, ``ab_schedule_variants``)."""
        super().__init__(device)
        self.ln_fold = int(ln_fold)  # 0 = separate LayerNorm kernels, 1 = both folded, 2 = only the attention-block one
        _check_supported(config)
        self.config = config
        self.model_dim = config.model_dim
        self.embedding_dim = _embedding_dim(config)
        self.pooling = getattr(Pooling, config.pooling.upper())
        pad_idx = config.vocab_info.pad_idx if config.vocab_info.pad_idx is not None else 1
        max_len = config.max_seq_len + (pad_idx + 1 if config._from_fairseq else 0)  # factory.py:53-59
        self.encoder_frontend = _FrontendInfo(max_len, config.model_dim)

        sd = state_dict
        d, L = config.model_dim, config.num_encoder_layers
        bf, f32 = self._bf16, self._f32

        embed = sd["encoder_frontend.embed.weight"]
        if embed.shape != (config.vocab_info.size, d):
            raise ValueError(f"embedding shape {tuple(embed.shape)} != ({config.vocab_info.size}, {d})")
        top = {"embed": bf(embed), "pos_table": f32(sinusoidal_position_table(max_len, d, pad_idx)),
               "final_ln_g": f32(sd["layer_norm.weight"]), "final_ln_b": f32(sd["layer_norm.bias"])}
        self._layer_bufs: List[Dict[str, Tensor]] = []
        for i in range(L):
            p = f"encoder.layers.{i}."
            a = p + "self_attn."
            self._layer_bufs.append({
                "wqkv": bf(torch.cat([sd[a + "q_proj.weight"], sd[a + "k_proj.weight"], sd[a + "v_proj.weight"]], 0)),
                "bqkv": f32(torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]], 0)),
                "wo": bf(sd[a + "output_proj.weight"]), "bo": f32(sd[a + "output_proj.bias"]),
                "w1": bf(sd[p + "ffn.inner_proj.weight"]), "b1": f32(sd[p + "ffn.inner_proj.bias"]),
                "w2": bf(sd[p + "ffn.output_proj.weight"]), "b2": f32(sd[p + "ffn.output_proj.bias"]),
                "ln1_g": f32(sd[p + "self_attn_layer_norm.weight"]), "ln1_b": f32(sd[p + "self_attn_layer_norm.bias"]),
                "ln2_g": f32(sd[p + "ffn_layer_norm.weight"]), "ln2_b": f32(sd[p + "ffn_layer_norm.bias"]),
            })

        attn = self.pooling == Pooling.ATTENTION
        pooler_layers = []
        if attn:
            pooler_top, pooler_layers = self._pooler_weights(sd, "pooler", 0, self.embedding_dim)
            top.update(pooler_top)
        cfg_c = _lib.SbEncoderConfig(
            model_dim=d, num_layers=L, num_heads=config.num_encoder_attn_heads, ffn_inner_dim=config.ffn_inner_dim,
            vocab_size=config.vocab_info.size, pos_rows=max_len, pooling=self.pooling.value, ln_eps=1e-5,
            embed_scale=1.0 if config.no_scale_embedding else math.sqrt(d), cta_group=cta_group, num_sms=0,
            ln_fold=int(ln_fold), embedding_dim=self.embedding_dim,
            pooler_layers=config.num_decoder_layers if attn else 0,
            pooler_heads=config.num_decoder_attn_heads if attn else 0,
            pooler_ffn_inner_dim=_pooler_ffn_inner_dim(config) if attn else 0)
        w_c = _lib.SbEncoderWeights(layers=self._layer_array(_lib.SbLayerWeights, self._layer_bufs),
                                    **{k: v.data_ptr() for k, v in top.items()})
        if attn:
            w_c.pooler = self._layer_array(_lib.SbPoolerLayerWeights, pooler_layers)
        self._create(cfg_c, w_c)
        self.return_encoded_seqs = False

    @torch.inference_mode()
    def forward(self, batch: SequenceBatch) -> SonarEncoderOutput:
        seqs = batch.seqs
        if seqs.dim() != 2:
            raise ValueError("expected token ids of shape [N, S]")
        seqs = self._on_device(seqs, torch.int64)
        if seqs.stride(1) != 1:
            seqs = seqs.contiguous()
        n, s = seqs.shape
        pm = batch.padding_mask
        if pm is not None:
            lens_np = np.ascontiguousarray(pm.seq_lens_host, dtype=np.int32)  # one vectorised conversion, no per-item Python
            lens_c = lens_np.ctypes.data_as(C.POINTER(C.c_int32))
            tokens = int(lens_np.sum(dtype=np.int64))
        else:
            lens_c = None
            tokens = n * s
        ws = self._ensure_workspace(n, max(tokens, 1), headroom=1.1)  # predict() grows it batch by batch
        out = torch.empty((n, self.embedding_dim), dtype=torch.float32, device=self.device)
        enc = (torch.empty((n, s, self.model_dim), dtype=torch.float32, device=self.device)
               if self.return_encoded_seqs else None)
        with torch.cuda.device(self.device):
            rc = self._lib.sb_encoder_forward(
                self._handle, seqs.data_ptr(), seqs.stride(0), lens_c, n, s, out.data_ptr(),
                enc.data_ptr() if enc is not None else None, ws.data_ptr(), ws.numel(), self._stream())
        _lib.check(rc, "sb_encoder_forward")
        return SonarEncoderOutput(encoded_seqs=enc, sentence_embeddings=out, padding_mask=pm)

    def profile_ffn1(self, start: Optional[torch.cuda.Event], stop: Optional[torch.cuda.Event]) -> None:
        """Record `start`/`stop` (timing-enabled events that have been recorded once, so their handles exist) around
        the FFN inner-projection GEMM of the middle layer in every following forward; (None, None) switches it off."""
        _lib.check(self._lib.sb_encoder_profile_ffn1(self._handle, start.cuda_event if start is not None else None,
                                                     stop.cuda_event if stop is not None else None),
                   "sb_encoder_profile_ffn1")

    def check_inputs(self) -> None:
        """Raise ``ValueError`` if a batch since the last check contained a token id outside the vocabulary."""
        _lib.check(self._lib.sb_encoder_check_inputs(self._handle, self._stream()), "sb_encoder_check_inputs")

    # ------------------------------------------------------------------ reference static API
    @staticmethod
    def static_pooling(seqs: Tensor, padding_mask: Optional[PaddingMask], pooling: Pooling) -> Tensor:
        """``SonarTextTransformerEncoderModel.static_pooling`` (``model.py:86-128``) on the GPU kernel.
        ``seqs`` is a padded CUDA tensor [N, S, D] with D a multiple of 128."""
        if pooling == Pooling.ATTENTION:
            raise NotImplementedError(pooling)
        ops._need_cuda(seqs)
        n, s, d = seqs.shape
        lens = padding_mask.seq_lens_host if padding_mask is not None else [s] * n
        valid = (torch.arange(s)[None, :] < torch.tensor(lens)[:, None]).to(seqs.device)
        packed = seqs.float()[valid].contiguous()  # [T, D] (layout change only)
        cu = ops.cu_seqlens_of(lens).to(seqs.device)
        return ops.pool_packed(packed, cu, pooling.name).to(seqs.dtype)
