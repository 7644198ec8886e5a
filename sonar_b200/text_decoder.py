"""Host-side mirror of the reference embedding->text decoder, backed by the CUDA engine.

``B200TextDecoderModel`` stands where fairseq2's ``ConditionalTransformerDecoderModel``
(``sonar/nn/conditional_decoder_model.py:26-94``, built by ``SonarTextDecoderFactory``,
``sonar/models/sonar_text/factory.py:229-315``) stands in ``EmbeddingToTextModelPipeline``
(``sonar/inference_pipelines/text.py:272-346``).  The reference generator calls ``decode``/``project`` once per
generated token with an incremental state bag; here the same step is one C-ABI call (``sb_decoder_step``) that
returns the 16 most probable next tokens per hypothesis (log-softmax over the full vocabulary) instead of the
``[R, 256206]`` logits tensor.
"""

from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass, field
from typing import Dict, Optional, Tuple, Union

import torch
from torch import Tensor

from . import _lib
from ._engine import EngineModel
from .text_encoder import VocabularyInfo, _FrontendInfo, sinusoidal_position_table

TOPK = 16  # candidates per row returned by sb_decoder_step (kTopkCandidates)


@dataclass
class SonarTextDecoderConfig:
    """Mirror of the reference dataclass (``sonar/models/sonar_text/config.py:130-194``); defaults = ``basic``."""

    model_dim: int = 1024
    max_seq_len: int = 512
    vocab_info: VocabularyInfo = field(
        default_factory=lambda: VocabularyInfo(size=256206, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1))
    activation_fn: str = "ReLU"
    layernorm_embedding: bool = False
    no_scale_embedding: bool = False
    no_token_positional_embeddings: bool = False
    learned_pos: bool = False
    emb_dropout_p: float = 0.1
    attention_dropout_p: float = 0.1
    activation_dropout_p: float = 0.1
    normalize_before: bool = True
    num_encoder_layers: int = 24
    num_decoder_layers: int = 24
    num_encoder_attn_heads: int = 16
    num_decoder_attn_heads: int = 16
    ffn_inner_dim: int = 1024 * 8
    input_dim: Optional[int] = None


def sonar_text_decoder_config(arch: str = "basic", **overrides) -> SonarTextDecoderConfig:
    """Named archs of ``register_sonar_text_decoder_configs`` (``config.py:197-255``; ``toy`` is too small for
    the 64-wide heads / 256-wide tiles of this engine and is not offered)."""
    if arch == "basic":
        cfg = SonarTextDecoderConfig()
    elif arch == "small":
        cfg = SonarTextDecoderConfig(
            vocab_info=VocabularyInfo(size=32005, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=1),
            num_encoder_layers=6, num_decoder_layers=6, ffn_inner_dim=1024 * 4)
    else:
        raise ValueError(f"unknown sonar text decoder arch {arch!r}")
    return dataclasses.replace(cfg, **overrides)


class B200TextDecoderModel(EngineModel):
    """SONAR text decoder (24 pre-LN layers + final LN + tied projection) on sm_90a kernels."""

    _abi = "decoder"
    _default_config = staticmethod(sonar_text_decoder_config)

    def __init__(self, config: SonarTextDecoderConfig, state_dict: Dict[str, Tensor],
                 device: Union[str, torch.device] = "cuda") -> None:
        super().__init__(device)
        if config.activation_fn != "ReLU" or config.layernorm_embedding or config.learned_pos \
                or config.no_token_positional_embeddings or not config.normalize_before:
            raise NotImplementedError("sonar_b200 text decoder supports the `basic`/`small` wiring only")
        if config.input_dim not in (None, config.model_dim):
            raise NotImplementedError("input_dim != model_dim is not supported by the CUDA decoder")
        self.config = config
        self.model_dim = config.model_dim
        self.target_vocab_info = config.vocab_info
        pad = config.vocab_info.pad_idx if config.vocab_info.pad_idx is not None else 1
        # SinusoidalPositionEncoder(max_seq_len, _legacy_pad_idx=pad) as built at factory.py:248-252
        self.max_target_seq_len = config.max_seq_len
        self.decoder_frontend = _FrontendInfo(config.max_seq_len, config.model_dim)
        sd, d, L = state_dict, config.model_dim, config.num_decoder_layers
        bf, f32 = self._bf16, self._f32

        embed = sd["decoder_frontend.embed.weight"]
        if "final_proj.weight" in sd and sd["final_proj.weight"].data_ptr() != embed.data_ptr() \
                and not torch.equal(sd["final_proj.weight"], embed):
            raise ValueError("final_proj.weight must be tied to decoder_frontend.embed.weight (factory.py:306-307)")
        top = {"embed": bf(embed), "pos_table": f32(sinusoidal_position_table(config.max_seq_len, d, pad)),
               "final_ln_g": f32(sd["decoder.layer_norm.weight"]), "final_ln_b": f32(sd["decoder.layer_norm.bias"])}
        layers = []
        for i in range(L):
            p = f"decoder.layers.{i}."
            a, c = p + "self_attn.", p + "encoder_decoder_attn."
            layers.append({
                "wqkv": bf(torch.cat([sd[a + "q_proj.weight"], sd[a + "k_proj.weight"], sd[a + "v_proj.weight"]], 0)),
                "bqkv": f32(torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]], 0)),
                "wo": bf(sd[a + "output_proj.weight"]), "bo": f32(sd[a + "output_proj.bias"]),
                "cross_wv": bf(sd[c + "v_proj.weight"]), "cross_bv": f32(sd[c + "v_proj.bias"]),
                "cross_wo": bf(sd[c + "output_proj.weight"]), "cross_bo": f32(sd[c + "output_proj.bias"]),
                "w1": bf(sd[p + "ffn.inner_proj.weight"]), "b1": f32(sd[p + "ffn.inner_proj.bias"]),
                "w2": bf(sd[p + "ffn.output_proj.weight"]), "b2": f32(sd[p + "ffn.output_proj.bias"]),
                "ln1_g": f32(sd[p + "self_attn_layer_norm.weight"]), "ln1_b": f32(sd[p + "self_attn_layer_norm.bias"]),
                "ln3_g": f32(sd[p + "ffn_layer_norm.weight"]), "ln3_b": f32(sd[p + "ffn_layer_norm.bias"]),
            })
        cfg_c = _lib.SbDecoderConfig(
            model_dim=d, num_layers=L, num_heads=config.num_decoder_attn_heads, ffn_inner_dim=config.ffn_inner_dim,
            input_dim=config.input_dim or d, vocab_size=config.vocab_info.size, pos_rows=config.max_seq_len,
            eos_idx=config.vocab_info.eos_idx, ln_eps=1e-5,
            embed_scale=1.0 if config.no_scale_embedding else math.sqrt(d))
        w_c = _lib.SbDecoderWeights(layers=self._layer_array(_lib.SbDecoderLayerWeights, layers),
                                    **{k: v.data_ptr() for k, v in top.items()})
        self._create(cfg_c, w_c)
        self._shape: Optional[Tuple[int, int, int]] = None

    @torch.inference_mode()
    def begin(self, embeddings: Tensor, beam: int, max_len: int) -> None:
        """Start decoding a batch of sentence embeddings [N, model_dim] with `beam` hypotheses each and at most
        `max_len` positions (prompt included)."""
        emb = self._on_device(embeddings, torch.float32).contiguous()
        if emb.dim() == 3 and emb.shape[1] == 1:
            emb = emb[:, 0].contiguous()
        n = emb.shape[0]
        if emb.dim() != 2 or emb.shape[1] != self.model_dim:
            raise ValueError(f"expected embeddings of shape [N, {self.model_dim}]")
        if max_len > self.max_target_seq_len:
            raise ValueError(f"max_len {max_len} exceeds the decoder's max_seq_len {self.max_target_seq_len}")
        ws = self._ensure_workspace(n, beam, max_len)
        self._shape = (n, beam, max_len)
        with torch.cuda.device(self.device):
            rc = self._lib.sb_decoder_begin(self._handle, emb.data_ptr(), n, beam, max_len, ws.data_ptr(), ws.numel(),
                                            self._stream())
        _lib.check(rc, "sb_decoder_begin")

    @torch.inference_mode()
    def step(self, tokens: Tensor, table: Tensor, t: int, probe: Optional[Tensor] = None):
        """tokens int64 [R] at position t, ancestry table int32 [R, max_len] ->
        (top-16 log-probs [R,16], their token ids int32 [R,16], log P(eos) [R]) and, when ``probe`` (int64 [R]) is given,
        a fourth tensor log P(probe[r]) [R]."""
        n, beam, max_len = self._shape
        r = n * beam
        assert tokens.shape == (r,) and tokens.dtype == torch.int64 and tokens.is_cuda and tokens.is_contiguous()
        assert table.shape == (r, max_len) and table.dtype == torch.int32 and table.is_contiguous()
        lp = torch.empty((r, TOPK), dtype=torch.float32, device=self.device)
        tok = torch.empty((r, TOPK), dtype=torch.int32, device=self.device)
        eos = torch.empty((r,), dtype=torch.float32, device=self.device)
        probe_lp = None
        if probe is not None:
            assert probe.shape == (r,) and probe.dtype == torch.int64 and probe.is_cuda and probe.is_contiguous()
            probe_lp = torch.empty((r,), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            rc = self._lib.sb_decoder_step(self._handle, tokens.data_ptr(), table.data_ptr(), t, n, beam, max_len,
                                           lp.data_ptr(), tok.data_ptr(), eos.data_ptr(),
                                           probe.data_ptr() if probe is not None else None,
                                           probe_lp.data_ptr() if probe_lp is not None else None,
                                           self._workspace.data_ptr(), self._workspace.numel(), self._stream())
        _lib.check(rc, "sb_decoder_step")
        return (lp, tok, eos) if probe is None else (lp, tok, eos, probe_lp)

    def check_inputs(self) -> None:
        """Raise ``ValueError`` if a step since the last check was fed a token id outside the vocabulary."""
        _lib.check(self._lib.sb_decoder_check_inputs(self._handle, self._stream()), "sb_decoder_check_inputs")
