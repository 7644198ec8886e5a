"""CPU oracle of the SONAR text encoder with attention pooling.  TEST INFRASTRUCTURE ONLY.

``pooling="attention"`` (``sonar/models/sonar_text/model.py:69-84``): the final-LayerNormed token states go through
``AttentionEncoderOutputPooler`` (``sonar/nn/encoder_pooler.py:47-89``) built by
``SonarTextEncoderFactory.create_attention_pooler`` (``sonar/models/sonar_text/factory.py:155-226``): one query, token
``bos_idx = 0`` of a one-row embedding of width E = ``embedding_dim or model_dim``, through ``num_decoder_layers``
POST-LN decoder layers whose encoder-decoder attention has key / value width ``model_dim``, then ``projection_out``
(E -> E, with bias).  State-dict names: ``pooler.decoder_frontend.embed.weight``, ``pooler.decoder.layers.{i}.*``,
``pooler.projection_out.*``.

The pooler itself is the speech oracle's (``OracleSpeechEncoder.pooler_query`` / ``pooler_layers``, pinned against
HuggingFace ``BartDecoderLayer`` through ``tests/golden/pooler_layers_small.pt``), run at width E; its key / value
projections are plain ``F.linear`` calls, so a key width D != E needs nothing else.  The encoder before it is
``OracleTextEncoder``.  Parity unpinned offline [fs2]: the zero-position sinusoid of the query, the sqrt(E) scaling of
the BOS row, and a POST stack with no final LayerNorm.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from .speech_encoder import OracleSpeechConfig, OracleSpeechEncoder
from .text_encoder import OracleEncoderConfig, OracleTextEncoder, make_synthetic_state_dict


@dataclass
class OracleAttentionEncoderConfig(OracleEncoderConfig):
    """``OracleEncoderConfig`` plus the pooler fields the reference factory reads (``factory.py:182-219``)."""

    embedding_dim: Optional[int] = None  # E; None = model_dim
    pooler_layers: int = 24  # num_decoder_layers
    pooler_heads: int = 16  # num_decoder_attn_heads
    pooler_ffn_inner_dim: Optional[int] = None  # decoder_ffn_inner_dim; None = ffn_inner_dim

    @property
    def out_dim(self) -> int:
        return self.embedding_dim or self.model_dim


def make_synthetic_pooler_state_dict(cfg: OracleAttentionEncoderConfig, seed: int,
                                     weight_std: float = 0.02) -> Dict[str, Tensor]:
    """Seeded ``pooler.*`` weights (distributions as ``make_synthetic_state_dict``), from their own generator."""
    g = torch.Generator().manual_seed(seed)
    d, e = cfg.model_dim, cfg.out_dim
    fp = cfg.pooler_ffn_inner_dim or cfg.ffn_inner_dim

    def rn(*shape, std=weight_std):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    sd: Dict[str, Tensor] = {"pooler.decoder_frontend.embed.weight": rn(1, e, std=e ** -0.5)}
    for i in range(cfg.pooler_layers):
        p = f"pooler.decoder.layers.{i}."
        for a, kv in (("self_attn", e), ("encoder_decoder_attn", d)):
            for name, cols in (("q_proj", e), ("k_proj", kv), ("v_proj", kv), ("output_proj", e)):
                sd[p + f"{a}.{name}.weight"] = rn(e, cols)
                sd[p + f"{a}.{name}.bias"] = rn(e)
            sd[p + f"{a}_layer_norm.weight"] = 1.0 + rn(e)
            sd[p + f"{a}_layer_norm.bias"] = rn(e)
        sd[p + "ffn.inner_proj.weight"] = rn(fp, e)
        sd[p + "ffn.inner_proj.bias"] = rn(fp)
        sd[p + "ffn.output_proj.weight"] = rn(e, fp)
        sd[p + "ffn.output_proj.bias"] = rn(e)
        sd[p + "ffn_layer_norm.weight"] = 1.0 + rn(e)
        sd[p + "ffn_layer_norm.bias"] = rn(e)
    sd["pooler.projection_out.weight"] = rn(e, e, std=e ** -0.5)
    sd["pooler.projection_out.bias"] = rn(e)
    return sd


def make_synthetic_attention_state_dict(cfg: OracleAttentionEncoderConfig, seed: int = 1, weight_std: float = 0.02,
                                        pooler_std: Optional[float] = None) -> Dict[str, Tensor]:
    """``make_synthetic_state_dict(cfg, seed)`` (the encoder weights are exactly those of the same seed without a
    pooler) plus the pooler's weights drawn from a second generator (seed + 1000), with std ``pooler_std`` if given."""
    sd = make_synthetic_state_dict(cfg, seed=seed, weight_std=weight_std)
    sd.update(make_synthetic_pooler_state_dict(cfg, seed + 1000, weight_std if pooler_std is None else pooler_std))
    return sd


class OracleAttentionTextEncoder:
    """``SonarTextTransformerEncoderModel.forward`` with ``Pooling.ATTENTION``, in fp32 or fp64."""

    def __init__(self, cfg: OracleAttentionEncoderConfig, state_dict: Dict[str, Tensor],
                 dtype: torch.dtype = torch.float32) -> None:
        self.cfg = cfg
        self.encoder = OracleTextEncoder(cfg, state_dict, dtype)
        # the speech oracle's pooler at width E, on the text weights under its parameter names
        self._pooler = OracleSpeechEncoder(
            OracleSpeechConfig(model_dim=cfg.out_dim, num_layers=0, pooler_layers=cfg.pooler_layers,
                               pooler_heads=cfg.pooler_heads, bos_idx=0, ln_eps=cfg.ln_eps), {})
        self._pooler.sd = {"encoder_" + k: v.to(dtype) for k, v in state_dict.items() if k.startswith("pooler.")}

    def pooler_layers(self, x: Tensor, enc: Tensor, key_ok: Optional[Tensor]) -> Tensor:
        """The POST-LN decoder layers: x [B, 1, E] over enc [B, S, model_dim] (``key_ok`` [B, S] or None)."""
        return self._pooler.pooler_layers(x, enc, key_ok)

    def pooler(self, enc: Tensor, key_ok: Optional[Tensor]) -> Tensor:
        """``AttentionEncoderOutputPooler.__call__`` (``encoder_pooler.py:70-83``) -> [B, E]."""
        sd = self._pooler.sd
        x = self.pooler_layers(self._pooler.pooler_query(enc.shape[0]), enc, key_ok)
        return F.linear(x, sd["encoder_pooler.projection_out.weight"], sd["encoder_pooler.projection_out.bias"]).squeeze(1)

    @torch.no_grad()
    def forward(self, ids: Tensor, seq_lens: Optional[Tensor]):
        """ids int64 [B,S] right-padded; seq_lens int64 [B] or None.  -> (sentence_embeddings [B,E], encoded_seqs
        [B,S,D] after the final LayerNorm)."""
        _, x = self.encoder(ids, seq_lens)
        key_ok = None if seq_lens is None else torch.arange(ids.shape[1])[None, :] < seq_lens[:, None]
        return self.pooler(x, key_ok), x

    __call__ = forward
