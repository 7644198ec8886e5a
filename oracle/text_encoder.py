"""CPU oracle for the SONAR text-embedding hot path.  TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import this module.  Nothing under ``sonar_b200/``
may import, call or fall back to it.

What it restates (reference = /root/reference, fairseq2 0.4.x is un-vendored):

* forward + pooling ........ ``sonar/models/sonar_text/model.py:86-143``
* graph wiring / flags ..... ``sonar/models/sonar_text/factory.py:53-153``
* hyper-parameters ......... ``sonar/models/sonar_text/config.py:92-116``
* state-dict key names ..... ``sonar/models/sonar_text/handler.py:71-92``
* the fairseq2 op sequence (``F.embedding``·sqrt(d) + sinusoid(offset 2) →
  24×[LN → q/k/v ``F.linear`` → ``F.scaled_dot_product_attention`` with a
  key-padding mask → out ``F.linear`` + residual; LN → linear → ReLU → linear +
  residual] → LN → masked mean) as written out in SURVEY.md Appendix A.2.

Parity pinning status: the reference's own numeric goldens for this path
(``tests/integration_tests/test_text_sonar.py:46-53``) need the downloaded
checkpoint + SentencePiece model, which do not exist offline, and fairseq2
cannot be imported here, so against the *reference itself* this oracle is
"parity unpinned".  It IS pinned (a) by the reference's pooling known-answer
tests (``tests/unit_tests/test_sonar_pooling.py:16-68``, restated in
``tests/test_oracle.py``) and (b) against an independent implementation
of the same network, HuggingFace ``M2M100Encoder`` -- the port the reference's
own notebook uses as *the* SONAR text encoder
(``examples/finetune_sonar_as_toxicity_classifier.ipynb`` cells 0/50/53) -- via
the committed fixture ``tests/golden/m2m100_small.pt`` produced by
``tests/golden/make_m2m100_golden.py``.
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor


@dataclass
class OracleEncoderConfig:
    """Mirror of the fields of ``SonarTextEncoderConfig`` that reach the math
    (``sonar/models/sonar_text/config.py:14-84``); defaults = arch ``basic``
    (``config.py:92-116``)."""

    model_dim: int = 1024
    vocab_size: int = 256206
    max_seq_len: int = 512  # fairseq value; +pad_idx+1 below (factory.py:56-59)
    pad_idx: int = 1  # model-config pad idx: only sets the sinusoid offset
    num_layers: int = 24
    num_heads: int = 16
    ffn_inner_dim: int = 8192
    ln_eps: float = 1e-5

    @property
    def pos_table_len(self) -> int:
        # `_from_fairseq=True` => max_seq_len += pad_idx + 1 (factory.py:53-59)
        return self.max_seq_len + self.pad_idx + 1


def sinusoidal_table(num_pos: int, dim: int, legacy_pad_idx: int = 1) -> Tensor:
    """fairseq2 ``SinusoidalPositionEncoder`` with ``_legacy_pad_idx`` [fs2]
    (built at ``factory.py:88-92``): row ``t`` holds the encoding of position
    index ``t + legacy_pad_idx + 1``; layout ``[sin | cos]`` halves with
    ``exp(-j * ln(1e4) / (half - 1))`` (SURVEY App. A.2 / F3; identical to HF
    ``M2M100SinusoidalPositionalEmbedding.get_embedding``)."""
    half = dim // 2
    start = legacy_pad_idx + 1
    steps = torch.arange(start, start + num_pos, dtype=torch.float32)
    freq = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000.0) / (half - 1)))
    ang = steps[:, None] * freq[None, :]
    return torch.cat([torch.sin(ang), torch.cos(ang)], dim=1)


def make_synthetic_state_dict(cfg: OracleEncoderConfig, seed: int = 1,
                              weight_std: float = 0.02) -> Dict[str, Tensor]:
    """Seeded synthetic weights under the fairseq2 state-dict names of
    SURVEY App. A.3 (``handler.py:71-92``); distributions per SURVEY §8(d):
    matrices/biases N(0, std²), LN γ = 1 + N(0, std²), β = N(0, std²),
    embedding N(0, 1/model_dim) (= ``init_scaled_embedding``, factory.py:77)."""
    g = torch.Generator().manual_seed(seed)
    d, f = cfg.model_dim, cfg.ffn_inner_dim

    def rn(*shape, std=weight_std):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    sd: Dict[str, Tensor] = {}
    sd["encoder_frontend.embed.weight"] = rn(cfg.vocab_size, d, std=d ** -0.5)
    for i in range(cfg.num_layers):
        p = f"encoder.layers.{i}."
        for name in ("q_proj", "k_proj", "v_proj", "output_proj"):
            sd[p + f"self_attn.{name}.weight"] = rn(d, d)
            sd[p + f"self_attn.{name}.bias"] = rn(d)
        sd[p + "self_attn_layer_norm.weight"] = 1.0 + rn(d)
        sd[p + "self_attn_layer_norm.bias"] = rn(d)
        sd[p + "ffn.inner_proj.weight"] = rn(f, d)
        sd[p + "ffn.inner_proj.bias"] = rn(f)
        sd[p + "ffn.output_proj.weight"] = rn(d, f)
        sd[p + "ffn.output_proj.bias"] = rn(d)
        sd[p + "ffn_layer_norm.weight"] = 1.0 + rn(d)
        sd[p + "ffn_layer_norm.bias"] = rn(d)
    sd["layer_norm.weight"] = 1.0 + rn(d)
    sd["layer_norm.bias"] = rn(d)
    return sd


def static_pooling(seqs: Tensor, seq_lens: Optional[Tensor], pooling: str) -> Tensor:
    """``SonarTextTransformerEncoderModel.static_pooling``
    (``sonar/models/sonar_text/model.py:86-128``).  ``seq_lens=None`` is the
    reference's ``padding_mask is None`` case.  ``seqs`` is [N,S,M,...]."""
    n, s = seqs.shape[0], seqs.shape[1]
    if seq_lens is not None:
        valid = torch.arange(s)[None, :] < seq_lens[:, None]  # [N,S]
        valid = valid.reshape(n, s, *([1] * (seqs.dim() - 2)))
    pooling = pooling.lower()
    if pooling == "last":  # model.py:100-108
        if seq_lens is None:
            return seqs[:, -1]
        return seqs[torch.arange(n), (seq_lens - 1).clip(0)]
    if pooling == "max":  # model.py:109-111
        if seq_lens is not None:
            seqs = torch.where(valid, seqs, torch.full_like(seqs, -torch.inf))
        return seqs.max(dim=1).values
    if pooling == "mean":  # model.py:112-124
        if seq_lens is not None:
            seqs = torch.where(valid, seqs, torch.zeros_like(seqs))
        out = seqs.sum(dim=1)
        if seq_lens is None:
            return out * (1.0 / (s + 1e-7))
        w = 1.0 / (seq_lens.to(out.dtype) + 1e-7)
        return torch.einsum("i...,i->i...", out, w)
    raise NotImplementedError(pooling)


def self_attention(q: Tensor, k: Tensor, v: Tensor, key_ok: Optional[Tensor]) -> Tensor:
    """The encoder layer's attention core (``F.scaled_dot_product_attention`` with a key-padding mask, scale
    1/sqrt(head_dim)): q, k, v [B, H, S, head_dim], key_ok bool [B, S] (True = a real token) or None (no padding)."""
    attn_mask = None
    if key_ok is not None:
        b, s = key_ok.shape
        attn_mask = torch.zeros(b, 1, 1, s, dtype=q.dtype, device=q.device)
        attn_mask.masked_fill_(~key_ok[:, None, None, :], -torch.inf)
    return F.scaled_dot_product_attention(q, k, v, attn_mask=attn_mask)


class OracleTextEncoder:
    """fp32 (or fp64) CPU restatement of ``SonarTextTransformerEncoderModel.forward``
    (``model.py:130-143``) for the ``basic`` wiring (pre-LN layers, no LN inside the
    stack, model-level final LN, MEAN pooling)."""

    def __init__(self, cfg: OracleEncoderConfig, state_dict: Dict[str, Tensor],
                 dtype: torch.dtype = torch.float32) -> None:
        self.cfg = cfg
        self.dtype = dtype
        self.sd = {k: v.to(dtype) for k, v in state_dict.items()}
        self.pos = sinusoidal_table(cfg.pos_table_len, cfg.model_dim, cfg.pad_idx)  # fp32

    @torch.no_grad()
    def forward(self, ids: Tensor, seq_lens: Optional[Tensor], *, return_layers: bool = False):
        """ids int64 [B,S] right-padded; seq_lens int64 [B] or None (no padding).
        Returns (sentence_embeddings [B,D], encoded_seqs [B,S,D][, per-layer list])."""
        cfg, sd = self.cfg, self.sd
        b, s = ids.shape
        d, h = cfg.model_dim, cfg.num_heads
        hd = d // h
        # frontend (factory.py:73-100): embed * sqrt(d) + sinusoid, fp32 add then cast [fs2]
        x = F.embedding(ids, sd["encoder_frontend.embed.weight"]) * math.sqrt(d)
        x = (x.float() + self.pos[:s][None]).to(self.dtype)
        key_ok = None if seq_lens is None else torch.arange(s)[None, :] < seq_lens[:, None]  # [B,S]
        layers = []
        for i in range(cfg.num_layers):
            p = f"encoder.layers.{i}."
            r = x
            y = F.layer_norm(x, (d,), sd[p + "self_attn_layer_norm.weight"],
                             sd[p + "self_attn_layer_norm.bias"], cfg.ln_eps)
            q = F.linear(y, sd[p + "self_attn.q_proj.weight"], sd[p + "self_attn.q_proj.bias"])
            k = F.linear(y, sd[p + "self_attn.k_proj.weight"], sd[p + "self_attn.k_proj.bias"])
            v = F.linear(y, sd[p + "self_attn.v_proj.weight"], sd[p + "self_attn.v_proj.bias"])
            q = q.view(b, s, h, hd).transpose(1, 2)
            k = k.view(b, s, h, hd).transpose(1, 2)
            v = v.view(b, s, h, hd).transpose(1, 2)
            a = self_attention(q, k, v, key_ok)
            a = a.transpose(1, 2).reshape(b, s, d)
            x = r + F.linear(a, sd[p + "self_attn.output_proj.weight"],
                             sd[p + "self_attn.output_proj.bias"])
            r = x
            y = F.layer_norm(x, (d,), sd[p + "ffn_layer_norm.weight"],
                             sd[p + "ffn_layer_norm.bias"], cfg.ln_eps)
            y = F.relu(F.linear(y, sd[p + "ffn.inner_proj.weight"], sd[p + "ffn.inner_proj.bias"]))
            x = r + F.linear(y, sd[p + "ffn.output_proj.weight"], sd[p + "ffn.output_proj.bias"])
            if return_layers:
                layers.append(x.clone())
        x = F.layer_norm(x, (d,), sd["layer_norm.weight"], sd["layer_norm.bias"], cfg.ln_eps)
        emb = static_pooling(x, seq_lens, "mean")
        if return_layers:
            return emb, x, layers
        return emb, x

    __call__ = forward


def encoder_flops(seq_len: int, d: int = 1024, f: int = 8192, layers: int = 24) -> float:
    """Algorithmic FLOPs per sentence, SURVEY §8(d):
    F(S) = L·S·(2·(4d² + 2df) + 4·S·d)."""
    return layers * seq_len * (2.0 * (4 * d * d + 2 * d * f) + 4.0 * seq_len * d)
