"""CPU oracle for the SONAR speech encoder (BASELINE.json config 3; SURVEY §8 rows a11-a12, App. B.2/B.3).
TEST INFRASTRUCTURE ONLY.

Restates ``SonarSpeechEncoderModel.forward`` (``sonar/models/sonar_speech/model.py:59-77``):
w2v-BERT frontend (stack 2 fbank frames -> LayerNorm(160) -> Linear 160->1024) -> 24 Conformer blocks
(macaron half-step SiLU FFNs, Transformer-XL relative-position self-attention with ``u_bias/v_bias/r_proj``,
convolution module with GLU / depthwise k=31 / BatchNorm / SiLU, final LayerNorm per block) -> ``model.layer_norm``
(the re-homed stack LayerNorm, ``sonar_speech/handler.py:102-108``) -> ``AttentionEncoderOutputPooler``
(``sonar/nn/encoder_pooler.py:47-89``): one BOS query through 3 (english) / 6 POST-LN decoder layers cross-attending
the encoder output, then a bias-free 1024->1024 projection (``sonar_speech/factory.py:73-152``,
``config.py:61-95``).  State-dict names: ``sonar_speech/handler.py:63-100``.

The Conformer internals live in fairseq2's w2v-BERT ``600m`` config, which is not on disk (SURVEY F7): the block is
restated from the identical-by-parameter-name HuggingFace ``SeamlessM4TConformerEncoderLayer`` and PINNED against it
through ``tests/golden/conformer_layer_small.pt`` (``tests/golden/make_conformer_golden.py``); the whole stack before the
pooler (2-frame stacking, LayerNorm + projection frontend, block composition, final LayerNorm) is PINNED against HuggingFace's
feature projection + ``SeamlessM4TConformerEncoder`` (``tests/golden/conformer_encoder_small.pt``).  The pooler's POST-LN
decoder-layer stack is PINNED against HuggingFace ``BartDecoderLayer`` (``tests/golden/pooler_layers_small.pt``,
``make_pooler_golden.py``); the fbank features are pinned against torchaudio on the reference's own audio clips
(``tests/test_reference_audio.py``).  What stays unpinned offline: the w2v-BERT ``600m`` hyper-parameters (SURVEY F7), the
pooler's one-token input (the reference's golden ``speech_embedding.pt`` needs the downloaded
checkpoint; ``tests/test_reference_audio.py`` runs it when ``SONAR_B200_CHECKPOINT_DIR`` is set).
"""

from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor


@dataclass
class OracleSpeechConfig:
    model_dim: int = 1024
    feature_dim: int = 160          # 2 stacked 80-bin frames
    num_layers: int = 24
    num_heads: int = 16
    ffn_inner_dim: int = 4096
    conv_kernel: int = 31
    pooler_layers: int = 3          # `english`; 6 for `non_english` (config.py:72,89)
    pooler_heads: int = 16
    pooler_ffn_inner_dim: int = 4096
    pooler_vocab: int = 1024        # Embedding(num_embeddings=w2v2 model_dim) (factory.py:102-108)
    bos_idx: int = 2
    ln_eps: float = 1e-5
    bn_eps: float = 1e-5


def rel_pos_table(seq_len: int, dim: int) -> Tensor:
    """[2S-1, dim]; row k encodes relative position (S-1-k); interleaved sin/cos (HF RelPositionalEmbedding)."""
    pos = torch.arange(seq_len, dtype=torch.float32)[:, None]
    div = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    p = torch.zeros(seq_len, dim)
    n = torch.zeros(seq_len, dim)
    p[:, 0::2], p[:, 1::2] = torch.sin(pos * div), torch.cos(pos * div)
    n[:, 0::2], n[:, 1::2] = torch.sin(-pos * div), torch.cos(-pos * div)
    return torch.cat([torch.flip(p, [0]), n[1:]], dim=0)


def relpos_attention(q: Tensor, k: Tensor, v: Tensor, r: Tensor, u_bias: Tensor, v_bias: Tensor, key_ok: Tensor) -> Tensor:
    """The Transformer-XL relative-position attention core of a Conformer block: q, k, v [B, S, H, hd]; r [2S-1, H, hd] =
    r_proj(rel_pos_table(S)), row c <-> relative position S-1-c; u_bias, v_bias [H, hd]; key_ok [B, S] -> [B, S, H*hd] =
    softmax_j(((q_i+u).k_j + (q_i+v).r[S-1-i+j]) / sqrt(hd), keys with key_ok False excluded) . v."""
    b, s, H, hd = q.shape
    k, v = k.transpose(1, 2), v.transpose(1, 2)  # [B,H,S,hd]
    qu = (q + u_bias).transpose(1, 2)
    qv = (q + v_bias).transpose(1, 2)
    ac = qu @ k.transpose(-2, -1)
    bd_full = qv @ r.permute(1, 2, 0)  # [B,H,S,2S-1]; column c <-> relative position S-1-c
    idx = (s - 1) - torch.arange(s)[:, None] + torch.arange(s)[None, :]  # column for (i,j): relpos i-j
    bd = torch.gather(bd_full, 3, idx[None, None].expand(b, H, s, s))
    scores = (ac + bd) / math.sqrt(hd)
    scores = scores.masked_fill(~key_ok[:, None, None, :], -torch.inf)
    return (torch.softmax(scores, dim=-1) @ v).transpose(1, 2).reshape(b, s, H * hd)


def conv_module_middle(y: Tensor, dw: Tensor, bn_mean: Tensor, bn_var: Tensor, bn_weight: Tensor, bn_bias: Tensor,
                       bn_eps: float) -> Tensor:
    """The convolution module between its pointwise convolutions: y [B, 2D, S] (pointwise_conv1 output, zero at padded
    positions) -> GLU -> depthwise conv (dw [D, 1, k], zero padding k//2) -> BatchNorm (running statistics) -> SiLU
    -> [B, D, S]."""
    y = F.glu(y, dim=1)
    y = F.conv1d(y, dw, padding=dw.shape[-1] // 2, groups=y.shape[1])
    y = F.batch_norm(y, bn_mean, bn_var, bn_weight, bn_bias, False, 0.0, bn_eps)
    return F.silu(y)


def make_synthetic_speech_state_dict(cfg: OracleSpeechConfig, seed: int = 3, std: float = 0.02) -> Dict[str, Tensor]:
    g = torch.Generator().manual_seed(seed)
    d, f, H = cfg.model_dim, cfg.ffn_inner_dim, cfg.num_heads

    def rn(*shape, s=std):
        return torch.randn(*shape, generator=g) * s

    def ln(prefix):
        sd[prefix + ".weight"] = 1.0 + rn(d)
        sd[prefix + ".bias"] = rn(d)

    sd: Dict[str, Tensor] = {}
    sd["encoder_frontend.post_extract_layer_norm.weight"] = 1.0 + rn(cfg.feature_dim)
    sd["encoder_frontend.post_extract_layer_norm.bias"] = rn(cfg.feature_dim)
    sd["encoder_frontend.model_dim_proj.weight"] = rn(d, cfg.feature_dim, s=cfg.feature_dim ** -0.5)
    sd["encoder_frontend.model_dim_proj.bias"] = rn(d)
    for i in range(cfg.num_layers):
        p = f"encoder.layers.{i}."
        for k in ("ffn1", "ffn2"):
            ln(p + f"{k}_layer_norm")
            sd[p + f"{k}.inner_proj.weight"], sd[p + f"{k}.inner_proj.bias"] = rn(f, d), rn(f)
            sd[p + f"{k}.output_proj.weight"], sd[p + f"{k}.output_proj.bias"] = rn(d, f), rn(d)
        ln(p + "self_attn_layer_norm")
        for n in ("q_proj", "k_proj", "v_proj", "output_proj"):
            sd[p + f"self_attn.{n}.weight"], sd[p + f"self_attn.{n}.bias"] = rn(d, d), rn(d)
        sd[p + "self_attn.sdpa.r_proj.weight"] = rn(d, d)
        sd[p + "self_attn.sdpa.u_bias"] = rn(H, d // H, s=0.1)
        sd[p + "self_attn.sdpa.v_bias"] = rn(H, d // H, s=0.1)
        ln(p + "conv_layer_norm")
        sd[p + "conv.pointwise_conv1.weight"] = rn(2 * d, d, 1)
        sd[p + "conv.depthwise_conv.weight"] = rn(d, 1, cfg.conv_kernel, s=0.2)
        sd[p + "conv.batch_norm.weight"] = 1.0 + rn(d)
        sd[p + "conv.batch_norm.bias"] = rn(d)
        sd[p + "conv.batch_norm.running_mean"] = rn(d)
        sd[p + "conv.batch_norm.running_var"] = 1.0 + rn(d).abs()
        sd[p + "conv.pointwise_conv2.weight"] = rn(d, d, 1)
        ln(p + "layer_norm")
    ln("layer_norm")
    sd["encoder_pooler.decoder_frontend.embed.weight"] = rn(cfg.pooler_vocab, d, s=d ** -0.5)
    fp = cfg.pooler_ffn_inner_dim
    for i in range(cfg.pooler_layers):
        p = f"encoder_pooler.decoder.layers.{i}."
        for a in ("self_attn", "encoder_decoder_attn"):
            for n in ("q_proj", "k_proj", "v_proj", "output_proj"):
                sd[p + f"{a}.{n}.weight"], sd[p + f"{a}.{n}.bias"] = rn(d, d), rn(d)
            ln(p + f"{a}_layer_norm")
        sd[p + "ffn.inner_proj.weight"], sd[p + "ffn.inner_proj.bias"] = rn(fp, d), rn(fp)
        sd[p + "ffn.output_proj.weight"], sd[p + "ffn.output_proj.bias"] = rn(d, fp), rn(d)
        ln(p + "ffn_layer_norm")
    sd["encoder_pooler.projection_out.weight"] = rn(d, d, s=d ** -0.5)
    return sd


class OracleSpeechEncoder:
    def __init__(self, cfg: OracleSpeechConfig, state_dict: Dict[str, Tensor]):
        self.cfg = cfg
        self.sd = {k: v.float() for k, v in state_dict.items()}

    # ------------------------------------------------------------------ conformer block (padded [B,S,D] + key mask)
    def conformer_block(self, i: int, x: Tensor, key_ok: Tensor) -> Tensor:
        cfg, sd = self.cfg, self.sd
        p = f"encoder.layers.{i}."
        d, H = cfg.model_dim, cfg.num_heads
        hd = d // H
        b, s, _ = x.shape

        def lnorm(t, name):
            return F.layer_norm(t, (d,), sd[p + name + ".weight"], sd[p + name + ".bias"], cfg.ln_eps)

        def ffn(t, name):
            t = F.silu(F.linear(t, sd[p + name + ".inner_proj.weight"], sd[p + name + ".inner_proj.bias"]))
            return F.linear(t, sd[p + name + ".output_proj.weight"], sd[p + name + ".output_proj.bias"])

        x = x + 0.5 * ffn(lnorm(x, "ffn1_layer_norm"), "ffn1")
        # --- relative-position self-attention ---
        y = lnorm(x, "self_attn_layer_norm")
        a = p + "self_attn."
        q = F.linear(y, sd[a + "q_proj.weight"], sd[a + "q_proj.bias"]).view(b, s, H, hd)
        k = F.linear(y, sd[a + "k_proj.weight"], sd[a + "k_proj.bias"]).view(b, s, H, hd)
        v = F.linear(y, sd[a + "v_proj.weight"], sd[a + "v_proj.bias"]).view(b, s, H, hd)
        r = F.linear(rel_pos_table(s, d), sd[a + "sdpa.r_proj.weight"]).view(2 * s - 1, H, hd)  # [2S-1,H,hd]
        o = relpos_attention(q, k, v, r, sd[a + "sdpa.u_bias"], sd[a + "sdpa.v_bias"], key_ok)
        x = x + F.linear(o, sd[a + "output_proj.weight"], sd[a + "output_proj.bias"])
        # --- convolution module ---
        y = lnorm(x, "conv_layer_norm")
        y = y.masked_fill(~key_ok[:, :, None], 0.0).transpose(1, 2)  # [B,D,S]
        bn = p + "conv.batch_norm."
        y = conv_module_middle(F.conv1d(y, sd[p + "conv.pointwise_conv1.weight"]), sd[p + "conv.depthwise_conv.weight"],
                               sd[bn + "running_mean"], sd[bn + "running_var"], sd[bn + "weight"], sd[bn + "bias"], cfg.bn_eps)
        y = F.conv1d(y, sd[p + "conv.pointwise_conv2.weight"]).transpose(1, 2)
        x = x + y
        x = x + 0.5 * ffn(lnorm(x, "ffn2_layer_norm"), "ffn2")
        return lnorm(x, "layer_norm")

    def pooler_query(self, batch: int) -> Tensor:
        """The pooler's single decoder input: TransformerEmbeddingFrontend(embed, SinusoidalPositionEncoder) of the BOS
        token = E[bos]*sqrt(d) + pos[0], pos[0] = [sin(0)... | cos(0)...] = [0.. | 1..]  [fs2]  (``encoder_pooler.py:70-76``)."""
        cfg, sd = self.cfg, self.sd
        d = cfg.model_dim
        pos0 = torch.cat([torch.zeros(d // 2), torch.ones(d // 2)])
        return (sd["encoder_pooler.decoder_frontend.embed.weight"][cfg.bos_idx] * math.sqrt(d) + pos0)[None, None].expand(batch, 1, d)

    def pooler_layers(self, x: Tensor, enc: Tensor, key_ok: Tensor) -> Tensor:
        """The POST-LN decoder-layer stack of the pooler (``sonar_speech/factory.py:110-137``): self-attention, encoder-decoder
        attention with a key-padding mask, ReLU FFN, each followed by residual + LayerNorm.  PINNED against HuggingFace
        ``BartDecoderLayer`` (post-LN, same sub-layer order) through ``tests/golden/pooler_layers_small.pt``."""
        cfg, sd = self.cfg, self.sd
        d, H = cfg.model_dim, cfg.pooler_heads
        hd = d // H
        b = enc.shape[0]

        def mha(pfx, q_in, kv_in, mask):
            q = F.linear(q_in, sd[pfx + "q_proj.weight"], sd[pfx + "q_proj.bias"]).view(b, -1, H, hd).transpose(1, 2)
            k = F.linear(kv_in, sd[pfx + "k_proj.weight"], sd[pfx + "k_proj.bias"]).view(b, -1, H, hd).transpose(1, 2)
            v = F.linear(kv_in, sd[pfx + "v_proj.weight"], sd[pfx + "v_proj.bias"]).view(b, -1, H, hd).transpose(1, 2)
            sc = q @ k.transpose(-2, -1) / math.sqrt(hd)
            if mask is not None:
                sc = sc.masked_fill(~mask[:, None, None, :], -torch.inf)
            o = (torch.softmax(sc, -1) @ v).transpose(1, 2).reshape(b, -1, d)
            return F.linear(o, sd[pfx + "output_proj.weight"], sd[pfx + "output_proj.bias"])

        for i in range(cfg.pooler_layers):
            p = f"encoder_pooler.decoder.layers.{i}."

            def lnorm(t, name):
                return F.layer_norm(t, (d,), sd[p + name + ".weight"], sd[p + name + ".bias"], cfg.ln_eps)

            x = lnorm(x + mha(p + "self_attn.", x, x, None), "self_attn_layer_norm")
            x = lnorm(x + mha(p + "encoder_decoder_attn.", x, enc, key_ok), "encoder_decoder_attn_layer_norm")
            f = F.linear(F.relu(F.linear(x, sd[p + "ffn.inner_proj.weight"], sd[p + "ffn.inner_proj.bias"])),
                         sd[p + "ffn.output_proj.weight"], sd[p + "ffn.output_proj.bias"])
            x = lnorm(x + f, "ffn_layer_norm")
        return x

    # ------------------------------------------------------------------ attention pooler
    def pooler(self, enc: Tensor, key_ok: Tensor) -> Tensor:
        x = self.pooler_layers(self.pooler_query(enc.shape[0]), enc, key_ok)
        return F.linear(x, self.sd["encoder_pooler.projection_out.weight"]).squeeze(1)  # bias-free (factory.py:146-152)

    @torch.no_grad()
    def encode(self, fbank: Tensor, frame_lens: List[int]) -> Tuple[Tensor, Tensor, List[int]]:
        """Everything before the pooler: fbank [B, T, 80] zero-padded, T even -> (encoder output [B, T/2, D] after
        model.layer_norm, key mask [B, T/2], positions per utterance).  Pinned against HuggingFace's SeamlessM4T Conformer
        encoder (tests/golden/conformer_encoder_small.pt)."""
        cfg, sd = self.cfg, self.sd
        b, t, nm = fbank.shape
        x = fbank.float().reshape(b, t // 2, nm * 2)  # stack 2 frames; seq_len // 2 (App. B.2)
        lens = [n // 2 for n in frame_lens]
        s = t // 2
        key_ok = torch.arange(s)[None, :] < torch.tensor(lens)[:, None]
        x = F.layer_norm(x, (cfg.feature_dim,), sd["encoder_frontend.post_extract_layer_norm.weight"],
                         sd["encoder_frontend.post_extract_layer_norm.bias"], cfg.ln_eps)
        x = F.linear(x, sd["encoder_frontend.model_dim_proj.weight"], sd["encoder_frontend.model_dim_proj.bias"])
        for i in range(cfg.num_layers):
            x = self.conformer_block(i, x, key_ok)
        x = F.layer_norm(x, (cfg.model_dim,), sd["layer_norm.weight"], sd["layer_norm.bias"], cfg.ln_eps)
        return x, key_ok, lens

    @torch.no_grad()
    def forward(self, fbank: Tensor, frame_lens: List[int]) -> Tuple[Tensor, Tensor, List[int]]:
        """fbank [B, T, 80] zero-padded, T even; frame_lens = true frame counts.
        -> (sentence_embeddings [B, D], encoder_output [B, T/2, D] after model.layer_norm, positions per utterance)."""
        x, key_ok, lens = self.encode(fbank, frame_lens)
        return self.pooler(x, key_ok), x, lens

    __call__ = forward
