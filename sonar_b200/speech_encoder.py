"""Host-side mirror of the reference speech encoder, backed by the CUDA engine.

``B200SpeechEncoderModel`` stands where ``SonarSpeechEncoderModel`` (``sonar/models/sonar_speech/model.py:20-77``) stands
in ``SpeechToEmbeddingModelPipeline`` (``sonar/inference_pipelines/speech.py:402-474``): ``model(SequenceBatch(fbank
[N,T,80], PaddingMask(frame lens))).sentence_embeddings``.  Weight repacking only (bf16, fused q|k|v, macaron 0.5
folded into the FFN output projections, BatchNorm folded to scale/shift, 160-wide frontend padded to 192); all
arithmetic is in ``sb_speech_encoder_forward`` (``csrc/conformer.cu``).
"""

from __future__ import annotations

import ctypes as C
import dataclasses
import math
from dataclasses import dataclass
from typing import Dict, Optional, Union

import torch
from torch import Tensor

from . import _lib
from ._engine import EngineModel
from .sequence import PaddingMask, SequenceBatch, SonarEncoderOutput


@dataclass
class SonarSpeechEncoderConfig:
    """The fields of ``SonarSpeechEncoderConfig`` + the w2v-BERT ``600m`` encoder config that reach the maths
    (``sonar/models/sonar_speech/config.py:20-95``; SURVEY App. B.2 / F7)."""

    model_dim: int = 1024
    num_encoder_layers: int = 24
    num_encoder_attn_heads: int = 16
    ffn_inner_dim: int = 4096          # Conformer FFN
    depthwise_conv_kernel_size: int = 31
    feature_dim: int = 160             # 80-bin fbank, stride 2
    max_seq_len: int = 1024            # pooler positions (unused by a 1-token query)
    pad_idx: Optional[int] = 1
    bos_idx: int = 2
    num_decoder_layers: int = 3        # `english`; `non_english` = 6
    num_decoder_attn_heads: int = 16
    decoder_ffn_inner_dim: int = 4096
    bn_eps: float = 1e-5


def sonar_speech_encoder_config(arch: str = "english", **overrides) -> SonarSpeechEncoderConfig:
    if arch == "english":
        cfg = SonarSpeechEncoderConfig()
    elif arch == "non_english":
        cfg = SonarSpeechEncoderConfig(num_decoder_layers=6)
    else:
        raise ValueError(f"unknown sonar speech encoder arch {arch!r}")
    return dataclasses.replace(cfg, **overrides)


def relpos_rows(max_len: int) -> int:
    """Rows of the relative-position table for a batch whose longest utterance has ``max_len`` positions: 2*max_len-1
    rounded up to a multiple of 256."""
    return ((2 * max_len - 1) + 255) // 256 * 256


def relative_position_table(max_len: int, dim: int, rows: int) -> Tensor:
    """fp32 [rows, dim]: row k (< 2*max_len-1) = sinusoid of relative position (max_len-1-k), interleaved sin/cos;
    remaining rows zero.  (fairseq2 ``RelativePositionalEncoding`` / Transformer-XL; SURVEY App. B.2.)"""
    pos = torch.arange(max_len, dtype=torch.float32)[:, None]
    div = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    p = torch.zeros(max_len, dim)
    n = torch.zeros(max_len, dim)
    p[:, 0::2], p[:, 1::2] = torch.sin(pos * div), torch.cos(pos * div)
    n[:, 0::2], n[:, 1::2] = torch.sin(-pos * div), torch.cos(-pos * div)
    out = torch.zeros(rows, dim)
    out[: 2 * max_len - 1] = torch.cat([torch.flip(p, [0]), n[1:]], dim=0)
    return out


class B200SpeechEncoderModel(EngineModel):
    _abi = "speech_encoder"
    _default_config = staticmethod(sonar_speech_encoder_config)

    def __init__(self, config: SonarSpeechEncoderConfig, state_dict: Dict[str, Tensor],
                 device: Union[str, torch.device] = "cuda", *, attn_impl: str = "mma_sync") -> None:
        """``attn_impl``: relative-position attention kernel -- "mma_sync" (default; the two have not been timed against each
        other on the H100) or "tcgen05" (the name the wgmma kernel keeps)
        (``csrc/attention_relpos_tc.cu``: band product, Q K^T and P V on the tensor cores (wgmma), bitwise independent of the
        batch an utterance is in; ``bench.py`` times both in its speech block)."""
        super().__init__(device)
        if attn_impl not in ("tcgen05", "mma_sync"):
            raise ValueError("attn_impl must be 'tcgen05' or 'mma_sync'")
        self.attn_impl = attn_impl
        self.config, self.model_dim = config, config.model_dim
        sd, d = state_dict, config.model_dim
        bf, f32 = self._bf16, self._f32

        layers = []
        for i in range(config.num_encoder_layers):
            p = f"encoder.layers.{i}."
            a = p + "self_attn."
            bn = p + "conv.batch_norm."
            scale = sd[bn + "weight"].float() / torch.sqrt(sd[bn + "running_var"].float() + config.bn_eps)
            layers.append({
                "ffn1_ln_g": f32(sd[p + "ffn1_layer_norm.weight"]), "ffn1_ln_b": f32(sd[p + "ffn1_layer_norm.bias"]),
                "ffn1_w1": bf(sd[p + "ffn1.inner_proj.weight"]), "ffn1_b1": f32(sd[p + "ffn1.inner_proj.bias"]),
                "ffn1_w2": bf(sd[p + "ffn1.output_proj.weight"].float() * 0.5), "ffn1_b2": f32(sd[p + "ffn1.output_proj.bias"].float() * 0.5),
                "attn_ln_g": f32(sd[p + "self_attn_layer_norm.weight"]), "attn_ln_b": f32(sd[p + "self_attn_layer_norm.bias"]),
                "wqkv": bf(torch.cat([sd[a + "q_proj.weight"], sd[a + "k_proj.weight"], sd[a + "v_proj.weight"]], 0)),
                "bqkv": f32(torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]], 0)),
                "wo": bf(sd[a + "output_proj.weight"]), "bo": f32(sd[a + "output_proj.bias"]),
                "wr": bf(sd[a + "sdpa.r_proj.weight"]),
                "u_bias": f32(sd[a + "sdpa.u_bias"].reshape(-1)), "v_bias": f32(sd[a + "sdpa.v_bias"].reshape(-1)),
                "conv_ln_g": f32(sd[p + "conv_layer_norm.weight"]), "conv_ln_b": f32(sd[p + "conv_layer_norm.bias"]),
                "pw1": bf(sd[p + "conv.pointwise_conv1.weight"].reshape(2 * d, d)),
                "dw": f32(sd[p + "conv.depthwise_conv.weight"].reshape(d, config.depthwise_conv_kernel_size)),
                "bn_scale": f32(scale), "bn_shift": f32(sd[bn + "bias"].float() - sd[bn + "running_mean"].float() * scale),
                "pw2": bf(sd[p + "conv.pointwise_conv2.weight"].reshape(d, d)),
                "ffn2_ln_g": f32(sd[p + "ffn2_layer_norm.weight"]), "ffn2_ln_b": f32(sd[p + "ffn2_layer_norm.bias"]),
                "ffn2_w1": bf(sd[p + "ffn2.inner_proj.weight"]), "ffn2_b1": f32(sd[p + "ffn2.inner_proj.bias"]),
                "ffn2_w2": bf(sd[p + "ffn2.output_proj.weight"].float() * 0.5), "ffn2_b2": f32(sd[p + "ffn2.output_proj.bias"].float() * 0.5),
                "ln_g": f32(sd[p + "layer_norm.weight"]), "ln_b": f32(sd[p + "layer_norm.bias"]),
            })
        fw = torch.zeros((d, 192), dtype=torch.float32)
        fw[:, : config.feature_dim] = sd["encoder_frontend.model_dim_proj.weight"].float()
        top, pooler = self._pooler_weights(sd, "encoder_pooler", config.bos_idx, d)  # projection_out has no bias
        top.update({
            "front_ln_g": f32(sd["encoder_frontend.post_extract_layer_norm.weight"]),
            "front_ln_b": f32(sd["encoder_frontend.post_extract_layer_norm.bias"]),
            "front_w": bf(fw), "front_b": f32(sd["encoder_frontend.model_dim_proj.bias"]),
            "final_ln_g": f32(sd["layer_norm.weight"]), "final_ln_b": f32(sd["layer_norm.bias"]),
            "zeros": f32(torch.zeros(8192)),
        })
        w_c = _lib.SbSpeechWeights(layers=self._layer_array(_lib.SbConformerLayerWeights, layers),
                                   pooler=self._layer_array(_lib.SbPoolerLayerWeights, pooler),
                                   **{k: v.data_ptr() for k, v in top.items()})
        cfg_c = _lib.SbSpeechConfig(model_dim=d, num_layers=config.num_encoder_layers, num_heads=config.num_encoder_attn_heads,
                                    ffn_inner_dim=config.ffn_inner_dim, conv_kernel=config.depthwise_conv_kernel_size,
                                    pooler_layers=config.num_decoder_layers,
                                    pooler_ffn_inner_dim=config.decoder_ffn_inner_dim, ln_eps=1e-5,
                                    attn_impl=1 if attn_impl == "mma_sync" else 0)
        self._create(cfg_c, w_c)
        self._relpos: Dict[int, Tensor] = {}
        self.return_encoded_seqs = False

    @torch.inference_mode()
    def forward(self, batch: SequenceBatch) -> SonarEncoderOutput:
        fb = batch.seqs
        if fb.dim() != 3 or fb.shape[2] != 80:
            raise ValueError("expected fbank features of shape [N, T, 80]")
        fb = self._on_device(fb, torch.float32).contiguous()
        n, t, _ = fb.shape
        frames = batch.padding_mask.seq_lens_host if batch.padding_mask is not None else [t] * n
        lens = [f // 2 for f in frames]  # Wav2Vec2FbankFeatureExtractor stride 2: seq_len // 2 (App. B.2)
        if min(lens) < 1:
            raise ValueError("every utterance needs at least 2 fbank frames")
        smax, total = max(lens), sum(lens)
        rows = relpos_rows(smax)
        if rows > 8192:
            raise ValueError("utterance too long for the relative-position workspace")
        if smax not in self._relpos:
            self._relpos = {smax: relative_position_table(smax, self.model_dim, rows).to(self.device, torch.bfloat16)}
        rel = self._relpos[smax]
        ws = self._ensure_workspace(n, total, smax)
        out = torch.empty((n, self.model_dim), dtype=torch.float32, device=self.device)
        enc = torch.empty((total, self.model_dim), dtype=torch.float32, device=self.device) if self.return_encoded_seqs else None
        lens_c = (C.c_int32 * n)(*lens)
        with torch.cuda.device(self.device):
            rc = self._lib.sb_speech_encoder_forward(
                self._handle, fb.data_ptr(), t, lens_c, n, rel.data_ptr(), rows, out.data_ptr(),
                enc.data_ptr() if enc is not None else None, ws.data_ptr(), ws.numel(), self._stream())
        _lib.check(rc, "sb_speech_encoder_forward")
        return SonarEncoderOutput(encoded_seqs=enc, sentence_embeddings=out, padding_mask=batch.padding_mask)
