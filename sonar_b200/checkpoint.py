"""Checkpoint converters: legacy fairseq layouts -> the fairseq2 state-dict names the CUDA models consume.

Host-side mirrors of the reference's converters (pure key renaming + one row permutation, no arithmetic):

* text encoder  -- ``convert_sonar_text_encoder_checkpoint``  (``sonar/models/sonar_text/handler.py:52-94``)
* text decoder  -- ``convert_sonar_text_decoder_checkpoint``  (``handler.py:119-172``)
* speech encoder -- ``convert_sonar_speech_checkpoint``        (``sonar/models/sonar_speech/handler.py:47-110``)

fairseq stored the control symbols as (BOS, PAD, EOS, UNK); the NLLB tokenizer of fairseq2 uses (PAD, UNK, BOS, EOS),
so rows 0-3 of the embedding matrix are permuted ``embeds[[0,1,2,3]] = embeds[[1,3,0,2]]`` (``handler.py:86-92,165-171``).
A checkpoint that already has the fairseq2 names (``{"model": {... "encoder_frontend.embed.weight" ...}}``) is returned
unchanged, like the reference.
"""

from __future__ import annotations

import re
from typing import Any, Dict, Mapping

import torch

_TEXT_ENCODER_KEY_MAP = {  # handler.py:71-84
    r"layers\.([0-9]+)\.self_attn\.q_proj\.": r"encoder.layers.\1.self_attn.q_proj.",
    r"layers\.([0-9]+)\.self_attn\.v_proj\.": r"encoder.layers.\1.self_attn.v_proj.",
    r"layers\.([0-9]+)\.self_attn\.k_proj\.": r"encoder.layers.\1.self_attn.k_proj.",
    r"layers\.([0-9]+)\.self_attn.out_proj\.": r"encoder.layers.\1.self_attn.output_proj.",
    r"layers\.([0-9]+)\.self_attn_layer_norm\.": r"encoder.layers.\1.self_attn_layer_norm.",
    r"layers\.([0-9]+)\.fc1\.": r"encoder.layers.\1.ffn.inner_proj.",
    r"layers\.([0-9]+)\.fc2\.": r"encoder.layers.\1.ffn.output_proj.",
    r"layers\.([0-9]+)\.final_layer_norm\.": r"encoder.layers.\1.ffn_layer_norm.",
    r"embed_tokens\.": r"encoder_frontend.embed.",
}

_TEXT_DECODER_KEY_MAP = {  # handler.py:136-158
    r"layers\.([0-9]+)\.self_attn\.k_proj\.": r"decoder.layers.\1.self_attn.k_proj.",
    r"layers\.([0-9]+)\.self_attn\.v_proj\.": r"decoder.layers.\1.self_attn.v_proj.",
    r"layers\.([0-9]+)\.self_attn\.q_proj\.": r"decoder.layers.\1.self_attn.q_proj.",
    r"layers\.([0-9]+)\.self_attn.out_proj\.": r"decoder.layers.\1.self_attn.output_proj.",
    r"layers\.([0-9]+)\.self_attn_layer_norm\.": r"decoder.layers.\1.self_attn_layer_norm.",
    r"layers\.([0-9]+).ffn\.inner_proj\.": r"decoder.layers.\1.ffn.inner_proj.",
    r"layers\.([0-9]+).ffn\.output_proj\.": r"decoder.layers.\1.ffn.output_proj.",
    r"layers\.([0-9]+)\.ffn_layer_norm\.": r"decoder.layers.\1.ffn_layer_norm.",
    r"layers\.([0-9]+).encoder_attn\.k_proj\.": r"decoder.layers.\1.encoder_decoder_attn.k_proj.",
    r"layers\.([0-9]+).encoder_attn\.v_proj\.": r"decoder.layers.\1.encoder_decoder_attn.v_proj.",
    r"layers\.([0-9]+).encoder_attn\.q_proj\.": r"decoder.layers.\1.encoder_decoder_attn.q_proj.",
    r"layers\.([0-9]+).encoder_attn\.out_proj\.": r"decoder.layers.\1.encoder_decoder_attn.output_proj.",
    r"layers\.([0-9]+)\.encoder_attn_layer_norm\.": r"decoder.layers.\1.encoder_decoder_attn_layer_norm.",
    r"layers\.([0-9]+)\.fc1\.": r"decoder.layers.\1.ffn.inner_proj.",
    r"layers\.([0-9]+)\.fc2\.": r"decoder.layers.\1.ffn.output_proj.",
    r"layers\.([0-9]+)\.final_layer_norm\.": r"decoder.layers.\1.ffn_layer_norm.",
    r"output_projection.": r"final_proj.",
    r"embed_tokens.": r"decoder_frontend.embed.",
    r"layer_norm.": r"decoder.layer_norm.",
}

_SPEECH_KEY_MAP = {  # sonar_speech/handler.py:63-100 (+ the LayerNorm re-homing, :102-108)
    r"^encoder.w2v_model.layer_norm\.": r"encoder_frontend.post_extract_layer_norm.",
    r"^encoder.w2v_model.post_extract_proj\.": r"encoder_frontend.model_dim_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.conv_module\.batch_norm\.": r"encoder.layers.\1.conv.batch_norm.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.conv_module\.depthwise_conv\.": r"encoder.layers.\1.conv.depthwise_conv.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.conv_module\.layer_norm\.": r"encoder.layers.\1.conv_layer_norm.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.conv_module\.pointwise_conv1\.": r"encoder.layers.\1.conv.pointwise_conv1.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.conv_module\.pointwise_conv2\.": r"encoder.layers.\1.conv.pointwise_conv2.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.ffn(1|2)\.layer_norm\.": r"encoder.layers.\1.ffn\2_layer_norm.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.ffn(1|2)\.w_1\.": r"encoder.layers.\1.ffn\2.inner_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.ffn(1|2)\.w_2\.": r"encoder.layers.\1.ffn\2.output_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn_layer_norm\.": r"encoder.layers.\1.self_attn_layer_norm.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn\.linear_q\.": r"encoder.layers.\1.self_attn.q_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn\.linear_k\.": r"encoder.layers.\1.self_attn.k_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn\.linear_v\.": r"encoder.layers.\1.self_attn.v_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn\.linear_out\.": r"encoder.layers.\1.self_attn.output_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn\.linear_pos\.": r"encoder.layers.\1.self_attn.sdpa.r_proj.",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn\.pos_bias_u": r"encoder.layers.\1.self_attn.sdpa.u_bias",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.self_attn\.pos_bias_v": r"encoder.layers.\1.self_attn.sdpa.v_bias",
    r"^encoder.w2v_model.encoder\.layers\.([0-9]+)\.final_layer_norm\.": r"encoder.layers.\1.layer_norm.",
    r"^encoder.w2v_model.encoder\.layer_norm\.": r"layer_norm.",  # re-homed to the SONAR model (conformer case)
    r"^decoder\.embed_tokens\.": r"encoder_pooler.decoder_frontend.embed.",
    r"^decoder\.layers\.([0-9]+)\.self_attn_layer_norm\.": r"encoder_pooler.decoder.layers.\1.self_attn_layer_norm.",
    r"^decoder\.layers\.([0-9]+)\.self_attn\.out_proj\.": r"encoder_pooler.decoder.layers.\1.self_attn.output_proj.",
    r"^decoder\.layers\.([0-9]+)\.self_attn\.": r"encoder_pooler.decoder.layers.\1.self_attn.",
    r"^decoder\.layers\.([0-9]+)\.encoder_attn_layer_norm\.": r"encoder_pooler.decoder.layers.\1.encoder_decoder_attn_layer_norm.",
    r"^decoder\.layers\.([0-9]+)\.encoder_attn\.out_proj\.": r"encoder_pooler.decoder.layers.\1.encoder_decoder_attn.output_proj.",
    r"^decoder\.layers\.([0-9]+)\.encoder_attn\.": r"encoder_pooler.decoder.layers.\1.encoder_decoder_attn.",
    r"^decoder\.layers\.([0-9]+)\.fc1\.": r"encoder_pooler.decoder.layers.\1.ffn.inner_proj.",
    r"^decoder\.layers\.([0-9]+)\.fc2\.": r"encoder_pooler.decoder.layers.\1.ffn.output_proj.",
    r"^decoder\.layers\.([0-9]+)\.final_layer_norm\.": r"encoder_pooler.decoder.layers.\1.ffn_layer_norm.",
    r"^decoder\.embed_out": r"encoder_pooler.projection_out.weight",
}


def _rename(state_dict: Mapping[str, Any], key_map: Mapping[str, str]) -> Dict[str, Any]:
    """fairseq2 ``convert_fairseq_checkpoint`` semantics [fs2]: the FIRST pattern that matches a key renames it."""
    compiled = [(re.compile(p), r) for p, r in key_map.items()]
    out: Dict[str, Any] = {}
    for k, v in state_dict.items():
        new = k
        for pat, rep in compiled:
            new, n = pat.subn(rep, k)
            if n:
                break
        out[new] = v
    return out


def _swap_control_rows(embed: torch.Tensor) -> torch.Tensor:
    e = embed.clone()
    e[[0, 1, 2, 3]] = embed[[1, 3, 0, 2]]  # (BOS, PAD, EOS, UNK) -> (PAD, UNK, BOS, EOS)
    return e


def convert_sonar_text_encoder_checkpoint(checkpoint: Dict[str, Any]) -> Dict[str, Any]:
    if "model" in checkpoint and "encoder_frontend.embed.weight" in checkpoint["model"]:
        return checkpoint
    sd = dict(checkpoint["state_dict"])
    sd.pop("version", None)
    sd.pop("embed_positions._float_tensor", None)
    if "embed_tokens" in checkpoint and "embed_tokens.weight" not in sd:  # pickled nn.Embedding (handler.py:86)
        sd["embed_tokens.weight"] = checkpoint["embed_tokens"].weight
    out = _rename(sd, _TEXT_ENCODER_KEY_MAP)
    out["encoder_frontend.embed.weight"] = _swap_control_rows(out["encoder_frontend.embed.weight"])
    return {"model": out}


def convert_sonar_text_decoder_checkpoint(checkpoint: Dict[str, Any]) -> Dict[str, Any]:
    if "model" in checkpoint and "decoder_frontend.embed.weight" in checkpoint["model"]:
        return checkpoint
    sd = dict(checkpoint["state_dict"])
    sd.pop("version", None)
    sd.pop("embed_positions._float_tensor", None)
    out = _rename(sd, _TEXT_DECODER_KEY_MAP)
    out["decoder_frontend.embed.weight"] = _swap_control_rows(out["decoder_frontend.embed.weight"])
    if "final_proj.weight" not in out:
        out["final_proj.weight"] = out["decoder_frontend.embed.weight"]  # TiedProjection (factory.py:306-307)
    return {"model": out}


def convert_sonar_speech_checkpoint(checkpoint: Dict[str, Any]) -> Dict[str, Any]:
    sd = checkpoint["model"] if "model" in checkpoint else checkpoint
    if "encoder_frontend.model_dim_proj.weight" in sd:
        return {"model": dict(sd)}
    sd = dict(sd)
    for k in ("encoder.w2v_model.mask_emb", "encoder.w2v_model.encoder.pos_conv.0.bias",
              "encoder.w2v_model.encoder.pos_conv.0.weight_g", "encoder.w2v_model.encoder.pos_conv.0.weight_v"):
        sd.pop(k, None)
    return {"model": _rename(sd, _SPEECH_KEY_MAP)}
