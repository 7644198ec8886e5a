"""ctypes binding of ``libsonar_b200.so`` (C ABI: ``include/sonar_b200.h``).

There is deliberately NO fallback: if the library is missing or a call fails, a
``RuntimeError`` / ``ValueError`` is raised -- this package has no CPU compute path.
"""

from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Optional

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libsonar_b200.so"
_lib: Optional[C.CDLL] = None

SB_POOL_MAX, SB_POOL_MEAN, SB_POOL_LAST, SB_POOL_ATTENTION = 1, 2, 3, 4
SB_EPI_BIAS, SB_EPI_BIAS_RELU, SB_EPI_BIAS_RESIDUAL, SB_EPI_BIAS_TANH = 0, 1, 2, 7
SB_BLASER_COMET, SB_BLASER_QE = 0, 1
SB_ERR_INVALID, SB_ERR_CUDA, SB_ERR_DRIVER, SB_ERR_INPUT = -1, -2, -3, -4


class SbEncoderConfig(C.Structure):
    _fields_ = [
        ("model_dim", C.c_int32), ("num_layers", C.c_int32), ("num_heads", C.c_int32),
        ("ffn_inner_dim", C.c_int32), ("vocab_size", C.c_int64), ("pos_rows", C.c_int32),
        ("pooling", C.c_int32), ("ln_eps", C.c_float), ("embed_scale", C.c_float),
        ("cta_group", C.c_int32), ("num_sms", C.c_int32), ("ln_fold", C.c_int32),
        ("embedding_dim", C.c_int32), ("pooler_layers", C.c_int32), ("pooler_heads", C.c_int32),
        ("pooler_ffn_inner_dim", C.c_int32),
    ]


class SbLayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "wqkv", "bqkv", "wo", "bo", "w1", "b1", "w2", "b2", "ln1_g", "ln1_b", "ln2_g", "ln2_b")]


class SbPoolerLayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "sa_wv", "sa_bv", "sa_wo", "sa_bo", "sa_ln_g", "sa_ln_b", "ca_wq", "ca_bq", "ca_wkv", "ca_bkv", "ca_wo", "ca_bo",
        "ca_ln_g", "ca_ln_b", "w1", "b1", "w2", "b2", "ffn_ln_g", "ffn_ln_b")]


class SbEncoderWeights(C.Structure):
    _fields_ = [("embed", C.c_void_p), ("pos_table", C.c_void_p), ("final_ln_g", C.c_void_p),
                ("final_ln_b", C.c_void_p), ("layers", C.POINTER(SbLayerWeights)),
                ("pooler_q0", C.c_void_p), ("proj_w", C.c_void_p), ("proj_b", C.c_void_p),
                ("pooler", C.POINTER(SbPoolerLayerWeights))]


class SbDecoderConfig(C.Structure):
    _fields_ = [
        ("model_dim", C.c_int32), ("num_layers", C.c_int32), ("num_heads", C.c_int32),
        ("ffn_inner_dim", C.c_int32), ("input_dim", C.c_int32), ("vocab_size", C.c_int64),
        ("pos_rows", C.c_int32), ("eos_idx", C.c_int32), ("ln_eps", C.c_float), ("embed_scale", C.c_float),
    ]


class SbDecoderLayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "wqkv", "bqkv", "wo", "bo", "cross_wv", "cross_bv", "cross_wo", "cross_bo", "w1", "b1", "w2", "b2",
        "ln1_g", "ln1_b", "ln3_g", "ln3_b")]


class SbDecoderWeights(C.Structure):
    _fields_ = [("embed", C.c_void_p), ("pos_table", C.c_void_p), ("final_ln_g", C.c_void_p),
                ("final_ln_b", C.c_void_p), ("layers", C.POINTER(SbDecoderLayerWeights))]


class SbSpeechConfig(C.Structure):
    _fields_ = [("model_dim", C.c_int32), ("num_layers", C.c_int32), ("num_heads", C.c_int32),
                ("ffn_inner_dim", C.c_int32), ("conv_kernel", C.c_int32), ("pooler_layers", C.c_int32),
                ("pooler_ffn_inner_dim", C.c_int32), ("ln_eps", C.c_float), ("attn_impl", C.c_int32)]


class SbConformerLayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "ffn1_ln_g", "ffn1_ln_b", "ffn1_w1", "ffn1_b1", "ffn1_w2", "ffn1_b2", "attn_ln_g", "attn_ln_b", "wqkv", "bqkv",
        "wo", "bo", "wr", "u_bias", "v_bias", "conv_ln_g", "conv_ln_b", "pw1", "dw", "bn_scale", "bn_shift", "pw2",
        "ffn2_ln_g", "ffn2_ln_b", "ffn2_w1", "ffn2_b1", "ffn2_w2", "ffn2_b2", "ln_g", "ln_b")]


class SbSpeechWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("front_ln_g", "front_ln_b", "front_w", "front_b", "final_ln_g", "final_ln_b",
                                          "pooler_q0", "proj_w", "zeros")] + \
               [("layers", C.POINTER(SbConformerLayerWeights)), ("pooler", C.POINTER(SbPoolerLayerWeights))]


class SbLaser2Config(C.Structure):
    _fields_ = [("vocab_size", C.c_int64), ("pad_idx", C.c_int64), ("embed_dim", C.c_int32), ("hidden_size", C.c_int32),
                ("num_layers", C.c_int32), ("bidirectional", C.c_int32), ("padding_value", C.c_float),
                ("num_sms", C.c_int32)]


class SbLstmLayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w_ih", "w_hh", "b_ih", "b_hh")]


class SbLaser2Weights(C.Structure):
    _fields_ = [("embed", C.c_void_p), ("layers", C.POINTER(SbLstmLayerWeights))]


class SbBlaserConfig(C.Structure):
    _fields_ = [("input_form", C.c_int32), ("embedding_dim", C.c_int32), ("num_hidden", C.c_int32),
                ("hidden_dims", C.POINTER(C.c_int32)), ("cta_group", C.c_int32), ("num_sms", C.c_int32)]


class SbBlaserWeights(C.Structure):
    _fields_ = [("w", C.POINTER(C.c_void_p)), ("b", C.POINTER(C.c_void_p))]


# name -> (restype, argtypes); must list every symbol include/sonar_b200.h declares
_SIGNATURES = {
    "sb_last_error": (C.c_char_p, []),
    "sb_version": (C.c_int, []),
    "sb_encoder_create": (C.c_int, [C.POINTER(SbEncoderConfig), C.POINTER(SbEncoderWeights),
                                    C.POINTER(C.c_void_p)]),
    "sb_encoder_destroy": (None, [C.c_void_p]),
    "sb_encoder_workspace_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_size_t)]),
    "sb_encoder_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sb_encoder_forward_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                          C.c_void_p]),
    "sb_encoder_profile_ffn1": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_encoder_check_inputs": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_gemm_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                               C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                               C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "sb_layernorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int64,
                               C.c_int32, C.c_void_p]),
    "sb_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    "sb_embed": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                           C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                           C.c_void_p, C.c_void_p]),
    "sb_layernorm_dual": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int64,
                                    C.c_int32, C.c_void_p]),
    "sb_pool": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_float,
                          C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "sb_pool_latent_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_void_p, C.c_void_p]),
    "sb_attention_relpos": (C.c_int, [C.c_void_p] * 5 + [C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_int32] +
                            [C.c_void_p] * 5),
    "sb_conformer_conv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 5),
    "sb_speech_frontend": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                     C.c_float, C.c_void_p, C.c_void_p]),
    "sb_decoder_create": (C.c_int, [C.POINTER(SbDecoderConfig), C.POINTER(SbDecoderWeights), C.POINTER(C.c_void_p)]),
    "sb_decoder_destroy": (None, [C.c_void_p]),
    "sb_decoder_workspace_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_size_t)]),
    "sb_decoder_begin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_size_t,
                                   C.c_void_p]),
    "sb_decoder_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.c_void_p]),
    "sb_decoder_check_inputs": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_decoder_embed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_int32,
                                   C.c_void_p, C.c_void_p]),
    "sb_decoder_attention": (C.c_int, [C.c_void_p] * 4 + [C.c_int32] * 4 + [C.c_void_p] * 2),
    "sb_decoder_add_const_layernorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                                 C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]),
    "sb_decoder_vocab_chunks": (C.c_int, [C.c_int32, C.c_int64, C.POINTER(C.c_int32)]),
    "sb_decoder_vocab_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_void_p,
                                        C.c_int32] + [C.c_void_p] * 8),
    "sb_fbank_tables_bytes": (C.c_size_t, []),
    "sb_fbank_build_tables": (C.c_int, [C.c_void_p]),
    "sb_fbank": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                           C.c_void_p, C.c_int32, C.c_void_p]),
    "sb_speech_encoder_create": (C.c_int, [C.POINTER(SbSpeechConfig), C.POINTER(SbSpeechWeights), C.POINTER(C.c_void_p)]),
    "sb_speech_encoder_destroy": (None, [C.c_void_p]),
    "sb_speech_encoder_workspace_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.POINTER(C.c_size_t)]),
    "sb_speech_encoder_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                            C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sb_xsim_workspace_bytes": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_size_t)]),
    "sb_xsim_knn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                              C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sb_xsim_margin_predict": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_int32, C.c_void_p, C.c_void_p]),
    "sb_fold_layernorm": (C.c_int, [C.c_void_p] * 4 + [C.c_int32, C.c_int32] + [C.c_void_p] * 4),
    "sb_gemm_ln_consumer": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p]),
    "sb_gemm_residual_stats": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                         C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "sb_gemm_residual_splitk": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                          C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]),
    "sb_xsim_bidir_workspace_bytes": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_size_t)]),
    "sb_xsim_knn_bidir": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sb_beam_step": (C.c_int, [C.c_void_p] * 13 + [C.c_int32] * 7 + [C.c_int64] + [C.c_int32] * 3 +
                     [C.c_float, C.c_float, C.c_int32, C.c_void_p]),
    "sb_laser2_create": (C.c_int, [C.POINTER(SbLaser2Config), C.POINTER(SbLaser2Weights), C.POINTER(C.c_void_p)]),
    "sb_laser2_destroy": (None, [C.c_void_p]),
    "sb_laser2_workspace_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_size_t)]),
    "sb_laser2_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p]),
    "sb_laser2_check_inputs": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sb_laser2_layer_weights": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                          C.POINTER(C.c_void_p)]),
    "sb_laser2_embed": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int32,
                                  C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_lstm_recurrent": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                    C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_float,
                                    C.c_void_p]),
    "sb_blaser_create": (C.c_int, [C.POINTER(SbBlaserConfig), C.POINTER(SbBlaserWeights), C.POINTER(C.c_void_p)]),
    "sb_blaser_destroy": (None, [C.c_void_p]),
    "sb_blaser_workspace_bytes": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_size_t)]),
    "sb_blaser_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p]),
    "sb_blaser_featurize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
}


def lib_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load the shared library (once) and bind every declared symbol."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise RuntimeError(
            f"sonar_b200: native library {_LIB_PATH} is missing -- run `python -m sonar_b200.build` "
            "(or `__graft_entry__.build()`); there is no CPU/PyTorch fallback path.")
    lib = C.CDLL(str(_LIB_PATH))
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == header/library mismatch
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def last_error() -> str:
    msg = load().sb_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def workspace_bytes(query, *args) -> int:
    """Bytes the ``sb_*_workspace_bytes`` entry point ``query`` (a function of the loaded library) asks for; ``args``
    are its arguments before the out-pointer."""
    need = C.c_size_t()
    check(query(*args, C.byref(need)), query.__name__)
    return need.value


def check(rc: int, what: str) -> None:
    """Map a C-ABI return code to the exception the reference API would raise."""
    if rc == 0:
        return
    msg = f"{what}: {last_error()} (code {rc})"
    if rc in (SB_ERR_INVALID, SB_ERR_INPUT):
        raise ValueError(msg)
    raise RuntimeError(msg)
