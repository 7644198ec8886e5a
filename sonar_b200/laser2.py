"""The LASER2 text encoder on the engine: ``B200LaserLstmEncoder`` stands in for the reference's ``LaserLstmEncoder``
(``sonar/nn/laser_lstm_encoder.py:15-116``, loaded through ``sonar/models/laser2_text/``).

The model is an embedding, a packed multi-layer (bidirectional) ``torch.nn.LSTM`` and a max over time in which positions
holding ``pad_idx`` are left out.  All arithmetic happens in ``libsonar_b200.so`` (``sb_laser2_forward``): the
embedding gather, the input projections on the wgmma GEMM and the recurrence on the cluster-resident LSTM kernel.  The
reference has no pipeline for this model; its own test calls the model on ``Collater(pad_value=1)`` batches.
"""

from __future__ import annotations

import ctypes as C
import dataclasses
from dataclasses import dataclass
from typing import Dict, List, Sequence, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib
from ._engine import EngineModel


@dataclass
class Laser2Config:
    """Field-for-field mirror of the reference dataclass (``sonar/models/laser2_text/config.py:12-20``)."""

    vocabulary_size: int
    pad_idx: int
    model_dim: int = 320
    hidden_size: int = 512
    num_layers: int = 1
    bidirectional: bool = False
    padding_value: float = 0.0


def laser2_config(arch: str = "laser2", **overrides) -> Laser2Config:
    """Named archs of ``register_laser2_configs`` (``config.py:23-38``)."""
    if arch != "laser2":
        raise ValueError(f"unknown laser2 arch {arch!r}")
    cfg = Laser2Config(vocabulary_size=50004, pad_idx=1, model_dim=320, hidden_size=512, num_layers=5, bidirectional=True,
                       padding_value=0.0)
    return dataclasses.replace(cfg, **overrides)


def _check_supported(cfg: Laser2Config) -> None:
    bad = []
    if cfg.hidden_size != 512:
        bad.append(f"hidden_size={cfg.hidden_size} (needs 512)")
    if cfg.model_dim <= 0 or cfg.model_dim % 64 != 0:
        bad.append(f"model_dim={cfg.model_dim} (needs a positive multiple of 64)")
    if cfg.num_layers < 1:
        bad.append(f"num_layers={cfg.num_layers} (needs >= 1)")
    if cfg.vocabulary_size < 1:
        bad.append(f"vocabulary_size={cfg.vocabulary_size}")
    if bad:
        raise NotImplementedError("sonar_b200 LASER2 encoder does not support: " + "; ".join(bad))


class B200LaserLstmEncoder(EngineModel):
    """LASER2 sentence encoder on sm_90a kernels: ``forward(seqs, seq_lens) -> [B, hidden_size * (1 + bidirectional)]``
    with the reference's semantics, including its masking by token value (see ``forward``)."""

    _abi = "laser2"
    _default_config = staticmethod(laser2_config)

    def __init__(self, config: Laser2Config, state_dict: Dict[str, Tensor],
                 device: Union[str, torch.device] = "cuda") -> None:
        super().__init__(device)
        _check_supported(config)
        self.config = config
        self.output_units = config.hidden_size * (2 if config.bidirectional else 1)
        sd = state_dict
        embed = sd["embed_tokens.weight"]
        if tuple(embed.shape) != (config.vocabulary_size, config.model_dim):
            raise ValueError(f"embedding shape {tuple(embed.shape)} != ({config.vocabulary_size}, {config.model_dim})")
        bf, f32 = self._bf16, self._f32
        self._layer_bufs: List[Dict[str, Tensor]] = []
        for k in range(config.num_layers):
            for suffix in ("", "_reverse")[: 2 if config.bidirectional else 1]:
                self._layer_bufs.append({
                    "w_ih": bf(sd[f"lstm.weight_ih_l{k}{suffix}"]), "w_hh": bf(sd[f"lstm.weight_hh_l{k}{suffix}"]),
                    "b_ih": f32(sd[f"lstm.bias_ih_l{k}{suffix}"]), "b_hh": f32(sd[f"lstm.bias_hh_l{k}{suffix}"]),
                })
        cfg_c = _lib.SbLaser2Config(vocab_size=config.vocabulary_size, pad_idx=config.pad_idx, embed_dim=config.model_dim,
                                    hidden_size=config.hidden_size, num_layers=config.num_layers,
                                    bidirectional=int(config.bidirectional), padding_value=config.padding_value, num_sms=0)
        w_c = _lib.SbLaser2Weights(embed=bf(embed).data_ptr(),
                                   layers=self._layer_array(_lib.SbLstmLayerWeights, self._layer_bufs))
        self._create(cfg_c, w_c)

    @torch.inference_mode()
    def forward(self, seqs: Tensor, seq_lens: Union[Tensor, Sequence[int]]) -> Tensor:
        """``seqs`` int64 CUDA [B, S] right-padded token ids, ``seq_lens`` [B] lengths in 1..S (any device) ->
        fp32 [B, output_units] sentence embeddings, in the input order.

        As in the reference, every position whose id equals ``pad_idx`` is left out of the max, including one inside
        a sentence, and a position at or beyond the sentence's length whose id is another value contributes
        ``padding_value``.  A zero length raises ``ValueError`` (``pack_padded_sequence`` refuses one)."""
        if not isinstance(seqs, Tensor) or not seqs.is_cuda:
            raise RuntimeError("B200LaserLstmEncoder takes token ids on a CUDA device (there is no CPU path)")
        if seqs.dim() != 2:
            raise ValueError("expected token ids of shape [N, S]")
        seqs = self._on_device(seqs, torch.int64)
        if seqs.stride(1) != 1:
            seqs = seqs.contiguous()
        n, s = seqs.shape
        lens = seq_lens.cpu().numpy() if isinstance(seq_lens, Tensor) else np.asarray(seq_lens)
        lens_np = np.ascontiguousarray(lens, dtype=np.int32)
        if lens_np.shape != (n,):
            raise ValueError(f"seq_lens has shape {tuple(lens_np.shape)}, expected ({n},)")
        tokens = int(lens_np.sum(dtype=np.int64))
        ws = self._ensure_workspace(n, max(tokens, 1), headroom=1.1)
        out = torch.empty((n, self.output_units), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            rc = self._lib.sb_laser2_forward(self._handle, seqs.data_ptr(), seqs.stride(0),
                                             lens_np.ctypes.data_as(C.POINTER(C.c_int32)), n, s, out.data_ptr(),
                                             ws.data_ptr(), ws.numel(), self._stream())
        _lib.check(rc, "sb_laser2_forward")
        return out

    def check_inputs(self) -> None:
        """Raise ``ValueError`` if a batch since the last check contained a token id outside the vocabulary."""
        _lib.check(self._lib.sb_laser2_check_inputs(self._handle, self._stream()), "sb_laser2_check_inputs")
