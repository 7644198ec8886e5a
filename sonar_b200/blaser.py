"""BLASER 2.0 on the engine: ``B200BlaserModel`` stands in for the reference's ``BlaserModel``
(``sonar/models/blaser/model.py:26-125``, cards ``blaser_2_0_ref`` / ``blaser_2_0_qe``), the translation-quality metric
that scores (source, translation[, reference]) sentence-embedding pairs.

The model normalises each embedding, concatenates products and differences of them, and runs a Tanh MLP down to one
score per pair.  All arithmetic happens in ``libsonar_b200.so`` (``sb_blaser_forward``): the featurization kernel, the
hidden layers on the wgmma GEMM with a tanh epilogue, and the final dot product.  There is no pipeline class, as in the
reference: the embeddings come from the text or speech pipelines.
"""

from __future__ import annotations

import ctypes as C
import dataclasses
import os
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, List, Optional, Union

import torch
from torch import Tensor

from . import _lib, ops
from ._engine import EngineModel

_INPUT_FORMS = {"COMET": _lib.SB_BLASER_COMET, "QE": _lib.SB_BLASER_QE}
_CARDS = {"blaser_2_0_ref": "basic_ref", "blaser_2_0_qe": "basic_qe"}  # sonar/cards/blaser_2_0.yaml
PASS_ROWS = 65536  # pairs per engine call: bounds the workspace (about 1.6 GB for basic_ref)


@dataclass
class BlaserConfig:
    """Field-for-field mirror of the reference dataclass (``sonar/models/blaser/config.py:15-24``)."""

    input_form: str = "COMET"
    norm_emb: bool = True
    embedding_dim: int = 1024
    output_dim: int = 1
    hidden_dims: List[int] = field(default_factory=lambda: [3072, 1536])
    dropout: float = 0.1
    activation: str = "TANH"
    output_act: bool = False


def blaser_config(arch: str = "basic_ref", **overrides) -> BlaserConfig:
    """Named archs of ``register_blaser_configs`` (``config.py:43-67``)."""
    if arch not in ("basic_ref", "basic_qe"):
        raise ValueError(f"unknown blaser arch {arch!r}")
    cfg = BlaserConfig(embedding_dim=1024, output_dim=1, norm_emb=True, input_form="COMET" if arch == "basic_ref" else "QE",
                       dropout=0.1, hidden_dims=[3072, 1536], activation="TANH", output_act=False)
    return dataclasses.replace(cfg, **overrides)


def linear_layer_indices(cfg: BlaserConfig) -> List[int]:
    """Indices in the reference's ``mlp`` Sequential of its Linear layers, the output layer last: the module list of
    ``model.py:63-79`` rebuilt (a Dropout first and after every activation when dropout > 0; hidden sizes <= 0 skipped)."""
    hidden = [h for h in cfg.hidden_dims if h > 0]
    if not cfg.hidden_dims:
        return [0]
    idx, out = (1 if cfg.dropout > 0 else 0), []
    for _ in hidden:
        out.append(idx)
        idx += 2 + (1 if cfg.dropout > 0 else 0)  # Linear, activation[, Dropout]
    return out + [idx]


def _check_supported(cfg: BlaserConfig) -> None:
    if cfg.input_form not in _INPUT_FORMS:
        raise ValueError(f"Input form '{cfg.input_form}' is invalid; should be one of {sorted(_INPUT_FORMS)}.")
    bad = []
    if cfg.activation != "TANH":
        bad.append(f"activation={cfg.activation!r} (needs 'TANH')")
    if not cfg.norm_emb:
        bad.append("norm_emb=False (needs True)")
    if cfg.output_act:
        bad.append("output_act=True (needs False)")
    if cfg.output_dim != 1:
        bad.append(f"output_dim={cfg.output_dim} (needs 1)")
    hidden = [h for h in cfg.hidden_dims if h > 0]
    if not hidden:
        bad.append(f"hidden_dims={cfg.hidden_dims} (needs at least one hidden layer)")
    if any(h % 256 for h in hidden):
        bad.append(f"hidden_dims={cfg.hidden_dims} (each needs to be a multiple of 256)")
    width = (6 if cfg.input_form == "COMET" else 4) * cfg.embedding_dim
    if cfg.embedding_dim <= 0 or cfg.embedding_dim % 16 or width % 64:
        bad.append(f"embedding_dim={cfg.embedding_dim} (needs a positive multiple of 16 whose feature width "
                   f"{width} is a multiple of 64)")
    if bad:
        raise NotImplementedError("sonar_b200 BLASER model does not support: " + "; ".join(bad))


class B200BlaserModel(EngineModel):
    """BLASER 2.0 scorer on sm_90a kernels: ``forward(src, mt, ref=None) -> fp32 [N, 1]`` with the reference's semantics
    in eval mode (dropout off)."""

    _abi = "blaser"
    _default_config = staticmethod(blaser_config)

    def __init__(self, config: BlaserConfig, state_dict: Dict[str, Tensor],
                 device: Union[str, torch.device] = "cuda") -> None:
        super().__init__(device)
        _check_supported(config)
        self.config = config
        hidden = [h for h in config.hidden_dims if h > 0]
        idx = linear_layer_indices(config)
        sd = state_dict
        widths = [(6 if config.input_form == "COMET" else 4) * config.embedding_dim] + hidden + [1]
        ws: List[Tensor] = []
        bs: List[Tensor] = []
        for i, j in enumerate(idx):
            w, b = sd[f"mlp.{j}.weight"], sd[f"mlp.{j}.bias"]
            if tuple(w.shape) != (widths[i + 1], widths[i]) or tuple(b.shape) != (widths[i + 1],):
                raise ValueError(f"mlp.{j}: weight {tuple(w.shape)} / bias {tuple(b.shape)}, expected "
                                 f"({widths[i + 1]}, {widths[i]}) / ({widths[i + 1]},)")
            last = i == len(idx) - 1
            ws.append(self._f32(w.reshape(-1)) if last else self._bf16(w))  # the output row stays fp32
            bs.append(self._f32(b))
        self._dims = (C.c_int32 * len(hidden))(*hidden)
        self._w_ptrs = (C.c_void_p * len(ws))(*[t.data_ptr() for t in ws])
        self._b_ptrs = (C.c_void_p * len(bs))(*[t.data_ptr() for t in bs])
        cfg_c = _lib.SbBlaserConfig(input_form=_INPUT_FORMS[config.input_form], embedding_dim=config.embedding_dim,
                                    num_hidden=len(hidden), hidden_dims=self._dims, cta_group=2, num_sms=0)
        self._create(cfg_c, _lib.SbBlaserWeights(w=self._w_ptrs, b=self._b_ptrs))

    def _inputs(self, src: Tensor, mt: Tensor, ref: Optional[Tensor]) -> List[Tensor]:
        """src, mt and, for COMET, ref as contiguous fp32 [N, E] tensors on the engine's device."""
        if self.config.input_form == "COMET" and ref is None:
            raise ValueError("With the COMET input form of BLASER, a reference embedding must be provided.")
        named = [("src", src), ("mt", mt)] + ([("ref", ref)] if self.config.input_form == "COMET" else [])
        e = self.config.embedding_dim
        for name, t in named:
            if not isinstance(t, Tensor) or t.dim() != 2 or t.shape[1] != e or t.shape[0] != named[0][1].shape[0]:
                raise ValueError(f"{name} has shape {tuple(getattr(t, 'shape', ()))}; src, mt and ref must all be "
                                 f"[N, {e}] with the same N")
        return [self._on_device(t, torch.float32).contiguous() for _, t in named]

    @torch.inference_mode()
    def forward(self, src: Tensor, mt: Tensor, ref: Optional[Tensor] = None) -> Tensor:
        """Scores of the pairs (src[i], mt[i]) (and ref[i] for COMET): fp32 [N, 1] on the engine's device.  Inputs may
        have any float dtype and device.  QE ignores ``ref``.  A pair's score does not depend on the rest of the batch."""
        x = self._inputs(src, mt, ref)
        n = x[0].shape[0]
        out = torch.empty((n, 1), dtype=torch.float32, device=self.device)
        if n == 0:
            return out
        ws = self._ensure_workspace(min(n, PASS_ROWS))
        e = self.config.embedding_dim
        with torch.cuda.device(self.device):
            for i0 in range(0, n, PASS_ROWS):
                rows = min(PASS_ROWS, n - i0)
                src_p, mt_p = x[0][i0].data_ptr(), x[1][i0].data_ptr()
                ref_p = x[2][i0].data_ptr() if len(x) == 3 else None
                rc = self._lib.sb_blaser_forward(self._handle, src_p, mt_p, ref_p, e, rows, out[i0].data_ptr(),
                                                 ws.data_ptr(), ws.numel(), self._stream())
                _lib.check(rc, "sb_blaser_forward")
        return out

    @torch.inference_mode()
    def featurize_input(self, src: Tensor, mt: Tensor, ref: Optional[Tensor] = None) -> Tensor:
        """The reference method of the same name (``model.py:96-125``): fp32 features of the inputs as given (not
        normalised), [N, 6E] for COMET and [N, 4E] for QE, on the engine's device."""
        x = self._inputs(src, mt, ref)
        with torch.cuda.device(self.device):
            return ops.blaser_featurize(x[0], x[1], x[2] if len(x) == 3 else None, self.config.input_form)


def load_blaser_model(name: str, device: Union[str, torch.device] = "cuda") -> B200BlaserModel:
    """Mirror of ``sonar/models/blaser/loader.py``: the card ``blaser_2_0_ref`` or ``blaser_2_0_qe`` from a local
    checkpoint ``$SONAR_B200_CHECKPOINT_DIR/<name>.pt`` (either the ``{"model": state_dict}`` layout or a bare state dict,
    as ``blaser/handler.py:37-45`` accepts).  There is no downloader."""
    root = os.environ.get("SONAR_B200_CHECKPOINT_DIR")
    if name not in _CARDS or not root or not (Path(root) / f"{name}.pt").exists():
        raise FileNotFoundError(f"blaser card {name!r}: set SONAR_B200_CHECKPOINT_DIR to a directory holding {name}.pt "
                                f"(one of {sorted(_CARDS)})")
    return B200BlaserModel.from_checkpoint(Path(root) / f"{name}.pt", blaser_config(_CARDS[name]), device)
