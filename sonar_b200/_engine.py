"""Host plumbing shared by ``B200TextEncoderModel``, ``B200TextDecoderModel`` and ``B200SpeechEncoderModel``."""

from __future__ import annotations

import ctypes as C
import math
from pathlib import Path
from typing import Any, Callable, Dict, List, Optional, Tuple, Union

import torch
from torch import Tensor

from . import _lib


class EngineModel(torch.nn.Module):
    """One C engine handle (``sb_<abi>_create`` / ``sb_<abi>_destroy``) on one CUDA device, the repacked weights it
    points into, and one grow-only workspace.

    The device and the weights' dtypes (bf16 matrices, fp32 vectors) are fixed at construction.  The engine keeps raw
    pointers to the weights, so they are held in plain attributes, not registered as buffers or parameters:
    ``.to()``, ``.half()``, ``.float()`` and ``.cuda()`` have nothing to convert and leave the model as it is.

    A subclass sets ``_abi`` (the ``sb_<abi>_*`` prefix of its entry points) and ``_default_config`` (the config
    function ``from_checkpoint`` uses when none is given).
    """

    _abi: str
    _default_config: Callable[[], Any]

    def __init__(self, device: Union[str, torch.device]) -> None:
        super().__init__()
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(f"{type(self).__name__} needs a CUDA device (there is no CPU path)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        self._lib = _lib.load()
        self._workspace_query = getattr(self._lib, f"sb_{self._abi}_workspace_bytes")
        self._weights: List[Tensor] = []  # every tensor whose pointer the engine holds
        self._handle: Optional[C.c_void_p] = None
        self._workspace: Optional[Tensor] = None

    @classmethod
    def from_checkpoint(cls, path: Union[str, Path], config: Any = None, device: Union[str, torch.device] = "cuda",
                        **kw) -> "EngineModel":
        """Load a fairseq2-layout checkpoint ``{"model": state_dict}`` (or a bare state dict); ``kw`` goes to the
        constructor."""
        ckpt = torch.load(str(path), map_location="cpu", weights_only=True)
        sd = ckpt["model"] if "model" in ckpt else ckpt
        return cls(config or cls._default_config(), sd, device, **kw)

    @property
    def dtype(self) -> torch.dtype:
        """Compute dtype of the engine (bf16 operands, fp32 accumulation)."""
        return torch.bfloat16

    def _bf16(self, t: Tensor) -> Tensor:
        return self._own(t, torch.bfloat16)

    def _f32(self, t: Tensor) -> Tensor:
        return self._own(t, torch.float32)

    def _own(self, t: Tensor, dtype: torch.dtype) -> Tensor:
        t = t.detach().to(device=self.device, dtype=dtype).contiguous()
        self._weights.append(t)
        return t

    @staticmethod
    def _layer_array(struct: type, layers: List[Dict[str, Tensor]]) -> C.Array:
        """ctypes array of ``struct``: each pointer field of entry i is the same-named tensor of ``layers[i]``."""
        arr = (struct * max(len(layers), 1))()
        for i, tensors in enumerate(layers):
            for name, _ in struct._fields_:
                setattr(arr[i], name, tensors[name].data_ptr())
        return arr

    def _pooler_weights(self, sd: Dict[str, Tensor], prefix: str, bos_idx: int,
                        width: int) -> Tuple[Dict[str, Tensor], List[Dict[str, Tensor]]]:
        """The ``<prefix>.*`` tensors of an ``AttentionEncoderOutputPooler`` of width ``width`` with
        ``self.config.num_decoder_layers`` layers, in the engine's layout: ``pooler_q0``, ``proj_w`` and, when the
        projection has a bias, ``proj_b``; and one ``SbPoolerLayerWeights`` dict per decoder layer."""
        bf, f32 = self._bf16, self._f32
        # the single decoder input: TransformerEmbeddingFrontend of token bos_idx = embed[bos_idx] * sqrt(width) + the
        # sinusoid of position 0, [sin 0 ... | cos 0 ...] = [0 ... | 1 ...]  [fs2]
        pos0 = torch.cat([torch.zeros(width // 2), torch.ones(width - width // 2)])
        top = {"pooler_q0": f32(sd[f"{prefix}.decoder_frontend.embed.weight"][bos_idx].float() * math.sqrt(width) + pos0),
               "proj_w": bf(sd[f"{prefix}.projection_out.weight"])}
        if f"{prefix}.projection_out.bias" in sd:
            top["proj_b"] = f32(sd[f"{prefix}.projection_out.bias"])
        layers = []
        for i in range(self.config.num_decoder_layers):
            p = f"{prefix}.decoder.layers.{i}."
            sa, ca = p + "self_attn.", p + "encoder_decoder_attn."
            layers.append({
                "sa_wv": bf(sd[sa + "v_proj.weight"]), "sa_bv": f32(sd[sa + "v_proj.bias"]),
                "sa_wo": bf(sd[sa + "output_proj.weight"]), "sa_bo": f32(sd[sa + "output_proj.bias"]),
                "sa_ln_g": f32(sd[p + "self_attn_layer_norm.weight"]), "sa_ln_b": f32(sd[p + "self_attn_layer_norm.bias"]),
                "ca_wq": bf(sd[ca + "q_proj.weight"]), "ca_bq": f32(sd[ca + "q_proj.bias"]),
                "ca_wkv": bf(torch.cat([sd[ca + "k_proj.weight"], sd[ca + "v_proj.weight"]], 0)),
                "ca_bkv": f32(torch.cat([sd[ca + "k_proj.bias"], sd[ca + "v_proj.bias"]], 0)),
                "ca_wo": bf(sd[ca + "output_proj.weight"]), "ca_bo": f32(sd[ca + "output_proj.bias"]),
                "ca_ln_g": f32(sd[p + "encoder_decoder_attn_layer_norm.weight"]),
                "ca_ln_b": f32(sd[p + "encoder_decoder_attn_layer_norm.bias"]),
                "w1": bf(sd[p + "ffn.inner_proj.weight"]), "b1": f32(sd[p + "ffn.inner_proj.bias"]),
                "w2": bf(sd[p + "ffn.output_proj.weight"]), "b2": f32(sd[p + "ffn.output_proj.bias"]),
                "ffn_ln_g": f32(sd[p + "ffn_layer_norm.weight"]), "ffn_ln_b": f32(sd[p + "ffn_layer_norm.bias"]),
            })
        return top, layers

    def _create(self, cfg: C.Structure, weights: C.Structure) -> None:
        name = f"sb_{self._abi}_create"
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(getattr(self._lib, name)(C.byref(cfg), C.byref(weights), C.byref(handle)), name)
        self._handle = handle

    def __del__(self) -> None:  # pragma: no cover - best effort
        try:
            if getattr(self, "_handle", None):
                getattr(self._lib, f"sb_{self._abi}_destroy")(self._handle)
                self._handle = None
        except Exception:
            pass

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _on_device(self, t: Tensor, dtype: torch.dtype) -> Tensor:
        """An input moved to the engine's device as ``dtype`` (``t`` itself when it is already there)."""
        return t.to(device=self.device, dtype=dtype, non_blocking=True)

    def _ensure_workspace(self, *shape: int, headroom: float = 1.0) -> Tensor:
        """The workspace, grown to ``headroom`` times what ``sb_<abi>_workspace_bytes(handle, *shape)`` asks for when
        the current one is smaller than that; it never shrinks."""
        need = _lib.workspace_bytes(self._workspace_query, self._handle, *shape)
        if self._workspace is None or self._workspace.numel() < need:
            self._workspace = None  # release before growing
            self._workspace = torch.empty(int(need * headroom), dtype=torch.uint8, device=self.device)
        return self._workspace
