"""CPU / float64 restatement of BLASER 2.0 (the reference's ``BlaserModel.forward``, ``sonar/models/blaser/model.py:82-125``),
pinned against the reference's own module by ``tests/golden/blaser_small.pt``:

* each input row is divided by ``max(||row||_2, 1e-12)`` (``F.normalize``, ``model.py:90-94``), so a zero row stays zero;
* ``featurize_input`` (``model.py:96-125``): COMET = ``[ref, mt, src*mt, ref*mt, |mt-src|, |mt-ref|]``,
  QE = ``[src, mt, src*mt, |mt-src|]``; COMET without ``ref`` raises ``ValueError``;
* the MLP (``model.py:63-80``): ``Linear -> activation`` per positive hidden size, then ``Linear(-> output_dim)``
  [``-> Tanh`` with ``output_act``].  Dropout is the identity in eval mode; it only shifts the ``mlp.<i>`` indices.

Also the synthetic weights and inputs the tests use: layer 1 ~ N(0, E / K), later layers ~ N(0, 1.5^2 / K), biases
~ N(0, 0.1^2) and (src, mt, ref) = a shared base row + 0.7 x independent N(0, 1) noise, which spreads the scores (std
about 0.76 at E = 1024) where ``nn.Linear``'s default init gives a near-constant score.
"""

from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor


def mlp_linear_indices(hidden_dims: List[int], dropout: float) -> List[int]:
    """Positions of the Linear layers (the output layer last) in the reference's ``nn.Sequential`` (``model.py:63-79``)."""
    if len(hidden_dims) == 0:
        return [0]
    pos = 0
    if dropout > 0:
        pos += 1  # leading Dropout
    out = []
    for h in hidden_dims:
        if h > 0:
            out.append(pos)
            pos += 2  # Linear, activation
            if dropout > 0:
                pos += 1
    return out + [pos]


def _normalize(x: Tensor) -> Tensor:
    return x / x.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def featurize(src: Tensor, mt: Tensor, ref: Optional[Tensor], input_form: str) -> Tensor:
    if input_form == "COMET":
        if ref is None:
            raise ValueError("With the COMET input form of BLASER, a reference embedding must be provided.")
        return torch.cat([ref, mt, src * mt, ref * mt, (mt - src).abs(), (mt - ref).abs()], dim=-1)
    if input_form == "QE":
        return torch.cat([src, mt, src * mt, (mt - src).abs()], dim=-1)
    raise ValueError(f"Unrecognized input format: {input_form}")


class OracleBlaser:
    def __init__(self, sd: Dict[str, Tensor], *, input_form: str, hidden_dims: List[int], dropout: float,
                 activation: str = "TANH", norm_emb: bool = True, output_act: bool = False) -> None:
        self.input_form, self.norm_emb, self.output_act = input_form, norm_emb, output_act
        self.act = {"TANH": torch.tanh, "RELU": torch.relu}[activation]
        self.layers: List[Tuple[Tensor, Tensor]] = [
            (sd[f"mlp.{i}.weight"].double(), sd[f"mlp.{i}.bias"].double()) for i in mlp_linear_indices(hidden_dims, dropout)]

    def featurize_input(self, src: Tensor, mt: Tensor, ref: Optional[Tensor] = None) -> Tensor:
        return featurize(src.double(), mt.double(), None if ref is None else ref.double(), self.input_form)

    def __call__(self, src: Tensor, mt: Tensor, ref: Optional[Tensor] = None) -> Tensor:
        src, mt = src.double(), mt.double()
        ref = None if ref is None else ref.double()
        if self.norm_emb:
            src, mt = _normalize(src), _normalize(mt)
            ref = None if ref is None else _normalize(ref)
        x = featurize(src, mt, ref, self.input_form)
        for i, (w, b) in enumerate(self.layers):
            x = x @ w.T + b
            if i + 1 < len(self.layers):
                x = self.act(x)
        return torch.tanh(x) if self.output_act else x


def make_synthetic_blaser_state_dict(input_form: str, embedding_dim: int, hidden_dims: List[int], dropout: float,
                                     seed: int = 0, output_dim: int = 1) -> Dict[str, Tensor]:
    """fp32 weights under the reference's ``mlp.<i>`` names, drawn by the recipe in the module docstring."""
    g = torch.Generator().manual_seed(seed)
    widths = [(6 if input_form == "COMET" else 4) * embedding_dim] + [h for h in hidden_dims if h > 0] + [output_dim]
    sd = {}
    for layer, idx in enumerate(mlp_linear_indices(hidden_dims, dropout)):
        k, n = widths[layer], widths[layer + 1]
        std = math.sqrt(embedding_dim) / math.sqrt(k) if layer == 0 else 1.5 / math.sqrt(k)
        sd[f"mlp.{idx}.weight"] = (torch.randn(n, k, generator=g, dtype=torch.float64) * std).float()
        sd[f"mlp.{idx}.bias"] = (torch.randn(n, generator=g, dtype=torch.float64) * 0.1).float()
    return sd


def make_blaser_inputs(n: int, embedding_dim: int, seed: int = 0) -> Tuple[Tensor, Tensor, Tensor]:
    """fp32 (src, mt, ref) [n, E]: one shared base row plus 0.7 x independent N(0, 1) noise each."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(1, embedding_dim, generator=g)
    return tuple(base + 0.7 * torch.randn(n, embedding_dim, generator=g) for _ in range(3))  # type: ignore[return-value]
