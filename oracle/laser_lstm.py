"""CPU / float64 restatement of the LASER2 text encoder (the reference's ``LaserLstmEncoder.forward``,
``sonar/nn/laser_lstm_encoder.py:60-116``), written from the definition of a multi-layer LSTM.

For one layer and direction, with the stacked gate matrices of ``torch.nn.LSTM`` in the order i, f, g, o:

    z_t = W_ih x_t + b_ih + W_hh h_{t-1} + b_hh
    i = sigmoid(z_i), f = sigmoid(z_f), g = tanh(z_g), o = sigmoid(z_o)
    c_t = f * c_{t-1} + i * g,   h_t = o * tanh(c_t),   h_{-1} = c_{-1} = 0

Sequence b runs over its own ``len_b`` positions only (packed sequences); the reverse direction starts at position
``len_b - 1``.  Layer l > 0 reads ``[forward | backward]`` of layer l - 1.  Then, over the padded time axis of width S:

* positions ``t >= len_b`` hold ``padding_value`` (``pad_packed_sequence``);
* every position whose token id equals ``pad_idx`` holds ``-inf``, also one inside ``len_b`` (the reference masks by value);
* the sentence embedding is the max over t.

A zero length raises ``ValueError`` (``pack_padded_sequence`` refuses one).  Runs on any device and dtype.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch
from torch import Tensor


@dataclass
class OracleLaser2Config:
    vocabulary_size: int = 50004
    pad_idx: int = 1
    model_dim: int = 320
    hidden_size: int = 512
    num_layers: int = 5
    bidirectional: bool = True
    padding_value: float = 0.0


def make_synthetic_laser2_state_dict(cfg: OracleLaser2Config, seed: int = 1, embed_std: float = 1.0,
                                     weight_bound: Optional[float] = None) -> Dict[str, Tensor]:
    """Seeded fp32 weights with the module's parameter names.  Defaults follow torch's own initialisation:
    ``nn.Embedding`` N(0, 1) with the ``pad_idx`` row zeroed, ``nn.LSTM`` U(-1/sqrt(H), 1/sqrt(H)); ``weight_bound``
    overrides the LSTM bound."""
    g = torch.Generator().manual_seed(seed)
    k = weight_bound if weight_bound is not None else cfg.hidden_size ** -0.5
    H = cfg.hidden_size

    def u(*shape):
        return (torch.rand(*shape, generator=g) * 2 - 1) * k

    emb = torch.randn(cfg.vocabulary_size, cfg.model_dim, generator=g) * embed_std
    emb[cfg.pad_idx] = 0
    sd = {"embed_tokens.weight": emb}
    dirs = 2 if cfg.bidirectional else 1
    for layer in range(cfg.num_layers):
        inp = cfg.model_dim if layer == 0 else dirs * H
        for suffix in ("", "_reverse")[:dirs]:
            sd[f"lstm.weight_ih_l{layer}{suffix}"] = u(4 * H, inp)
            sd[f"lstm.weight_hh_l{layer}{suffix}"] = u(4 * H, H)
            sd[f"lstm.bias_ih_l{layer}{suffix}"] = u(4 * H)
            sd[f"lstm.bias_hh_l{layer}{suffix}"] = u(4 * H)
    return sd


class OracleLaser2:
    def __init__(self, cfg: OracleLaser2Config, state_dict: Dict[str, Tensor], dtype: torch.dtype = torch.float64,
                 device="cpu") -> None:
        self.cfg = cfg
        self.sd = {k: v.detach().to(device=device, dtype=dtype) for k, v in state_dict.items()}
        self.dtype, self.device = dtype, torch.device(device)

    def direction(self, x: Tensor, lens: Tensor, layer: int, reverse: bool) -> Tensor:
        """One LSTM layer and direction over padded inputs x [B, S, in] -> outputs [B, S, H], zero at t >= len_b."""
        suffix = "_reverse" if reverse else ""
        w_ih, w_hh = self.sd[f"lstm.weight_ih_l{layer}{suffix}"], self.sd[f"lstm.weight_hh_l{layer}{suffix}"]
        b = self.sd[f"lstm.bias_ih_l{layer}{suffix}"] + self.sd[f"lstm.bias_hh_l{layer}{suffix}"]
        B, S, _ = x.shape
        H = w_hh.shape[1]
        gx = x @ w_ih.T + b  # [B, S, 4H]: the input half of z for every position at once
        h = x.new_zeros(B, H)
        c = x.new_zeros(B, H)
        y = x.new_zeros(B, S, H)
        rows = torch.arange(B, device=x.device)
        for s in range(int(lens.max())):
            idx = rows[lens > s]  # the sequences still running at step s
            pos = lens[idx] - 1 - s if reverse else torch.full_like(idx, s)
            z = gx[idx, pos] + h[idx] @ w_hh.T
            zi, zf, zg, zo = z.split(H, dim=1)
            c_new = torch.sigmoid(zf) * c[idx] + torch.sigmoid(zi) * torch.tanh(zg)
            h_new = torch.sigmoid(zo) * torch.tanh(c_new)
            c[idx], h[idx] = c_new, h_new
            y[idx, pos] = h_new
        return y

    def layers(self, seqs: Tensor, seq_lens: Tensor) -> Tensor:
        """The last layer's [fwd | bwd] outputs [B, S, dirs * H], zero at t >= len_b."""
        lens = torch.as_tensor(seq_lens, dtype=torch.int64, device=self.device)
        if bool((lens < 1).any()):
            raise ValueError("a zero sequence length (pack_padded_sequence refuses it)")
        seqs = seqs.to(self.device)
        x = self.sd["embed_tokens.weight"][seqs]
        for layer in range(self.cfg.num_layers):
            outs: List[Tensor] = [self.direction(x, lens, layer, False)]
            if self.cfg.bidirectional:
                outs.append(self.direction(x, lens, layer, True))
            x = torch.cat(outs, dim=-1)
        return x

    def __call__(self, seqs: Tensor, seq_lens: Tensor) -> Tensor:
        """seqs int64 [B, S], seq_lens [B] -> [B, dirs * H] sentence embeddings."""
        y = self.layers(seqs, seq_lens)
        S = seqs.shape[1]
        lens = torch.as_tensor(seq_lens, dtype=torch.int64, device=self.device)
        y = y.clone()
        y[torch.arange(S, device=self.device)[None, :] >= lens[:, None]] = self.cfg.padding_value
        y[seqs.to(self.device) == self.cfg.pad_idx] = float("-inf")
        return y.max(dim=1).values
