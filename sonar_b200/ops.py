"""Thin torch-tensor wrappers over the kernel-level C-ABI entry points.

Used by the parity tests, the micro-benchmarks and ``static_pooling``.  Every
function requires CUDA tensors and launches on torch's current stream; there is
no CPU implementation behind any of them.
"""

from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
from torch import Tensor

from . import _lib
from .speech_encoder import relpos_rows

POOLING_MODES = {"max": _lib.SB_POOL_MAX, "mean": _lib.SB_POOL_MEAN, "last": _lib.SB_POOL_LAST}


def _need_cuda(*tensors: Optional[Tensor]) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("sonar_b200 runs on CUDA tensors only (no CPU fallback exists)")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _out_rows(out: Optional[Tensor], t: int, d: int, device) -> Tensor:
    if out is None:
        return torch.empty((t, d), dtype=torch.bfloat16, device=device)
    assert out.dtype == torch.bfloat16 and out.shape == (t, d) and out.is_contiguous()
    return out


def gemm_bf16(a: Tensor, w: Tensor, bias: Tensor, *, epilogue: str = "bias", residual: Optional[Tensor] = None,
              out_dtype: torch.dtype = torch.bfloat16, out: Optional[Tensor] = None, cta_group: int = 2) -> Tensor:
    """out[M,N] = epi(a[M,K] @ w[N,K]^T + bias[N]); epilogue in {bias, relu, silu, tanh, residual}."""
    _need_cuda(a, w, bias, residual, out)
    assert a.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and bias.dtype == torch.float32
    assert a.dim() == 2 and w.dim() == 2 and a.stride(1) == 1 and w.stride(1) == 1
    m, k = a.shape
    n = w.shape[0]
    assert w.shape[1] == k and bias.numel() == n
    epi = {"bias": _lib.SB_EPI_BIAS, "relu": _lib.SB_EPI_BIAS_RELU, "residual": _lib.SB_EPI_BIAS_RESIDUAL, "silu": 5,
           "tanh": _lib.SB_EPI_BIAS_TANH}[epilogue]
    if out is None:
        out = torch.empty((m, n), dtype=out_dtype, device=a.device)
    assert out.dtype in (torch.bfloat16, torch.float32) and out.stride(1) == 1
    if epilogue == "residual":
        assert residual is not None and residual.dtype == out.dtype and residual.stride(1) == 1
    rc = _lib.load().sb_gemm_bf16(
        a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), out.data_ptr(), out.stride(0),
        1 if out.dtype == torch.float32 else 0, bias.data_ptr(), _ptr(residual),
        residual.stride(0) if residual is not None else 0, m, n, k, epi, cta_group, _stream())
    _lib.check(rc, "sb_gemm_bf16")
    return out


def layernorm(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5) -> Tensor:
    """bf16 LayerNorm(x fp32 [T,D])."""
    _need_cuda(x, gamma, beta)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    rc = _lib.load().sb_layernorm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps, y.data_ptr(),
                                  x.shape[0], x.shape[1], _stream())
    _lib.check(rc, "sb_layernorm")
    return y


def layernorm_dual(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5, *, out32: Optional[Tensor] = None,
                   out16: Optional[Tensor] = None):
    """LayerNorm(x fp32 [T,D]) as fp32 and bf16 rows (``sb_layernorm_dual``, the in-place LayerNorm of the attention
    pooling path) -> (y32, y16).  ``out32`` may be ``x`` itself."""
    _need_cuda(x, gamma, beta, out32, out16)
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
    t, d = x.shape
    assert gamma.dtype == beta.dtype == torch.float32 and gamma.numel() == beta.numel() == d
    if out32 is None:
        out32 = torch.empty((t, d), dtype=torch.float32, device=x.device)
    assert out32.dtype == torch.float32 and out32.shape == (t, d) and out32.is_contiguous()
    out16 = _out_rows(out16, t, d, x.device)
    rc = _lib.load().sb_layernorm_dual(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps, out32.data_ptr(),
                                       out16.data_ptr(), t, d, _stream())
    _lib.check(rc, "sb_layernorm_dual")
    return out32, out16


def cu_seqlens_of(seq_lens) -> Tensor:
    lens = torch.as_tensor(seq_lens, dtype=torch.int64).cpu()
    cu = torch.zeros(lens.numel() + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(lens, 0).to(torch.int32)
    return cu


def fold_layernorm(w: Tensor, bias: Tensor, gamma: Tensor, beta: Tensor):
    """LayerNorm folding, weight side: -> (Wf bf16 [N,K], colsum fp32 [N], bias_f fp32 [N])."""
    _need_cuda(w, bias, gamma, beta)
    assert w.dtype == torch.bfloat16 and w.is_contiguous()
    n, k = w.shape
    wf = torch.empty_like(w)
    colsum = torch.empty((n,), dtype=torch.float32, device=w.device)
    bias_f = torch.empty((n,), dtype=torch.float32, device=w.device)
    rc = _lib.load().sb_fold_layernorm(w.data_ptr(), bias.data_ptr(), gamma.data_ptr(), beta.data_ptr(), n, k, wf.data_ptr(),
                                       colsum.data_ptr(), bias_f.data_ptr(), _stream())
    _lib.check(rc, "sb_fold_layernorm")
    return wf, colsum, bias_f


def gemm_residual_stats(a: Tensor, w: Tensor, bias: Tensor, x: Tensor):
    """x += a . w^T + bias in place (fp32); -> (h = bf16(x) [M,N], stats fp32 [M, N/128, 2]): partial 2*t + g holds (mean, M2)
    of column half g of 256-column tile t of the new row, i.e. of columns 256 t + 128 g ... 256 t + 128 g + 127."""
    _need_cuda(a, w, bias, x)
    m, k = a.shape
    n = w.shape[0]
    assert x.shape == (m, n) and x.dtype == torch.float32 and x.is_contiguous() and n % 256 == 0
    h = torch.empty((m, n), dtype=torch.bfloat16, device=a.device)
    stats = torch.empty((m, n // 128, 2), dtype=torch.float32, device=a.device)
    rc = _lib.load().sb_gemm_residual_stats(a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), x.data_ptr(), n,
                                            bias.data_ptr(), h.data_ptr(), n, stats.data_ptr(), m, n, k, _stream())
    _lib.check(rc, "sb_gemm_residual_stats")
    return h, stats


def gemm_residual_splitk(a: Tensor, w: Tensor, bias: Tensor, x: Tensor, counters: Tensor) -> Tensor:
    """x += a . w^T + bias in place (fp32) with the decoder step's ordered split-K (``sb_gemm_residual_splitk``);
    ``counters``: zero-initialised int32 device tensor with >= 4 * (M/256 * N/256) entries, left zero."""
    _need_cuda(a, w, bias, x, counters)
    m, k = a.shape
    n = w.shape[0]
    assert x.shape == (m, n) and x.dtype == torch.float32 and x.is_contiguous() and counters.dtype == torch.int32
    rc = _lib.load().sb_gemm_residual_splitk(a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), x.data_ptr(), n,
                                             bias.data_ptr(), m, n, k, counters.data_ptr(), counters.numel(), _stream())
    _lib.check(rc, "sb_gemm_residual_splitk")
    return x


def gemm_ln_consumer(a: Tensor, wf: Tensor, bias_f: Tensor, colsum: Tensor, stats: Tensor, eps: float = 1e-5,
                     relu: bool = False) -> Tensor:
    """bf16 [M,N] = [relu](rstd * (a . wf^T - mean * colsum) + bias_f), (mean, rstd) merged from stats [M, K/128, 2]
    (any partition of the row into 128-column subsets)."""
    _need_cuda(a, wf, bias_f, colsum, stats)
    m, k = a.shape
    n = wf.shape[0]
    out = torch.empty((m, n), dtype=torch.bfloat16, device=a.device)
    rc = _lib.load().sb_gemm_ln_consumer(a.data_ptr(), a.stride(0), wf.data_ptr(), wf.stride(0), out.data_ptr(), n,
                                         bias_f.data_ptr(), colsum.data_ptr(), stats.data_ptr(), eps, m, n, k,
                                         1 if relu else 0, _stream())
    _lib.check(rc, "sb_gemm_ln_consumer")
    return out


def attention(qkv: Tensor, cu_seqlens: Tensor, num_heads: int, *, out: Optional[Tensor] = None) -> Tensor:
    """Packed bidirectional MHA: qkv bf16 [T, 3*64*H] -> bf16 [T, 64*H]."""
    _need_cuda(qkv, cu_seqlens, out)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and cu_seqlens.dtype == torch.int32
    t = qkv.shape[0]
    d = 64 * num_heads
    assert qkv.shape[1] == 3 * d
    out = _out_rows(out, t, d, qkv.device)
    rc = _lib.load().sb_attention(qkv.data_ptr(), cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, num_heads, t,
                                  out.data_ptr(), _stream())
    _lib.check(rc, "sb_attention")
    return out


def embed(ids: Tensor, cu_seqlens: Tensor, table: Tensor, pos_table: Tensor, scale: float, total_tokens: int, *,
          lnfold: bool = False, out: Optional[Tensor] = None, flag: Optional[Tensor] = None):
    """x[cu[b]+t] = table[ids[b,t]] * scale + pos_table[t]  (fp32 [T, D]).  With ``lnfold`` -> (x, h, stats): also the
    LnFold outputs h = bf16(x) [T, D] and stats fp32 [T, D/128, 2], the (mean, M2) of each 128-column chunk of a row.
    An id outside [0, vocab) raises ValueError, unless ``flag`` (int32 device tensor) is given: the kernel then sets
    flag[0] to 1 and embeds row 0 for that id."""
    _need_cuda(ids, cu_seqlens, table, pos_table, out, flag)
    assert ids.dtype == torch.int64 and ids.stride(1) == 1 and table.dtype == torch.bfloat16
    b, s = ids.shape
    d = table.shape[1]
    if out is None:
        out = torch.empty((total_tokens, d), dtype=torch.float32, device=ids.device)
    assert out.dtype == torch.float32 and out.shape == (total_tokens, d) and out.is_contiguous()
    h = stats = None
    if lnfold:
        h = torch.empty((total_tokens, d), dtype=torch.bfloat16, device=ids.device)
        stats = torch.empty((total_tokens, d // 128, 2), dtype=torch.float32, device=ids.device)
    err = torch.zeros(1, dtype=torch.int32, device=ids.device) if flag is None else flag
    assert err.dtype == torch.int32
    rc = _lib.load().sb_embed(ids.data_ptr(), ids.stride(0), cu_seqlens.data_ptr(), b, s, table.data_ptr(),
                              table.shape[0], pos_table.data_ptr(), pos_table.shape[0], d, scale, out.data_ptr(),
                              err.data_ptr(), _ptr(h), _ptr(stats), _stream())
    _lib.check(rc, "sb_embed")
    if flag is None and int(err.item()) != 0:
        raise ValueError("sb_embed: token id outside [0, vocab_size)")
    return (out, h, stats) if lnfold else out


def pool_packed(x: Tensor, cu_seqlens: Tensor, pooling: str, *, gamma: Optional[Tensor] = None,
                beta: Optional[Tensor] = None, eps: float = 1e-5, encoded_seq_len: int = 0):
    """(optional LayerNorm +) pooling of packed rows fp32 [T,D] -> fp32 [B,D]
    (and, if ``encoded_seq_len`` > 0, the padded [B,S,D] states)."""
    _need_cuda(x, cu_seqlens, gamma, beta)
    assert x.dtype == torch.float32 and x.is_contiguous()
    b = cu_seqlens.numel() - 1
    d = x.shape[1]
    out = torch.empty((b, d), dtype=torch.float32, device=x.device)
    enc = torch.empty((b, encoded_seq_len, d), dtype=torch.float32, device=x.device) if encoded_seq_len > 0 else None
    rc = _lib.load().sb_pool(x.data_ptr(), cu_seqlens.data_ptr(), b, d, _ptr(gamma), _ptr(beta), eps,
                             1 if gamma is not None else 0, POOLING_MODES[pooling.lower()], out.data_ptr(),
                             _ptr(enc), encoded_seq_len, _stream())
    _lib.check(rc, "sb_pool")
    return (out, enc) if enc is not None else out


def pool_latent_attention(qt: Tensor, mem: Tensor, cu_seqlens: Tensor, *, out: Optional[Tensor] = None) -> Tensor:
    """The attention pooler's cross-attention on the absorbed form: qt bf16 [B, Hd, D] (Hd <= 16 queries per sentence),
    mem bf16 [T, D] packed rows, cu_seqlens int32 [B+1] -> u bf16 [B, Hd, D] with
    u[b, h] = softmax_t(qt[b, h] . mem[t] / 8) . mem over the rows of sentence b (zeros for an empty sentence)."""
    _need_cuda(qt, mem, cu_seqlens, out)
    assert qt.dtype == torch.bfloat16 and mem.dtype == torch.bfloat16 and cu_seqlens.dtype == torch.int32
    assert qt.is_contiguous() and mem.is_contiguous() and qt.dim() == 3 and mem.dim() == 2
    b, hd, d = qt.shape
    assert mem.shape[1] == d and cu_seqlens.numel() == b + 1
    u = torch.empty_like(qt) if out is None else out
    assert u.dtype == torch.bfloat16 and u.shape == qt.shape and u.is_contiguous()
    rc = _lib.load().sb_pool_latent_attention(qt.data_ptr(), mem.data_ptr(), cu_seqlens.data_ptr(), b, hd, d,
                                              u.data_ptr(), _stream())
    _lib.check(rc, "sb_pool_latent_attention")
    return u


RELPOS_IMPLS = {"wgmma": 0, "mma_sync": 1}


def attention_relpos(qkv: Tensor, p: Tensor, u_bias: Tensor, v_bias: Tensor, cu_seqlens: Tensor, num_heads: int, *,
                     impl: str = "wgmma", out: Optional[Tensor] = None) -> Tensor:
    """The Conformer's Transformer-XL relative-position self-attention over packed utterances (``sb_attention_relpos``):
    qkv bf16 [T, 3D] (q | k | v), p bf16 [Npad, D] (row k = r_proj of relative position S_center - 1 - k, S_center = the
    longest utterance, Npad = ``relpos_rows(S_center)``), u_bias / v_bias fp32 [D], cu_seqlens int32 [B+1] -> bf16 [T, D];
    ``impl`` "wgmma" (at most 2047 utterances) or "mma_sync"."""
    _need_cuda(qkv, p, u_bias, v_bias, cu_seqlens, out)
    d = 64 * num_heads
    t = qkv.shape[0]
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (t, 3 * d)
    assert u_bias.dtype == torch.float32 and v_bias.dtype == torch.float32 and u_bias.numel() == v_bias.numel() == d
    assert cu_seqlens.dtype == torch.int32
    s_center = int(cu_seqlens.cpu().diff().max())
    npad = relpos_rows(s_center)
    assert p.dtype == torch.bfloat16 and p.is_contiguous() and p.shape == (npad, d), (tuple(p.shape), npad)
    out = _out_rows(out, t, d, qkv.device)
    code = RELPOS_IMPLS[impl]
    qu = qv = vp = None
    if code == 0:
        qu = torch.empty((t, d), dtype=torch.bfloat16, device=qkv.device)
        qv = torch.empty_like(qu)
    else:
        vp = torch.empty((num_heads, npad), dtype=torch.float32, device=qkv.device)
    rc = _lib.load().sb_attention_relpos(qkv.data_ptr(), p.data_ptr(), u_bias.data_ptr(), v_bias.data_ptr(),
                                         cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, num_heads, t, npad, s_center, code,
                                         _ptr(qu), _ptr(qv), _ptr(vp), out.data_ptr(), _stream())
    _lib.check(rc, "sb_attention_relpos")
    return out


def conformer_conv(g: Tensor, cu_seqlens: Tensor, dw: Tensor, bn_scale: Tensor, bn_shift: Tensor, *,
                   out: Optional[Tensor] = None) -> Tensor:
    """The Conformer convolution module between its pointwise convolutions (``sb_conformer_conv``): g bf16 [T, 2D]
    (value | gate) -> bf16 [T, D] = SiLU(bn_scale * depthwise_conv(value * sigmoid(gate)) + bn_shift), dw fp32 [D, 31],
    zero padding at each utterance's ends."""
    _need_cuda(g, cu_seqlens, dw, bn_scale, bn_shift, out)
    t, d2 = g.shape
    d = d2 // 2
    assert g.dtype == torch.bfloat16 and g.is_contiguous() and cu_seqlens.dtype == torch.int32
    assert dw.dtype == torch.float32 and dw.is_contiguous() and dw.shape == (d, 31)
    assert bn_scale.dtype == bn_shift.dtype == torch.float32 and bn_scale.numel() == bn_shift.numel() == d
    max_len = int(cu_seqlens.cpu().diff().max())
    out = _out_rows(out, t, d, g.device)
    rc = _lib.load().sb_conformer_conv(g.data_ptr(), cu_seqlens.data_ptr(), cu_seqlens.numel() - 1, max_len, d, dw.data_ptr(),
                                       bn_scale.data_ptr(), bn_shift.data_ptr(), out.data_ptr(), _stream())
    _lib.check(rc, "sb_conformer_conv")
    return out


def speech_frontend(fbank: Tensor, cu_seqlens: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5, *,
                    out: Optional[Tensor] = None) -> Tensor:
    """The speech frontend's frame stacking and LayerNorm (``sb_speech_frontend``): fbank fp32 [B, padded_frames, 80],
    cu_seqlens int32 [B+1] of positions (= frames // 2) -> bf16 [T, 192], row cu[b] + t = LayerNorm(160) of frames 2t, 2t+1,
    columns 160..191 zero."""
    _need_cuda(fbank, cu_seqlens, gamma, beta, out)
    assert fbank.dtype == torch.float32 and fbank.is_contiguous() and fbank.dim() == 3 and fbank.shape[2] == 80
    assert gamma.dtype == beta.dtype == torch.float32 and gamma.numel() == beta.numel() == 160
    assert cu_seqlens.dtype == torch.int32 and cu_seqlens.numel() == fbank.shape[0] + 1
    cu = cu_seqlens.cpu()
    max_len, t = int(cu.diff().max()), int(cu[-1])
    out = _out_rows(out, t, 192, fbank.device)
    rc = _lib.load().sb_speech_frontend(fbank.data_ptr(), fbank.shape[1], cu_seqlens.data_ptr(), fbank.shape[0], max_len,
                                        gamma.data_ptr(), beta.data_ptr(), eps, out.data_ptr(), _stream())
    _lib.check(rc, "sb_speech_frontend")
    return out


def decoder_embed(tokens: Tensor, embed: Tensor, pos_row: Tensor, scale: float, *, out: Optional[Tensor] = None):
    """The decoder step's embedding (``sb_decoder_embed``): tokens int64 [R], embed bf16 [V, D], pos_row fp32 [D] ->
    (x fp32 [R, D] = embed[tokens] * scale + pos_row, flag): flag is True if an id lay outside [0, V) (row 0 embedded)."""
    _need_cuda(tokens, embed, pos_row, out)
    assert tokens.dtype == torch.int64 and tokens.is_contiguous() and tokens.dim() == 1
    assert embed.dtype == torch.bfloat16 and embed.is_contiguous() and pos_row.dtype == torch.float32 and pos_row.is_contiguous()
    r, (v, d) = tokens.numel(), embed.shape
    assert pos_row.numel() == d
    if out is None:
        out = torch.empty((r, d), dtype=torch.float32, device=tokens.device)
    assert out.dtype == torch.float32 and out.shape == (r, d) and out.is_contiguous()
    err = torch.zeros(1, dtype=torch.int32, device=tokens.device)
    rc = _lib.load().sb_decoder_embed(tokens.data_ptr(), embed.data_ptr(), v, pos_row.data_ptr(), d, scale, out.data_ptr(), r,
                                      err.data_ptr(), _stream())
    _lib.check(rc, "sb_decoder_embed")
    return out, bool(err.item())


def decoder_attention(qkv: Tensor, kcache: Tensor, vcache: Tensor, table: Tensor, t: int, num_heads: int, *,
                      out: Optional[Tensor] = None) -> Tensor:
    """The decoder step's cached self-attention at position t of one layer (``sb_decoder_attention``): qkv bf16 [R, 3D],
    kcache / vcache bf16 [R, Tmax, D] (updated in place: row r, position t <- k / v of qkv row r), table int32 [R, Tmax]
    (table[r, t'] = cache row of position t' < t of hypothesis r) -> bf16 [R, D] = softmax(q . k / 8) . v over 0..t."""
    _need_cuda(qkv, kcache, vcache, table, out)
    d = 64 * num_heads
    r = qkv.shape[0]
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape == (r, 3 * d)
    tmax = kcache.shape[1]
    for c in (kcache, vcache):
        assert c.dtype == torch.bfloat16 and c.is_contiguous() and c.shape == (r, tmax, d)
    assert table.dtype == torch.int32 and table.is_contiguous() and table.shape == (r, tmax)
    out = _out_rows(out, r, d, qkv.device)
    rc = _lib.load().sb_decoder_attention(qkv.data_ptr(), kcache.data_ptr(), vcache.data_ptr(), table.data_ptr(), t, r, tmax,
                                          num_heads, out.data_ptr(), _stream())
    _lib.check(rc, "sb_decoder_attention")
    return out


def decoder_add_const_layernorm(x: Tensor, c: Tensor, beam: int, gamma: Tensor, beta: Tensor, eps: float = 1e-5, *,
                                out: Optional[Tensor] = None) -> Tensor:
    """The decoder layer's cross-attention residual and FFN LayerNorm (``sb_decoder_add_const_layernorm``): x fp32 [R, D]
    += c[r // beam] in place (c fp32 [R / beam, D]) -> h bf16 [R, D] = LayerNorm(x) * gamma + beta."""
    _need_cuda(x, c, gamma, beta, out)
    r, d = x.shape
    assert x.dtype == c.dtype == torch.float32 and x.is_contiguous() and c.is_contiguous()
    assert c.shape == ((r + beam - 1) // beam, d) and gamma.numel() == beta.numel() == d
    out = _out_rows(out, r, d, x.device)
    rc = _lib.load().sb_decoder_add_const_layernorm(x.data_ptr(), c.data_ptr(), r, beam, d, gamma.data_ptr(), beta.data_ptr(),
                                                    eps, out.data_ptr(), _stream())
    _lib.check(rc, "sb_decoder_add_const_layernorm")
    return out


def decoder_vocab_chunks(rows: int, vocab: int) -> int:
    """The number of column chunks the decoder step splits a vocabulary sweep of `rows` rows into."""
    n = C.c_int32()
    _lib.check(_lib.load().sb_decoder_vocab_chunks(rows, vocab, C.byref(n)), "sb_decoder_vocab_chunks")
    return n.value


def decoder_vocab_head(h: Tensor, embed: Tensor, eos_idx: int, probe_tokens: Optional[Tensor] = None, *, n_chunks: int = 0,
                       out: Optional[tuple] = None):
    """The decoder step's vocabulary head (``sb_decoder_vocab_head``): h bf16 [R, D], embed bf16 [V, D] ->
    (lprob fp32 [R, 16], tok int32 [R, 16], eos fp32 [R], probe fp32 [R] or None): the 16 best log-softmax values of
    h . embed^T by (value desc, token asc), log P(eos_idx) and log P(probe_tokens[r]).  ``n_chunks`` = 0 is the step's own
    split of the vocabulary; ``out`` optionally gives the four output tensors."""
    _need_cuda(h, embed, probe_tokens)
    assert h.dtype == embed.dtype == torch.bfloat16 and h.is_contiguous() and embed.is_contiguous()
    (r, d), v = h.shape, embed.shape[0]
    assert embed.shape[1] == d
    chunks = n_chunks if n_chunks > 0 else decoder_vocab_chunks(r, v)
    lists = 2 * chunks
    cand_val = torch.empty((r, lists, 16), dtype=torch.float32, device=h.device)
    cand_idx = torch.empty((r, lists, 16), dtype=torch.int32, device=h.device)
    lse_part = torch.empty((r, lists, 2), dtype=torch.float32, device=h.device)
    if out is None:
        out = (torch.empty((r, 16), dtype=torch.float32, device=h.device), torch.empty((r, 16), dtype=torch.int32, device=h.device),
               torch.empty((r,), dtype=torch.float32, device=h.device),
               None if probe_tokens is None else torch.empty((r,), dtype=torch.float32, device=h.device))
    lprob, tok, eos, probe = out
    _need_cuda(lprob, tok, eos, probe)
    assert lprob.shape == tok.shape == (r, 16) and eos.shape == (r,) and lprob.is_contiguous() and tok.is_contiguous()
    assert lprob.dtype == eos.dtype == torch.float32 and tok.dtype == torch.int32
    assert (probe is None) == (probe_tokens is None)
    if probe_tokens is not None:
        assert probe_tokens.dtype == torch.int64 and probe_tokens.shape == (r,) and probe.shape == (r,)
        assert probe.dtype == torch.float32
    rc = _lib.load().sb_decoder_vocab_head(h.data_ptr(), embed.data_ptr(), r, v, d, eos_idx, _ptr(probe_tokens), n_chunks,
                                           cand_val.data_ptr(), cand_idx.data_ptr(), lse_part.data_ptr(), lprob.data_ptr(),
                                           tok.data_ptr(), eos.data_ptr(), _ptr(probe), _stream())
    _lib.check(rc, "sb_decoder_vocab_head")
    return lprob, tok, eos, probe


LSTM_TILE_ROWS = 64  # sequences per tile of the LSTM recurrent kernel


def lstm_gate_rows(hidden_size: int = 512, num_dirs: int = 1) -> Tensor:
    """int64 [num_dirs * 4H]: entry n is the row of torch.nn.LSTM's stacked [i | f | g | o] gate matrices (of direction
    n // 4H) that row n of the LSTM kernels' gate order holds: row 128 c + 32 gate + u is gate `gate` of hidden unit
    32 c + u, so each 16th of the hidden units has its four gates together."""
    n = torch.arange(4 * hidden_size)
    one = (n % 128) // 32 * hidden_size + n // 128 * 32 + n % 32
    return torch.cat([one + d * 4 * hidden_size for d in range(num_dirs)])


def lstm_recurrent(g: Tensor, w_hh: Tensor, cu_seqlens: Tensor, tile_seqs: Tensor, num_dirs: int, *,
                   pool: bool = False, pad_mask: Optional[Tensor] = None, tail_keep: Optional[Tensor] = None,
                   padding_value: float = 0.0, out: Optional[Tensor] = None) -> Tensor:
    """The LSTM recurrence (H = 512) of one layer on packed tokens, everything in ``lstm_gate_rows`` order:
    g bf16 [T, num_dirs * 4H] input pre-activations (x . W_ih^T + b_ih + b_hh; may be a column view of a wider buffer),
    w_hh bf16 [num_dirs * 4H, H], cu_seqlens int32 [B + 1], tile_seqs int32 [tiles * 64] (sequence per tile row,
    -1 = empty).  Returns the outputs bf16 [T, num_dirs * H], or with ``pool`` fp32 [B, num_dirs * H]: the max over each
    sequence's tokens, skipping those with pad_mask (uint8 [T]) set, then max with ``padding_value`` where tail_keep
    (uint8 [B]) is set; rows of sequences missing from tile_seqs are left uninitialised.  ``out`` may give that output
    as a caller-owned view with unit column stride (its row stride may be wider than the data); only its rows and
    columns are written."""
    _need_cuda(g, w_hh, cu_seqlens, tile_seqs, pad_mask, tail_keep, out)
    assert g.dtype == torch.bfloat16 and w_hh.dtype == torch.bfloat16 and g.stride(1) == 1 and w_hh.is_contiguous()
    assert cu_seqlens.dtype == torch.int32 and tile_seqs.dtype == torch.int32 and tile_seqs.numel() % LSTM_TILE_ROWS == 0
    h = w_hh.shape[1]
    assert w_hh.shape[0] == num_dirs * 4 * h and g.shape[1] >= num_dirs * 4 * h
    for m in (pad_mask, tail_keep):
        assert m is None or m.dtype == torch.uint8
    t, b = g.shape[0], cu_seqlens.numel() - 1
    shape, dtype = ((b, num_dirs * h), torch.float32) if pool else ((t, num_dirs * h), torch.bfloat16)
    if out is None:
        out = torch.empty(shape, dtype=dtype, device=g.device)
    assert out.dtype == dtype and tuple(out.shape) == shape and out.stride(1) == 1
    y, pool_out, ld = (None, out, out.stride(0)) if pool else (out, None, out.stride(0))
    rc = _lib.load().sb_lstm_recurrent(g.data_ptr(), g.stride(0), w_hh.data_ptr(), cu_seqlens.data_ptr(), tile_seqs.data_ptr(),
                                       tile_seqs.numel() // LSTM_TILE_ROWS, num_dirs, _ptr(y), ld, _ptr(pool_out), ld,
                                       _ptr(pad_mask), _ptr(tail_keep), padding_value, _stream())
    _lib.check(rc, "sb_lstm_recurrent")
    return out


def laser_embed(ids: Tensor, cu_seqlens: Tensor, table: Tensor, pad_idx: int, *, seq_len: Optional[int] = None,
                out: Optional[tuple] = None, flag: Optional[Tensor] = None):
    """The LASER2 embedding gather (``sb_laser2_embed``): ids int64 [B, W] with unit column stride (seq_len <= W,
    default W), cu_seqlens int32 [B + 1] (lengths <= seq_len), table bf16 [V, D] -> (x bf16 [T, D], pad uint8 [T],
    tail uint8 [B], flag int32 [1]): x row cu[b] + t = table[ids[b, t]], pad = (id == pad_idx), tail[b] = some id at
    len_b <= t < seq_len differs from pad_idx; an id outside [0, V) gathers zeros and sets flag[0] to 1 (``flag`` is
    not cleared first).  ``out`` optionally gives (x, pad, tail), pad and tail contiguous with at least T and B
    entries."""
    _need_cuda(ids, cu_seqlens, table, flag)
    assert ids.dtype == torch.int64 and ids.dim() == 2 and ids.stride(1) == 1 and cu_seqlens.dtype == torch.int32
    assert table.dtype == torch.bfloat16 and table.is_contiguous()
    b = ids.shape[0]
    s = ids.shape[1] if seq_len is None else seq_len
    (v, d), t = table.shape, int(cu_seqlens[-1])
    assert cu_seqlens.numel() == b + 1 and s <= ids.shape[1] <= ids.stride(0)
    if out is None:
        out = (torch.empty((t, d), dtype=torch.bfloat16, device=ids.device), torch.empty(t, dtype=torch.uint8, device=ids.device),
               torch.empty(b, dtype=torch.uint8, device=ids.device))
    x, pad, tail = out
    _need_cuda(x, pad, tail)
    assert x.dtype == torch.bfloat16 and x.shape == (t, d) and x.is_contiguous()
    assert pad.dtype == tail.dtype == torch.uint8 and pad.is_contiguous() and tail.is_contiguous()
    assert pad.numel() >= t and tail.numel() >= b
    if flag is None:
        flag = torch.zeros(1, dtype=torch.int32, device=ids.device)
    assert flag.dtype == torch.int32
    rc = _lib.load().sb_laser2_embed(ids.data_ptr(), ids.stride(0), cu_seqlens.data_ptr(), b, s, table.data_ptr(), v, d,
                                     pad_idx, x.data_ptr(), pad.data_ptr(), tail.data_ptr(), flag.data_ptr(), _stream())
    _lib.check(rc, "sb_laser2_embed")
    return x, pad, tail, flag


class _DeviceArray:
    """A borrowed device buffer seen through ``__cuda_array_interface__`` (no copy)."""

    def __init__(self, ptr: int, shape: tuple, typestr: str) -> None:
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3}


def laser2_layer_weights(model, layer: int):
    """Copies of a ``B200LaserLstmEncoder``'s repacked weights of one layer (``sb_laser2_layer_weights``):
    (w_ih bf16 [dirs * 4H, in], bias fp32 [dirs * 4H], w_hh bf16 [dirs * 4H, H]), rows in ``lstm_gate_rows`` order."""
    cfg = model.config
    dirs, h = (2 if cfg.bidirectional else 1), cfg.hidden_size
    n, k = dirs * 4 * h, (cfg.model_dim if layer == 0 else dirs * h)
    w_ih, bias, w_hh = C.c_void_p(), C.c_void_p(), C.c_void_p()
    _lib.check(model._lib.sb_laser2_layer_weights(model._handle, layer, C.byref(w_ih), C.byref(bias), C.byref(w_hh)),
               "sb_laser2_layer_weights")
    dev = model.device

    def view(p, shape, typestr):
        return torch.as_tensor(_DeviceArray(p.value, shape, typestr), device=dev).clone()

    return (view(w_ih, (n, k), "<i2").view(torch.bfloat16), view(bias, (n,), "<f4"),
            view(w_hh, (n, h), "<i2").view(torch.bfloat16))


def blaser_featurize(src: Tensor, mt: Tensor, ref: Optional[Tensor], input_form: str, *, normalize: bool = False,
                     out_dtype: torch.dtype = torch.float32) -> Tensor:
    """BLASER's feature rows of fp32 [N, E] embeddings (``sb_blaser_featurize``): COMET [ref, mt, src*mt, ref*mt,
    |mt-src|, |mt-ref|] or QE [src, mt, src*mt, |mt-src|] (ref unused), of the rows as given or, with ``normalize``,
    after ``F.normalize``; out_dtype fp32 or bf16."""
    _need_cuda(src, mt, ref)
    qe = {"COMET": False, "QE": True}[input_form]
    for t in (src, mt) + (() if qe else (ref,)):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.shape == src.shape and t.dim() == 2
    n, e = src.shape
    out = torch.empty((n, (4 if qe else 6) * e), dtype=out_dtype, device=src.device)
    rc = _lib.load().sb_blaser_featurize(src.data_ptr(), mt.data_ptr(), None if qe else ref.data_ptr(), e, n, e,
                                         _lib.SB_BLASER_QE if qe else _lib.SB_BLASER_COMET, int(normalize),
                                         out.data_ptr(), int(out_dtype == torch.float32), _stream())
    _lib.check(rc, "sb_blaser_featurize")
    return out
