"""xsim cosine-margin mining over sentence embeddings on the H100 (BASELINE.json config 5).

``knn`` / ``knn_bidir`` / ``xsim`` run entirely in ``libsonar_b200.so`` (``sb_xsim_knn``: wgmma GEMM with a fused
running top-k, exact fp64 re-rank; ``sb_xsim_knn_bidir``: both directions from one pass; ``sb_xsim_margin_predict``).
``xsim_distributed`` shards the query rows over the ranks of a ``torch.distributed`` group: one all-gather assembles the
y matrix on every rank (the single exchange step of the path, SURVEY §8e), each rank scores its row block against it once
(forward k-NN + its share of the reverse k-NN), and a second, small all-gather merges the reverse lists.
"""

from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _lib
from .ops import _need_cuda

_MARGINS = {"absolute": 0, "ratio": 1, "distance": 2}


def _need_cuda_f32(t: Tensor) -> Tensor:
    _need_cuda(t)
    return t.float().contiguous()


def knn(x: Tensor, y: Tensor, k: int = 4) -> Tuple[Tensor, Tensor]:
    """Exact-cosine k nearest rows of ``y`` for every row of ``x`` -> (cos fp64 [n,k], idx int32 [n,k])."""
    x, y = _need_cuda_f32(x), _need_cuda_f32(y)
    n, d = x.shape
    m = y.shape[0]
    assert y.shape[1] == d
    lib = _lib.load()
    ws = torch.empty(_lib.workspace_bytes(lib.sb_xsim_workspace_bytes, n, m, d), dtype=torch.uint8, device=x.device)
    val = torch.empty((n, k), dtype=torch.float64, device=x.device)
    idx = torch.empty((n, k), dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        rc = lib.sb_xsim_knn(x.data_ptr(), y.data_ptr(), n, m, d, k, val.data_ptr(), idx.data_ptr(), ws.data_ptr(),
                             ws.numel(), torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, "sb_xsim_knn")
    return val, idx


def knn_bidir(x: Tensor, y: Tensor, k: int = 4, stats: Optional[dict] = None) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """Both k-NN directions from ONE pass over the similarity matrix (``sb_xsim_knn_bidir``):
    -> (cos_xy fp64 [n,k], idx_xy int32 [n,k], cos_yx fp64 [m,k], idx_yx int32 [m,k]); ``idx_yx`` indexes rows of ``x``.
    The reverse direction's candidates are the products above per-column thresholds -- a y row's 16th best bf16 score
    against every 8th x row, which cannot exceed its 16th best over all of them, so the result equals ``knn(y, x)`` for any
    data; the few y rows that collect more candidates than their buffer holds (ties, duplicates; marked
    ``idx = -2`` by the kernel) are redone with the plain one-direction search against all of x (``stats["overflow_rows"]``
    reports how many, when a dict is passed)."""
    x, y = _need_cuda_f32(x), _need_cuda_f32(y)
    n, d = x.shape
    m = y.shape[0]
    assert y.shape[1] == d
    lib = _lib.load()
    ws = torch.empty(_lib.workspace_bytes(lib.sb_xsim_bidir_workspace_bytes, n, m, d), dtype=torch.uint8, device=x.device)
    val_xy = torch.empty((n, k), dtype=torch.float64, device=x.device)
    idx_xy = torch.empty((n, k), dtype=torch.int32, device=x.device)
    val_yx = torch.empty((m, k), dtype=torch.float64, device=x.device)
    idx_yx = torch.empty((m, k), dtype=torch.int32, device=x.device)
    overflow = torch.zeros(1, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        rc = lib.sb_xsim_knn_bidir(x.data_ptr(), y.data_ptr(), n, m, d, k, val_xy.data_ptr(), idx_xy.data_ptr(),
                                   val_yx.data_ptr(), idx_yx.data_ptr(), overflow.data_ptr(), ws.data_ptr(), ws.numel(),
                                   torch.cuda.current_stream(x.device).cuda_stream)
    _lib.check(rc, "sb_xsim_knn_bidir")
    del ws
    n_over = int(overflow.item())
    if stats is not None:
        stats["overflow_rows"] = n_over
    if n_over != 0:  # rows of y whose candidate buffer overflowed: one-direction search for just those rows
        rows = (idx_yx[:, 0] == -2).nonzero(as_tuple=True)[0]
        v2, i2 = knn(y[rows].contiguous(), x, k)
        val_yx[rows] = v2
        idx_yx[rows] = i2
    return val_xy, idx_xy, val_yx, idx_yx


def margin_predict(val_xy: Tensor, idx_xy: Tensor, val_yx: Optional[Tensor], m: int, margin: str = "ratio") -> Tensor:
    n, k = val_xy.shape
    pred = torch.empty((n,), dtype=torch.int32, device=val_xy.device)
    lib = _lib.load()
    with torch.cuda.device(val_xy.device):
        rc = lib.sb_xsim_margin_predict(val_xy.data_ptr(), idx_xy.data_ptr(),
                                        val_yx.data_ptr() if val_yx is not None else None, n, m, k, _MARGINS[margin],
                                        pred.data_ptr(), torch.cuda.current_stream(val_xy.device).cuda_stream)
    _lib.check(rc, "sb_xsim_margin_predict")
    return pred


def xsim(x: Tensor, y: Tensor, margin: str = "ratio", k: int = 4) -> Tuple[int, int, Tensor]:
    """LASER-style xsim: row i of ``x`` should retrieve row i of ``y``.  -> (errors, n, predictions int32 [n])."""
    if margin not in _MARGINS:
        raise ValueError(f"margin must be one of {sorted(_MARGINS)}")
    if margin == "absolute":
        val_xy, idx_xy = knn(x, y, k)
        val_yx = None
    else:  # both directions from one pass over x . y^T
        val_xy, idx_xy, val_yx, _ = knn_bidir(x, y, k)
    pred = margin_predict(val_xy, idx_xy, val_yx, y.shape[0], margin)
    n = x.shape[0]
    err = int((pred.long() != torch.arange(n, device=pred.device)).sum().item())
    return err, n, pred


def _xsim_distributed_impl(x_shard: Tensor, y_shard: Tensor, margin: str, k: int, group, knn_fn, margin_fn, knn_bidir_fn):
    """Collective plumbing of ``xsim_distributed`` with the compute steps passed in as callables (the gloo test in
    ``tests/test_distributed_gloo.py`` drives it with a CPU checker; the public function below binds the CUDA kernels).

    Only the y matrix is gathered (the one exchange step of the path, SURVEY §8e).  Every rank scores its x rows against
    all of y ONCE and gets both its forward k-NN and, for every y row, the k best of ITS x rows; the reverse lists
    (``[N, k]`` per rank) are all-gathered and merged per y row -- 1/16 of the bytes of gathering x as well."""
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    ns, d = x_shard.shape
    y_all = torch.empty((world * ns, d), dtype=torch.float32, device=x_shard.device)
    dist.all_gather_into_tensor(y_all, y_shard, group=group)  # the exchange step: [N,1024] on every rank
    val_yx_all = None
    if margin == "absolute":
        val_xy, idx_xy = knn_fn(x_shard, y_all, k)
    else:
        val_xy, idx_xy, val_yx_loc, _ = knn_bidir_fn(x_shard, y_all, k)  # reverse lists over this rank's x rows: [N, k]
        val_yx_loc = val_yx_loc.contiguous()
        m_all = val_yx_loc.shape[0]
        gathered = torch.empty((world * m_all, k), dtype=val_yx_loc.dtype, device=val_yx_loc.device)
        dist.all_gather_into_tensor(gathered, val_yx_loc, group=group)  # rank-major blocks of [N, k]
        merged = gathered.view(world, m_all, k).permute(1, 0, 2).reshape(m_all, world * k)
        val_yx_all = torch.topk(merged, k, dim=1).values.contiguous()  # k best cosines of every y row over ALL x rows
    pred = margin_fn(val_xy, idx_xy, val_yx_all, world * ns, margin)
    target = torch.arange(rank * ns, (rank + 1) * ns, device=pred.device)
    err = (pred.long() != target).sum()
    dist.all_reduce(err, group=group)
    return int(err.item()), world * ns, pred


def xsim_distributed(x_shard: Tensor, y_shard: Tensor, margin: str = "ratio", k: int = 4, group=None):
    """Every rank holds the same number of rows of x and y (its batch shard of the encoded sentences).
    -> (global errors, global n, predictions for this rank's rows as GLOBAL y indices).  CUDA tensors only."""
    if margin not in _MARGINS:
        raise ValueError(f"margin must be one of {sorted(_MARGINS)}")
    x_shard, y_shard = _need_cuda_f32(x_shard), _need_cuda_f32(y_shard)
    return _xsim_distributed_impl(x_shard, y_shard, margin, k, group, knn, margin_predict, knn_bidir)
