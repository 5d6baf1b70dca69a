"""Tensor-level wrappers over the C ABI (include/b200rec.h) and the autograd nodes built on them.

PyTorch is plumbing here: it owns device memory, streams and the autograd graph the reference's unchanged
runner expects (helpers/BaseRunner.py:193-206).  Every arithmetic step is a kernel in libb200rec.so.

Embedding-table gradients can leave the autograd graph in three forms, selected per table with
``set_table_mode(param, mode)``:
  'dense'   a dense [n_rows, d] tensor, bit-reproducible (one writer per row) -- what the reference's
            nn.Embedding(sparse=False) hands to stock torch.optim (exact reference semantics);
  'sparse'  a coalesced torch.sparse_coo tensor (unique rows only) for torch.optim.SparseAdam/SGD/Adagrad;
  'fused'   nothing is materialised: the contribution streams are parked on the parameter and
            ``rechorus_b200.optim.RowSparseOptimizer.step()`` reduces and applies them in one kernel.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from . import lib as _lib

# --------------------------------------------------------------------------------------------------
# plumbing
# --------------------------------------------------------------------------------------------------


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise _lib.B200RecError(
                "rechorus_b200 runs on a CUDA device only (got a %s tensor); there is no CPU fallback" % t.device)


def _f32c(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise TypeError(f"{what} must be float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _i64c(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.dtype != torch.int64:
        raise TypeError(f"{what} must be int64 (the reference's collate dtype), got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


_err_flags = {}


def err_flag(device: torch.device) -> torch.Tensor:
    """Per-device int32 counter of out-of-range ids seen by the kernels (they clamp, never read OOB)."""
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key not in _err_flags:
        _err_flags[key] = torch.zeros(1, dtype=torch.int32, device=device)
    return _err_flags[key]


def check_ids(device: Optional[torch.device] = None) -> None:
    """Synchronising poll of the out-of-range counter; raises IndexError like ATen's embedding would."""
    device = device or torch.device("cuda", torch.cuda.current_device())
    flag = err_flag(device)
    bad = int(flag.item())
    if bad:
        flag.zero_()
        raise IndexError(f"{bad} embedding id(s) out of range (kernels clamped them to row 0)")


def poll_ids(device: torch.device) -> None:
    """check_ids, but only if a kernel has used this device's counter yet (cheap no-op before the first forward)"""
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key in _err_flags:
        check_ids(device)


# --------------------------------------------------------------------------------------------------
# kernels, no autograd
# --------------------------------------------------------------------------------------------------

def rowdot(Q: torch.Tensor, qid: Optional[torch.Tensor], T: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """pred[b,c] = <Q[qid[b]], T[ids[b,c]]> (qid None: row b).  BPRMF.py:39-42 / SASRec.py:80-81."""
    _need_cuda(Q, T, ids, qid)
    Q, T, ids = _f32c(Q, "Q"), _f32c(T, "T"), _i64c(ids, "ids")
    if ids.dim() != 2:
        raise ValueError("ids must be [B, C]")
    B, Cn = ids.shape
    d = T.shape[1]
    if Q.shape[1] != d:
        raise ValueError(f"emb width mismatch: Q {Q.shape[1]} vs T {d}")
    if qid is not None:
        qid = _i64c(qid, "qid")
        if qid.numel() != B:
            raise ValueError("qid must have B entries")
    elif Q.shape[0] != B:
        raise ValueError("dense Q must have B rows")
    pred = torch.empty((B, Cn), dtype=torch.float32, device=T.device)
    L = _lib.load()
    _lib.check(L.b2r_rowdot_fwd(_p(Q), _p(qid), Q.shape[0], _p(T), _p(ids), T.shape[0], _p(pred), B, Cn, d,
                                _p(err_flag(T.device)), _stream()), "b2r_rowdot_fwd")
    return pred


def rowdot_bwd_query(g: torch.Tensor, T: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """dQ[b,:] = sum_c g[b,c] * T[ids[b,c],:]  -> dense [B, d], fixed summation order."""
    _need_cuda(g, T, ids)
    g, T, ids = _f32c(g, "g"), _f32c(T, "T"), _i64c(ids, "ids")
    B, Cn = ids.shape
    d = T.shape[1]
    dQ = torch.empty((B, d), dtype=torch.float32, device=T.device)
    L = _lib.load()
    _lib.check(L.b2r_rowdot_bwd_query(_p(g), _p(T), _p(ids), T.shape[0], _p(dQ), B, Cn, d, _stream()),
               "b2r_rowdot_bwd_query")
    return dQ


def gather_rows(T: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """out[..., :] = T[ids[...], :]   (nn.Embedding forward)."""
    _need_cuda(T, ids)
    T, ids = _f32c(T, "T"), _i64c(ids, "ids")
    d = T.shape[1]
    out = torch.empty(tuple(ids.shape) + (d,), dtype=torch.float32, device=T.device)
    L = _lib.load()
    _lib.check(L.b2r_gather_rows(_p(T), _p(ids), T.shape[0], _p(out), ids.numel(), d, _p(err_flag(T.device)),
                                 _stream()), "b2r_gather_rows")
    return out


def pairdot(Q: torch.Tensor, qidx: torch.Tensor, T: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """out[e] = <Q[qidx[e]], T[rows[e]]>, rows[e] < 0 -> 0   (b2r_pairdot_fwd; sharded-table owner side)"""
    _need_cuda(Q, T, qidx, rows)
    Q, T = _f32c(Q, "Q"), _f32c(T, "T")
    qidx, rows = _i64c(qidx.reshape(-1), "qidx"), _i64c(rows.reshape(-1), "rows")
    n = rows.numel()
    out = torch.empty(n, dtype=torch.float32, device=T.device)
    L = _lib.load()
    _lib.check(L.b2r_pairdot_fwd(_p(Q), _p(qidx), Q.shape[0], _p(T), _p(rows), T.shape[0], _p(out), n, T.shape[1],
                                 _p(err_flag(T.device)), _stream()), "b2r_pairdot_fwd")
    return out


def pairdot_p2p(Q: torch.Tensor, qidx: torch.Tensor, T: torch.Tensor, rows: torch.Tensor, out_tab: torch.Tensor,
                seg: int) -> None:
    """pairdot whose score for pair e goes to out_tab[e // seg][e % seg]; out_tab: int64 device tensor of float*
    addresses (peer-mapped receive buffers).  The scoring hop of config 5's default exchange (b2r_pairdot_fwd_p2p)."""
    _need_cuda(Q, qidx, T, rows, out_tab)
    Q, T = _f32c(Q, "Q"), _f32c(T, "T")
    qidx, rows = _i64c(qidx.reshape(-1), "qidx"), _i64c(rows.reshape(-1), "rows")
    out_tab = _i64c(out_tab, "out_tab")
    n = rows.numel()
    if n != out_tab.numel() * int(seg):
        raise ValueError("pairdot_p2p: n must equal len(out_tab) * seg")
    _lib.check(_lib.load().b2r_pairdot_fwd_p2p(_p(Q), _p(qidx), Q.shape[0], _p(T), _p(rows), T.shape[0], _p(out_tab),
                                               int(seg), n, T.shape[1], _p(err_flag(Q.device)), _stream()),
               "b2r_pairdot_fwd_p2p")


def pair_runs_sum(out: torch.Tensor, key: torch.Tensor, rows: torch.Tensor, coef: torch.Tensor, T: torch.Tensor) -> None:
    """out[key[e]] = sum over each contiguous run of valid pairs with that key of coef[e] * T[rows[e]]
    (b2r_pair_runs_sum; rows < 0 = unused slot)"""
    _need_cuda(out, key, rows, coef, T)
    key, rows = _i64c(key.reshape(-1), "key"), _i64c(rows.reshape(-1), "rows")
    coef, T = _f32c(coef.reshape(-1), "coef"), _f32c(T, "T")
    L = _lib.load()
    _lib.check(L.b2r_pair_runs_sum(_p(key), _p(rows), _p(coef), _p(T), T.shape[0], _p(out), out.shape[0], rows.numel(),
                                   T.shape[1], _stream()), "b2r_pair_runs_sum")


def gt_rank(pred: torch.Tensor) -> torch.Tensor:
    """rank[r] = #{c : pred[r, c] >= pred[r, 0]} as int64 on the device (helpers/BaseRunner.py:63)."""
    _need_cuda(pred)
    pred = _f32c(pred, "pred")
    if pred.dim() != 2 or pred.shape[1] < 1:
        raise ValueError("pred must be [N, C] with C >= 1")
    N, Cn = pred.shape
    rank = torch.empty(N, dtype=torch.int64, device=pred.device)
    _lib.check(_lib.load().b2r_gt_rank(_p(pred), N, Cn, Cn, _p(rank), _stream()), "b2r_gt_rank")
    return rank


def rank_histogram(rank: torch.Tensor, kmax: int) -> torch.Tensor:
    """hist[k] = #{rank == k} for k <= kmax, hist[kmax + 1] = #{rank > kmax}; int64 [kmax + 2] on the device."""
    _need_cuda(rank)
    rank = _i64c(rank.reshape(-1), "rank")
    hist = torch.empty(kmax + 2, dtype=torch.int64, device=rank.device)
    _lib.check(_lib.load().b2r_rank_histogram(_p(rank), rank.numel(), int(kmax), _p(hist), _stream()),
               "b2r_rank_histogram")
    return hist


def metrics_from_histogram(hist, n_rows: int, topk, metrics) -> dict:
    """HR@k / NDCG@k of helpers/BaseRunner.py:64-76 from the rank histogram: every row of rank r <= k contributes
    1 (HR) or 1/log2(r+1) (NDCG); the mean is over all n_rows rows."""
    import numpy as np
    h = np.asarray(hist.cpu() if isinstance(hist, torch.Tensor) else hist, dtype=np.int64)
    out = {}
    for k in topk:
        r = np.arange(1, int(k) + 1)
        cnt = h[1:int(k) + 1].astype(np.float64)
        for metric in metrics:
            key = f"{metric}@{k}"
            if metric == "HR":
                out[key] = cnt.sum() / n_rows
            elif metric == "NDCG":
                out[key] = (cnt / np.log2(r + 1)).sum() / n_rows
            else:
                raise ValueError(f"Undefined evaluation metric: {metric}.")
    return out


def rank_all_items(q: torch.Tensor, table: torch.Tensor, target: torch.Tensor,
                   mask_row: Optional[torch.Tensor] = None, mask_item: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Ranks under the test_all protocol (BaseModel.py:194-198 + BaseRunner.py:244-251) without the [B, n_items]
    score matrix: q [B, d] query rows, table [n_items, d], target [B]; (mask_row, mask_item) unique (batch row,
    item id) pairs whose scores the reference overwrites with -inf."""
    _need_cuda(q, table, target, mask_row, mask_item)
    q, table, target = _f32c(q, "q"), _f32c(table, "table"), _i64c(target.reshape(-1), "target")
    if q.dim() != 2 or table.dim() != 2 or q.shape[1] != table.shape[1] or target.numel() != q.shape[0]:
        raise ValueError("rank_all_items: q [B, d], table [n_items, d], target [B]")
    n_mask = 0
    if mask_row is not None:
        mask_row, mask_item = _i64c(mask_row.reshape(-1), "mask_row"), _i64c(mask_item.reshape(-1), "mask_item")
        if mask_row.numel() != mask_item.numel():
            raise ValueError("mask_row and mask_item must have the same length")
        n_mask = mask_row.numel()
    B, d = q.shape
    rank = torch.empty(B, dtype=torch.int64, device=q.device)
    s0 = torch.empty(B, dtype=torch.float32, device=q.device)
    _lib.check(_lib.load().b2r_rank_all_items(_p(q), d, _p(table), _p(target), B, table.shape[0], d,
                                              _p(mask_row) if n_mask else None, _p(mask_item) if n_mask else None,
                                              n_mask, _p(s0), _p(rank), _p(err_flag(q.device)), _stream()),
               "b2r_rank_all_items")
    return rank


def clicked_csr(sets: Sequence[dict], n_users: int):
    """The union of per-user item sets ({user: iterable of item ids}, e.g. corpus.train_clicked_set) as a CSR over
    users: ptr int64 [n_users + 1] and items int64 (at least one slot), user u's items sorted ascending without
    duplicates at items[ptr[u]:ptr[u + 1]].  Users outside [0, n_users) are ignored.  NumPy arrays."""
    import numpy as np
    parts = {}
    for s in sets:
        for u, items in s.items():
            if 0 <= int(u) < n_users and len(items):
                parts.setdefault(int(u), []).append(np.fromiter(items, dtype=np.int64, count=len(items)))
    rows = {u: (np.unique(np.concatenate(p)) if len(p) > 1 else np.sort(p[0])) for u, p in parts.items()}
    ptr = np.zeros(int(n_users) + 1, dtype=np.int64)
    for u, r in rows.items():
        ptr[u + 1] = len(r)
    ptr = np.cumsum(ptr)
    flat = np.zeros(max(int(ptr[-1]), 1), dtype=np.int64)
    for u, r in rows.items():
        flat[ptr[u]:ptr[u + 1]] = r
    return ptr, flat


class ClickedSets:
    """The items BaseRunner.py:244-251 masks under test_all -- train_clicked_set[u] | residual_clicked_set[u] -- as a
    device CSR (clicked_csr): the input of mask_clicked and topk_all_items."""

    def __init__(self, train_clicked_set: dict, residual_clicked_set: dict, n_users: int, device):
        ptr, items = clicked_csr([train_clicked_set, residual_clicked_set], n_users)
        self.n_users = int(n_users)
        self.ptr = torch.from_numpy(ptr).to(device)
        self.items = torch.from_numpy(items).to(device)


def rank_all_items_clicked(q: torch.Tensor, table: torch.Tensor, target: torch.Tensor, users: torch.Tensor,
                           clicked: ClickedSets) -> torch.Tensor:
    """rank_all_items with the masked pairs taken from the clicked-item CSR: row b excludes every item of
    train_clicked_set[users[b]] | residual_clicked_set[users[b]] (BaseRunner.py:244-251).  Same ranks as
    rank_all_items given those pairs as COO lists; a user outside [0, n_users) makes check_ids raise IndexError."""
    if q.dim() != 2 or table.dim() != 2 or q.shape[1] != table.shape[1] or target.numel() != q.shape[0] \
            or users.numel() != q.shape[0]:
        raise ValueError("rank_all_items_clicked: q [B, d], table [n_items, d], target [B], users [B]")
    if clicked.ptr.numel() != clicked.n_users + 1:
        raise ValueError(f"rank_all_items_clicked: the clicked sets cover {clicked.ptr.numel() - 1} users, "
                         f"n_users says {clicked.n_users}")
    _need_cuda(q, table, target, users, clicked.ptr, clicked.items)
    q, table = _f32c(q, "q"), _f32c(table, "table")
    target, users = _i64c(target.reshape(-1), "target"), _i64c(users.reshape(-1), "users")
    B, d = q.shape
    rank = torch.empty(B, dtype=torch.int64, device=q.device)
    if B == 0:
        return rank
    s0 = torch.empty(B, dtype=torch.float32, device=q.device)
    _lib.check(_lib.load().b2r_rank_all_items_clicked(_p(q), d, _p(table), table.shape[0], d, _p(target), _p(users), B,
                                                      _p(clicked.ptr), _p(clicked.items), clicked.n_users, _p(s0),
                                                      _p(rank), _p(err_flag(q.device)), _stream()),
               "b2r_rank_all_items_clicked")
    return rank


def _topk_k(k: int) -> int:
    k = int(k)
    if not 1 <= k <= 1024:
        raise ValueError(f"top-k lists support 1 <= k <= 1024, got k={k}")
    return k


def topk_rows(pred: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Top-k' (k' = min(k, C)) of every row of pred [N, C] in the order of Python's stable
    sorted(..., key=score, reverse=True) (include/b200rec.h): (columns int64 [N, k'], scores float32 [N, k'])."""
    _need_cuda(pred)
    pred = _f32c(pred, "pred")
    if pred.dim() != 2 or pred.shape[1] < 1:
        raise ValueError("topk_rows: pred must be [N, C] with C >= 1")
    k = _topk_k(k)
    N, Cn = pred.shape
    kk = min(k, Cn)
    idx = torch.empty((N, kk), dtype=torch.int64, device=pred.device)
    val = torch.empty((N, kk), dtype=torch.float32, device=pred.device)
    L = _lib.load()
    nb = L.b2r_topk_rows_workspace_bytes(N, Cn, k)
    ws = _ws(nb, pred.device) if nb else None
    _lib.check(L.b2r_topk_rows(_p(pred), N, Cn, Cn, k, _p(idx), _p(val), _p(ws), nb, _stream()), "b2r_topk_rows")
    return idx, val


def mask_clicked(pred: torch.Tensor, users: torch.Tensor, clicked: ClickedSets) -> torch.Tensor:
    """pred[b, j] = -inf in place for every item j the user users[b] clicked, 1 <= j < C (BaseRunner.py:244-251 for
    the test_all candidate list, where column j is item j).  Returns pred."""
    _need_cuda(pred, users, clicked.ptr)
    if pred.dtype != torch.float32 or not pred.is_contiguous() or pred.dim() != 2:
        raise TypeError("mask_clicked: pred must be a contiguous float32 [N, C] tensor")
    users = _i64c(users.reshape(-1), "users")
    if users.numel() != pred.shape[0]:
        raise ValueError("mask_clicked: one user per row")
    N, Cn = pred.shape
    _lib.check(_lib.load().b2r_mask_clicked(_p(pred), N, Cn, Cn, _p(users), _p(clicked.ptr), _p(clicked.items),
                                            clicked.n_users, _p(err_flag(pred.device)), _stream()), "b2r_mask_clicked")
    return pred


def topk_all_items(q: torch.Tensor, table: torch.Tensor, target: torch.Tensor, users: torch.Tensor,
                   clicked: ClickedSets, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The test_all top-k' lists (k' = min(k, n_items)) of dot-product models without the [B, n_items] scores:
    candidates [target] + arange(1, n_items) scored <q[b], table[j]>, clicked items masked (-inf), ordered as
    topk_rows orders them.  Returns (item ids int64 [B, k'], scores float32 [B, k'])."""
    _need_cuda(q, table, target, users, clicked.ptr)
    q, table = _f32c(q, "q"), _f32c(table, "table")
    target, users = _i64c(target.reshape(-1), "target"), _i64c(users.reshape(-1), "users")
    if q.dim() != 2 or table.dim() != 2 or q.shape[1] != table.shape[1] or target.numel() != q.shape[0] \
            or users.numel() != q.shape[0]:
        raise ValueError("topk_all_items: q [B, d], table [n_items, d], target [B], users [B]")
    k = _topk_k(k)
    B, d = q.shape
    n_items = table.shape[0]
    kk = min(k, n_items)
    items = torch.empty((B, kk), dtype=torch.int64, device=q.device)
    scores = torch.empty((B, kk), dtype=torch.float32, device=q.device)
    if B == 0:
        return items, scores
    L = _lib.load()
    nb = L.b2r_topk_all_items_workspace_bytes(B, n_items, k)
    ws = _ws(nb, q.device)
    _lib.check(L.b2r_topk_all_items(_p(q), d, _p(table), n_items, d, _p(target), _p(users), B, _p(clicked.ptr),
                                    _p(clicked.items), clicked.n_users, k, _p(items), _p(scores),
                                    _p(err_flag(q.device)), _p(ws), nb, _stream()), "b2r_topk_all_items")
    return items, scores


def neumf_all_items_error(d: int, layers: Sequence[int], Bn: int, n_items: int) -> Optional[str]:
    """None when NeuMF's test_all scores of a batch of Bn rows can come from neumf_score_rows (d in {32, 64}, at least
    4096 candidate rows, every hidden layer on the forward's tensor-core Linear, the fused CTA within shared memory), else
    why not (b2r_neumf_score_rows_check; host only)"""
    layers = [int(w) for w in layers]
    if not 1 <= len(layers) <= _lib.NEUMF_MAX_LAYERS:
        return f"{len(layers)} hidden layers, the fused scorer takes 1..{_lib.NEUMF_MAX_LAYERS}"
    widths = (C.c_int32 * len(layers))(*layers)
    L = _lib.load()
    if L.b2r_neumf_score_rows_check(int(d), len(layers), widths, int(Bn), int(n_items)) == 0:
        return None
    return L.b2r_last_error().decode("utf-8", "replace")


def neumf_window_rows(Bn: int, n_items: int) -> int:
    """rows of one neumf_score_rows window: a [rows, n_items] float32 block within 32 MB, at least one row"""
    return int(_lib.load().b2r_neumf_window_rows(int(Bn), int(n_items)))


def neumf_score_rows(mf_u: torch.Tensor, mf_i: torch.Tensor, mlp_u: torch.Tensor, mlp_i: torch.Tensor,
                     mlp: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor]]], w_out: torch.Tensor, users: torch.Tensor,
                     targets: torch.Tensor, b0: int, b1: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Rows [b0, b1) of NeuMF's test_all scores for one evaluation batch (users [Bn], targets [Bn]): the [b1 - b0,
    n_items] block NeuMF's forward gives on the candidate list [target | arange(1, n_items)], bit for bit (column 0 the
    target, column j >= 1 item j), without the [Bn * n_items, 2d] concat input (b2r_neumf_score_rows).  mlp: the hidden
    layers' (weight [N, K], bias [N] or None); w_out: prediction.weight [1, d + last].  Raises B200RecError for shapes
    outside neumf_all_items_error's envelope; out-of-range user / target ids make check_ids raise IndexError."""
    _need_cuda(mf_u, mf_i, mlp_u, mlp_i, w_out, users, targets)
    mf_u, mf_i, mlp_u, mlp_i = (_f32c(t, n) for t, n in ((mf_u, "mf_u"), (mf_i, "mf_i"), (mlp_u, "mlp_u"), (mlp_i, "mlp_i")))
    w_out = _f32c(w_out.reshape(-1), "w_out")
    users, targets = _i64c(users.reshape(-1), "users"), _i64c(targets.reshape(-1), "targets")
    n_users, d = mf_u.shape
    n_items = mf_i.shape[0]
    Bn = users.numel()
    if targets.numel() != Bn or mlp_u.shape != mf_u.shape or mlp_i.shape != mf_i.shape or mf_i.shape[1] != d:
        raise ValueError("neumf_score_rows: tables [n_users, d] / [n_items, d], users and targets [Bn]")
    if not 0 <= b0 < b1 <= Bn:
        raise ValueError(f"neumf_score_rows: window [{b0}, {b1}) outside the batch of {Bn} rows")
    if not 1 <= len(mlp) <= _lib.NEUMF_MAX_LAYERS:
        raise ValueError(f"neumf_score_rows: {len(mlp)} hidden layers, the fused scorer takes 1..{_lib.NEUMF_MAX_LAYERS}")
    Ws = [_f32c(W, f"W{l}") for l, (W, _) in enumerate(mlp)]
    bs = [None if b is None else _f32c(b, f"bias{l}") for l, (_, b) in enumerate(mlp)]
    for l, (W, b) in enumerate(zip(Ws, bs)):
        K = 2 * d if l == 0 else Ws[l - 1].shape[0]
        if W.dim() != 2 or W.shape[1] != K or (b is not None and b.numel() != W.shape[0]):
            raise ValueError(f"neumf_score_rows: hidden layer {l} must be a [N, {K}] weight with an [N] bias")
    if w_out.numel() != d + Ws[-1].shape[0]:
        raise ValueError("neumf_score_rows: w_out must hold d + the last hidden width")
    if out is None:
        out = torch.empty((b1 - b0, n_items), dtype=torch.float32, device=mf_u.device)
    elif out.dtype != torch.float32 or out.dim() != 2 or out.shape != (b1 - b0, n_items) or out.stride(1) != 1:
        raise ValueError("neumf_score_rows: out must be float32 [b1 - b0, n_items] with contiguous rows")
    a = _lib.NeumfRows()
    a.mf_u, a.mf_i, a.mlp_u, a.mlp_i = _p(mf_u), _p(mf_i), _p(mlp_u), _p(mlp_i)
    a.n_users, a.n_items, a.d, a.n_layers = n_users, n_items, d, len(Ws)
    for l, (W, b) in enumerate(zip(Ws, bs)):
        a.widths[l], a.W[l], a.bias[l] = W.shape[0], _p(W), _p(b)
    a.w_out, a.users, a.targets = _p(w_out), _p(users), _p(targets)
    a.Bn, a.b0, a.b1 = Bn, int(b0), int(b1)
    a.out, a.ld_out = _p(out), out.stride(0)
    _lib.check(_lib.load().b2r_neumf_score_rows(C.byref(a), _p(err_flag(mf_u.device)), _stream()), "b2r_neumf_score_rows")
    return out


class DeviceNegativeSampler:
    """Groundwork for SURVEY.md §8 f3: models/BaseModel.py:206-214 on the device.  Holds the training clicks as a CSR
    on the GPU and draws ``num_neg`` non-clicked items per training row with b2r_sample_negatives.  Same distribution
    as the reference's NumPy loop, a different (counter-based, reproducible from (seed, epoch)) random stream."""

    def __init__(self, train_clicked_set: dict, n_users: int, n_items: int, device, seed: int = 0):
        ptr, flat = clicked_csr([train_clicked_set], n_users)
        self.ptr = torch.from_numpy(ptr).to(device)
        self.items = torch.from_numpy(flat).to(device)
        self.n_users, self.n_items, self.seed = int(n_users), int(n_items), int(seed)

    def sample(self, user_ids: torch.Tensor, num_neg: int, epoch: int) -> torch.Tensor:
        _need_cuda(user_ids, self.ptr)
        user_ids = _i64c(user_ids.reshape(-1), "user_ids")
        out = torch.empty((user_ids.numel(), int(num_neg)), dtype=torch.int64, device=user_ids.device)
        _lib.check(_lib.load().b2r_sample_negatives(_p(user_ids), user_ids.numel(), int(num_neg), _p(self.ptr),
                                                    _p(self.items), self.n_users, self.n_items,
                                                    self.seed & 0xFFFFFFFFFFFFFFFF, int(epoch) & 0xFFFFFFFF, _p(out),
                                                    _p(err_flag(user_ids.device)), _stream()), "b2r_sample_negatives")
        return out


def collate_general(users: torch.Tensor, items: torch.Tensor, neg: torch.Tensor, perm: Optional[torch.Tensor], start: int,
                    Bn: int, out_uid: torch.Tensor, out_iid: torch.Tensor) -> None:
    """b2r_collate_general: one GeneralModel training batch assembled on the device (BaseModel.py:192-203,135-152)"""
    _need_cuda(users, items, neg, perm, out_uid, out_iid)
    K = neg.shape[1]
    if out_iid.shape[1] != K + 1 or out_iid.shape[0] < Bn or out_uid.numel() < Bn:
        raise ValueError("collate_general: output buffers do not fit the batch")
    for t in (users, items, neg, out_uid, out_iid):
        if t.dtype != torch.int64 or not t.is_contiguous():
            raise TypeError("collate_general: contiguous int64 tensors expected")
    if perm is not None and (perm.dtype != torch.int64 or not perm.is_contiguous()):
        raise TypeError("collate_general: perm must be contiguous int64")
    _lib.check(_lib.load().b2r_collate_general(_p(users), _p(items), _p(neg), _p(perm), int(start), int(Bn), int(K),
                                               _p(out_uid), _p(out_iid), _stream()), "b2r_collate_general")


def history_csr(user_his: dict, n_users: int):
    """corpus.user_his ({u: [(item, time), ...]}, helpers/SeqReader.py:14-33) as a CSR over users: his_ptr int64
    [n_users + 1] and his_items int64 [total] (items only), user u's history at his_items[his_ptr[u]:his_ptr[u + 1]].
    NumPy arrays; one pass over the interactions."""
    import numpy as np
    ptr = np.zeros(int(n_users) + 1, dtype=np.int64)
    for u, h in user_his.items():
        if not 0 <= int(u) < n_users:
            raise ValueError(f"history_csr: user {u} outside [0, {n_users})")
        ptr[int(u) + 1] = len(h)
    ptr = np.cumsum(ptr)
    items = np.zeros(int(ptr[-1]), dtype=np.int64)
    for u, h in user_his.items():
        if len(h):
            items[ptr[int(u)]:ptr[int(u) + 1]] = np.fromiter((x[0] for x in h), dtype=np.int64, count=len(h))
    return ptr, items


def history_width(positions, history_max: int) -> int:
    """the fixed padded width of device-collated histories: min(H, max position), or max position when H <= 0"""
    import numpy as np
    top = int(np.max(positions)) if len(positions) else 1
    return max(1, min(int(history_max), top) if int(history_max) > 0 else top)


class DeviceHistory:
    """The inputs of b2r_collate_history for one SequentialModel training set, on the device: the history CSR of
    ``corpus.user_his`` (``history_csr``) and the dataset's ``position`` column.  Every row's position is checked once,
    here, to lie in [1, len(user_his[u])]; ``width`` (``history_width``) is the padded history width of every batch."""

    def __init__(self, user_his: dict, n_users: int, users, positions, history_max: int, device):
        import numpy as np
        users = np.asarray(users, dtype=np.int64)
        positions = np.asarray(positions, dtype=np.int64)
        ptr, items = history_csr(user_his, n_users)
        if users.shape != positions.shape:
            raise ValueError("DeviceHistory: users and positions differ in length")
        if len(users) and (users.min() < 0 or users.max() >= n_users):
            raise ValueError("DeviceHistory: a training row's user is outside [0, n_users)")
        have = ptr[users + 1] - ptr[users]
        bad = np.flatnonzero((positions < 1) | (positions > have))
        if len(bad):
            r = int(bad[0])
            raise ValueError(f"DeviceHistory: {len(bad)} training row(s) with a position outside [1, len(user_his[u])] "
                             f"(first: row {r}, user {int(users[r])}, position {int(positions[r])}, history {int(have[r])})")
        self.n_users, self.history_max = int(n_users), int(history_max)
        self.width = history_width(positions, history_max)
        self.ptr = torch.from_numpy(ptr).to(device)
        self.items = torch.from_numpy(items if len(items) else np.zeros(1, dtype=np.int64)).to(device)
        self.positions = torch.from_numpy(positions).to(device)

    def collate(self, users: torch.Tensor, perm: Optional[torch.Tensor], start: int, Bn: int, out_hist: torch.Tensor,
                out_len: torch.Tensor) -> None:
        collate_history(users, self.positions, self.ptr, self.items, self.n_users, perm, start, Bn, self.history_max,
                        out_hist, out_len)


def collate_history(users: torch.Tensor, positions: torch.Tensor, his_ptr: torch.Tensor, his_items: torch.Tensor,
                    n_users: int, perm: Optional[torch.Tensor], start: int, Bn: int, history_max: int,
                    out_hist: torch.Tensor, out_len: torch.Tensor) -> None:
    """b2r_collate_history: the history part of one SequentialModel training batch assembled on the device
    (BaseModel.py:236-245,135-152), right-padded with 0 to out_hist's width Lp.  Bad rows are clamped and counted in the
    out-of-range counter (check_ids raises IndexError)."""
    _need_cuda(users, positions, his_ptr, his_items, perm, out_hist, out_len)
    if out_hist.dim() != 2 or out_hist.shape[0] < Bn or out_len.numel() < Bn or his_ptr.numel() != int(n_users) + 1:
        raise ValueError("collate_history: output buffers do not fit the batch")
    for t in (users, positions, his_ptr, his_items, out_hist, out_len):
        if t.dtype != torch.int64 or not t.is_contiguous():
            raise TypeError("collate_history: contiguous int64 tensors expected")
    if perm is not None and (perm.dtype != torch.int64 or not perm.is_contiguous()):
        raise TypeError("collate_history: perm must be contiguous int64")
    _lib.check(_lib.load().b2r_collate_history(_p(users), _p(positions), _p(his_ptr), _p(his_items), int(n_users), _p(perm),
                                               int(start), int(Bn), int(history_max), int(out_hist.shape[1]), _p(out_hist),
                                               _p(out_len), _p(err_flag(users.device)), _stream()), "b2r_collate_history")


def list_csr(lists, width: int):
    """Ragged per-row lists (e.g. an impression phase's ``pos_items`` column) cut to their first ``width`` entries, as a
    CSR over the rows: ptr int64 [N + 1] and items int64 (at least one slot).  NumPy arrays; one pass over the lists."""
    import itertools

    import numpy as np
    width = int(width)
    lens = np.fromiter((min(len(x), width) for x in lists), dtype=np.int64, count=len(lists))
    ptr = np.zeros(len(lists) + 1, dtype=np.int64)
    np.cumsum(lens, out=ptr[1:])
    items = np.fromiter(itertools.chain.from_iterable(x[:width] for x in lists), dtype=np.int64, count=int(ptr[-1]))
    return ptr, (items if len(items) else np.zeros(1, dtype=np.int64))


def collate_impression(users: torch.Tensor, pos_ptr: torch.Tensor, pos_items: torch.Tensor, neg_ptr: torch.Tensor,
                       neg_items: torch.Tensor, n_users: int, start: int, Bn: int, mp: int, mn: int, out_uid: torch.Tensor,
                       out_iid: torch.Tensor) -> None:
    """b2r_collate_impression: rows [start, start + Bn) of an impression evaluation phase as ImpressionModel.Dataset's
    collate_batch builds them (models/BaseImpressionModel.py:152-184): out_uid[t] = users[start + t], out_iid[t] =
    [pos[:mp] | 0-pad | neg[:mn] | 0-pad], the lists read from the CSRs (pos_ptr, pos_items) / (neg_ptr, neg_items) over
    the phase's rows (list_csr).  A user outside [0, n_users) makes check_ids raise IndexError."""
    _need_cuda(users, pos_ptr, pos_items, neg_ptr, neg_items, out_uid, out_iid)
    for t in (users, pos_ptr, pos_items, neg_ptr, neg_items, out_uid, out_iid):
        if t.dtype != torch.int64 or not t.is_contiguous():
            raise TypeError("collate_impression: contiguous int64 tensors expected")
    N = users.numel()
    if not 0 <= start <= start + Bn <= N or pos_ptr.numel() != N + 1 or neg_ptr.numel() != N + 1:
        raise ValueError("collate_impression: rows outside the phase, or CSRs that do not cover its rows")
    if out_iid.dim() != 2 or out_iid.shape[1] != mp + mn or out_iid.shape[0] < Bn or out_uid.numel() < Bn:
        raise ValueError("collate_impression: output buffers do not fit the batch")
    _lib.check(_lib.load().b2r_collate_impression(_p(users), _p(pos_ptr), _p(pos_items), _p(neg_ptr), _p(neg_items),
                                                  int(n_users), int(start), int(Bn), int(mp), int(mn), _p(out_uid),
                                                  _p(out_iid), _p(err_flag(users.device)), _stream()),
               "b2r_collate_impression")


def collate_impression_train(users: torch.Tensor, pos_ptr: torch.Tensor, pos_items: torch.Tensor, neg_ptr: torch.Tensor,
                             neg_items: torch.Tensor, pos_num: torch.Tensor, neg_num: torch.Tensor,
                             perm: Optional[torch.Tensor], n_users: int, start: int, Bn: int, mp: int, mn: int, out_uid: torch.Tensor,
                             out_iid: torch.Tensor, out_labels: torch.Tensor) -> None:
    """b2r_collate_impression_train: one training batch of ImpressionRunner.fit (helpers/ImpressionRunner.py:181-190), the
    rows perm[start:start + Bn] of the training set (perm None: rows start .. start + Bn - 1): ``user_id`` and ``item_id`` as collate_impression builds them, and
    out_labels[t, c] = 1 / -1 for c < mp (c < min(pos_num, mp)) and 0 / -1 after it (c - mp < min(neg_num, mn)).
    pos_num / neg_num are the raw int64 data columns of the whole set.  A user outside [0, n_users) makes check_ids
    raise IndexError."""
    tensors = (users, pos_ptr, pos_items, neg_ptr, neg_items, pos_num, neg_num, perm, out_uid, out_iid, out_labels)
    _need_cuda(*tensors)
    for t in tensors:
        if t is not None and (t.dtype != torch.int64 or not t.is_contiguous()):
            raise TypeError("collate_impression_train: contiguous int64 tensors expected")
    N = users.numel()
    if pos_ptr.numel() != N + 1 or neg_ptr.numel() != N + 1 or pos_num.numel() != N or neg_num.numel() != N:
        raise ValueError("collate_impression_train: CSRs and pos_num / neg_num that do not cover the set's rows")
    if (perm is not None and perm.numel() != N) or not 0 <= start <= start + Bn <= N:
        raise ValueError("collate_impression_train: perm must order the set's rows, and the batch must lie within it")
    if (out_iid.dim() != 2 or out_iid.shape[1] != mp + mn or out_iid.shape[0] < Bn or out_uid.numel() < Bn
            or out_labels.shape != out_iid.shape):
        raise ValueError("collate_impression_train: output buffers do not fit the batch")
    _lib.check(_lib.load().b2r_collate_impression_train(
        _p(users), _p(pos_ptr), _p(pos_items), _p(neg_ptr), _p(neg_items), _p(pos_num), _p(neg_num), _p(perm),
        int(n_users), int(start), int(Bn), int(mp), int(mn), _p(out_uid), _p(out_iid), _p(out_labels),
        _p(err_flag(users.device)), _stream()), "b2r_collate_impression_train")


_imp_ws = {}


def impression_metrics(pred: torch.Tensor, pos_num: torch.Tensor, neg_num: torch.Tensor, mp: int, topk: Sequence[int],
                       acc: torch.Tensor) -> torch.Tensor:
    """b2r_impression_metrics: adds the per-row NDCG@k, MAP@k and HR@k sums of one batch of impression predictions
    pred [Bn, mp + mn] into acc float64 [3 * len(topk)] (NDCG for every k, then MAP, then HR), the metrics of
    ImpressionRunner.evaluate (helpers/ImpressionRunner.py:135-171, :74-133) as include/b200rec.h restates them.
    pos_num / neg_num: the batch rows' raw int64 data columns.  Fixed summation order: the same inputs give the same
    bits.  Returns acc."""
    _need_cuda(pred, pos_num, neg_num, acc)
    if pred.dtype != torch.float32 or pred.dim() != 2 or pred.stride(1) != 1:
        raise TypeError("impression_metrics: pred must be float32 [Bn, C] with contiguous rows")
    pos_num, neg_num = _i64c(pos_num.reshape(-1), "pos_num"), _i64c(neg_num.reshape(-1), "neg_num")
    Bn, Cn = pred.shape
    ks = [int(k) for k in topk]
    nk = len(ks)
    if not 1 <= nk <= _lib.IMPRESSION_MAX_TOPK or min(ks) < 1:
        raise ValueError(f"impression_metrics: 1 to {_lib.IMPRESSION_MAX_TOPK} cut-offs >= 1 expected, got {ks}")
    if not 0 <= int(mp) <= Cn or pos_num.numel() != Bn or neg_num.numel() != Bn:
        raise ValueError("impression_metrics: mp within the row, one pos_num / neg_num per row")
    if acc.dtype != torch.float64 or not acc.is_contiguous() or acc.numel() != 3 * nk:
        raise ValueError("impression_metrics: acc must be a contiguous float64 [3 * len(topk)] tensor")
    if Bn == 0:
        return acc
    L = _lib.load()
    nb = int(L.b2r_impression_metrics_workspace_bytes(Bn, Cn, nk))
    key = acc.device.index if acc.device.index is not None else torch.cuda.current_device()
    ws = _imp_ws.get(key)
    if ws is None or ws.numel() < nb:
        ws = _imp_ws[key] = torch.zeros(nb, dtype=torch.uint8, device=acc.device)   # the counter starts at zero
    kk = (C.c_int * nk)(*ks)
    _lib.check(L.b2r_impression_metrics(_p(pred), pred.stride(0), Bn, Cn, int(mp), _p(pos_num), _p(neg_num), kk, nk,
                                        _p(acc), _p(ws), ws.numel(), _stream()), "b2r_impression_metrics")
    return acc


def adam_exact_advance(W: torch.Tensor, m: torch.Tensor, v: torch.Tensor, last: torch.Tensor, upto: int, opt,
                       rows: Optional[torch.Tensor] = None, stamp: int = 0, state_ld: int = 0) -> None:
    """Groundwork for the exact dense-Adam mode (b2r_adam_exact_advance): bring the listed unique rows (all rows when
    ``rows`` is None) of a row-sparsely updated table to optimizer step ``upto``, as torch.optim.Adam over the whole
    table would have moved them on zero data gradients.  ``last`` int32 [n_rows] is read and re-stamped."""
    _need_cuda(W, m, v, last, rows)
    if last.dtype != torch.int32 or not last.is_contiguous():
        raise TypeError("last must be a contiguous int32 tensor")
    n = 0
    if rows is not None:
        rows = _i64c(rows.reshape(-1), "rows")
        n = rows.numel()
    o = _lib.Optim(1, opt.lr, opt.betas[0], opt.betas[1], opt.eps, opt.weight_decay, 1.0, 1.0, state_ld)
    _lib.check(_lib.load().b2r_adam_exact_advance(_p(rows), n, W.shape[0], W.shape[1], _p(W), _p(m), _p(v), _p(last),
                                                  int(upto), int(stamp), C.byref(o), _p(err_flag(W.device)), _stream()),
               "b2r_adam_exact_advance")


def bpr_loss_and_grad(pred: torch.Tensor, want_grad: bool = True) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """BaseModel.py:175-189 value and closed-form d loss / d pred in one pass."""
    _need_cuda(pred)
    pred = _f32c(pred, "pred")
    if pred.dim() != 2:
        raise ValueError("pred must be [B, C]")
    B, Cn = pred.shape
    loss = torch.empty((), dtype=torch.float32, device=pred.device)
    grad = torch.empty_like(pred) if want_grad else None
    rows = torch.empty(B, dtype=torch.float32, device=pred.device)
    L = _lib.load()
    _lib.check(L.b2r_bpr_loss(_p(pred), _p(loss), _p(grad), _p(rows), B, Cn, _stream()), "b2r_bpr_loss")
    return loss, grad


# --------------------------------------------------------------------------------------------------
# index plan + contribution sources
# --------------------------------------------------------------------------------------------------

@dataclass
class Source:
    """One contribution stream into a table gradient (b2r_grad_source): position p adds
    coef[p] * src[row(p)], row(p) = src_id[p // div] if src_id is given else p // div."""
    src: torch.Tensor                      # [*, d] float32
    n: int                                 # number of positions
    coef: Optional[torch.Tensor] = None    # [n] float32
    src_id: Optional[torch.Tensor] = None  # int64
    div: int = 1
    ld: int = 0                            # leading dimension of src in floats (0: d)

    def c_struct(self) -> _lib.GradSource:
        return _lib.GradSource(_p(self.src), _p(self.coef), _p(self.src_id), self.n, self.div, self.ld)


class IndexPlan:
    """Sorted, de-duplicated view of the ids a batch touches in one table (b2r_plan_build_ex)."""

    def __init__(self, ids: torch.Tensor, n_rows: int, ignore_id: int = -1, ignore_n: int = 0):
        _need_cuda(ids)
        ids = _i64c(ids.reshape(-1), "ids")
        n = ids.numel()
        if n == 0:
            raise ValueError("empty id list")
        dev = ids.device
        self.n, self.n_rows, self.device = n, int(n_rows), dev
        self.sorted_key = torch.empty(n, dtype=torch.int32, device=dev)   # uint32 bits
        self.sorted_pos = torch.empty(n, dtype=torch.int32, device=dev)   # uint32 bits
        self.seg_start = torch.empty(n, dtype=torch.int32, device=dev)
        self.n_uniq = torch.empty(1, dtype=torch.int32, device=dev)
        L = _lib.load()
        nbytes = L.b2r_plan_workspace_bytes(n, self.n_rows)
        if nbytes == 0:
            raise _lib.B200RecError(f"b2r_plan_workspace_bytes({n}, {n_rows}) = 0: " + L.b2r_last_error().decode())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(L.b2r_plan_build_ex(_p(ids), n, self.n_rows, int(ignore_id), int(ignore_n), _p(self.sorted_key),
                                       _p(self.sorted_pos), _p(self.seg_start), _p(self.n_uniq), _p(ws), nbytes,
                                       _p(err_flag(dev)), _stream()), "b2r_plan_build_ex")
        self._ws = ws   # keep alive until the stream has consumed it

    def count(self) -> int:
        """number of unique rows (synchronises)"""
        return int(self.n_uniq.item())

    def _apply(self, d: int, sources: Sequence[Source], mode: int, uniq=None, rows=None, dense=None, W=None,
               m=None, v=None, opt: Optional[_lib.Optim] = None) -> None:
        if not 1 <= len(sources) <= 2:
            raise ValueError("one or two sources")
        if sum(s.n for s in sources) != self.n:
            raise ValueError("sources do not cover the plan")
        s0 = sources[0].c_struct()
        s1 = sources[1].c_struct() if len(sources) == 2 else None
        L = _lib.load()
        _lib.check(L.b2r_segment_apply(_p(self.sorted_key), _p(self.sorted_pos), _p(self.seg_start),
                                       _p(self.n_uniq), self.n, self.n_rows, d, C.byref(s0),
                                       C.byref(s1) if s1 is not None else None, mode, _p(uniq), _p(rows),
                                       _p(dense), _p(W), _p(m), _p(v),
                                       C.byref(opt) if opt is not None else None, _stream()),
                   "b2r_segment_apply")

    def reduce_rows(self, d: int, sources: Sequence[Source]) -> Tuple[torch.Tensor, torch.Tensor]:
        """row-sparse gradient: (unique row ids [nu] int64 ascending, grad rows [nu, d]); synchronises once."""
        uniq = torch.empty(self.n, dtype=torch.int64, device=self.device)
        rows = torch.empty((self.n, d), dtype=torch.float32, device=self.device)
        self._apply(d, sources, 0, uniq=uniq, rows=rows)
        nu = self.count()
        if nu > 0 and int(uniq[nu - 1].item()) >= self.n_rows:      # trailing sentinel run of ignored positions
            nu -= 1
        return uniq[:nu], rows[:nu]

    def add_to_dense(self, dense: torch.Tensor, sources: Sequence[Source]) -> None:
        self._apply(dense.shape[1], sources, 1, dense=dense)

    def apply_optimizer(self, W: torch.Tensor, m, v, opt: _lib.Optim, sources: Sequence[Source]) -> None:
        self._apply(W.shape[1], sources, 2, W=W, m=m, v=v, opt=opt)


_direct_ws = {}


class DirectPlan:
    """b2r_direct_plan_build / _apply: bucketed partition of a batch's (row id, position) pairs -- the hot-path sibling of
    IndexPlan for the dense-add and fused-optimizer outputs (d in {32, 64, 128}): a scatter into fixed-capacity bucket
    regions and one per-bucket sort.  Workspace cached per (device, stream, n, n_rows) and reused in stream order."""

    SUPPORTED_D = (32, 64, 128)

    def __init__(self, ids: torch.Tensor, n_rows: int, ignore_id: int = -1, ignore_n: int = 0):
        _need_cuda(ids)
        ids = _i64c(ids.reshape(-1), "ids")
        n = ids.numel()
        if n == 0:
            raise ValueError("empty id list")
        self.n, self.n_rows, self.device = n, int(n_rows), ids.device
        L = _lib.load()
        key = (ids.device.index, _stream(), n, self.n_rows)
        ws = _direct_ws.get(key)
        if ws is None:
            nbytes = L.b2r_direct_plan_workspace_bytes(n, self.n_rows)
            if nbytes == 0:
                raise _lib.B200RecError(f"b2r_direct_plan_workspace_bytes({n}, {n_rows}) = 0")
            ws = torch.empty(nbytes, dtype=torch.uint8, device=ids.device)
            _lib.check(L.b2r_direct_plan_init(_p(ws), nbytes, n, self.n_rows, _stream()), "b2r_direct_plan_init")
            _direct_ws[key] = ws
        self.ws, self._ids = ws, ids
        _lib.check(L.b2r_direct_plan_build(_p(ids), n, self.n_rows, int(ignore_id), int(ignore_n), _p(ws), ws.numel(),
                                           _p(err_flag(ids.device)), _stream()), "b2r_direct_plan_build")

    @staticmethod
    def available(n: int, n_rows: int) -> bool:
        return _lib.load().b2r_direct_plan_workspace_bytes(int(n), int(n_rows)) != 0

    def _apply(self, d, sources, mode, dense=None, W=None, m=None, v=None, opt=None):
        if not 1 <= len(sources) <= 2:
            raise ValueError("one or two sources")
        s0 = sources[0].c_struct()
        s1 = sources[1].c_struct() if len(sources) == 2 else None
        _lib.check(_lib.load().b2r_direct_plan_apply(_p(self.ws), self.n, self.n_rows, d, C.byref(s0),
                                                     C.byref(s1) if s1 is not None else None, mode, _p(dense), _p(W), _p(m),
                                                     _p(v), C.byref(opt) if opt is not None else None, _stream()),
                   "b2r_direct_plan_apply")

    def add_to_dense(self, dense: torch.Tensor, sources: Sequence[Source]) -> None:
        self._apply(dense.shape[1], sources, 1, dense=dense)

    def apply_optimizer(self, W: torch.Tensor, m, v, opt: _lib.Optim, sources: Sequence[Source]) -> None:
        self._apply(W.shape[1], sources, 2, W=W, m=m, v=v, opt=opt)


def make_plan(ids: torch.Tensor, n_rows: int, d: int, ignore_id: int = -1, ignore_n: int = 0):
    """DirectPlan (two launches) where its kernels exist (d = 32/64/128) and it can be sized, IndexPlan (device radix
    sort) otherwise"""
    if d in DirectPlan.SUPPORTED_D and DirectPlan.available(ids.numel(), n_rows):
        return DirectPlan(ids, n_rows, ignore_id, ignore_n)
    return IndexPlan(ids, n_rows, ignore_id, ignore_n)


def dense_optim(W: torch.Tensor, grad: torch.Tensor, m, v, opt: _lib.Optim) -> None:
    L = _lib.load()
    _lib.check(L.b2r_dense_optim(_p(W), _p(grad), _p(m), _p(v), W.numel(), C.byref(opt), _stream()),
               "b2r_dense_optim")


# --------------------------------------------------------------------------------------------------
# how a table's gradient leaves autograd
# --------------------------------------------------------------------------------------------------

TABLE_MODES = ("dense", "sparse", "fused")


def set_table_mode(param: torch.nn.Parameter, mode: str) -> None:
    if mode not in TABLE_MODES:
        raise ValueError(f"table mode must be one of {TABLE_MODES}")
    param._b2r_mode = mode
    if not hasattr(param, "_b2r_pending"):
        param._b2r_pending = []


def table_mode(param: torch.Tensor) -> str:
    return getattr(param, "_b2r_mode", "dense")


def _table_grad(table: torch.Tensor, ids: torch.Tensor, source: Source, ignore_id: int = -1
                ) -> Optional[torch.Tensor]:
    """ignore_id: positions holding this id contribute exactly zero (padding) and are dropped from the plan"""
    mode = table_mode(table)
    if mode == "fused":
        table._b2r_pending.append((ids.reshape(-1), source, ignore_id))
        return None
    ign_n = ids.numel() if ignore_id >= 0 else 0
    if mode == "sparse":
        plan = IndexPlan(ids, table.shape[0], ignore_id, ign_n)
        uniq, rows = plan.reduce_rows(table.shape[1], [source])
        return torch.sparse_coo_tensor(uniq.unsqueeze(0), rows, size=tuple(table.shape), is_coalesced=True)
    dense = torch.zeros_like(table)
    make_plan(ids, table.shape[0], table.shape[1], ignore_id, ign_n).add_to_dense(dense, [source])
    return dense


# --------------------------------------------------------------------------------------------------
# autograd nodes
# --------------------------------------------------------------------------------------------------

class _Gather(torch.autograd.Function):
    """out = T[ids]; backward: row-sparse scatter of grad_out (nn.Embedding fwd/bwd)."""

    @staticmethod
    def forward(ctx, table, ids):
        ctx.save_for_backward(ids)
        ctx.table = table
        return gather_rows(table, ids)

    @staticmethod
    def backward(ctx, gout):
        (ids,) = ctx.saved_tensors
        table = ctx.table
        gout = _f32c(gout, "grad").reshape(-1, table.shape[1])
        g = _table_grad(table, ids, Source(src=gout, n=ids.numel()))
        return g, None


class _Score(torch.autograd.Function):
    """pred[b,c] = <q[b], T[ids[b,c]]> with q a dense [B,d] activation; backward gives dq and the
    row-sparse table gradient g[b,c] * q[b] (BPRMF.py:42 / SASRec.py:81 and their autograd)."""

    @staticmethod
    def forward(ctx, q, table, ids):
        q = _f32c(q, "q")
        ctx.save_for_backward(q, ids)
        ctx.table = table
        return rowdot(q, None, table, ids)

    @staticmethod
    def backward(ctx, g):
        q, ids = ctx.saved_tensors
        table = ctx.table
        g = _f32c(g, "grad_pred")
        dq = rowdot_bwd_query(g, table, ids) if ctx.needs_input_grad[0] else None
        gt = None
        if ctx.needs_input_grad[1]:
            gt = _table_grad(table, ids, Source(src=q, n=ids.numel(), coef=g.reshape(-1), div=ids.shape[1]))
        return dq, gt, None


class _BprLoss(torch.autograd.Function):
    """GeneralModel.loss (BaseModel.py:175-189): value and closed-form gradient from one kernel."""

    @staticmethod
    def forward(ctx, pred):
        loss, grad = bpr_loss_and_grad(pred, want_grad=True)
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, gl):
        (grad,) = ctx.saved_tensors
        return grad * gl


def listwise_kind(loss_n: str) -> Tuple[int, int]:
    """(kind, hard) of b2r_listwise_loss for a reference --loss_n string (BaseImpressionModel.py:26-27,58-128)"""
    if "BPR" in loss_n:
        if "simple" in loss_n:
            raise ValueError("loss 'BPR...simple' returns a vector in the reference (BaseImpressionModel.py:79-81) and cannot "
                             "be back-propagated there; not provided")
        kind = 1 if "after" in loss_n else (2 if "before" in loss_n else 0)
        return kind, 1 if "hard" in loss_n else 0
    table = {"listnet": 3, "softmaxCE": 4, "attention_rank": 5}
    if loss_n not in table:
        raise ValueError("Undefined loss function: {}".format(loss_n))
    return table[loss_n], 0


class _ListwiseLoss(torch.autograd.Function):
    """ImpressionModel.loss (BaseImpressionModel.py:44-128): value and closed-form gradient from b2r_listwise_loss."""

    @staticmethod
    def forward(ctx, pred, target, kind, hard, max_pos):
        _need_cuda(pred, target)
        pred, target = _f32c(pred, "prediction"), _i64c(target, "target")
        if pred.dim() != 2 or tuple(target.shape) != tuple(pred.shape):
            raise ValueError("prediction and target must both be [B, Cn]")
        B, Cn = pred.shape
        loss = torch.empty((), dtype=torch.float32, device=pred.device)
        grad = torch.empty_like(pred)
        L = _lib.load()
        ws = _ws(L.b2r_listwise_workspace_bytes(B), pred.device)
        _lib.check(L.b2r_listwise_loss(_p(pred), _p(target), B, Cn, int(max_pos), int(kind), int(hard), _p(loss), _p(grad),
                                       _p(ws), ws.numel(), _stream()), "b2r_listwise_loss")
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, gl):
        (grad,) = ctx.saved_tensors
        return grad * gl, None, None, None, None


def listwise_loss(pred: torch.Tensor, target: torch.Tensor, loss_n: str, max_pos: int) -> torch.Tensor:
    kind, hard = listwise_kind(loss_n)
    return _ListwiseLoss.apply(pred, target, kind, hard, max_pos)


def embedding(table: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    return _Gather.apply(table, ids)


def score(q: torch.Tensor, table: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    return _Score.apply(q, table, ids)


def bpr_loss(pred: torch.Tensor) -> torch.Tensor:
    return _BprLoss.apply(pred)


# --------------------------------------------------------------------------------------------------
# whole-step entry points (one C call per training step)
# --------------------------------------------------------------------------------------------------

def bprmf_fused_fwd_bwd(U, uid, I, iid):
    """b2r_bprmf_fused_fwd_bwd -> (pred [B,C], grad_pred [B,C], row_loss [B], dQ [B,d]); raises when the shape is
    outside the streaming kernel's class."""
    _need_cuda(U, I, uid, iid)
    U, I, uid, iid = _f32c(U, "U"), _f32c(I, "I"), _i64c(uid, "uid"), _i64c(iid, "iid")
    B, Cn = iid.shape
    d = U.shape[1]
    pred = torch.empty((B, Cn), dtype=torch.float32, device=U.device)
    gp = torch.empty((B, Cn), dtype=torch.float32, device=U.device)
    rl = torch.empty(B, dtype=torch.float32, device=U.device)
    dq = torch.empty((B, d), dtype=torch.float32, device=U.device)
    L = _lib.load()
    _lib.check(L.b2r_bprmf_fused_fwd_bwd(_p(U), _p(uid), U.shape[0], _p(I), _p(iid), I.shape[0], _p(pred), _p(gp),
                                         _p(rl), _p(dq), B, Cn, d, _p(err_flag(U.device)), _stream()),
               "b2r_bprmf_fused_fwd_bwd")
    return pred, gp, rl, dq


_step_ctx = {}


class _StepContext:
    """b2r_bprmf_ctx: workspace + side stream + double-buffered index plans for one (B, C, d, table sizes)."""

    def __init__(self, device, B, Cn, d, n_users, n_items):
        L = _lib.load()
        nbytes = L.b2r_bprmf_step_workspace_bytes(B, Cn, d, n_users, n_items)
        if nbytes == 0:
            raise _lib.B200RecError("b2r_bprmf_step_workspace_bytes returned 0")
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.handle = C.c_void_p()
        _lib.check(L.b2r_bprmf_ctx_create(C.byref(self.handle), B, Cn, d, n_users, n_items, _p(self.ws), nbytes),
                   "b2r_bprmf_ctx_create")

    def __del__(self):
        try:
            if self.handle:
                _lib.load().b2r_bprmf_ctx_destroy(self.handle)
        except Exception:
            pass


def bprmf_step_reset() -> None:
    """Drop every step context's prefetched plan (b2r_bprmf_ctx_reset).  Runners call this at the start of an epoch
    and when one is aborted: a prefetched plan is recognised by the id tensors' addresses, which the caching
    allocator may reuse for another batch."""
    L = _lib.load()
    for ctx in _step_ctx.values():
        L.b2r_bprmf_ctx_reset(ctx.handle)


def bprmf_train_step(U: torch.nn.Parameter, I: torch.nn.Parameter, optimizer, uid: torch.Tensor,
                     iid: torch.Tensor, next_uid: Optional[torch.Tensor] = None,
                     next_iid: Optional[torch.Tensor] = None) -> torch.Tensor:
    """b2r_bprmf_train_step: forward + BPR loss + backward + fused row-sparse optimizer, in place.
    next_uid/next_iid (optional): the NEXT batch's id tensors, already on the device and left untouched until
    the next call -- their index plan is built on the side stream while this step's kernels run."""
    from .optim import RowSparseOptimizer
    if not isinstance(optimizer, RowSparseOptimizer):
        raise _lib.B200RecError("train_step needs model.optimizer to be a rechorus_b200.optim.RowSparseOptimizer")
    _need_cuda(U, I, uid, iid, next_uid, next_iid)
    uid, iid = _i64c(uid, "user_id"), _i64c(iid, "item_id")
    B, Cn = iid.shape
    d = U.shape[1]
    eu, ei = optimizer.entry(U), optimizer.entry(I)
    if eu["wd"] != ei["wd"] or eu["state_ld"] != ei["state_ld"]:
        raise _lib.B200RecError("fused step expects one weight decay / state layout for both tables")
    L = _lib.load()
    key = (U.device.index, B, Cn, d, U.shape[0], I.shape[0], _stream())
    ctx = _step_ctx.get(key)
    if ctx is None:
        ctx = _step_ctx[key] = _StepContext(U.device, B, Cn, d, U.shape[0], I.shape[0])
    if next_uid is not None and next_iid is not None:
        if tuple(next_iid.shape) != (B, Cn) or next_uid.numel() != B:
            raise ValueError("prefetched batch must have the same shape as the current one")
        if not (next_uid.is_contiguous() and next_iid.is_contiguous()) or next_uid.dtype != torch.int64 \
                or next_iid.dtype != torch.int64:
            # the side stream reads these after this call returns: a temporary contiguous copy would be freed under it
            raise ValueError("prefetched id tensors must be contiguous int64 tensors that stay alive until the next step")
    else:
        next_uid = next_iid = None
    optimizer.advance()
    opt = optimizer._opt(ei["wd"], ei["state_ld"])
    tables = _lib.BprmfTables(_p(U.data), _p(I.data), _p(eu["m"]), _p(eu["v"]), _p(ei["m"]), _p(ei["v"]),
                              U.shape[0], I.shape[0], d, 0)
    loss = torch.empty((), dtype=torch.float32, device=U.device)
    _lib.check(L.b2r_bprmf_train_step(ctx.handle, C.byref(tables), _p(uid), _p(iid), _p(next_uid), _p(next_iid),
                                      C.byref(opt), _p(loss), _p(err_flag(U.device)), _stream()),
               "b2r_bprmf_train_step")
    return loss


# --------------------------------------------------------------------------------------------------
# dense layers (NeuMF MLP tower, SASRec q/k/v + FFN, LayerNorm, attention) -- kernels + autograd nodes
# --------------------------------------------------------------------------------------------------

def _ws(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def _rows_ld(t: torch.Tensor) -> Tuple[int, int]:
    """(rows, leading dimension) of a 2-D float32 tensor whose last dim is contiguous"""
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError("expected a 2-D tensor with a contiguous last dimension")
    return t.shape[0], t.stride(0)


def linear_fwd(x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor], relu: bool) -> torch.Tensor:
    """y = act(x W^T + b); x [M, K] (row stride may exceed K), W [N, K] contiguous (nn.Linear layout)."""
    _need_cuda(x, W)
    M, ldx = _rows_ld(x)
    N, K = W.shape
    W = _f32c(W, "W")
    y = torch.empty((M, N), dtype=torch.float32, device=x.device)
    L = _lib.load()
    _lib.check(L.b2r_linear_fwd(_p(x), ldx, _p(W), _p(bias), _p(y), N, M, N, K, 1 if relu else 0, _stream()),
               "b2r_linear_fwd")
    return y


def linear_fwd_uses_tc(M: int, N: int, K: int) -> bool:
    """whether the Linear forward of X[M, K] W^T with W [N, K] runs on the tensor-core kernel (b2r_linear_fwd_uses_tc)
    rather than the SGEMM -- the library's one copy of that decision"""
    return bool(_lib.load().b2r_linear_fwd_uses_tc(int(M), int(N), int(K)))


def linear_fwd_tc(x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor], relu: bool, strict: bool = True):
    """same as linear_fwd on the tensor cores (wgmma, TF32 hi/lo split, fp32-class accuracy); for shapes outside the
    kernel's class it raises (strict) or returns None"""
    _need_cuda(x, W)
    M, ldx = _rows_ld(x)
    N, K = W.shape
    W = _f32c(W, "W")
    y = torch.empty((M, N), dtype=torch.float32, device=x.device)
    L = _lib.load()
    rc = L.b2r_linear_fwd_tc(_p(x), ldx, _p(W), _p(bias), _p(y), N, M, N, K, 1 if relu else 0, _stream())
    if rc == -3 and not strict:
        return None
    _lib.check(rc, "b2r_linear_fwd_tc")
    return y


# --------------------------------------------------------------------------------------------------
# dropout (NeuMF.py:70-72, utils/layers.py:113-117) fused into the Linear and residual-LayerNorm kernels
# --------------------------------------------------------------------------------------------------

class DropoutState:
    """One model's dropout stream on the device: int64 {seed, step} (b2r_dropout in include/b200rec.h).  ``tick()``
    enqueues b2r_dropout_tick, which copies {seed, step} into a fresh 16-byte snapshot and advances step; every kernel of
    that forward and of its backward reads the snapshot.  Captured in a CUDA graph, the tick advances on every replay."""

    def __init__(self, seed: int, device):
        self.state = torch.tensor([_i64(seed), 0], dtype=torch.int64, device=device)

    def tick(self) -> torch.Tensor:
        snap = torch.empty(2, dtype=torch.int64, device=self.state.device)
        _lib.check(_lib.load().b2r_dropout_tick(_p(self.state), _p(snap), _stream()), "b2r_dropout_tick")
        return snap

    def get(self) -> Tuple[int, int]:
        """(seed, step) -- the step the next training forward uses (synchronises)"""
        seed, step = (int(v) for v in self.state.cpu())
        return seed & 0xFFFFFFFFFFFFFFFF, step

    def set(self, seed: int, step: int) -> None:
        self.state.copy_(torch.tensor([_i64(seed), int(step)], dtype=torch.int64))


def _i64(v: int) -> int:
    v = int(v) & 0xFFFFFFFFFFFFFFFF
    return v - (1 << 64) if v >= (1 << 63) else v


def check_dropout_p(p: float) -> float:
    """nn.Dropout's validation (the reference builds nn.Dropout(p): ValueError outside [0, 1])"""
    if not 0.0 <= float(p) <= 1.0:
        raise ValueError(f"dropout probability has to be between 0 and 1, but got {p}")
    return float(p)


@dataclass
class Drop:
    """One dropout site of one forward: the snapshot DropoutState.tick() returned, the probability and the site index
    (NeuMF layer l: l; SASRec block i: 2i after the attention, 2i + 1 after linear2)."""
    snapshot: torch.Tensor
    p: float
    site: int

    def c_struct(self, L: int = 0, lengths: Optional[torch.Tensor] = None) -> _lib.Dropout:
        return _lib.Dropout(_p(self.snapshot), _p(lengths), float(self.p), int(self.site), int(L))

    @property
    def scale(self) -> float:
        """s = float(1 / (1 - p)), 0 at p = 1"""
        import numpy as np
        return 0.0 if self.p >= 1.0 else float(np.float32(1.0 / (1.0 - self.p)))


def linear_fwd_dropout(x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor], relu: bool, drop: Drop,
                       tc: bool) -> torch.Tensor:
    """y = dropout(act(x W^T + b)) in one kernel, rows = activation rows (NeuMF's r = b*C + c); tc: the tensor-core kernel
    where the shape is in its class, else the CUDA-core one"""
    _need_cuda(x, W, drop.snapshot)
    M, ldx = _rows_ld(x)
    N, K = W.shape
    W = _f32c(W, "W")
    y = torch.empty((M, N), dtype=torch.float32, device=x.device)
    L = _lib.load()
    dc = drop.c_struct()
    rc = -3
    if tc:
        rc = L.b2r_linear_fwd_tc_dropout(_p(x), ldx, _p(W), _p(bias), _p(y), N, M, N, K, 1 if relu else 0, C.byref(dc),
                                         _stream())
        if rc not in (0, -3):
            _lib.check(rc, "b2r_linear_fwd_tc_dropout")
    if rc != 0:
        _lib.check(L.b2r_linear_fwd_dropout(_p(x), ldx, _p(W), _p(bias), _p(y), N, M, N, K, 1 if relu else 0, C.byref(dc),
                                            _stream()), "b2r_linear_fwd_dropout")
    return y


def linear_bwd(dy: torch.Tensor, x: torch.Tensor, W: torch.Tensor, y_relu: Optional[torch.Tensor],
               need_dx: bool, need_dw: bool, need_db: bool, drop: Optional[Drop] = None):
    """gradients of y = act(x W^T + b) given dy; y_relu = saved post-ReLU output (None when no ReLU).  drop: the layer's
    output went through that dropout (y_relu is then the saved post-dropout output, > 0 exactly where ReLU and mask
    passed): dz = s * dy * [y > 0], with s folded into the weight for dX and into the final reduction for dW / dbias."""
    M, lddy = _rows_ld(dy)
    _, ldx = _rows_ld(x)
    N, K = W.shape
    L = _lib.load()
    dx = dW = db = None
    if y_relu is not None and _rows_ld(y_relu)[1] != lddy:
        y_relu = y_relu.contiguous()
        dy = dy.contiguous()
        lddy = N
    if need_dx:
        dx = torch.empty((M, K), dtype=torch.float32, device=dy.device)
        done = False
        Wd = W if drop is None else W * drop.scale
        if M >= 4096 and N % 32 == 0 and N <= 128 and K % 16 == 0 and K <= 256 and lddy % 4 == 0:
            # dX = (dY o mask) W = (dY o mask) (W^T)^T on the tensor-core kernel: the transposed weight (N*K floats) is a copy
            Wt = Wd.t().contiguous()
            rc = L.b2r_linear_tc(_p(dy), lddy, _p(y_relu), _p(Wt), None, _p(dx), K, M, K, N, 0, _stream())
            done = rc == 0
            if rc not in (0, -3):
                _lib.check(rc, "b2r_linear_tc")
        if not done:
            _lib.check(L.b2r_linear_bwd_input(_p(dy), lddy, _p(y_relu), _p(Wd), _p(dx), K, M, N, K, _stream()),
                       "b2r_linear_bwd_input")
    if need_dw or need_db:
        dW = torch.empty((N, K), dtype=torch.float32, device=dy.device)
        db = torch.empty((N,), dtype=torch.float32, device=dy.device) if need_db else None
        if M >= 4096 and N % 4 == 0 and N <= 128 and K % 16 == 0 and K <= 240 and lddy % 4 == 0 and ldx % 4 == 0:
            # long reductions (M = B*L rows) on the tensor cores: k_linear_dw_tc
            ws = _ws(L.b2r_linear_bwd_weight_tc_workspace_bytes(M, N, K), dy.device)
            if drop is None:
                rc = L.b2r_linear_bwd_weight_tc(_p(dy), lddy, _p(y_relu), _p(x), ldx, _p(dW), _p(db), M, N, K, _p(ws),
                                                ws.numel(), _stream())
            else:
                dc = drop.c_struct()
                rc = L.b2r_linear_bwd_weight_tc_dropout(_p(dy), lddy, _p(y_relu), _p(x), ldx, _p(dW), _p(db), M, N, K,
                                                        C.byref(dc), _p(ws), ws.numel(), _stream())
            if rc == 0:
                return dx, dW, db
            if rc != -3:                                   # B2R_E_UNSUPPORTED falls through to the CUDA-core kernel
                _lib.check(rc, "b2r_linear_bwd_weight_tc")
        nbytes = L.b2r_linear_bwd_weight_workspace_bytes(M, N, K)
        ws = _ws(nbytes, dy.device)
        if drop is None:
            _lib.check(L.b2r_linear_bwd_weight(_p(dy), lddy, _p(y_relu), _p(x), ldx, _p(dW), _p(db), M, N, K, _p(ws),
                                               ws.numel(), _stream()), "b2r_linear_bwd_weight")
        else:
            dc = drop.c_struct()
            _lib.check(L.b2r_linear_bwd_weight_dropout(_p(dy), lddy, _p(y_relu), _p(x), ldx, _p(dW), _p(db), M, N, K,
                                                       C.byref(dc), _p(ws), ws.numel(), _stream()),
                       "b2r_linear_bwd_weight_dropout")
    return dx, dW, db


class _Linear(torch.autograd.Function):
    """nn.Linear (+ optional ReLU, + optional dropout after the ReLU) on the library's SGEMM: NeuMF.py:70-71 /
    layers.py:26-28,106-107."""

    @staticmethod
    def forward(ctx, x, W, bias, relu, drop=None):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        if x2.stride(1) != 1:
            x2 = x2.contiguous()
        N, K = W.shape
        # a long batch dimension (M >= 4096) runs on the tensor cores (csrc/linear_tc.cu: wgmma, TF32 hi/lo split,
        # 3 products, fp32-class accuracy checked in tests/test_gpu_tc.py); linear_bwd picks dX and dW the same way
        tc = linear_fwd_uses_tc(x2.shape[0], N, K)
        if drop is not None:
            if not relu:
                raise ValueError("fused dropout follows a ReLU (its backward reads the mask off the saved output)")
            y = linear_fwd_dropout(x2, W, bias, relu, drop, tc)
        elif tc:
            y = linear_fwd_tc(x2, W, bias, relu, strict=False)          # wgmma TF32-split forward
        else:
            y = None
        if y is None:
            y = linear_fwd(x2, W, bias, relu)
        ctx.save_for_backward(x2, W, y if relu else None)
        ctx.has_bias, ctx.shape, ctx.drop = bias is not None, shape, drop
        return y.view(*shape[:-1], W.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, W, y_relu = ctx.saved_tensors
        dy2 = _f32c(dy.reshape(-1, W.shape[0]), "dy")
        dx, dW, db = linear_bwd(dy2, x2, W, y_relu, ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                                ctx.has_bias and ctx.needs_input_grad[2], ctx.drop)
        if dx is not None:
            dx = dx.view(*ctx.shape)
        return dx, dW, db, None, None


def linear(x, W, bias=None, relu=False, drop: Optional[Drop] = None):
    """drop: dropout after the ReLU (NeuMF.py:71), fused into the kernel; needs relu=True"""
    return _Linear.apply(x, W, bias, relu, drop)


class _AddLayerNorm(torch.autograd.Function):
    """LayerNorm(x + res) with affine (layers.py:113,117); with ``drop``, LayerNorm(dropout(x) + res)."""

    @staticmethod
    def forward(ctx, x, res, gamma, beta, eps, drop=None, lengths=None, L_seq=0):
        _need_cuda(x, res, gamma, beta)
        d = x.shape[-1]
        x2, r2 = _f32c(x.reshape(-1, d), "x"), _f32c(res.reshape(-1, d), "res")
        rows = x2.shape[0]
        y = torch.empty_like(x2)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        L = _lib.load()
        if drop is None:
            _lib.check(L.b2r_add_layernorm_fwd(_p(x2), _p(r2), _p(gamma), _p(beta), _p(y), _p(mean), _p(rstd), rows, d,
                                               float(eps), _stream()), "b2r_add_layernorm_fwd")
        else:
            _need_cuda(drop.snapshot, lengths)
            dc = drop.c_struct(L_seq, lengths)
            _lib.check(L.b2r_add_layernorm_fwd_dropout(_p(x2), _p(r2), _p(gamma), _p(beta), _p(y), _p(mean), _p(rstd), rows,
                                                       d, float(eps), C.byref(dc), _stream()), "b2r_add_layernorm_fwd_dropout")
        ctx.save_for_backward(x2, r2, gamma, mean, rstd, lengths)
        ctx.shape, ctx.drop, ctx.L_seq = x.shape, drop, L_seq
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, r2, gamma, mean, rstd, lengths = ctx.saved_tensors
        d = x2.shape[1]
        rows = x2.shape[0]
        dy2 = _f32c(dy.reshape(-1, d), "dy")
        dz = torch.empty_like(x2)
        dg = torch.empty(d, dtype=torch.float32, device=dy.device)
        db = torch.empty(d, dtype=torch.float32, device=dy.device)
        L = _lib.load()
        ws = _ws(L.b2r_add_layernorm_bwd_workspace_bytes(rows, d), dy.device)
        if ctx.drop is None:
            _lib.check(L.b2r_add_layernorm_bwd(_p(dy2), _p(x2), _p(r2), _p(gamma), _p(mean), _p(rstd), _p(dz), _p(dg),
                                               _p(db), rows, d, _p(ws), ws.numel(), _stream()), "b2r_add_layernorm_bwd")
            dz = dz.view(ctx.shape)
            return dz, dz, dg, db, None, None, None, None
        dx = torch.empty_like(x2)
        dc = ctx.drop.c_struct(ctx.L_seq, lengths)
        _lib.check(L.b2r_add_layernorm_bwd_dropout(_p(dy2), _p(x2), _p(r2), _p(gamma), _p(mean), _p(rstd), _p(dz), _p(dx),
                                                   _p(dg), _p(db), rows, d, C.byref(dc), _p(ws), ws.numel(), _stream()),
                   "b2r_add_layernorm_bwd_dropout")
        return dx.view(ctx.shape), dz.view(ctx.shape), dg, db, None, None, None, None


def add_layernorm(x, res, gamma, beta, eps=1e-5, drop: Optional[Drop] = None, lengths: Optional[torch.Tensor] = None,
                  seq_len: int = 0):
    """drop: LayerNorm(dropout(x) + res) (layers.py:113,117).  Rows map to (sequence, position) for the mask: x [B, L, d]
    gives row b*L + t -> (b, t); x [B, d] with ``lengths`` and ``seq_len`` (the batch's padded width) gives row b ->
    (b, clamp(lengths[b] - 1, 0, seq_len - 1)), the position select_last reads"""
    if drop is not None and lengths is None:
        if x.dim() != 3:
            raise ValueError("add_layernorm with dropout: x must be [B, L, d], or [B, d] with lengths")
        seq_len = x.shape[1]
    elif lengths is not None:
        lengths = _i64c(lengths, "lengths")
    return _AddLayerNorm.apply(x, res, gamma, beta, eps, drop, lengths, int(seq_len))


class _CausalAttention(torch.autograd.Function):
    """layers.py:52-63 for q,k,v [B, L, d] with H heads (contiguous d/H chunks), causal mask, no W_o.  ``live`` (optional
    int64 [B]): positions >= live[b] are dead rows (nothing downstream reads them): skipped, written as zeros."""

    @staticmethod
    def forward(ctx, q, k, v, H, live):
        _need_cuda(q, k, v, live)
        B, Ln, d = q.shape
        q, k, v = _f32c(q, "q"), _f32c(k, "k"), _f32c(v, "v")
        live = None if live is None else _i64c(live, "live lengths")
        out = torch.empty((B, Ln, d), dtype=torch.float32, device=q.device)
        L = _lib.load()
        lse = None
        if d % H == 0 and d // H in (8, 16, 32) and Ln <= 128:
            # register-resident kernels (csrc/attention_rt.cu); the row log-sum-exp is kept for the backward
            lse = torch.empty((B, Ln, H), dtype=torch.float32, device=q.device)
            rc = L.b2r_attention_fwd_rt(_p(q), _p(k), _p(v), d, _p(live), _p(out), _p(lse), B, Ln, d, H, _stream())
            if rc == -3:                                   # B2R_E_UNSUPPORTED: shape / alignment outside the fast path
                lse = None
            else:
                _lib.check(rc, "b2r_attention_fwd_rt")
        if lse is None:                                    # shared-memory kernels (csrc/attention.cu)
            _lib.check(L.b2r_attention_fwd_live(_p(q), _p(k), _p(v), d, _p(live), _p(out), B, Ln, d, H, _stream()),
                       "b2r_attention_fwd_live")
        ctx.save_for_backward(q, k, v, live, out if lse is not None else None, lse)
        ctx.H = H
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, live, out, lse = ctx.saved_tensors
        B, Ln, d = q.shape
        dout = _f32c(dout, "dctx")
        dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
        L = _lib.load()
        if lse is not None:
            _lib.check(L.b2r_attention_bwd_rt(_p(q), _p(k), _p(v), d, _p(live), _p(out), _p(lse), _p(dout), _p(dq), _p(dk),
                                              _p(dv), d, B, Ln, d, ctx.H, _stream()), "b2r_attention_bwd_rt")
        else:
            _lib.check(L.b2r_attention_bwd_live(_p(q), _p(k), _p(v), d, _p(live), _p(dout), _p(dq), _p(dk), _p(dv), d, B, Ln,
                                                d, ctx.H, _stream()), "b2r_attention_bwd_live")
        return dq, dk, dv, None, None


def causal_attention(q, k, v, num_heads, live=None):
    return _CausalAttention.apply(q, k, v, num_heads, live)


def seq_train_error(L: int, d: int, H: int, num_layers: int, last_query: bool) -> Optional[str]:
    """None when a SASRec training step on batches of width up to L runs on the kernels (b2r_seq_train_check), else the
    library's reason.  last_query: the last block runs for the one query per sequence (attention_last)."""
    last_query = bool(last_query) and num_layers > 0
    flags = _lib.SEQ_LAST_QUERY if last_query else 0
    L_ = _lib.load()
    rc = L_.b2r_seq_train_check(int(L), int(d), int(H), int(num_layers) - int(last_query), flags)
    return None if rc == 0 else L_.b2r_last_error().decode("utf-8", "replace")


class _AttentionLast(torch.autograd.Function):
    """Attention for the one query per sequence that SASRec's last block needs (position len-1): q_last [B, d] against
    k, v [B, L, d]; identical to row len-1 of _CausalAttention.  SASRec's last block runs on it; L <= 256."""

    @staticmethod
    def forward(ctx, q_last, k, v, lengths, H):
        _need_cuda(q_last, k, v, lengths)
        B, Ln, d = k.shape
        q_last, k, v = _f32c(q_last, "q_last"), _f32c(k, "k"), _f32c(v, "v")
        lengths = _i64c(lengths, "lengths")
        out = torch.empty((B, d), dtype=torch.float32, device=k.device)
        prob = torch.empty((B, H, Ln), dtype=torch.float32, device=k.device)
        _lib.check(_lib.load().b2r_attention_last_fwd(_p(q_last), _p(k), _p(v), d, _p(lengths), _p(out), _p(prob), B, Ln,
                                                      d, H, _stream()), "b2r_attention_last_fwd")
        ctx.save_for_backward(q_last, k, v, lengths, prob)
        ctx.H = H
        return out

    @staticmethod
    def backward(ctx, dout):
        q_last, k, v, lengths, prob = ctx.saved_tensors
        B, Ln, d = k.shape
        dout = _f32c(dout, "dctx_last")
        dq, dk, dv = torch.empty_like(q_last), torch.empty_like(k), torch.empty_like(k)
        _lib.check(_lib.load().b2r_attention_last_bwd(_p(q_last), _p(k), _p(v), d, _p(lengths), _p(prob), _p(dout), _p(dq),
                                                      _p(dk), _p(dv), d, B, Ln, d, ctx.H, _stream()),
                   "b2r_attention_last_bwd")
        return dq, dk, dv, None, None


def attention_last(q_last, k, v, lengths, num_heads):
    return _AttentionLast.apply(q_last, k, v, lengths, num_heads)


class _EmbedHistory(torch.autograd.Function):
    """x = I[hist] + P[(len - t) * valid]  (SASRec.py:58-66); backward: row-sparse scatter into I (padding
    positions dropped: their gradient is exactly zero) and the dense small-table gradient of P."""

    @staticmethod
    def forward(ctx, I, P, hist, lengths):
        _need_cuda(I, P, hist, lengths)
        hist, lengths = _i64c(hist, "history_items"), _i64c(lengths, "lengths")
        B, Ln = hist.shape
        d = I.shape[1]
        x = torch.empty((B, Ln, d), dtype=torch.float32, device=I.device)
        pos = torch.empty((B, Ln), dtype=torch.int64, device=I.device)
        L = _lib.load()
        _lib.check(L.b2r_embed_history(_p(I), I.shape[0], _p(P), P.shape[0], _p(hist), _p(lengths), _p(x), _p(pos),
                                       B, Ln, d, _p(err_flag(I.device)), _stream()), "b2r_embed_history")
        ctx.save_for_backward(hist, pos)
        ctx.I, ctx.P = I, P
        return x

    @staticmethod
    def backward(ctx, dx):
        hist, pos = ctx.saved_tensors
        I, P = ctx.I, ctx.P
        d = I.shape[1]
        dx2 = _f32c(dx.reshape(-1, d), "dx")
        gI = gP = None
        if ctx.needs_input_grad[0]:
            gI = _table_grad(I, hist, Source(src=dx2, n=hist.numel()), ignore_id=0)
        if ctx.needs_input_grad[1]:
            n = pos.numel()
            gP = torch.empty_like(P)
            L = _lib.load()
            ws = _ws(L.b2r_small_table_grad_workspace_bytes(n, P.shape[0], d), dx.device)
            rc = L.b2r_small_table_grad(_p(dx2), d, _p(pos), n, P.shape[0], d, _p(gP), _p(ws), ws.numel(), _stream())
            if rc == -3:                    # B2R_E_UNSUPPORTED: the table's shared-memory copies do not fit
                gP = _table_grad(P, pos, Source(src=dx2, n=n))
            else:
                _lib.check(rc, "b2r_small_table_grad")
        return gI, gP, None, None


def embed_history(I, P, hist, lengths):
    return _EmbedHistory.apply(I, P, hist, lengths)


class _SelectLast(torch.autograd.Function):
    """h[b] = y[b, len[b]-1] * valid  (SASRec.py:74-76)."""

    @staticmethod
    def forward(ctx, y, hist, lengths):
        _need_cuda(y, hist, lengths)
        y = _f32c(y, "y")
        B, Ln, d = y.shape
        h = torch.empty((B, d), dtype=torch.float32, device=y.device)
        L = _lib.load()
        _lib.check(L.b2r_select_last(_p(y), _p(hist), _p(lengths), _p(h), B, Ln, d, _stream()), "b2r_select_last")
        ctx.save_for_backward(hist, lengths)
        ctx.shape = (B, Ln, d)
        return h

    @staticmethod
    def backward(ctx, dh):
        hist, lengths = ctx.saved_tensors
        B, Ln, d = ctx.shape
        dy = torch.empty((B, Ln, d), dtype=torch.float32, device=dh.device)
        L = _lib.load()
        _lib.check(L.b2r_select_last_bwd(_p(_f32c(dh, "dh")), _p(hist), _p(lengths), _p(dy), B, Ln, d, _stream()),
                   "b2r_select_last_bwd")
        return dy, None, None


def select_last(y, hist, lengths):
    return _SelectLast.apply(y, _i64c(hist, "history_items"), _i64c(lengths, "lengths"))


class _ColScale(torch.autograd.Function):
    """out[r,k] = a[r,k] * w[k]  (the GMF half of NeuMF's bias-free output layer, NeuMF.py:68,74-75)."""

    @staticmethod
    def forward(ctx, a, w):
        _need_cuda(a, w)
        a, w = _f32c(a, "a"), _f32c(w, "w")
        out = torch.empty_like(a)
        L = _lib.load()
        _lib.check(L.b2r_colscale(_p(a), _p(w), _p(out), a.shape[0], a.shape[1], _stream()), "b2r_colscale")
        ctx.save_for_backward(a, w)
        return out

    @staticmethod
    def backward(ctx, g):
        a, w = ctx.saved_tensors
        g = _f32c(g, "g")
        L = _lib.load()
        da = dw = None
        if ctx.needs_input_grad[0]:
            da = torch.empty_like(a)
            _lib.check(L.b2r_colscale(_p(g), _p(w), _p(da), a.shape[0], a.shape[1], _stream()), "b2r_colscale")
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            _lib.check(L.b2r_colsum_prod(_p(g), _p(a), _p(dw), a.shape[0], a.shape[1], _stream()), "b2r_colsum_prod")
        return da, dw


def colscale(a, w):
    return _ColScale.apply(a, w)


class _GatherConcat(torch.autograd.Function):
    """x[p, :] = [ Tu[uid[p // C]] ; Ti[iid[p]] ]  (NeuMF.py:61-69: repeated user ids + concat), written by two
    strided gathers into one [B*C, 2d] buffer; backward: one row-sparse scatter per table reading its column
    block of the dense gradient in place."""

    @staticmethod
    def forward(ctx, Tu, Ti, uid, iid):
        _need_cuda(Tu, Ti, uid, iid)
        uid, iid = _i64c(uid, "user_id"), _i64c(iid, "item_id")
        B, Cn = iid.shape
        d = Tu.shape[1]
        n = B * Cn
        x = torch.empty((n, 2 * d), dtype=torch.float32, device=Tu.device)
        L = _lib.load()
        ef = _p(err_flag(Tu.device))
        _lib.check(L.b2r_gather_rows_strided(_p(Tu), _p(uid), Tu.shape[0], _p(x), 2 * d, n, d, Cn, ef, _stream()),
                   "b2r_gather_rows_strided")
        _lib.check(L.b2r_gather_rows_strided(_p(Ti), _p(iid), Ti.shape[0], x.data_ptr() + 4 * d, 2 * d, n, d, 1, ef,
                                             _stream()), "b2r_gather_rows_strided")
        ctx.save_for_backward(uid, iid)
        ctx.Tu, ctx.Ti = Tu, Ti
        return x

    @staticmethod
    def backward(ctx, dx):
        uid, iid = ctx.saved_tensors
        Tu, Ti = ctx.Tu, ctx.Ti
        B, Cn = iid.shape
        d = Tu.shape[1]
        n = B * Cn
        dx = _f32c(dx, "dx")
        gu = gi = None
        if ctx.needs_input_grad[0]:
            # one position per sample-candidate pair, id = uid[p // C]: materialise the repeated ids for the plan
            rep = uid.repeat_interleave(Cn)
            gu = _table_grad(Tu, rep, Source(src=dx, n=n, ld=2 * d))
        if ctx.needs_input_grad[1]:
            gi = _table_grad(Ti, iid, Source(src=dx[:, d:], n=n, ld=2 * d))
        return gu, gi, None, None


def gather_concat(Tu, Ti, uid, iid):
    return _GatherConcat.apply(Tu, Ti, uid, iid)
