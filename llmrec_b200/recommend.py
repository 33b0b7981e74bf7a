"""Recommendations from a trained model: top-K item lists for trained users and for interaction histories folded in at call time,
over the trained catalog or a catalog grown by items added after training, item-to-item neighbours, and the `candidate_indices` file of
the reference's augmentation stage.

Scoring is `ops.score_topk` (llmrec_score_topk_f32): <U[u], I[i]> over the whole catalog, items of the user's mask row excluded, ties to
the lowest item id, K <= 64; a row with fewer than K candidates is padded with id -1 and score -inf.  Histories go through
`engine.HotPath.fold_in`, new items (lists of the trained users who interacted with each) through `engine.HotPath.fold_in_items`; new
item j gets catalog id n_items + j.  The host side only builds CSRs (the mask rows, the folded-in histories and item lists) and the
output file.
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import scipy.sparse as sp
import torch

from . import ops
from .graph import histories_csr, history_matrix

MAX_K = 64                 # the selection of llmrec_score_topk_f32
EXCLUDE = ("train", "none")
USER_BLOCK = 32768         # users scored per launch (as utility/batch_test.test_torch)


def check_k(K, n_items, what="n_items"):
    if isinstance(K, bool) or not isinstance(K, (int, np.integer)) or not 1 <= int(K) <= min(MAX_K, int(n_items)):
        raise ValueError(f"K = {K!r}: recommendations take K in 1..{min(MAX_K, int(n_items))} (at most {MAX_K}, the scoring kernel's "
                         f"selection width, and at most {what} = {int(n_items)})")
    return int(K)


def check_engine(engine):
    from .engine import HotPath
    if not isinstance(engine, HotPath):
        raise ValueError(f"recommendations come from the single-GPU engines (engine.HotPath, hoist.HoistedHotPath); {type(engine).__name__} "
                         "keeps its user rows per rank")
    return engine


def _i32(a, dev):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(np.int32))).to(dev)


def _score(U, I, users, mask_rowptr, mask_col, K, mode):
    """score_topk over `users` (int32 device rows of U) in blocks -> (ids int64 [n x K], scores fp32 [n x K]) on the device"""
    n, dev = int(users.numel()), U.device
    ids = torch.empty((n, K), dtype=torch.int64, device=dev)
    vals = torch.empty((n, K), dtype=torch.float32, device=dev)
    for s in range(0, n, USER_BLOCK):
        idx, v = ops.score_topk(U, I, users[s:s + USER_BLOCK], mask_rowptr, mask_col, K, mode=mode, want_vals=True)
        ids[s:s + USER_BLOCK].copy_(idx)
        vals[s:s + USER_BLOCK].copy_(v)
    return ids, vals


def new_items_csr(new_items, n_users):
    """The user lists of items added after training -- a sequence of user-id lists or a (rowptr, col) pair, as for histories, or a
    scipy CSR -- as the binary [m x n_users] CSR (ids checked against [0, n_users), repeats collapsed); None stays None."""
    if new_items is None:
        return None
    if sp.issparse(new_items):
        R = sp.csr_matrix(new_items)
        return history_matrix(R.indptr, R.indices, n_users, what="new_items", unit="user id")
    return histories_csr(new_items, n_users, what="new_items", unit="user id")


def _catalog(engine, Rn):
    """I over the trained items, then the m new items of Rn (HotPath.fold_in_items) as rows n_items .. n_items + m - 1"""
    if Rn is None or Rn.shape[0] == 0:
        return engine.I
    return torch.cat([engine.I, engine.fold_in_items(Rn.indptr, Rn.indices)])


def select_rows(rowptr, col, rows):
    """Rows `rows` (int64, -1 = an empty row) of an int32 CSR, in that order -> (rowptr, col) int32 on the CSR's device."""
    dev = col.device
    rp, rows = rowptr.long(), rows.to(dev).long()
    r = rows.clamp(min=0)
    cnt = torch.where(rows >= 0, rp[r + 1] - rp[r], torch.zeros_like(r))
    out = torch.zeros(rows.numel() + 1, dtype=torch.long, device=dev)
    out[1:] = torch.cumsum(cnt, 0)
    owner = torch.repeat_interleave(torch.arange(rows.numel(), device=dev), cnt)
    src = rp[r[owner]] + torch.arange(int(out[-1]), device=dev) - out[owner]
    return out.to(torch.int32), col[src].to(torch.int32)


def append_rows(a_rowptr, a_col, b_rowptr, b_col, offset):
    """Row r of the result = row r of a, then row r of b with `offset` added (two int32 CSRs with the same rows).  An offset above
    every id of a keeps sorted rows sorted: the mask of a grown catalog is a training row (or history) followed by new items."""
    dev = a_col.device
    a, b = a_rowptr.to(dev).long(), b_rowptr.to(dev).long()
    n = a.numel() - 1
    rp = a + b
    col = torch.empty(int(rp[-1]), dtype=torch.int32, device=dev)
    ra = torch.repeat_interleave(torch.arange(n, device=dev), a[1:] - a[:-1])
    col[torch.arange(int(a[-1]), device=dev) + b[ra]] = a_col.to(torch.int32)           # row r starts at a[r] + b[r]
    rb = torch.repeat_interleave(torch.arange(n, device=dev), b[1:] - b[:-1])
    col[torch.arange(int(b[-1]), device=dev) + a[rb + 1]] = b_col.to(dev).to(torch.int32) + int(offset)
    return rp.to(torch.int32), col


def top_k(engine, train_rowptr, train_col, users=None, K=10, exclude="train", histories=None, mode=0, new_items=None):
    """Top-K of a model whose last full `forward()` is current (U, I and the item side).
    users: trained user ids (default every user), scored from U's rows; with `histories` they name the trained id of each history (or
    -1), and may be omitted.  histories: a sequence of item-id lists or a (rowptr, col) pair; they are folded in (HotPath.fold_in).
    new_items: the user lists of m items added after training (`new_items_csr`); they are folded in (HotPath.fold_in_items) and scored
    after the trained catalog as ids n_items + j.
    exclude: "train" masks the training row of a trained user, and the history itself for a folded-in one, plus every new item whose
    list names that user (for a history: its trained id); "none" masks nothing.
    train_rowptr / train_col: the training rows (int32 device CSR, rows sorted), the mask of exclude="train".
    mode: ops.SCORE_MODE.  -> (ids int64 [m x K], scores fp32 [m x K]) on the engine's device."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    K = check_k(K, engine.ni + (0 if Rn is None else Rn.shape[0]))
    if exclude not in EXCLUDE:
        raise ValueError(f"exclude = {exclude!r}: one of {EXCLUDE}")
    dev = engine.E_u.device
    if histories is None:
        u = np.arange(engine.nu) if users is None else np.asarray(users, dtype=np.int64).reshape(-1)
        if u.size and (u.min() < 0 or u.max() >= engine.nu):
            raise ValueError(f"users: trained user ids are in [0, {engine.nu})")
        U, rows, rp, col = engine.U, u, train_rowptr, train_col
    else:
        R = histories_csr(histories, engine.ni)
        m = R.shape[0]
        U = engine.fold_in(R.indptr, R.indices, known=users)                 # checks `users`
        rows, rp, col = np.arange(m), _i32(R.indptr, dev), _i32(R.indices, dev)
    I = _catalog(engine, Rn)
    if exclude == "none":
        rp, col = torch.zeros(rp.numel(), dtype=torch.int32, device=dev), col[:0]      # no row read
    elif Rn is not None and Rn.nnz:
        Rt = sp.csr_matrix(Rn.T)                                              # row u: the new items whose list names trained user u
        Rt.sort_indices()
        nrp, ncol = _i32(Rt.indptr, dev), _i32(Rt.indices, dev)
        if histories is not None:                                             # a history's row: that of its trained id, or none
            kn = np.full(m, -1) if users is None else (users.detach().cpu().numpy() if hasattr(users, "detach") else np.asarray(users))
            nrp, ncol = select_rows(nrp, ncol, torch.from_numpy(kn.astype(np.int64).reshape(-1)))
        rp, col = append_rows(rp, col, nrp, ncol, engine.ni)
    return _score(U, I, _i32(rows, dev), rp, col, K, mode)


def similar_items(engine, items, K=10, new_items=None, mode=0):
    """Item-to-item neighbours of a model whose last full `forward()` is current: each query's K nearest items by cosine of the fused
    item rows, over the trained catalog and the m new items of `new_items` (ids n_items + j, as in `top_k`); the query itself is never
    returned.  items: query ids in [0, n_items + m).  -> (ids int64 [q x K], cosines fp32 [q x K]) on the engine's device, ties to the
    lowest id, padded with -1 / -inf.  The rows are normalised by llmrec_row_normalize_f32 and scored against each other by
    score_topk; the mask row of catalog item i holds i alone."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    n = engine.ni + (0 if Rn is None else Rn.shape[0])
    K = check_k(K, n - 1, "the catalog size - 1")
    q = (items.detach().cpu().numpy() if hasattr(items, "detach") else np.asarray(items)).reshape(-1)
    if q.size and (q.dtype.kind not in "iu" or q.min() < 0 or q.max() >= n):
        raise ValueError(f"items: query ids are integers in [0, {n}) (trained items, then the new ones)")
    dev = engine.E_u.device
    X = ops.row_normalize(_catalog(engine, Rn))
    eye_rp, eye_col = torch.arange(n + 1, dtype=torch.int32, device=dev), torch.arange(n, dtype=torch.int32, device=dev)
    return _score(X, X, _i32(q, dev), eye_rp, eye_col, K, mode)


def write_candidates(path, ids):
    """The reference's stage-1 file (`data/<dataset>/candidate_indices`, read by gpt_ui_aug.py with pickle.load): pickle.dump of a CPU
    int64 tensor [n_users x K].  Written to `path + ".tmp"`, flushed and fsync'ed, then renamed over `path`, as checkpoint.write does:
    a reader never sees half a file."""
    ids = torch.as_tensor(ids).to("cpu", torch.int64).contiguous()
    path = os.fspath(path)
    folder = os.path.dirname(os.path.abspath(path))
    os.makedirs(folder, exist_ok=True)
    tmp = path + ".tmp"
    try:
        with open(tmp, "wb") as f:
            pickle.dump(ids, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    return path
