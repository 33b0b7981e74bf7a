"""Recommendations from a trained model: top-K item lists for trained users and for interaction histories folded in at call time,
over the trained catalog or a catalog grown by items added after training, item-to-item neighbours, and the `candidate_indices` file of
the reference's augmentation stage.

Scoring is `ops.score_topk` (llmrec_score_topk_f32): <U[u], I[i]> over the whole catalog, items of the user's mask row excluded, ties to
the lowest item id, K <= 64; a row with fewer than K candidates is padded with id -1 and score -inf.  Histories go through
`engine.HotPath.fold_in`, new items (lists of the trained users who interacted with each) through `engine.HotPath.fold_in_items`; new
item j gets catalog id n_items + j.  The host side only builds CSRs (the mask rows, the folded-in histories and item lists) and the
output file.

`among` restricts the catalog to given item ids and `exclude_items` adds per-query ids to the mask rows: the catalog rows are the
argument of `ops.score_topk_among` (llmrec_score_topk_among_f32, the same kernels with the catalog given by ids), and the caller's rows
are merged with the rows of `exclude` on the device (`merge_rows`).

Explanations (`explain`) split scores exactly over the query's history items and the model's channels with `ops.explain`
(llmrec_explain_f32), reading the per-row operands of the user side: the forward's rows for trained users, `HotPath.fold_in_operands`
for histories.

Diversified lists (`diversity=`, `pool=` of `top_k` and `rerank`) take the call's own top-P list as each query's pool and select K
of it by maximal marginal relevance with `ops.diversify` (llmrec_diversify_f32), whose cosines are those of `similar_items`.

Scores of given (user, item) pairs are `ops.score_pairs` (llmrec_score_pairs_f32) and re-ranking of given candidate lists is
`ops.rerank` (llmrec_rerank_f32, K <= 1024): the same sequential fp32 chain as score_topk's returned scores, so the bits agree, and the
same mask rows (`exclusion_mask`) for exclude="train".

Group lists (`top_k_groups`) rank the catalog for sets of trained users who choose together, by the mean, minimum or maximum of the
members' scores, with `ops.score_topk_group` (llmrec_score_topk_group_f32): every member is scored, the group scores are aggregated
inside the scoring kernel and no score matrix is stored.  A group's mask row is the union of its members' rows (`group_rows`).
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import scipy.sparse as sp
import torch

from . import ops
from .engine import _known_ids
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


def _score(U, I, users, mask_rowptr, mask_col, K, mode, among=None):
    """score_topk over `users` (int32 device rows of U) in blocks -> (ids int64 [n x K], scores fp32 [n x K]) on the device; among:
    None (the whole catalog I) or the catalog's ids (int32 device, strictly ascending; score_topk_among)"""
    n, dev = int(users.numel()), U.device
    ids = torch.empty((n, K), dtype=torch.int64, device=dev)
    vals = torch.empty((n, K), dtype=torch.float32, device=dev)
    for s in range(0, n, USER_BLOCK):
        if among is None:
            idx, v = ops.score_topk(U, I, users[s:s + USER_BLOCK], mask_rowptr, mask_col, K, mode=mode, want_vals=True)
        else:
            idx, v = ops.score_topk_among(U, I, users[s:s + USER_BLOCK], among, mask_rowptr, mask_col, K, mode=mode, want_vals=True)
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


def _queries(engine, train_rowptr, train_col, users, histories):
    """The query rows of `top_k` / `rerank`, checked, before anything is folded in -> (R, rows int [m], own_rowptr, own_col, known):
    trained users are rows `users` of U (default every user) with their training rows (R and known None); histories (R, their CSR) will
    be rows 0..m-1 of their fold-in, with their own items, `users` naming each one's trained id or -1 (known)."""
    dev = engine.E_u.device
    if histories is None:
        u = np.arange(engine.nu) if users is None else np.asarray(users, dtype=np.int64).reshape(-1)
        if u.size and (u.min() < 0 or u.max() >= engine.nu):
            raise ValueError(f"users: trained user ids are in [0, {engine.nu})")
        return None, u, train_rowptr, train_col, None
    R = histories_csr(histories, engine.ni)
    m = R.shape[0]
    kn = _known_ids(users, m, engine.nu, "fold_in: known must hold one trained user id in [0, {n}) or -1 per history ({m})")
    return R, np.arange(m), _i32(R.indptr, dev), _i32(R.indices, dev), kn


def _query_rows(engine, R, known):
    """U for trained users (R None), else the fold-in of the histories R (HotPath.fold_in)"""
    return engine.U if R is None else engine.fold_in(R.indptr, R.indices, known=known)


def exclusion_mask(engine, rowptr, col, exclude, Rn=None, known=None):
    """The mask rows (int32 device CSR, rows sorted) of exclude="train": each query's own row of (rowptr, col) -- a trained user's
    training row, indexed by user id, or a history's own items -- followed by every new item n_items + j of Rn whose list names that user
    (for a history: the list names its trained id `known`; -1 names none).  exclude="none": empty rows."""
    dev = col.device
    if exclude == "none":
        return torch.zeros(rowptr.numel(), dtype=torch.int32, device=dev), col[:0]          # no row read
    if Rn is not None and Rn.nnz:
        Rt = sp.csr_matrix(Rn.T)                                              # row u: the new items whose list names trained user u
        Rt.sort_indices()
        nrp, ncol = _i32(Rt.indptr, dev), _i32(Rt.indices, dev)
        if known is not None:                                                 # a history's row: that of its trained id, or none
            nrp, ncol = select_rows(nrp, ncol, torch.from_numpy(known))
        rowptr, col = append_rows(rowptr, col, nrp, ncol, engine.ni)
    return rowptr, col


def check_exclude(exclude):
    if exclude not in EXCLUDE:
        raise ValueError(f"exclude = {exclude!r}: one of {EXCLUDE}")


def catalog_ids(among, n_catalog, device, what="among"):
    """The item ids of a restricted catalog (int list, ndarray or tensor) -> int32 device tensor, sorted with repeats removed on the
    device; raises ValueError on non-integers, ids outside [0, n_catalog) or an empty set."""
    a = _ids(among, what)
    if a.numel() == 0:
        raise ValueError(f"{what}: the catalog to rank is empty; give at least one item id")
    _check_range(a, 0, n_catalog, what, "item id")
    return torch.unique(a.to(device)).to(torch.int32)


def merge_rows(a_rowptr, a_col, b_rowptr, b_col, n_catalog):
    """Row r of the result = the sorted union of row r of a and row r of b without repeats (CSRs with the same number of rows, ids in
    [0, n_catalog); ids < 0 in b are padding and dropped) -> (rowptr, col) int32 on a's device."""
    dev = a_col.device
    a, b = a_rowptr.to(dev).long(), b_rowptr.to(dev).long()
    m = a.numel() - 1
    ra = torch.repeat_interleave(torch.arange(m, device=dev), a[1:] - a[:-1])
    rb = torch.repeat_interleave(torch.arange(m, device=dev), b[1:] - b[:-1])
    bc = b_col.to(dev).long()
    keep = bc >= 0
    keys = torch.unique(torch.cat([ra * n_catalog + a_col.long(), rb[keep] * n_catalog + bc[keep]]))      # sorted: by row, then id
    rp = torch.zeros(m + 1, dtype=torch.long, device=dev)
    rp[1:] = torch.cumsum(torch.bincount(keys // n_catalog, minlength=m), 0)
    return rp.to(torch.int32), (keys % n_catalog).to(torch.int32)


def prepare_top_k(engine, train_rowptr, train_col, users=None, K=10, exclude="train", histories=None, new_items=None, among=None,
                  exclude_items=None, diversity=None, pool=None):
    """Every check of `top_k`, and its host-side inputs, before anything is launched: -> a dict for `run_top_k`."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    n = engine.ni + (0 if Rn is None else Rn.shape[0])
    dev = engine.E_u.device
    S = None if among is None else catalog_ids(among, n, dev)
    K = check_k(K, n) if S is None else check_k(K, S.numel(), "|among|")
    lam = _check_pool_use(diversity, pool)
    div = None
    if lam is not None:                                       # the pool is the top-P list of the same call
        rankable = n if S is None else S.numel()
        cap = min(MAX_K, rankable)
        P = cap if pool is None else check_pool(pool, K, cap, f"at most {MAX_K}, the scoring kernel's selection width, and at most the "
                                                               f"{rankable} rankable ids")
        div, K = (K, lam), P
    check_exclude(exclude)
    extra = None if exclude_items is None else candidates_csr(exclude_items, n)
    R, rows, rp, col, kn = _queries(engine, train_rowptr, train_col, users, histories)
    if extra is not None and extra[0].numel() - 1 != len(rows):
        raise ValueError(f"exclude_items: {extra[0].numel() - 1} rows for {len(rows)} " + ("users" if R is None else "histories"))
    rp, col = exclusion_mask(engine, rp, col, exclude, Rn, kn)
    qrow = _i32(rows, dev)
    if extra is not None:                                    # per-query mask rows: query b reads mask row b, and U row b of its own copy
        rp, col = merge_rows(*select_rows(rp, col, qrow), extra[0], extra[1], n)
    return dict(R=R, known=kn, Rn=Rn, qrow=qrow, per_query=extra is not None, mask_rowptr=rp, mask_col=col, K=K, among=S, diversify=div)


def run_top_k(engine, job, mode=0):
    """The launches of `top_k` for a `prepare_top_k` job: fold-ins, then the scoring launches."""
    U = _query_rows(engine, job["R"], job["known"])
    I = _catalog(engine, job["Rn"])
    qrow = job["qrow"]
    if job["per_query"]:
        U = U[qrow.long()].contiguous()                      # the same fp32 rows, so the same score bits
        qrow = torch.arange(qrow.numel(), dtype=torch.int32, device=qrow.device)
    ids, vals = _score(U, I, qrow, job["mask_rowptr"], job["mask_col"], job["K"], mode, job["among"])
    if job["diversify"] is None:
        return ids, vals
    return diversify(engine, job["Rn"], ids, vals, *job["diversify"], I=I)[:2]


def top_k(engine, train_rowptr, train_col, users=None, K=10, exclude="train", histories=None, mode=0, new_items=None, among=None,
          exclude_items=None, diversity=None, pool=None):
    """Top-K of a model whose last full `forward()` is current (U, I and the item side).
    users: trained user ids (default every user), scored from U's rows; with `histories` they name the trained id of each history (or
    -1), and may be omitted.  histories: a sequence of item-id lists or a (rowptr, col) pair; they are folded in (HotPath.fold_in).
    new_items: the user lists of m items added after training (`new_items_csr`); they are folded in (HotPath.fold_in_items) and scored
    after the trained catalog as ids n_items + j.
    exclude: "train" masks the training row of a trained user, and the history itself for a folded-in one, plus every new item whose
    list names that user (for a history: its trained id); "none" masks nothing.
    among: None (the whole catalog), or the item ids to rank (int list, ndarray or tensor; ids in [0, n_items + m), repeats collapsed);
    K is then at most the number of distinct ids.
    exclude_items: None, or one row of item ids per query (`candidates_csr` forms; -1 = padding) masked on top of what `exclude` masks.
    diversity: None, or lambda in [0, 1]: the K items are then picked by `diversify` from the call's own top-`pool` list (K <= pool <= 64,
    default the smallest of 64 and the number of rankable ids), in pick order.
    train_rowptr / train_col: the training rows (int32 device CSR, rows sorted), the mask of exclude="train".
    mode: ops.SCORE_MODE.  -> (ids int64 [m x K], scores fp32 [m x K]) on the engine's device; ids are catalog ids."""
    job = prepare_top_k(engine, train_rowptr, train_col, users, K, exclude, histories, new_items, among, exclude_items, diversity, pool)
    return run_top_k(engine, job, mode)


def similar_items(engine, items, K=10, new_items=None, mode=0, among=None):
    """Item-to-item neighbours of a model whose last full `forward()` is current: each query's K nearest items by cosine of the fused
    item rows, over the trained catalog and the m new items of `new_items` (ids n_items + j, as in `top_k`); the query itself is never
    returned.  items: query ids in [0, n_items + m).  among: None (the whole catalog), or the ids the neighbours come from (as in
    `top_k`; a query need not be one of them); K is then at most the number of distinct ids.  -> (ids int64 [q x K], cosines fp32
    [q x K]) on the engine's device, ties to the lowest id, padded with -1 / -inf.  The rows are normalised by
    llmrec_row_normalize_f32 and scored against each other by score_topk; the mask row of catalog item i holds i alone."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    n = engine.ni + (0 if Rn is None else Rn.shape[0])
    dev = engine.E_u.device
    S = None if among is None else catalog_ids(among, n, dev)
    K = check_k(K, n - 1, "the catalog size - 1") if S is None else check_k(K, S.numel(), "|among|")
    q = (items.detach().cpu().numpy() if hasattr(items, "detach") else np.asarray(items)).reshape(-1)
    if q.size and (q.dtype.kind not in "iu" or q.min() < 0 or q.max() >= n):
        raise ValueError(f"items: query ids are integers in [0, {n}) (trained items, then the new ones)")
    X = ops.row_normalize(_catalog(engine, Rn))
    eye_rp, eye_col = torch.arange(n + 1, dtype=torch.int32, device=dev), torch.arange(n, dtype=torch.int32, device=dev)
    return _score(X, X, _i32(q, dev), eye_rp, eye_col, K, mode, S)


def _ids(a, what):
    """An integer id array (list, ndarray or tensor on any device) -> int64 CPU tensor, flattened; anything else raises ValueError."""
    t = a.detach().cpu() if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
    if t.numel() == 0:
        return t.reshape(-1).to(torch.int64)
    if t.dtype == torch.bool or t.dtype.is_floating_point or t.dtype.is_complex:
        raise ValueError(f"{what}: ids must be integers, got {t.dtype}")
    return t.reshape(-1).to(torch.int64)


def _check_range(ids, lo, n, what, unit):
    if ids.numel() and (int(ids.min()) < lo or int(ids.max()) >= n):
        bad = int(ids[(ids < lo) | (ids >= n)][0])
        raise ValueError(f"{what}: {unit} {bad} is outside [{max(lo, 0)}, {n})" + (" (-1 = padding)" if lo < 0 else ""))


def candidates_csr(candidates, n_catalog):
    """A caller's candidate lists -> (rowptr int64 CPU tensor [m+1], col int64 CPU tensor [nnz]), ids checked against [0, n_catalog)
    with -1 allowed as padding.  Three forms: a 2-D integer tensor / ndarray [m x C] (the `candidate_indices` layout, row r = query r's
    candidates), a (rowptr, col) pair (a tuple of two arrays / tensors), or a sequence of id lists, one per query."""
    if isinstance(candidates, tuple) and len(candidates) == 2 and all(hasattr(a, "shape") for a in candidates):
        rp, col = _ids(candidates[0], "candidates rowptr"), _ids(candidates[1], "candidates")
        if rp.numel() < 1 or int(rp[0]) != 0 or bool((rp[1:] < rp[:-1]).any()) or int(rp[-1]) != col.numel():
            raise ValueError(f"candidates: rowptr must start at 0, never decrease and end at len(col) = {col.numel()}")
    elif hasattr(candidates, "shape"):
        if len(candidates.shape) != 2:
            raise ValueError(f"candidates: a tensor / ndarray of candidates is 2-D [queries x C], got shape {tuple(candidates.shape)}")
        m, c = (int(x) for x in candidates.shape)
        col = _ids(candidates, "candidates")
        rp = torch.arange(m + 1, dtype=torch.int64) * c
    else:
        rows = [_ids(list(r) if not hasattr(r, "shape") else r, "candidates") for r in candidates]
        rp = torch.zeros(len(rows) + 1, dtype=torch.int64)
        rp[1:] = torch.cumsum(torch.tensor([r.numel() for r in rows], dtype=torch.int64), 0)
        col = torch.cat(rows) if rows else torch.zeros(0, dtype=torch.int64)
    _check_range(col, -1, n_catalog, "candidates", "item id")
    return rp, col


def check_rerank_k(K):
    if K is not None and (isinstance(K, bool) or not isinstance(K, (int, np.integer)) or not 1 <= int(K) <= ops.RERANK_MAX_K):
        raise ValueError(f"K = {K!r}: re-ranking takes K in 1..{ops.RERANK_MAX_K} (the re-ranking kernel's selection width), or None")
    return None if K is None else int(K)


CAND_BLOCK = 1 << 30       # candidates per rerank launch at most (the kernel's CSR is int32)


def _blocks(rp, limit):
    """Query blocks [s, e) of a CSR's rows (int64 CPU rowptr) holding at most `limit` candidates each (at least one row)."""
    m, s = rp.numel() - 1, 0
    while s < m:
        e = int(torch.searchsorted(rp, rp[s] + limit, right=True)) - 1
        e = min(max(e, s + 1), m)
        if int(rp[e] - rp[s]) >= 2 ** 31:
            raise ValueError(f"candidates: row {s} holds {int(rp[e] - rp[s])} candidates (at most 2^31 - 1 per row)")
        yield s, e
        s = e


def _survivors(rp, col, qrow, mrp, mcol, n):
    """The longest row of distinct candidates left after padding and the mask (the K of K=None), on the device."""
    dev = mcol.device
    m = rp.numel() - 1
    col = col.to(dev)
    r = torch.repeat_interleave(torch.arange(m, device=dev), (rp[1:] - rp[:-1]).to(dev))
    keep = col >= 0
    keys = torch.unique(r[keep] * n + col[keep])
    if mcol.numel():
        q_rp, q_col = select_rows(mrp, mcol, qrow)
        q_rp = q_rp.long()
        mr = torch.repeat_interleave(torch.arange(m, device=dev), q_rp[1:] - q_rp[:-1])
        keys = keys[~torch.isin(keys, mr * n + q_col.long())]
    return int(torch.bincount(keys // n, minlength=1).max()) if keys.numel() else 0


def prepare_rerank(engine, train_rowptr, train_col, candidates, users=None, K=None, exclude="none", histories=None, new_items=None,
                   diversity=None, pool=None):
    """Every check of `rerank`, and its host-side inputs, before anything is launched: -> a dict for `run_rerank`."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    n = engine.ni + (0 if Rn is None else Rn.shape[0])
    K = check_rerank_k(K)
    lam = _check_pool_use(diversity, pool)
    if lam is not None and pool is not None:
        pool = check_pool(pool, K or 1, ops.RERANK_MAX_K, f"at most {ops.RERANK_MAX_K}, the re-ranking kernel's selection width")
    check_exclude(exclude)
    rp, col = candidates_csr(candidates, n)
    m = rp.numel() - 1
    if histories is None and users is None and m != engine.nu:
        raise ValueError(f"candidates: {m} rows; without `users` (or `histories`) there is one row per trained user ({engine.nu})")
    R, rows, mrp, mcol, kn = _queries(engine, train_rowptr, train_col, users, histories)
    if len(rows) != m:
        raise ValueError(f"candidates: {m} rows for {len(rows)} " + ("users" if R is None else "histories"))
    qrow = _i32(rows, engine.E_u.device)
    mrp, mcol = exclusion_mask(engine, mrp, mcol, exclude, Rn, kn)
    div = None
    if lam is not None:                                       # the pool is the call's own re-ranked top-P list
        if pool is None:
            pool = max(min(ops.RERANK_MAX_K, _survivors(rp, col, qrow, mrp, mcol, n)), K or 1)
        div, K = (pool if K is None else K, lam), pool
    elif K is None:
        K = _survivors(rp, col, qrow, mrp, mcol, n)
        if K > ops.RERANK_MAX_K:
            raise ValueError(f"K = None: the longest candidate row keeps {K} ids, more than {ops.RERANK_MAX_K}; give K")
        K = max(K, 1)
    return dict(R=R, known=kn, Rn=Rn, rowptr=rp, col=col, qrow=qrow, mask_rowptr=mrp, mask_col=mcol, K=K, diversify=div)


def run_rerank(engine, job):
    """The launches of `rerank` for a `prepare_rerank` job: fold-ins, then one re-ranking launch per query block."""
    U = _query_rows(engine, job["R"], job["known"])
    I = _catalog(engine, job["Rn"])
    rp, col, qrow, K = job["rowptr"], job["col"], job["qrow"], job["K"]
    dev = qrow.device
    m = qrow.numel()
    ids = torch.empty((m, K), dtype=torch.int64, device=dev)
    vals = torch.empty((m, K), dtype=torch.float32, device=dev)
    for s, e in _blocks(rp, CAND_BLOCK):
        brp = (rp[s:e + 1] - rp[s]).to(torch.int32).to(dev)
        bcol = col[int(rp[s]):int(rp[e])].to(torch.int32).to(dev)
        idx, v = ops.rerank(U, I, qrow[s:e], brp, bcol, job["mask_rowptr"], job["mask_col"], K)
        ids[s:e].copy_(idx)
        vals[s:e].copy_(v)
    if job["diversify"] is None:
        return ids, vals
    return diversify(engine, job["Rn"], ids, vals, *job["diversify"], I=I)[:2]


def rerank(engine, train_rowptr, train_col, candidates, users=None, K=None, exclude="none", histories=None, new_items=None, diversity=None,
           pool=None):
    """Re-rank given candidate lists with a model whose last full `forward()` is current: query r's candidates (`candidates_csr` forms)
    scored against its user row by the exact fp32 chain of score_topk's returned scores, the K best by (score desc, id asc).
    users / histories / new_items / exclude as in `top_k` (exclude="train" masks exactly what `top_k` masks); queries are trained users
    (default: every user, when there are n_users candidate rows) or folded-in histories, one per candidate row.  Padding (-1), masked ids
    and repeats are dropped; a NaN score ranks after every number, a real candidate before padding.  K: 1..1024, or None for the longest
    surviving row.  diversity: None, or lambda in [0, 1]: the K items are then picked by `diversify` from the call's own re-ranked
    top-`pool` list (K <= pool <= 1024, default the smallest of 1024 and the longest surviving row, and at least K; K=None means K = pool),
    in pick order.  -> (ids int64 [m x K], scores fp32 [m x K]) on the engine's device, padded with -1 / -inf."""
    job = prepare_rerank(engine, train_rowptr, train_col, candidates, users, K, exclude, histories, new_items, diversity, pool)
    return run_rerank(engine, job)


# ---- diversified lists -------------------------------------------------------------------------------------------------------
def check_diversity(diversity):
    """None, or the trade-off lambda of `diversify`: a real number in [0, 1] -> float."""
    if diversity is None:
        return None
    if isinstance(diversity, (bool, np.bool_)) or not isinstance(diversity, (int, float, np.integer, np.floating)) or \
            not 0 <= float(diversity) <= 1:
        raise ValueError(f"diversity = {diversity!r}: lambda is a number in [0, 1] (1 ranks by score alone, 0 by dissimilarity to the "
                         "items picked before), or None")
    return float(diversity)


def check_pool(pool, K, cap, why):
    """The pool size P of a diversified call: an integer with K <= P <= cap."""
    if isinstance(pool, (bool, np.bool_)) or not isinstance(pool, (int, np.integer)) or not K <= int(pool) <= cap:
        raise ValueError(f"pool = {pool!r}: a diversified call picks K = {K} items from a pool of P, P in {K}..{cap} ({why})")
    return int(pool)


def _check_pool_use(diversity, pool):
    lam = check_diversity(diversity)
    if lam is None and pool is not None:
        raise ValueError(f"pool = {pool!r}: the pool of a diversified list; give diversity too")
    return lam


def diversify(engine, Rn, pool_ids, pool_scores, K, lam, I=None):
    """K items of each query's pool (ids int64 [m x P], -1 = padding; scores fp32 [m x P], the exact scores of `top_k` / `rerank`) picked
    greedily by maximal marginal relevance (llmrec_diversify_f32): first the best-scored, then each round the item with the largest
    lam * score - (1 - lam) * (its largest cosine to an item picked before), ties to the lowest id; a repeated id is picked once.
    Cosines are the fmaf chain over ops.row_normalize of the catalog (the trained items, then the new items of Rn; I: that catalog when
    the caller has it already), the cosines `similar_items` returns.  -> (ids int64 [m x K], scores fp32 [m x K], sims fp32 [m x K]:
    each pick's largest cosine to an earlier pick, -inf for the first), padded with -1 / -inf / -inf."""
    X = ops.row_normalize(_catalog(engine, Rn) if I is None else I)
    return ops.diversify(X, pool_ids, pool_scores, K, lam)


def check_pairs(users, items, n_users, n_catalog):
    """(users, items) of `score_pairs` -> int64 CPU tensors, checked: equal lengths, integers, trained users, catalog items."""
    u, i = _ids(users, "users"), _ids(items, "items")
    if u.numel() != i.numel():
        raise ValueError(f"score: {u.numel()} users but {i.numel()} items (one pair per position)")
    _check_range(u, 0, n_users, "users", "user id")
    _check_range(i, 0, n_catalog, "items", "item id")
    return u, i


def score_pairs(engine, users, items, new_items=None):
    """Scores of (user, item) pairs with a model whose last full `forward()` is current: <U[users[p]], I[items[p]]> by the exact fp32
    chain of score_topk's returned scores.  users: trained ids; items: trained ids or n_items + j for the j-th of `new_items` (folded in as
    in `top_k`).  -> fp32 [n] on the engine's device."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    n_cat = engine.ni + (0 if Rn is None else Rn.shape[0])
    u, i = check_pairs(users, items, engine.nu, n_cat)
    dev = engine.E_u.device
    I = _catalog(engine, Rn)
    out = torch.empty(u.numel(), dtype=torch.float32, device=dev)
    for s in range(0, u.numel(), CAND_BLOCK):
        out[s:s + CAND_BLOCK] = ops.score_pairs(engine.U, I, _i32(u[s:s + CAND_BLOCK], dev), _i32(i[s:s + CAND_BLOCK], dev))
    return out


def read_candidates(path, n_users, n_catalog):
    """A `candidate_indices` file (pickle of a 2-D integer tensor or ndarray [n_users x C], row u = user u's candidates, -1 = padding)
    -> that array, checked: the file loads, is 2-D with n_users rows and holds item ids in [0, n_catalog) or -1."""
    try:
        with open(os.fspath(path), "rb") as f:
            cand = pickle.load(f)
    except Exception as e:                                                  # noqa: BLE001 -- any unreadable file is a flag error
        raise ValueError(f"--rerank_in {path}: cannot read a pickled candidate array ({type(e).__name__}: {e})") from e
    if not hasattr(cand, "shape") or len(cand.shape) != 2 or int(cand.shape[0]) != n_users:
        raise ValueError(f"--rerank_in {path}: need a 2-D integer tensor / ndarray [n_users = {n_users} x C], got "
                         f"{type(cand).__name__} {tuple(getattr(cand, 'shape', ()))}")
    _check_range(_ids(cand, f"--rerank_in {path}"), -1, n_catalog, f"--rerank_in {path}", "item id")
    return cand


def read_among(path, n_catalog):
    """The --candidates_among file (a pickled 1-D integer tensor, ndarray or list of item ids) -> int64 CPU tensor of the distinct ids,
    sorted, checked: the file loads, is 1-D, holds integers in [0, n_catalog) and at least one id."""
    flag = f"--candidates_among {path}"
    try:
        with open(os.fspath(path), "rb") as f:
            ids = pickle.load(f)
    except Exception as e:                                                  # noqa: BLE001 -- any unreadable file is a flag error
        raise ValueError(f"{flag}: cannot read a pickled id list ({type(e).__name__}: {e})") from e
    if isinstance(ids, list):
        try:
            ids = np.asarray(ids)
        except ValueError:                                                  # a ragged list of lists
            ids = None
    if not hasattr(ids, "shape") or len(ids.shape) != 1:
        raise ValueError(f"{flag}: need a 1-D integer tensor / ndarray or a list of item ids, got {type(ids).__name__} "
                         f"{tuple(getattr(ids, 'shape', ()))}")
    return catalog_ids(ids, n_catalog, "cpu", flag).long()


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


# ---- explanations ---------------------------------------------------------------------------------------------------------------
def channels(engine):
    """The channels an explanation splits a score over: "id" (the ID layers l = 1..L-1), then the side terms of the fusion in its
    order -- "image", "text", "profile" and one per attribute key (SideLayout.fused)."""
    return ["id"] + (["image", "text", "profile"] + list(engine.keys) if engine.has_feats else [])


def check_top(top):
    if top is not None and (isinstance(top, bool) or not isinstance(top, (int, np.integer)) or not 1 <= int(top) <= ops.EXPLAIN_MAX_TOP):
        raise ValueError(f"top = {top!r}: explanations select the top 1..{ops.EXPLAIN_MAX_TOP} history items per target, or None")
    return None if top is None else int(top)


class Explanation:
    """The result of `explain` (tensors on the engine's device; m queries, P targets each, C channels):
    channels: the C channel names.  hist_rowptr int64 [m+1], hist int64 [nnz]: each query's history ids (ascending, repeats collapsed).
    contrib fp32 [P * nnz x C]: query q's block, rows P * hist_rowptr[q] .. P * hist_rowptr[q+1], is [P x H_q x C] (target, history item,
    channel).  own, last fp32 [m x P]: the user's own ID layer and the softmax layer l = L.  top_ids int64 / top_vals fp32 [m x P x N]:
    with top=N, each target's N history items with the largest summed contribution (ties to the lowest id; -1 / -inf past the history;
    a padding target -1 / 0); else None.  targets int64 [m x P]: the targets, -1 = padding (whose outputs are zeros)."""

    def __init__(self, channels, hist_rowptr, hist, contrib, own, last, top_ids, top_vals, targets):
        self.channels, self.hist_rowptr, self.hist, self.contrib = list(channels), hist_rowptr, hist, contrib
        self.own, self.last, self.top_ids, self.top_vals, self.targets = own, last, top_ids, top_vals, targets
        self._rp = hist_rowptr.cpu().tolist()

    def __len__(self):
        return len(self._rp) - 1

    def of(self, q):
        """Query q's views: dict(targets [P], hist [H], contrib [P x H x C], own [P], last [P], top_ids / top_vals [P x N] or None)."""
        if not 0 <= q < len(self):
            raise IndexError(f"query {q} of {len(self)}")
        a, b = self._rp[q], self._rp[q + 1]
        P = int(self.own.shape[1])
        return dict(targets=self.targets[q], hist=self.hist[a:b], contrib=self.contrib[P * a:P * b].view(P, b - a, len(self.channels)),
                    own=self.own[q], last=self.last[q], top_ids=None if self.top_ids is None else self.top_ids[q],
                    top_vals=None if self.top_vals is None else self.top_vals[q])


def prepare_explain(engine, train_rowptr, train_col, items, users=None, histories=None, new_items=None, top=None):
    """Every check of `explain`, and its host-side inputs, before anything is launched: -> a dict for `run_explain`."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    n = engine.ni + (0 if Rn is None else Rn.shape[0])
    top = check_top(top)
    rp, col = candidates_csr(items, n)
    m = rp.numel() - 1
    if histories is None and users is None and m != engine.nu:
        raise ValueError(f"items: {m} rows; without `users` (or `histories`) there is one row per trained user ({engine.nu})")
    R, rows, hrp, hcol, kn = _queries(engine, train_rowptr, train_col, users, histories)
    if len(rows) != m:
        raise ValueError(f"items: {m} rows for {len(rows)} " + ("users" if R is None else "histories"))
    dev = engine.E_u.device
    lens = rp[1:] - rp[:-1]
    P = int(lens.max()) if m else 0
    targets = torch.full((m, P), -1, dtype=torch.int64)                        # ragged rows padded to the longest
    if col.numel():
        owner = torch.repeat_interleave(torch.arange(m), lens)
        targets[owner, torch.arange(col.numel()) - rp[owner]] = col
    qrow = _i32(rows, dev)
    if R is None:                                                              # a trained user's history: its training row
        hrp, hcol = select_rows(train_rowptr, train_col, qrow)
    return dict(R=R, known=kn, Rn=Rn, qrow=qrow, hist_rowptr=hrp, hist_col=hcol, targets=targets.to(dev), top=top)


def explain_args(engine, job):
    """The positional arguments of `ops.explain` for a `prepare_explain` job, after the launches that produce them: the new items'
    fold-in (the catalog), and the histories' fold-in operands (or, for trained users, the forward's own rows)."""
    dev, L = engine.E_u.device, engine.L
    I = _catalog(engine, job["Rn"])
    R, qrow = job["R"], job["qrow"]
    if R is None:                                                              # trained users: the forward's own rows
        engine._fold_in_sources(True, sp.csr_matrix((qrow.numel(), engine.ni), dtype=np.float32))    # (the hoisted engine's Pi)
        layers, F, prof = engine.Ul, engine.Fu if engine.has_feats else None, engine.prof_u if engine.has_feats else None
        su = engine.ui.rs[qrow.long()].contiguous()
    else:                                                                      # histories: the operands of their fold-in
        layers, F, prof, su = engine._fold_in_operands(True, R, job["known"])
        qrow = torch.arange(qrow.numel(), dtype=torch.int32, device=dev)
    side_usr, side_src, coefs = [], [], []
    if engine.has_feats:
        side_usr, side_src, coefs = engine.sides.fused(F, prof), engine.sides.fused(engine.Pi, engine.prof_i), engine._side_coefs()
    return (layers[0], layers[L], side_usr, side_src, coefs, engine.Il[:L - 1], I, qrow, su, job["hist_rowptr"], job["hist_col"],
            job["targets"].to(torch.int32), L + 1, job["top"] or 0)


def run_explain(engine, job):
    """The launches of `explain` for a `prepare_explain` job: the new items' and histories' fold-ins, then the explanation kernel."""
    dev = engine.E_u.device
    m, P = job["targets"].shape
    top, N = job["top"] is not None, job["top"] or 0
    if m and P:
        contrib, own, last, tids, tvals = ops.explain(*explain_args(engine, job))
    else:                                                                      # nothing to launch
        contrib = torch.zeros((0, len(channels(engine))), dtype=torch.float32, device=dev)
        own, last = (torch.zeros((m, P), dtype=torch.float32, device=dev) for _ in range(2))
        tids, tvals = torch.full((m, P, N), -1, dtype=torch.int32, device=dev), torch.zeros((m, P, N), dtype=torch.float32, device=dev)
    return Explanation(channels(engine), job["hist_rowptr"].long(), job["hist_col"].long(), contrib, own, last,
                       tids.long() if top else None, tvals if top else None, job["targets"])


def explain(engine, train_rowptr, train_col, items, users=None, histories=None, new_items=None, top=None):
    """Explain scores of a model whose last full `forward()` is current: <U[u], I[i]> of every query u and each of its targets i, split
    exactly over u's history items and the model's channels (`channels`), plus the user's own ID layer and the softmax layer (see
    `Explanation` and llmrec_explain_f32).  items: each query's targets in the forms `rerank` takes for candidates (a 2-D [m x P] array
    with -1 padding, id lists padded to the longest, or a (rowptr, col) pair); ids in [0, n_items + m_new).  users / histories /
    new_items as in `top_k`: trained users (default every user, with one row per user) have their training rows as history, histories
    are folded in (repeats collapse; an unknown user has no ID layer, so own = 0) and new item j is target n_items + j.  top: None, or
    N in 1..64 to also select each target's N most helpful history items on the device.  -> Explanation."""
    return run_explain(engine, prepare_explain(engine, train_rowptr, train_col, items, users, histories, new_items, top))


# ---- group recommendations ------------------------------------------------------------------------------------------------------
GROUP_AGGS = tuple(ops.GROUP_AGG)


def check_agg(agg):
    if not isinstance(agg, str) or agg not in GROUP_AGGS:
        raise ValueError(f"agg = {agg!r}: one of {GROUP_AGGS} (the mean of the members' scores, the least misery, the most pleasure)")
    return agg


def groups_csr(groups, n_users, what="groups"):
    """Groups of trained users -- a sequence of user-id lists or a (rowptr, col) pair -- checked and made canonical: ids are integers in
    [0, n_users), repeats collapse and members come in ascending id, each group has 1..64 distinct members (64 = one tile of the
    scoring kernel).  -> (rowptr int64 CPU tensor [g+1], col int64 CPU tensor)."""
    if isinstance(groups, tuple) and len(groups) == 2 and all(hasattr(a, "shape") for a in groups):
        rp, col = _ids(groups[0], f"{what} rowptr"), _ids(groups[1], what)
    else:
        if isinstance(groups, (str, bytes)) or not hasattr(groups, "__iter__"):
            raise ValueError(f"{what}: a sequence of user-id lists or a (rowptr, col) pair, got {type(groups).__name__}")
        rows = []
        for r in groups:
            if isinstance(r, (str, bytes)) or not (hasattr(r, "shape") or hasattr(r, "__iter__")):
                raise ValueError(f"{what}: each group is a list of user ids, got {type(r).__name__}")
            rows.append(_ids(r if hasattr(r, "shape") else list(r), what))
        rp = torch.zeros(len(rows) + 1, dtype=torch.int64)
        rp[1:] = torch.cumsum(torch.tensor([r.numel() for r in rows], dtype=torch.int64), 0)
        col = torch.cat(rows) if rows else torch.zeros(0, dtype=torch.int64)
    R = history_matrix(rp, col, n_users, what=what, unit="user id")
    sizes = np.diff(R.indptr)
    if sizes.size and sizes.min() < 1:
        raise ValueError(f"{what}: group {int(np.argmin(sizes))} is empty; a group has 1..{ops.GROUP_MAX_MEMBERS} members")
    if sizes.size and sizes.max() > ops.GROUP_MAX_MEMBERS:
        g = int(np.argmax(sizes))
        raise ValueError(f"{what}: group {g} has {int(sizes[g])} distinct members; at most {ops.GROUP_MAX_MEMBERS} (one tile of the "
                         "scoring kernel)")
    return torch.from_numpy(R.indptr.astype(np.int64)), torch.from_numpy(R.indices.astype(np.int64))


def group_rows(rowptr, col, members, member_rowptr, n_catalog):
    """Row g = the sorted union of rows members[member_rowptr[g] .. member_rowptr[g+1]) of an int32 CSR (int64 CPU member_rowptr)
    -> (rowptr, col) int32 on the CSR's device."""
    dev = col.device
    mrp, mcol = select_rows(rowptr, col, members.long())
    mrp = mrp.long()
    ng, nm = member_rowptr.numel() - 1, members.numel()
    group_of = torch.repeat_interleave(torch.arange(ng, device=dev), (member_rowptr[1:] - member_rowptr[:-1]).to(dev))
    owner = torch.repeat_interleave(torch.arange(nm, device=dev), mrp[1:] - mrp[:-1])
    keys = torch.unique(group_of[owner] * n_catalog + mcol.long())                        # sorted: by group, then id
    rp = torch.zeros(ng + 1, dtype=torch.long, device=dev)
    rp[1:] = torch.cumsum(torch.bincount(keys // n_catalog, minlength=ng), 0)
    return rp.to(torch.int32), (keys % n_catalog).to(torch.int32)


def prepare_group_top_k(engine, train_rowptr, train_col, groups, K=10, agg="mean", exclude="train", new_items=None, among=None,
                        exclude_items=None):
    """Every check of `top_k_groups`, and its host-side inputs, before anything is launched: -> a dict for `run_group_top_k`."""
    check_engine(engine)
    Rn = new_items_csr(new_items, engine.nu)
    n = engine.ni + (0 if Rn is None else Rn.shape[0])
    dev = engine.E_u.device
    S = None if among is None else catalog_ids(among, n, dev)
    K = check_k(K, n) if S is None else check_k(K, S.numel(), "|among|")
    check_agg(agg)
    check_exclude(exclude)
    extra = None if exclude_items is None else candidates_csr(exclude_items, n)
    grp_rp, grp_col = groups_csr(groups, engine.nu)
    ng = grp_rp.numel() - 1
    if extra is not None and extra[0].numel() - 1 != ng:
        raise ValueError(f"exclude_items: {extra[0].numel() - 1} rows for {ng} groups")
    members = _i32(grp_col.numpy(), dev)
    if exclude == "train":                                   # each member's training row and the new items naming it, united
        urp, ucol = exclusion_mask(engine, train_rowptr, train_col, "train", Rn)
        rp, col = group_rows(urp, ucol, members, grp_rp, n)
    else:
        rp, col = torch.zeros(ng + 1, dtype=torch.int32, device=dev), torch.zeros(0, dtype=torch.int32, device=dev)
    if extra is not None:
        rp, col = merge_rows(rp, col, extra[0], extra[1], n)
    return dict(Rn=Rn, member_rowptr=grp_rp, members=members, mask_rowptr=rp, mask_col=col, K=K, agg=agg, among=S)


def run_group_top_k(engine, job, mode=0):
    """The launches of `top_k_groups` for a `prepare_group_top_k` job: the new items' fold-in, then one group launch per block of
    groups holding at most USER_BLOCK members."""
    I = _catalog(engine, job["Rn"])
    grp_rp, members, mrp, K = job["member_rowptr"], job["members"], job["mask_rowptr"], job["K"]
    ng, dev = grp_rp.numel() - 1, members.device
    ids = torch.empty((ng, K), dtype=torch.int64, device=dev)
    vals = torch.empty((ng, K), dtype=torch.float32, device=dev)
    for s, e in _blocks(grp_rp, USER_BLOCK):
        a, b = int(grp_rp[s]), int(grp_rp[e])
        idx, v = ops.score_topk_group(engine.U, I, grp_rp[s:e + 1] - a, members[a:b], job["among"], mrp[s:e + 1], job["mask_col"], K,
                                      agg=job["agg"], mode=mode, want_vals=True)
        ids[s:e].copy_(idx)
        vals[s:e].copy_(v)
    return ids, vals


def top_k_groups(engine, train_rowptr, train_col, groups, K=10, agg="mean", exclude="train", mode=0, new_items=None, among=None,
                 exclude_items=None):
    """Top-K for groups of trained users of a model whose last full `forward()` is current.  groups: user-id lists or a (rowptr, col)
    pair (`groups_csr`: repeats collapse, members taken in ascending id, 1..64 per group).  A group's score of item i, with s(u, i) the
    exact fp32 chain of `score_pairs`: agg="mean" the fp32 sum of s(u, i) over the members in ascending id, then one division by their
    number; "min" / "max" the exact minimum / maximum (a NaN member score makes it NaN).  exclude: "train" masks every member's
    training row and every new item whose list names a member; "none" masks nothing.  new_items / among / exclude_items (one row per
    group) as in `top_k`.  -> (ids int64 [g x K], scores fp32 [g x K]) on the engine's device by (score desc, id asc); NaN and -inf
    group scores are never returned; padded with -1 / -inf."""
    job = prepare_group_top_k(engine, train_rowptr, train_col, groups, K, agg, exclude, new_items, among, exclude_items)
    return run_group_top_k(engine, job, mode)


def read_groups(path, n_users):
    """The --groups_in file (a pickled sequence of trained-user-id lists, one per group) -> (rowptr, col) of `groups_csr`, checked: the
    file loads, and every group holds 1..64 distinct ids in [0, n_users)."""
    flag = f"--groups_in {path}"
    try:
        with open(os.fspath(path), "rb") as f:
            groups = pickle.load(f)
    except Exception as e:                                                  # noqa: BLE001 -- any unreadable file is a flag error
        raise ValueError(f"{flag}: cannot read a pickled sequence of user-id lists ({type(e).__name__}: {e})") from e
    if isinstance(groups, tuple) or not isinstance(groups, (list, np.ndarray, torch.Tensor)):
        raise ValueError(f"{flag}: need a list (or 2-D array) of user-id lists, one per group, got {type(groups).__name__}")
    return groups_csr(groups, n_users, flag)
