"""Recommendations from a trained model: top-K item lists for trained users and for interaction histories folded in at call time, and
the `candidate_indices` file of the reference's augmentation stage.

Scoring is `ops.score_topk` (llmrec_score_topk_f32): <U[u], I[i]> over the whole catalog, items of the user's mask row excluded, ties to
the lowest item id, K <= 64; a row with fewer than K candidates is padded with id -1 and score -inf.  Histories go through
`engine.HotPath.fold_in`.  The host side only builds CSRs (the mask rows, the folded-in histories) and the output file.
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import torch

from . import ops
from .graph import histories_csr

MAX_K = 64                 # the selection of llmrec_score_topk_f32
EXCLUDE = ("train", "none")
USER_BLOCK = 32768         # users scored per launch (as utility/batch_test.test_torch)


def check_k(K, n_items):
    if isinstance(K, bool) or not isinstance(K, (int, np.integer)) or not 1 <= int(K) <= min(MAX_K, int(n_items)):
        raise ValueError(f"K = {K!r}: recommendations take K in 1..{min(MAX_K, int(n_items))} (at most {MAX_K}, the scoring kernel's "
                         f"selection width, and at most n_items = {int(n_items)})")
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


def top_k(engine, train_rowptr, train_col, users=None, K=10, exclude="train", histories=None, mode=0):
    """Top-K of a model whose last full `forward()` is current (U, I and the item side).
    users: trained user ids (default every user), scored from U's rows; with `histories` they name the trained id of each history (or
    -1), and may be omitted.  histories: a sequence of item-id lists or a (rowptr, col) pair; they are folded in (HotPath.fold_in).
    exclude: "train" masks the training row of a trained user, and the history itself for a folded-in one; "none" masks nothing.
    train_rowptr / train_col: the training rows (int32 device CSR, rows sorted), the mask of exclude="train".
    mode: ops.SCORE_MODE.  -> (ids int64 [m x K], scores fp32 [m x K]) on the engine's device."""
    check_engine(engine)
    K = check_k(K, engine.ni)
    if exclude not in EXCLUDE:
        raise ValueError(f"exclude = {exclude!r}: one of {EXCLUDE}")
    dev = engine.E_u.device
    if histories is None:
        u = np.arange(engine.nu) if users is None else np.asarray(users, dtype=np.int64).reshape(-1)
        if u.size and (u.min() < 0 or u.max() >= engine.nu):
            raise ValueError(f"users: trained user ids are in [0, {engine.nu})")
        if exclude == "train":
            mrp, mcol = train_rowptr, train_col
        else:
            mrp, mcol = torch.zeros(engine.nu + 1, dtype=torch.int32, device=dev), torch.zeros(0, dtype=torch.int32, device=dev)   # no row read
        return _score(engine.U, engine.I, _i32(u, dev), mrp, mcol, K, mode)
    R = histories_csr(histories, engine.ni)
    m = R.shape[0]
    rp, col = _i32(R.indptr, dev), _i32(R.indices, dev)
    U_new = engine.fold_in(R.indptr, R.indices, known=users)
    if exclude == "none":
        rp, col = torch.zeros(m + 1, dtype=torch.int32, device=dev), col[:0]
    return _score(U_new, engine.I, _i32(np.arange(m), dev), rp, col, K, mode)


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
