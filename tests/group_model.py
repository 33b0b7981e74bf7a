"""Host restatement of group recommendations (llmrec_score_topk_group_f32): the exact group rule over member scores, and the ranking
with masks and padding.  Used by the CPU tests (through the `score_topk_group` stand-in below) and the GPU tests."""
import numpy as np
import torch


def aggregate(S, agg):
    """S float32 [n_members x n] (member scores, members in ascending id) -> float32 [n]: mean = the fp32 sum 0 + s_0 + s_1 + ...,
    then one division by n_members; min / max = the exact extreme taken in member order, a NaN member making it NaN."""
    S = np.asarray(S, dtype=np.float32)
    if agg == "mean":
        v = np.zeros(S.shape[1], np.float32)
        for r in S:
            v = v + r                                                   # float32 + float32: one IEEE rounding
        return v / np.float32(S.shape[0])
    v = np.full(S.shape[1], np.inf if agg == "min" else -np.inf, np.float32)
    with np.errstate(invalid="ignore"):
        for r in S:
            take = ((r < v) if agg == "min" else (r > v)) | np.isnan(r)
            v = np.where(take & ~np.isnan(v), r, v)
    return v


def rank(scores, ids, K):
    """scores float32 [n] of the catalog ids `ids` (masked ones already removed) -> (ids int64 [K], scores float32 [K]) by (score desc,
    id asc); NaN and -inf never returned; padded with -1 / -inf."""
    scores, ids = np.asarray(scores, np.float32), np.asarray(ids, np.int64)
    ok = ~np.isnan(scores) & (scores != -np.inf)
    s, i = scores[ok], ids[ok]
    o = np.lexsort((i, -s.astype(np.float64)))[:K]
    out_i, out_s = np.full(K, -1, np.int64), np.full(K, -np.inf, np.float32)
    out_i[:o.size], out_s[:o.size] = i[o], s[o]
    return out_i, out_s


def member_scores(U, I, rows):
    """Stand-in member scores: float64 products summed in float64, rounded once to fp32 (independent of which rows share a call)."""
    return (U[torch.as_tensor(rows).long()].double() @ I.double().t()).float()


def score_topk_standin(U, I, users, mask_rowptr, mask_col, K, mode=0, want_vals=False):          # llmrec_score_topk_f32
    """score_topk on `member_scores` arithmetic, so a singleton group and its member's list see the same bits"""
    S = member_scores(U, I, users).numpy()
    ids = np.arange(I.shape[0])
    rp, col = mask_rowptr.long().numpy(), mask_col.long().numpy()
    out = [rank(S[b][~np.isin(ids, col[rp[u]:rp[u + 1]])], ids[~np.isin(ids, col[rp[u]:rp[u + 1]])], K)
           for b, u in enumerate(users.long().tolist())]
    idx = torch.tensor(np.stack([o[0] for o in out]) if out else np.zeros((0, K), np.int64), dtype=torch.int32)
    val = torch.tensor(np.stack([o[1] for o in out]) if out else np.zeros((0, K), np.float32))
    return (idx, val) if want_vals else idx


def score_topk_group_standin(U, I, member_rowptr, members, among, mask_rowptr, mask_col, K, agg="mean", mode=0, want_vals=False):
    """llmrec_score_topk_group_f32 on the host: member scores (`member_scores`), `aggregate`, group mask rows, `rank`"""
    cat = np.arange(I.shape[0]) if among is None else among.long().numpy()
    rp, mem = member_rowptr.long().numpy(), members.long().numpy()
    mrp, mcol = mask_rowptr.long().numpy(), mask_col.long().numpy()
    S = member_scores(U, I, mem).numpy()[:, cat]
    ids, vals = [], []
    for g in range(rp.size - 1):
        s = aggregate(S[rp[g]:rp[g + 1]], agg)
        keep = ~np.isin(cat, mcol[mrp[g]:mrp[g + 1]])
        i, v = rank(s[keep], cat[keep], K)
        ids.append(i); vals.append(v)
    idx = torch.tensor(np.stack(ids) if ids else np.zeros((0, K), np.int64), dtype=torch.int32)
    val = torch.tensor(np.stack(vals) if vals else np.zeros((0, K), np.float32))
    return (idx, val) if want_vals else idx
