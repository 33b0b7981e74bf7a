"""Host restatement of llmrec_diversify_f32 (include/llmrec_b200.h), shared by the diversify tests: `mmr_select` is the selection rule
of one pool in numpy fp32, and `diversify` is a torch-CPU stand-in for ops.diversify built on it (cosines from an fp32 matmul, not the
fmaf chain), which the CPU tests install in a child process next to tests/ops_emulator.py.  The product never imports this file."""
import numpy as np
import torch


def mmr_select(ids, s, G, K, lam):
    """The selection of llmrec_diversify_f32 for one pool, in numpy fp32: ids int64 [P] (< 0 = padding), s fp32 [P], G fp32 [P x P] the
    cosines between pool entries (G[p, q] = cos(ids[p], ids[q])).  Each round's key is (obj, NaN last, score desc, -0 == +0), then id,
    then pool position; obj = s in round 1, lam * s - mu * m after (numpy rounds each fp32 op once).  -> (ids [K], scores [K], sims [K])."""
    lam = np.float32(lam)
    mu = np.float32(1) - lam
    P = ids.size
    pos = np.arange(P)
    alive = ids >= 0
    m = np.full(P, -np.inf, dtype=np.float32)
    out_i, out_v, out_s = np.full(K, -1, np.int64), np.full(K, -np.inf, np.float32), np.full(K, -np.inf, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(K):
            c = pos[alive]
            if c.size == 0:
                break
            obj = s[c] if t == 0 else lam * s[c] - mu * m[c]
            nan = np.isnan(obj)
            k = c[np.lexsort((c, ids[c], -np.where(nan, 0, obj).astype(np.float64), nan))[0]]
            out_i[t], out_v[t], out_s[t] = ids[k], s[k], m[k]
            alive &= ids != ids[k]
            g = G[:, k]
            upd = alive & (g > m)
            m[upd] = g[upd]
    return out_i, out_v, out_s


def diversify(X, pool_ids, pool_scores, K, lam):         # stands in for ops.diversify (llmrec_diversify_f32)
    n = X.shape[0]
    ids = pool_ids.long().clone()
    ids[(ids < 0) | (ids >= n)] = -1
    outs = []
    for b in range(ids.shape[0]):
        r = ids[b]
        xr = X[r.clamp(min=0)]
        outs.append(mmr_select(r.numpy(), pool_scores[b].numpy().astype(np.float32), (xr @ xr.t()).numpy(), K, lam))
    return tuple(torch.from_numpy(np.stack([o[j] for o in outs]) if outs else np.zeros((0, K), dt))
                 for j, dt in enumerate((np.int64, np.float32, np.float32)))
