"""Exact host restatement of `llmrec_device_sample_batch` (csrc/device_sampler.cu, `--device_sampler 1`).  TEST INFRASTRUCTURE ONLY.

`sample(...)` returns the [4 x cap] index buffer one launch leaves behind and the step after it, bit for bit, written in numpy uint64
with wrapping arithmetic.  It states the kernel's definition, not its mechanism (no radix select, no ballots):

    base          = splitmix64(seed ^ splitmix64(step))
    Rng{b0, c0}   word k (k = 1, 2, ...) = splitmix64(b0 + 0xD1342543DE82EF95 * (c0 + k)) >> 32;  below(n) = (word * n) >> 32
    users         batch <= n_exist: the `batch` smallest of key(i) = splitmix64(base ^ (0xA5A5A5A5 + i * 0x9E3779B97F4A7C15)) >> 32 over
                  the exist indices i, ties to the lower index, emitted in ascending i;
                  batch > n_exist: users[b] = exist[below(n_exist)] of Rng{base ^ 0x1111, 4b}
    pos / neg     Rng{base ^ 0x2222, b << 20}: pos = col[e0 + below(deg)]; then up to 2^16 candidates below(n_items) until one is not in
                  the (sorted) row; if all 2^16 were train items, the r-th non-member for r = below(n_items - deg)
    augmented     the min(n_aug, batch) smallest of key2(i) = splitmix64(base ^ (0x3333 + i * 0xD6E8FEB86659FD93)) >> 32 over the batch
                  positions, ties to the lower position; a position is kept when uid in [0, n_aug_table) and both table ids are in
                  [0, aug_limit); kept edges are appended in position order, up to cap
    meta          out[3, 0:2] = meta_table[B'] for B' = batch + kept; the step advances by one
"""
from __future__ import annotations

import numpy as np

U64 = np.uint64
M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15
RNG_MUL = 0xD1342543DE82EF95
KEY2_MUL = 0xD6E8FEB86659FD93
TRIES = 1 << 16


def splitmix64(x):
    """elementwise over a uint64 array (or a Python int), wrapping"""
    with np.errstate(over="ignore"):
        x = np.asarray(x, dtype=U64) + U64(GOLDEN)
        x = (x ^ (x >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> U64(27))) * U64(0x94D049BB133111EB)
        return x ^ (x >> U64(31))


def batch_base(seed, step):
    return int(splitmix64(U64(int(seed) & M64) ^ splitmix64(int(step) & M64)))


def rng_words(b0, ctr):
    """word number ctr (the value of ++ctr) of Rng{b0, .}: uint64 array of 32-bit values"""
    with np.errstate(over="ignore"):
        return splitmix64(U64(b0) + U64(RNG_MUL) * np.asarray(ctr, dtype=U64)) >> U64(32)


def below(word, n):
    return ((np.asarray(word, dtype=U64) * np.asarray(n, dtype=U64)) >> U64(32)).astype(np.int64)


def user_keys(base, n):
    i = np.arange(n, dtype=U64)
    return splitmix64(U64(base) ^ (U64(0xA5A5A5A5) + i * U64(GOLDEN))) >> U64(32)


def aug_keys(base, n):
    i = np.arange(n, dtype=U64)
    return splitmix64(U64(base) ^ (U64(0x3333) + i * U64(KEY2_MUL))) >> U64(32)


def smallest(keys, k):
    """indices of the k smallest keys, ties to the lower index, ascending"""
    k = min(int(k), len(keys))
    if k <= 0:
        return np.zeros(0, dtype=np.int64)
    if k == len(keys):
        return np.arange(k, dtype=np.int64)
    T = np.partition(keys, k - 1)[k - 1]
    less = np.flatnonzero(keys < T)
    ties = np.flatnonzero(keys == T)[:k - len(less)]
    return np.sort(np.concatenate([less, ties]))


def threshold_ties(keys, k):
    """(number of keys equal to the k-th smallest, how many of them the selection takes)"""
    T = np.partition(keys, k - 1)[k - 1]
    return int((keys == T).sum()), k - int((keys < T).sum())


def draw_users(base, exist, batch):
    exist = np.asarray(exist)
    n = len(exist)
    if batch <= n:
        return exist[smallest(user_keys(base, n), batch)].astype(np.int64)
    b = np.arange(batch, dtype=U64)
    return exist[below(rng_words(int(base) ^ 0x1111, b * U64(4) + U64(1)), n)].astype(np.int64)


def _member(rows, r, c):
    """c[a, j] in row rows[r[a]] (each row sorted ascending)"""
    out = np.zeros(c.shape, dtype=bool)
    for a in range(len(r)):
        row = rows[r[a]]
        if len(row):
            j = np.minimum(np.searchsorted(row, c[a]), len(row) - 1)
            out[a] = row[j] == c[a]
    return out


def draw_pos_neg(base, users, rowptr, col, n_items):
    """pos, neg and the number of words each position consumed"""
    B = len(users)
    b0 = int(base) ^ 0x2222
    ctr = np.arange(B, dtype=U64) << U64(20)
    e0 = rowptr[users].astype(np.int64)
    deg = rowptr[users + 1].astype(np.int64) - e0
    rows = [np.asarray(col[e0[b]:e0[b] + deg[b]]) for b in range(B)]
    pos = np.zeros(B, dtype=np.int64)
    has = deg > 0
    ctr[has] += U64(1)
    pos[has] = col[e0[has] + below(rng_words(b0, ctr[has]), deg[has])]
    neg = np.zeros(B, dtype=np.int64)
    active = np.arange(B)
    tries, k = 0, 4
    while len(active) and tries < TRIES:                       # every active position has drawn `tries` candidates so far
        k = min(k, TRIES - tries)
        c = below(rng_words(b0, ctr[active, None] + np.arange(1, k + 1, dtype=U64)[None, :]), n_items)
        miss = ~_member(rows, active, c)
        found = miss.any(1)
        first = miss.argmax(1)
        neg[active[found]] = c[found, first[found]]
        ctr[active[found]] += (first[found] + 1).astype(U64)
        ctr[active[~found]] += U64(k)
        neg[active[~found]] = c[~found, -1]
        active = active[~found]
        tries += k
        k *= 4
    for b in active:                                           # 2^16 train items in a row: the r-th non-member
        if deg[b] >= n_items:
            continue
        ctr[b] += U64(1)
        r = int(below(rng_words(b0, ctr[b]), n_items - deg[b]))
        neg[b] = np.setdiff1d(np.arange(n_items), rows[b])[r]
    return pos, neg, ctr - (np.arange(B, dtype=U64) << U64(20))


def sample(state, exist, rowptr, col_sorted, n_items, batch, n_aug, aug_pos, aug_neg, n_aug_table, aug_limit, meta_table, cap, out=None):
    """One launch.  state = (seed, step); meta_table: [cap + 1, 2]; out: the buffer before the launch ([4, cap], default all -7).
    Returns (buffer after the launch as int32 [4, cap], new step)."""
    seed, step = (int(x) for x in state)
    exist, rowptr, col = np.asarray(exist), np.asarray(rowptr, dtype=np.int64), np.asarray(col_sorted)
    buf = np.full((4, cap), -7, dtype=np.int64) if out is None else np.array(out, dtype=np.int64)
    base = batch_base(seed, step)
    B = int(batch)
    users = draw_users(base, exist, B)
    pos, neg, _ = draw_pos_neg(base, users, rowptr, col, int(n_items))
    buf[0, :B], buf[1, :B], buf[2, :B] = users, pos, neg
    kept = 0
    if n_aug > 0 and aug_pos is not None:
        sel = smallest(aug_keys(base, B), min(int(n_aug), B))
        u = users[sel]
        ok = (u >= 0) & (u < n_aug_table)
        uc = np.where(ok, u, 0)
        ap = np.where(ok, np.asarray(aug_pos, dtype=np.int64)[uc], -1)
        an = np.where(ok, np.asarray(aug_neg, dtype=np.int64)[uc], -1)
        ok &= (ap >= 0) & (an >= 0) & (ap < aug_limit) & (an < aug_limit)
        kept = min(int(ok.sum()), cap - B)
        buf[0, B:B + kept], buf[1, B:B + kept], buf[2, B:B + kept] = u[ok][:kept], ap[ok][:kept], an[ok][:kept]
    Bp = B + kept
    buf[3, 0:2] = np.asarray(meta_table).reshape(-1, 2)[Bp]
    return buf.astype(np.int32), step + 1


def sorted_rows(rowptr, col):
    rows = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
    return np.asarray(col)[np.lexsort((col, rows))].astype(np.int32)


def csr(rows):
    rowptr = np.zeros(len(rows) + 1, dtype=np.int32)
    np.cumsum([len(r) for r in rows], out=rowptr[1:])
    col = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows]) if rows else np.zeros(0, np.int32)
    return rowptr, col


def meta_table_for(cap):
    """{B', n_keep} with a recognisable n_keep (B' * 3 + 1) so a wrong row shows"""
    bp = np.arange(cap + 1)
    return np.stack([bp, 3 * bp + 1], 1).astype(np.int32)
