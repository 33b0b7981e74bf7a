"""The rest of a training step and of evaluation against exact fp64 references: the embedding fusion (csrc/fuse.cu), the BPR / prune
heads with `grad_init` and `sqnorm_grad` (csrc/bpr.cu), AdamW (csrc/adamw.cu), the hoisted-feature helpers (csrc/hoist.cu) and the
SIMT scoring, AUC and hit kernels (csrc/score_simt.cu).  Every output element is held to its own bound, worked out from the magnitudes
of the terms it is made of (u = 2^-24), never to a blanket tolerance:

    fusion forward    |y^ - y| <= 2u (L + T + d + 4) (sum_l |x_l| / L + sum_t |c_t x_t| / max(|x_t|, eps))
    fusion backward   |dx^ - dx| <= 2u (d + 8) S + 2u |old|,  S = |c| / n (|g| + |x| sum_j |x_j g_j| / n^2)  (n = |x| > eps),
                      S = |c g| / eps in the clamped branch (torch's clamp_min backward: the norm gets no gradient);
                      d_layer = g / L within 2u |g| / L
    BPR x             2u (d + 6) (sum |u p| + sum |u n|); pos == neg gives exactly fp32(1e-8)
    BPR maxi          2u 4 |logsigmoid(x^)| + 2^-140, against fp64 logsigmoid of the kernel's own x
    BPR sums          2u (d + 5) sum a^2;  kept set == stable argsort of the kernel's maxi, exactly
    BPR mf            2u (ceil(B/256) + 16) sum_kept |maxi| / n_keep      (fp64 mean of the kernel's maxi over its kept set)
    BPR emb, e-coefs  2u (d + ceil(B/256) + 24) |emb|  (twice that for the squared denominators of the e-coefficients)
    BPR row grads     2u (n_c + 2d + 2 ceil(B/256) + 60) (sum_contrib (|g| (|q| + |r|) + |e| |a|) + |G0|)   (float atomics, any order)
    grad_init loss    2u (ceil(n w / (132 * 256)) + 48) sum 0.5 |c| x^2;  G = c x within u |c x|
    sqnorm_grad loss  2u (ceil(n d / (1024 * 256)) + 40) sum 0.5 |c| x^2 + 2u |loss0|
    AdamW (one step)  m: 8u (|m| + (1-b1)(|g| + |m|)),  v: 8u (b2 v + (1-b2) g^2),
                      p: 2u (2 |p decay| + |p'|) + step/den * bound(m) + 24u |update|
    rank1_add         u |Y + s b|   (one fma)
    scaled_colsum     2u (ceil(n/1024) + n_terms + 140) (sum |s G| + |out0|)
    feat_reg_gram     dW: 2u (k + 12) |c| (|W| |G| + |b| |h|^T) + 2u |dW0|;  db: 2u (k + 24) |c| (|W| |h| + |n2 b|) + 2u |db0|;
                      loss: 2u (2k + d + 40) |c|/2 sum_i (|W_i| |G| |W_i|^T + 2 |b_i| |W_i| |h| + |n2| b_i^2) + 2u |loss0|
    score_topk / auc  integer-valued embeddings make every score exact: rankings (score desc, id asc) and Mann-Whitney counts are
                      compared exactly (AUC within 1 ulp of fp32 of the exact fraction); with random fp32 embeddings two items may swap
                      only where their fp64 scores lie within 2u d sum |u_j i_j| of each other

AdamW's reference takes the hyper-parameters as the fp32 values the kernel receives (1 - beta is formed from fp32 beta, as the kernel
does) and the bias corrections from Python's 1 - beta^t.  Rows and columns a kernel must not read hold NaN; output views sit between NaN
columns and rows a kernel must not write keep their bits.  Where a kernel promises determinism (the fixed-order tickets of the BPR heads,
grad_init, scaled_colsum and feat_reg_gram) a second call gives identical bits, also after a call of another shape.

Each bound has a self-test that runs without a GPU: an fp32 emulation of the kernel's summation order passes it, and a deliberately
wrong emulation (a term dropped or doubled, a wrong tie rule, an off-by-one chunk) fails it.  The largest error / bound ratio of each
family is printed at the end of the module (run with -s)."""
import ctypes as C
import math
import os
import sys
import zlib
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fp64_bounds import RATIOS, U, adamw_ref, check, passes, ratio_of, state_ok  # noqa: E402,F401

gpu = pytest.mark.gpu
cuda = "cuda"

EPS = 1e-12


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    if RATIOS:
        print("\nlargest error / bound per family: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def x_values(rng, n, d):
    """magnitudes in [0.5, 2), random signs"""
    return (rng.uniform(0.5, 2.0, (n, d)) * rng.choice([-1.0, 1.0], (n, d))).astype(np.float32)


def wide(a, off=4, gap=4, fill=np.nan, round4=True):
    """the fp32 block `a` as a column view of a device buffer whose other columns hold `fill` -> (buffer, view); round4: the buffer's
    row length is a multiple of 4"""
    a = np.asarray(a, np.float32)
    n, d = a.shape
    W = off + d + gap
    W += (-W) % 4 if round4 else 0
    buf = np.full((n, W), fill, np.float32)
    buf[:, off:off + d] = a
    t = torch.from_numpy(buf).to(cuda) if n else torch.empty((1, W), device=cuda)[:0]  # an empty block: row-major, non-null base
    return t, t[:, off:off + d]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def i32(a):
    return dev(np.asarray(a, np.int32))


def seq_sum_sq(x, y=None):
    """fp32 sequential sum over the columns of x*y (x*x): the order of one lane of the kernels, the worst case for a bound"""
    y = x if y is None else y
    s = np.zeros(x.shape[0], np.float32)
    for j in range(x.shape[1]):
        s = s + x[:, j] * y[:, j]
    return s


# =================================================================================================================================
# 1. fusion
# =================================================================================================================================
def fuse_fwd_ref(layers, sides, coefs):
    nl, d = len(layers), layers[0].shape[1]
    L = np.stack([l.astype(np.float64) for l in layers])
    y, mag = L.sum(0) / nl, np.abs(L).sum(0) / nl
    for x, c in zip(sides, coefs):
        x = x.astype(np.float64)
        s = float(np.float32(c)) / np.maximum(np.linalg.norm(x, axis=1), EPS)[:, None]
        y, mag = y + s * x, mag + np.abs(s * x)
    return y, 2 * U * (nl + len(sides) + d + 4) * mag


def fuse_bwd_ref(g, sides, coefs, nl, olds):
    """[(dx_t, bound)] and (d_layer, bound); olds[t]: the accumulated-into values or None"""
    g = g.astype(np.float64)
    d = g.shape[1]
    out = []
    for x, c, old in zip(sides, coefs, olds):
        c, x = float(np.float32(c)), x.astype(np.float64)
        n = np.linalg.norm(x, axis=1)[:, None]
        big = n > EPS
        nn = np.where(big, n, 1.0)
        dt, adt = (x * g).sum(1, keepdims=True), np.abs(x * g).sum(1, keepdims=True)
        r = np.where(big, c / nn * (g - dt / nn ** 2 * x), c * g / EPS)
        S = np.where(big, abs(c) / nn * (np.abs(g) + np.abs(x) * adt / nn ** 2), np.abs(c * g) / EPS)
        o = 0.0 if old is None else old.astype(np.float64)
        out.append((r + o, 2 * U * (d + 8) * S + 2 * U * np.abs(o)))
    return out, (g / nl, 2 * U * np.abs(g) / nl)


def fuse_fwd_emul(layers, sides, coefs, wrong=None):
    """fp32, the kernel's order; wrong: 'drop_side' | 'mean_off_by_one' | 'no_clamp'"""
    f = np.float32
    nl = len(layers)
    a = np.zeros_like(layers[0])
    for l in layers:
        a = a + l
    a = a * f(1.0 / (nl + (wrong == "mean_off_by_one")))
    for t, (x, c) in enumerate(zip(sides, coefs)):
        if wrong == "drop_side" and t == len(sides) - 1:
            continue
        nrm = np.sqrt(seq_sum_sq(x))
        with np.errstate(divide="ignore", invalid="ignore"):
            sc = f(c) / (nrm if wrong == "no_clamp" else np.maximum(nrm, f(EPS)))
            a = a + sc[:, None] * x
    return a


def fuse_bwd_emul(g, sides, coefs, olds, wrong=None):
    """fp32, the kernel's order; wrong: 'sb0' (no projection term) | 'clamp_b' (projection term kept when clamped) | 'no_acc'"""
    f = np.float32
    res = []
    for x, c, old in zip(sides, coefs, olds):
        ss, dt = seq_sum_sq(x), seq_sum_sq(x, g)
        nrm = np.sqrt(ss)
        big = nrm > f(EPS)
        with np.errstate(divide="ignore", invalid="ignore"):
            a = np.where(big, f(c) / nrm, f(c) / f(EPS)).astype(np.float32)
            b = np.where(big, dt / (nrm * nrm), dt / f(EPS) ** 2 if wrong == "clamp_b" else f(0)).astype(np.float32)
        if wrong == "sb0":
            b = np.zeros_like(b)
        r = a[:, None] * (g - b[:, None] * x)
        res.append(r if old is None or wrong == "no_acc" else old + r)
    return res


def fuse_sides(rng, n, d, n_sides):
    """side operands: row 0 exactly zero, rows 1 and 2 of norm 1e-14 and 3e-14 (clamped), the rest of norm ~1"""
    out = []
    for _ in range(n_sides):
        x = x_values(rng, n, d) / np.float32(math.sqrt(d))
        x[0] = 0
        for r, nrm in ((1, 1e-14), (2, 3e-14)):
            if r < n:
                x[r] = (x[r] * (nrm / np.linalg.norm(x[r].astype(np.float64)))).astype(np.float32)
        out.append(x)
    return out


def fuse_coefs(rng, n_sides):
    c = (rng.uniform(0.2, 2.0, n_sides) * rng.choice([-1.0, 1.0], n_sides)).astype(np.float32)
    if n_sides >= 2:
        c[1] = 0.0
    if n_sides >= 1:
        c[0] = -abs(c[0])
    return c


@pytest.mark.parametrize("d", [4, 13, 64])
def test_fuse_bounds_accept_fp32_and_reject_wrong_fusions(d):
    rng = np.random.default_rng(d)
    n, nl = 64, 3
    layers = [x_values(rng, n, d) for _ in range(nl)]
    sides = fuse_sides(rng, n, d, 4)
    coefs = fuse_coefs(rng, 4)
    coefs[1] = 0.7                                            # every side term visible
    y, b = fuse_fwd_ref(layers, sides, coefs)
    assert passes(fuse_fwd_emul(layers, sides, coefs), y, b)
    for wrong in ("drop_side", "mean_off_by_one", "no_clamp"):
        assert not passes(fuse_fwd_emul(layers, sides, coefs, wrong), y, b), wrong
    g = x_values(rng, n, d)
    olds = [x_values(rng, n, d), None, x_values(rng, n, d), None]
    refs, _ = fuse_bwd_ref(g, sides, coefs, nl, olds)
    for got, (y, b) in zip(fuse_bwd_emul(g, sides, coefs, olds), refs):
        assert passes(got, y, b)
    for wrong in ("sb0", "clamp_b", "no_acc"):
        bad = fuse_bwd_emul(g, sides, coefs, olds, wrong)
        assert not all(passes(got, y, b) for got, (y, b) in zip(bad, refs)), wrong
    # the projection term alone must show on every unclamped row
    bad = fuse_bwd_emul(g, sides, coefs, olds, "sb0")[0]
    y, b = refs[0]
    assert (ratio_of(bad, y, b)[3:].max(1) > 1).all()


FUSE_CFGS = [  # (n_layers, n_sides, accumulate, with d_layer)
    (1, 0, False, True), (2, 1, True, False), (3, 3, False, True), (8, 16, True, True), (4, 16, False, False), (5, 2, True, True),
    (7, 5, False, True), (6, 9, True, False)]
FUSE_FORMS = ["full", "list", "neg", "count_eq", "count_lt", "count_gt", "count_cap", "count_0", "compact"]
FUSE_N, FUSE_M = 160, 120


def fuse_rows(form, rng):
    """-> (rows | None, count | None, max_rows | None, live list entries)"""
    lst = np.concatenate([[0, 1, 2], 3 + rng.permutation(FUSE_N - 3)[:FUSE_M - 3]]).astype(np.int32)   # the zero and the clamped rows
    if form not in ("full", "list"):
        lst[[5, 50, FUSE_M - 1]] = (-1, -7, np.iinfo(np.int32).min)
    if form == "full":
        return None, None, None, np.arange(FUSE_N)
    if form in ("list", "neg", "compact"):
        return lst, None, None, lst
    cnt, mx = {"count_eq": (FUSE_M, FUSE_M), "count_lt": (FUSE_M // 2, FUSE_M), "count_gt": (FUSE_M + 37, FUSE_M),
               "count_cap": (FUSE_M, FUSE_M - 10), "count_0": (0, FUSE_M)}[form]
    return lst, cnt, mx, lst[:min(cnt, mx)]


def nan_except(a, keep_rows):
    a = a.copy()
    dead = np.ones(a.shape[0], bool)
    dead[keep_rows] = False
    a[dead] = np.nan
    return a


@gpu
@pytest.mark.parametrize("shift", [False, True], ids=["aligned", "shifted"])
@pytest.mark.parametrize("d", [4, 8, 20, 32, 36, 64, 128, 132, 256, 7, 13])
def test_fuse_fwd_bwd_match_fp64(d, shift):
    from llmrec_b200 import ops
    off = 5 if shift else 4                                   # one float off: the scalar path even when d % 4 == 0
    for ci, form in enumerate(FUSE_FORMS):
        nl, ns, acc, with_dl = FUSE_CFGS[(ci + d) % len(FUSE_CFGS)]
        rng = np.random.default_rng(1000 * d + ci + shift)
        rows, cnt, mx, live = fuse_rows(form, rng)
        valid = live[live >= 0]
        compact = form == "compact"
        what = f"d={d} shift={shift} form={form} L={nl} T={ns}"
        layers = [x_values(rng, FUSE_N, d) for _ in range(nl)]
        sides = fuse_sides(rng, FUSE_N, d, ns)
        coefs = fuse_coefs(rng, ns)
        # ---- forward -------------------------------------------------------------------------------------------------------
        if compact:                                            # sides and out are [len(rows) x d] blocks indexed by the list position
            csides = [np.where((rows >= 0)[:, None], x[np.maximum(rows, 0)], np.float32(np.nan)) for x in sides]
            y, b = fuse_fwd_ref([l[np.maximum(rows, 0)] for l in layers], [np.nan_to_num(x) for x in csides], coefs)
            y[rows < 0], b[rows < 0] = 0.0, 0.0
            dl = [wide(nan_except(l, valid), off) for l in layers]
            ds = [wide(x, off) for x in csides]
            ob, ov = wide(np.full((FUSE_M, d), np.nan, np.float32), off)
            written = np.arange(FUSE_M)
        else:
            y, b = fuse_fwd_ref(layers, sides, coefs)
            dl = [wide(nan_except(l, valid), off) for l in layers]
            ds = [wide(nan_except(x, valid), off) for x in sides]
            ob, ov = wide(np.full((FUSE_N, d), np.nan, np.float32), off)
            written = valid
        before = ob.cpu().numpy()
        ops.fuse_fwd([v for _, v in dl], [v for _, v in ds], coefs, ov, rows=None if rows is None else i32(rows), compact=compact,
                     count=None if cnt is None else i32([cnt]), max_rows=mx)
        after = ob.cpu().numpy()
        mask = np.zeros(after.shape, bool)
        mask[written, off:off + d] = True
        assert same_bits(after[~mask], before[~mask]), f"{what}: fuse_fwd wrote outside its rows / view"
        check(after[written, off:off + d], y[written], b[written], "fuse fwd", what)
        if compact:
            continue
        # ---- backward ------------------------------------------------------------------------------------------------------
        g = x_values(rng, FUSE_N, d)
        olds = [x_values(rng, FUSE_N, d) if acc else None for _ in range(ns)]
        has = [t % 3 != 2 for t in range(ns)]                 # d_sides[t] = None for every third side
        refs, (gl, gb) = fuse_bwd_ref(g, sides, coefs, nl, olds)
        gbuf = wide(nan_except(g, valid), off)
        dsb = [wide(o if acc else np.full((FUSE_N, d), np.nan, np.float32), off) if h else None for o, h in zip(olds, has)]
        dlb = wide(np.full((FUSE_N, d), np.nan, np.float32), off) if with_dl else None
        befores = [t[0].cpu().numpy() if t is not None else None for t in dsb + [dlb]]
        ops.fuse_bwd(gbuf[1], nl, dlb[1] if dlb else None, [v for _, v in ds], coefs, [t[1] if t else None for t in dsb], acc,
                     rows=None if rows is None else i32(rows), count=None if cnt is None else i32([cnt]), max_rows=mx)
        for t, (buf, bef) in enumerate(zip(dsb + [dlb], befores)):
            if buf is None:
                continue
            aft = buf[0].cpu().numpy()
            mask = np.zeros(aft.shape, bool)
            mask[valid, off:off + d] = True
            assert same_bits(aft[~mask], bef[~mask]), f"{what}: fuse_bwd wrote outside its rows / view (operand {t})"
            yy, bb = refs[t] if t < ns else (gl, gb)
            check(aft[valid, off:off + d], yy[valid], bb[valid], "fuse bwd", f"{what} operand {t}")


@gpu
def test_fuse_bwd_skips_negative_row_entries():
    """a negative entry of the backward's row list is skipped like the forward's: no row is read or written for it"""
    from llmrec_b200 import ops
    rng = np.random.default_rng(5)
    d, n = 32, 40
    x, g = x_values(rng, n, d), x_values(rng, n, d)
    rows = np.array([-1, 3, -2, 7, np.iinfo(np.int32).min], np.int32)
    xb, gbuf = wide(nan_except(x, [3, 7])), wide(nan_except(g, [3, 7]))
    dx = wide(np.full((n, d), np.nan, np.float32))
    ops.fuse_bwd(gbuf[1], 2, None, [xb[1]], [0.5], [dx[1]], False, rows=i32(rows))
    got = dx[0].cpu().numpy()
    refs, _ = fuse_bwd_ref(g, [x], [0.5], 2, [None])
    check(got[[3, 7], 4:4 + d], refs[0][0][[3, 7]], refs[0][1][[3, 7]], "fuse bwd", "negative entries")
    others = np.setdiff1d(np.arange(n), [3, 7])
    assert np.isnan(got[others]).all() and np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + d:]).all()


# =================================================================================================================================
# 2. BPR heads, grad_init, sqnorm_grad
# =================================================================================================================================
def logsigmoid64(x):
    x = np.asarray(x, np.float64)
    return np.minimum(x, 0.0) - np.log1p(np.exp(-np.abs(x)))


def sigmoid64(x):
    return 0.5 * (1.0 + np.tanh(0.5 * np.asarray(x, np.float64)))


def kept_set(maxi, n_keep):
    """the prune loss's kept set: the n_keep smallest values, ties to the lower batch position (stable argsort)"""
    keep = np.zeros(maxi.size, bool)
    keep[np.argsort(maxi, kind="stable")[:max(0, min(n_keep, maxi.size))]] = True
    return keep


def bpr_ref_head(XU, XI, users, pos, neg, d):
    """fp64 x and the per-triplet sums with their bounds"""
    a, q, r = (t.astype(np.float64) for t in (XU[users], XI[pos], XI[neg]))
    x = (a * q).sum(1) - (a * r).sum(1) + 1e-8
    bx = 2 * U * (d + 6) * (np.abs(a * q).sum(1) + np.abs(a * r).sum(1) + 1e-8)
    sums = [(t * t).sum(1) for t in (a, q, r)]
    return x, bx, sums, [2 * U * (d + 5) * s for s in sums]


def mf_ref(maxi, keep, B):
    nk = int(keep.sum())
    if nk == 0:
        return np.nan, 0.0
    m = maxi[keep].astype(np.float64)
    return -m.sum() / nk, 2 * U * (math.ceil(B / 256) + 16) * np.abs(m).sum() / nk


def bpr_grad_ref(g, e, a, q, r):
    """per-triplet row-gradient contributions and their magnitudes: (user, pos, neg) x (value, magnitude)"""
    eu, ep, en = e
    gc = g[:, None]
    return ((gc * (q - r) + eu * a, np.abs(gc) * (np.abs(q) + np.abs(r)) + abs(eu) * np.abs(a)),
            (gc * a + ep * q, np.abs(gc * a) + abs(ep) * np.abs(q)),
            (-gc * a + en * r, np.abs(gc * a) + abs(en) * np.abs(r)))


def test_bpr_bounds_accept_fp32_and_reject_wrong_heads():
    rng = np.random.default_rng(3)
    B, d = 700, 20
    XU, XI = x_values(rng, 50, d) / 4, x_values(rng, 80, d) / 4
    users, pos, neg = rng.integers(0, 50, B), rng.integers(0, 80, B), rng.integers(0, 80, B)
    neg[:5] = pos[:5]
    x, bx, sums, bs = bpr_ref_head(XU, XI, users, pos, neg, d)
    a, q, r = XU[users], XI[pos], XI[neg]
    x32 = (seq_sum_sq(a, q) - seq_sum_sq(a, r)) + np.float32(1e-8)
    assert passes(x32, x, bx) and (x32[:5] == np.float32(1e-8)).all()
    assert not (((seq_sum_sq(a, q) - seq_sum_sq(a, r)))[:5] == np.float32(1e-8)).any()     # dropping +1e-8 shows on pos == neg
    assert passes(seq_sum_sq(a), sums[0], bs[0]) and not passes(seq_sum_sq(a[:, 1:]), sums[0], bs[0])
    # maxi: fp32 logsigmoid is within a few ulp; the kept set's tie rule is exact
    m32 = (np.minimum(x32, 0) - np.log1p(np.exp(-np.abs(x32)))).astype(np.float32)
    assert passes(m32, logsigmoid64(x32), 8 * U * np.abs(logsigmoid64(x32)) + 2.0 ** -140)
    tied = np.round(m32 * 4) / 4
    nk = 201
    k = kept_set(tied, nk)
    later = np.zeros(B, bool)
    later[(B - 1 - np.argsort(tied[::-1], kind="stable"))[:nk]] = True                    # ties to the higher position
    assert k.sum() == nk and not np.array_equal(k, later)
    mf, bm = mf_ref(tied, k, B)
    assert passes(-np.float32(np.cumsum(tied[k].astype(np.float32))[-1] / np.float32(nk)), mf, bm)
    kk = k.copy()
    kk[np.nonzero(k)[0][np.argmin(tied[k])]] = False
    kk[np.nonzero(~k)[0][np.argmax(tied[~k])]] = True                                      # the smallest kept triplet swapped out
    assert not passes(mf_ref(tied, kk, B)[0], mf, bm)
    # row gradients: an fp32 accumulation in any order passes, a wrong coefficient (1/B instead of 1/n_keep) fails
    g = np.where(k, -sigmoid64(-x32) / nk, 0.0)
    e = (-4 * 0.05 / (2 * sums[0].sum()) ** 2,) * 3
    (cu, mu), _, _ = bpr_grad_ref(g, e, a, q, r)
    S = sp.csr_matrix((np.ones(B), (users, np.arange(B))), shape=(50, B))
    cnt = np.asarray(S.sum(1)).ravel()[:, None]
    ref, mag = S @ cu, S @ mu
    bound = 2 * U * (cnt + 2 * d + 2 * math.ceil(B / 256) + 60) * mag
    acc = np.zeros((50, d), np.float32)
    for b in rng.permutation(B):
        acc[users[b]] += cu[b].astype(np.float32)
    assert passes(acc, ref, bound)
    (cu2, _), _, _ = bpr_grad_ref(np.where(k, -sigmoid64(-x32) / B, 0.0), e, a, q, r)
    assert not passes(S @ cu2, ref, bound)


def work_arrays(work, h, cap):
    base = 32 + h * (7 * cap + 8)
    w = work[base: base + 7 * cap + 8]
    return {k: w[i * cap:(i + 1) * cap] for i, k in enumerate(("x", "maxi", "su", "sp", "sn", "gcoef", "keep"))} | {"e": w[7 * cap:7 * cap + 8]}


BPR_CASES = [  # (d, B, n_heads, n_keep, meta)
    (1, 1, 1, "B", None), (20, 255, 3, "B-1", None), (32, 256, 16, "1", None), (64, 257, 5, "above", None), (100, 257, 8, "0", None),
    (256, 255, 2, "B", "below"), (20, 256, 9, "frac", "equal"), (1, 257, 16, "frac", "below"), (100, 1, 2, "0", None),
    (32, 40000, 2, "frac", None), (64, 40000, 4, "B-1", "above"), (256, 40000, 1, "1", None), (64, 256, 12, "frac", "above")]


class BprCase:
    def __init__(self, d, B, n_heads, keep_spec, meta_spec, seed):
        rng = np.random.default_rng(seed)
        self.d, self.cap, self.H = d, B, n_heads
        bp = {None: B, "below": max(1, B - B // 3 - 1), "equal": B, "above": B + 100}[meta_spec]
        self.Bl = Bl = min(bp, B)
        self.nk = {"0": 0, "1": 1, "B-1": Bl - 1, "B": Bl, "above": Bl + 3, "frac": int(0.29 * Bl)}[keep_spec]
        self.meta = i32([bp, self.nk]) if meta_spec else None
        self.nu, self.ni = nu, ni = max(6, B // 3 + 6), max(8, B // 2 + 8)
        users, pos, neg = rng.integers(0, nu - 2, B), rng.integers(0, ni - 3, B), rng.integers(0, ni - 3, B)
        neg[0] = pos[0]                                       # pos == neg: x is exactly 1e-8
        if Bl >= 3:                                           # logits of +100 and -100 (logsigmoid saturates)
            users[1:3], pos[1:3], neg[1:3] = nu - 1, (ni - 1, ni - 2), (ni - 2, ni - 1)
        if Bl >= 6:
            users[4], pos[4], neg[4] = users[3], pos[3], neg[3]   # a repeated triplet
        users[Bl:], pos[Bl:], neg[Bl:] = nu - 2, ni - 3, ni - 3   # stale slots point at NaN rows
        self.users, self.pos, self.neg = users, pos, neg
        live_u, live_i = np.unique(users[:Bl]), np.unique(np.concatenate([pos[:Bl], neg[:Bl]]))
        s = np.float32(1 / math.sqrt(d))
        self.XU, self.XI = [], []
        for _ in range(n_heads):
            xu, xi = x_values(rng, nu, d) * s, x_values(rng, ni, d) * s
            xu[nu - 1], xi[ni - 1], xi[ni - 2] = 0, 0, 0
            xu[nu - 1, 0], xi[ni - 1, 0] = 10, 10
            self.XU.append(nan_except(xu, live_u))
            self.XI.append(nan_except(xi, live_i))
        self.n_g = max(1, (n_heads + 1) // 2)                 # several heads add into one gradient buffer
        self.GU0 = [x_values(rng, nu, d) for _ in range(self.n_g)]
        self.GI0 = [x_values(rng, ni, d) for _ in range(self.n_g)]
        self.wmf = np.where(np.arange(n_heads) % 4 == 2, 0.0, rng.uniform(0.5, 1.5, n_heads)).astype(np.float32)
        self.wemb = np.where(np.arange(n_heads) % 6 == 5, 0.0, rng.uniform(0.2, 1.0, n_heads)).astype(np.float32)
        self.has_gu = [h % 5 != 3 for h in range(n_heads)]
        self.has_gi = [h % 5 != 4 for h in range(n_heads)]
        self.c, self.L0 = np.float32(0.05), np.float32(1.25)

    def launch(self, heads=None, n_keep=None, work=None):
        """one bpr_heads call on fresh gradient buffers; -> dict of host results"""
        from llmrec_b200 import ops
        H = self.H if heads is None else heads
        xu = [wide(t) for t in self.XU[:H]]
        xi = [wide(t) for t in self.XI[:H]]
        gu = [wide(t) for t in self.GU0]
        gi = [wide(t) for t in self.GI0]
        hs = [(xu[h][1], xi[h][1], gu[h % self.n_g][1] if self.has_gu[h] else None, gi[h % self.n_g][1] if self.has_gi[h] else None,
               float(self.wmf[h]), float(self.wemb[h])) for h in range(H)]
        if work is None:
            work = torch.full((int(ops.N.lib().llmrec_bpr_work_elems(self.H, self.cap)),), float("nan"), device=cuda)
            work[:32] = 0
        out = torch.full((4 * H,), float("nan"), device=cuda)
        loss = torch.tensor([self.L0], device=cuda)
        ops.bpr_heads(hs, i32(self.users), i32(self.pos), i32(self.neg), self.nk if n_keep is None else n_keep, float(self.c), out, loss,
                      work, meta=self.meta if n_keep is None else None)
        return dict(out=out.cpu().numpy(), loss=loss.cpu().numpy(), work=work.cpu().numpy(), gu=[t[0].cpu().numpy() for t in gu],
                    gi=[t[0].cpu().numpy() for t in gi], work_t=work)


@gpu
@pytest.mark.parametrize("case", BPR_CASES, ids=lambda c: "-".join(map(str, c)))
def test_bpr_heads_match_fp64(case):
    d, B, H, ks, ms = case
    cs = BprCase(d, B, H, ks, ms, seed=zlib.crc32(str(case).encode()))
    res = cs.launch()
    Bl, cap, nk = cs.Bl, cs.cap, max(0, min(cs.nk, cs.Bl))
    what = f"d={d} B={B} B'={Bl} heads={H} n_keep={cs.nk}"
    work = res["work"]
    assert (work[:32] == 0).all(), "tickets not reset"
    u, p, n = cs.users[:Bl], cs.pos[:Bl], cs.neg[:Bl]
    nb = math.ceil(Bl / 256)
    grads_u = [np.zeros((cs.nu, d)) for _ in range(cs.n_g)]
    mags_u = [np.zeros((cs.nu, d)) for _ in range(cs.n_g)]
    cnt_u = [np.zeros((cs.nu, 1)) for _ in range(cs.n_g)]
    grads_i = [np.zeros((cs.ni, d)) for _ in range(cs.n_g)]
    mags_i = [np.zeros((cs.ni, d)) for _ in range(cs.n_g)]
    cnt_i = [np.zeros((cs.ni, 1)) for _ in range(cs.n_g)]
    Su = sp.csr_matrix((np.ones(Bl), (u, np.arange(Bl))), shape=(cs.nu, Bl))
    Sp = sp.csr_matrix((np.ones(Bl), (p, np.arange(Bl))), shape=(cs.ni, Bl))
    Sn = sp.csr_matrix((np.ones(Bl), (n, np.arange(Bl))), shape=(cs.ni, Bl))
    loss_ref, loss_mag = float(cs.L0), abs(float(cs.L0))
    for h in range(H):
        w = work_arrays(work, h, cap)
        for k in ("x", "maxi", "su", "sp", "sn", "gcoef", "keep"):
            assert np.isnan(w[k][Bl:]).all(), f"{what}: head {h} wrote {k} past B'"
        assert np.isnan(w["e"][3:]).all()
        x, bx, sums, bs = bpr_ref_head(cs.XU[h], cs.XI[h], u, p, n, d)
        check(w["x"][:Bl], x, bx, "bpr x", f"{what} head {h}")
        assert same_bits(w["x"][:1], np.float32([1e-8])), f"{what}: pos == neg must give x = fp32(1e-8) exactly"
        xk = w["x"][:Bl].astype(np.float64)
        ls = logsigmoid64(xk)
        check(w["maxi"][:Bl], ls, 8 * U * np.abs(ls) + 2.0 ** -140, "bpr maxi", f"{what} head {h}")
        for k, s, b in zip(("su", "sp", "sn"), sums, bs):
            check(w[k][:Bl], s, b, "bpr sums", f"{what} head {h} {k}")
        keep = kept_set(w["maxi"][:Bl], nk)
        assert np.array_equal(w["keep"][:Bl] == 1.0, keep) and np.isin(w["keep"][:Bl], (0.0, 1.0)).all(), f"{what}: kept set, head {h}"
        o = res["out"][4 * h:4 * h + 4]
        mf, bm = mf_ref(w["maxi"][:Bl], keep, Bl)
        if nk == 0:
            assert np.isnan(o[0]), "mean of an empty kept set is NaN"
        else:
            check(o[0:1], mf, bm, "bpr mf/emb", f"{what} head {h} mf")
        den = [2 * s.sum() + 1e-8 for s in sums]
        emb = float(cs.c) * sum(1 / t for t in den)
        check(o[1:2], emb, 2 * U * (d + nb + 24) * emb, "bpr mf/emb", f"{what} head {h} emb")
        assert o[2] == nk and o[3] == 0.0
        e = [-4.0 * float(cs.wemb[h]) * float(cs.c) / t ** 2 for t in den]
        check(w["e"][:3], np.array(e), 4 * U * (d + nb + 30) * np.abs(e), "bpr mf/emb", f"{what} head {h} e-coefficients")
        g = np.where(keep, -float(cs.wmf[h]) * sigmoid64(-xk) / max(nk, 1), 0.0)
        check(w["gcoef"][:Bl], g, 16 * U * np.abs(g) + 2.0 ** -126, "bpr grad", f"{what} head {h} gradient coefficients")
        if not np.isnan(o[0]):
            loss_ref += float(cs.wmf[h]) * float(o[0]) + float(cs.wemb[h]) * float(o[1])
            loss_mag += abs(float(cs.wmf[h]) * float(o[0])) + abs(float(cs.wemb[h]) * float(o[1]))
        (cu, mu), (cp, mp), (cn, mn) = bpr_grad_ref(g, e, *(t.astype(np.float64) for t in (cs.XU[h][u], cs.XI[h][p], cs.XI[h][n])))
        k = h % cs.n_g
        if cs.has_gu[h]:
            grads_u[k] += Su @ cu; mags_u[k] += Su @ mu; cnt_u[k] += Su @ np.ones((Bl, 1))
        if cs.has_gi[h]:
            grads_i[k] += Sp @ cp + Sn @ cn; mags_i[k] += Sp @ mp + Sn @ mn; cnt_i[k] += (Sp + Sn) @ np.ones((Bl, 1))
    if nk == 0:
        assert np.isnan(res["loss"][0])
    else:
        check(res["loss"], loss_ref, 2 * U * (H + 2) * loss_mag, "bpr mf/emb", f"{what} loss")
    for k in range(cs.n_g):
        for got, G0, ref, mag, cnt in ((res["gu"][k], cs.GU0[k], grads_u[k], mags_u[k], cnt_u[k]),
                                       (res["gi"][k], cs.GI0[k], grads_i[k], mags_i[k], cnt_i[k])):
            touched = cnt[:, 0] > 0
            v = got[:, 4:4 + d]
            assert np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + d:]).all()
            assert same_bits(v[~touched], G0[~touched]), f"{what}: an untouched gradient row changed"
            g0 = G0[touched].astype(np.float64)
            bound = 2 * U * (cnt[touched] + 2 * d + 2 * nb + 60) * (mag[touched] + np.abs(g0))
            check(v[touched], g0 + ref[touched], bound, "bpr grad", f"{what} gradient buffer {k}")
    # deterministic: the same bits on a second call, and after a call of another shape on the same work buffer
    live = lambda r: np.concatenate([np.concatenate([work_arrays(r["work"], h, cap)[k][:Bl] for k in ("x", "maxi", "gcoef", "keep")])
                                     for h in range(H)])
    again = cs.launch(work=res["work_t"])
    cs.launch(heads=max(1, H // 2), n_keep=1, work=res["work_t"])
    third = cs.launch(work=res["work_t"])
    for r in (again, third):
        assert same_bits(r["out"], res["out"]) and same_bits(r["loss"], res["loss"]) and same_bits(live(r), live(res)), what


@gpu
def test_grad_init_matches_fp64_and_is_deterministic():
    from llmrec_b200 import ops
    rng = np.random.default_rng(11)
    specs = [  # (n, width, off, with X, c)
        (300, 64, 4, True, 0.5), (77, 13, 4, True, -1.5), (50, 8, 4, True, 2.0), (3, 16, 4, True, 1.0), (129, 32, 5, True, 0.25),
        (40, 12, 4, False, 3.0), (64, 20, 4, True, 0.0), (1, 1, 4, True, 1.0), (4000, 100, 4, True, 0.125), (33, 7, 5, False, 1.0),
        (500, 4, 4, True, -0.75), (2, 256, 4, True, 1.0), (100, 36, 6, True, 0.5), (9, 3, 4, True, 4.0), (250, 48, 4, True, 1.0),
        (1000, 24, 4, True, 0.3)]
    for nreg in (1, 2, 5, 16):
        regions, refs = [], []
        for i, (n, w, off, hx, c) in enumerate(specs[:nreg]):
            X = x_values(rng, n, w)
            xb = wide(X, off, 4) if hx else None
            gb = wide(np.full((n, w), np.nan, np.float32), off, 2, round4=w != 8)    # width 8 with ld = 14: the scalar path
            regions.append((gb[1], xb[1] if hx else None, c))
            refs.append((gb, X if hx else np.zeros_like(X), c, off))
        loss = torch.tensor([123.0], device=cuda)
        ops.grad_init(regions, loss)
        tot, mag = 0.0, 0.0
        for gb, X, c, off in refs:
            got = gb[0].cpu().numpy()
            n, w = X.shape
            cx = float(np.float32(c)) * X.astype(np.float64)
            check(got[:, off:off + w], cx, U * np.abs(cx), "grad_init", f"{nreg} regions, region {w}x{n}")
            assert np.isnan(got[:, :off]).all() and np.isnan(got[:, off + w:]).all()
            tot += 0.5 * float(np.float32(c)) * (X.astype(np.float64) ** 2).sum()
            mag += 0.5 * abs(float(np.float32(c))) * (X.astype(np.float64) ** 2).sum()
        nmax = max(X.size for _, X, _, _ in refs)
        first = loss.cpu().numpy()
        check(first, tot, 2 * U * (math.ceil(nmax / (132 * 256)) + 48) * mag, "grad_init", f"{nreg} regions, loss (overwritten)")
        ops.grad_init(regions, loss)
        assert same_bits(loss.cpu().numpy(), first)
        ops.grad_init(regions[:1], torch.zeros(1, device=cuda))    # another shape on the same scratch
        loss.fill_(7.0)
        ops.grad_init(regions, loss)
        assert same_bits(loss.cpu().numpy(), first), "grad_init's loss changed bits"


@gpu
@pytest.mark.parametrize("with_g,acc", [(True, False), (True, True), (False, False)])
def test_sqnorm_grad_matches_fp64(with_g, acc):
    from llmrec_b200 import ops
    rng = np.random.default_rng(12 + acc)
    n, d, c = 2500, 1000, np.float32(0.37)                   # 2.5e6 > 1024 * 2048 elements: 1024 blocks stride over the table
    X = x_values(rng, n, d)
    G0 = x_values(rng, n, d) if acc else np.full((n, d), np.nan, np.float32)
    xb, gb = wide(X, 4, 4), wide(G0, 4, 4)
    loss = torch.tensor([2.5], device=cuda)
    ops.sqnorm_grad(xb[1], gb[1] if with_g else None, float(c), acc, loss)
    x64 = X.astype(np.float64)
    s = 0.5 * float(c) * (x64 ** 2).sum()
    check(loss.cpu().numpy(), 2.5 + s, 2 * U * (math.ceil(n * d / (1024 * 256)) + 40) * abs(s) + 2 * U * 2.5, "sqnorm_grad", "loss")
    got = gb[0].cpu().numpy()
    if with_g:
        ref = float(c) * x64 + (G0.astype(np.float64) if acc else 0.0)
        check(got[:, 4:4 + d], ref, 2 * U * np.abs(ref) + 2 * U * np.abs(float(c) * x64), "sqnorm_grad", f"G acc={acc}")
    else:
        assert np.isnan(got).all()
    assert np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + d:]).all()


# =================================================================================================================================
# 3. AdamW
# =================================================================================================================================
def adamw_emul(p, g, m, v, t, lr, b1, b2, eps, wd, wrong=None):
    """fp32 adam1 of the kernel; wrong: 'no_bc2' | 'step_t_minus_1' | 'skip' (the element is not updated)"""
    f = np.float32
    if wrong == "skip":
        return p, m, v
    tt = t - 1 if wrong == "step_t_minus_1" else t
    step = f(lr / (1.0 - b1 ** tt)) if tt > 0 else f(lr)
    bc2s = f(1.0) if wrong == "no_bc2" else f(math.sqrt(1.0 - b2 ** t))
    p = p * (f(1) - f(lr) * f(wd))
    m = m + (f(1) - f(b1)) * (g - m)
    v = v * f(b2) + (f(1) - f(b2)) * g * g
    den = np.sqrt(v) / bc2s + f(eps)
    return p - step * (m / den), m, v


@pytest.mark.parametrize("t", [1, 2, 10, 10000])
def test_adamw_bound_accepts_fp32_and_rejects_wrong_steps(t):
    rng = np.random.default_rng(t)
    n = 4096
    p, g = x_values(rng, n, 1)[:, 0], (rng.standard_normal(n) * 1e-2).astype(np.float32)
    m, v = (rng.standard_normal(n) * 1e-2).astype(np.float32), (rng.uniform(0, 1e-4, n)).astype(np.float32)
    if t == 1:
        m[:], v[:] = 0, 0
    hp = (1e-3, 0.9, 0.999, 1e-8, 0.01)
    refs = adamw_ref(p, g, m, v, t, *hp)
    for got, (y, b) in zip(adamw_emul(p, g, m, v, t, *hp), refs):
        assert passes(got, y, b)
    for wrong in ("no_bc2", "step_t_minus_1", "skip"):
        if wrong != "skip" and t == 10000:
            continue                                           # both bias corrections are 1 to within rounding by then
        got = adamw_emul(p, g, m, v, t, *hp, wrong=wrong)
        assert (ratio_of(got[0], *refs[0]) > 1).mean() > 0.5, wrong


ADAM_NUMELS = [1, 2, 3, 4, 5, 6, 7, 9, 1023, 1025, 1026, 1027, 4096, 4097, 33, 64, 65, 130, 131, 100003]   # 20 tensors: two launches


@gpu
@pytest.mark.parametrize("hp", [(1e-3, (0.9, 0.999), 1e-8, 0.01), (1e-2, (0.8, 0.95), 1e-6, 0.0)], ids=["defaults", "betas-wd0"])
def test_adamw_dense_steps_match_fp64(hp):
    from llmrec_b200 import ops
    lr, (b1, b2), eps, wd = hp
    rng = np.random.default_rng(int(lr * 1e4))
    params = [dev(x_values(rng, k, 1)[:, 0]) for k in ADAM_NUMELS]
    opt = ops.AdamW(params, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    for t in range(1, 11):
        grads = [dev((rng.standard_normal(k) * 1e-2).astype(np.float32)) for k in ADAM_NUMELS]
        snap = [(p.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()) for p, m, v in zip(params, opt.m, opt.v)]
        opt.step(grads)
        st = opt.state.cpu().numpy()
        assert st[0] == t
        assert state_ok(st, t, lr, b1, b2), (t, st)
        if t in (1, 2, 10):
            for i, (p0, m0, v0) in enumerate(snap):
                refs = adamw_ref(p0, grads[i].cpu().numpy(), m0, v0, t, lr, b1, b2, eps, wd)
                for name, got, (y, b) in zip("pmv", (params[i], opt.m[i], opt.v[i]), refs):
                    check(got, y, b, "adamw", f"step {t} tensor {i} (numel {ADAM_NUMELS[i]}) {name}")
    opt.state[0] = 9999.0                                     # late step: 1 - b1^t rounds to 1
    grads = [dev((rng.standard_normal(k) * 1e-2).astype(np.float32)) for k in ADAM_NUMELS]
    snap = [(p.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()) for p, m, v in zip(params, opt.m, opt.v)]
    opt.step(grads)
    st = opt.state.cpu().numpy()
    assert st[0] == 10000 and state_ok(st, 10000, lr, b1, b2), st
    for i, (p0, m0, v0) in enumerate(snap):
        refs = adamw_ref(p0, grads[i].cpu().numpy(), m0, v0, 10000, lr, b1, b2, eps, wd)
        for name, got, (y, b) in zip("pmv", (params[i], opt.m[i], opt.v[i]), refs):
            check(got, y, b, "adamw", f"step 10000 tensor {i} {name}")


def mask_words(keep):
    """uint32 bitmask over rows (RowSet layout: (n + 31) // 32 + 1 words) as an int32 CUDA tensor"""
    words = np.zeros((keep.size + 31) // 32 + 1, np.uint32)
    idx = np.nonzero(keep)[0]
    np.bitwise_or.at(words, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
    return torch.from_numpy(words.view(np.int32)).to(cuda)


@gpu
@pytest.mark.parametrize("width", [4, 1536])
def test_adamw_rows_equals_dense_with_zeroed_gradient(width):
    """the row-sparse kernel reads the gradient only on flagged rows (the others hold NaN) and gives the dense kernel's bits"""
    from llmrec_b200 import ops
    rng = np.random.default_rng(width)
    n = 100                                                    # not a multiple of 32
    keep = rng.random(n) < 0.4
    keep[[30, 31, 32, 33, 62, 63, 64, 65, 99]] = (False, True, True, False, False, True, True, False, True)
    p0 = x_values(rng, n, width)
    pr, pd = dev(p0), dev(p0)
    a, b = ops.AdamW([pr], lr=1e-2, weight_decay=0.05), ops.AdamW([pd], lr=1e-2, weight_decay=0.05)
    for step in range(3):
        g = (rng.standard_normal((n, width)) * 1e-2).astype(np.float32)
        gz = np.where(keep[:, None], g, np.float32(0))
        gn = np.where(keep[:, None], g, np.float32(np.nan))
        snap = (pd.cpu().numpy(), b.m[0].cpu().numpy(), b.v[0].cpu().numpy())
        a.step([dev(gn)], row_masks=[mask_words(keep)])
        b.step([dev(gz)])
        for x, y in ((pr, pd), (a.m[0], b.m[0]), (a.v[0], b.v[0])):
            assert same_bits(x.cpu().numpy(), y.cpu().numpy()), f"width {width} step {step + 1}"
        refs = adamw_ref(*snap[:1], gz, *snap[1:], step + 1, 1e-2, 0.9, 0.999, 1e-8, 0.05)
        for got, (y, bnd) in zip((pr, a.m[0], a.v[0]), refs):
            check(got, y, bnd, "adamw", f"rows width {width} step {step + 1}")


# =================================================================================================================================
# 4. hoisted-feature helpers
# =================================================================================================================================
def colsum_ref(terms, out0=None):
    """terms: [(G, scale | None)] -> (out, bound)"""
    w = terms[0][0].shape[1]
    y, mag = np.zeros(w), np.zeros(w)
    for G, s in terms:
        sG = G.astype(np.float64) * (1.0 if s is None else s.astype(np.float64)[:, None])
        y, mag = y + sG.sum(0), mag + np.abs(sG).sum(0)
    nmax = max(G.shape[0] for G, _ in terms)
    o = 0.0 if out0 is None else out0.astype(np.float64)
    return y + o, 2 * U * (math.ceil(nmax / 1024) + len(terms) + 140) * (mag + np.abs(o))


def colsum_emul(terms, slices=128):
    """fp32 in the kernel's order: 128 slices of 8 warps, rows strided by 1024, 4 chains; the finish loop adds `slices` slice partials"""
    w = terms[0][0].shape[1]
    part = np.zeros((128, w), np.float32)
    for sl in range(128):
        wsum = np.zeros((8, w), np.float32)
        for wp in range(8):
            acc = np.zeros(w, np.float32)
            for G, s in terms:
                a = np.zeros((4, w), np.float32)
                rows = np.arange(sl * 8 + wp, G.shape[0], 1024)
                for j, r in enumerate(rows):
                    a[j % 4] = a[j % 4] + (np.float32(1) if s is None else s[r]) * G[r]
                acc = acc + ((a[0] + a[1]) + (a[2] + a[3]))
            wsum[wp] = acc
        t = np.zeros(w, np.float32)
        for wp in range(8):
            t = t + wsum[wp]
        part[sl] = t
    out = np.zeros(w, np.float32)
    for sl in range(slices):
        out = out + part[sl]
    return out


def test_colsum_bound_accepts_fp32_and_rejects_a_missing_slice():
    rng = np.random.default_rng(4)
    for n in (1024, 4097, 20000):
        terms = [(x_values(rng, n, 5), x_values(rng, n, 1)[:, 0]), (x_values(rng, n // 3, 5), None)]
        y, b = colsum_ref(terms)
        assert passes(colsum_emul(terms), y, b)
        assert not passes(colsum_emul(terms, slices=127), y, b), n


def gram_ref(W, b, G, h, n2, c, dW0, db0, L0):
    W64, G64 = W.astype(np.float64), G.astype(np.float64)
    d, k = W.shape
    b64 = np.zeros(d) if b is None else b.astype(np.float64)
    h64 = np.zeros(k) if h is None else h.astype(np.float64)
    c, n2 = float(np.float32(c)), float(np.float32(n2))
    WG, aWG = W64 @ G64, np.abs(W64) @ np.abs(G64)
    dW = dW0 + c * (WG + np.outer(b64, h64))
    bdW = 2 * U * (k + 12) * abs(c) * (aWG + np.abs(np.outer(b64, h64))) + 2 * U * np.abs(dW0)
    Wh, aWh = W64 @ h64, np.abs(W64) @ np.abs(h64)
    db = db0 + c * (Wh + n2 * b64)
    bdb = 2 * U * (k + 24) * abs(c) * (aWh + abs(n2) * np.abs(b64)) + 2 * U * np.abs(db0)
    loss = L0 + 0.5 * c * ((WG * W64).sum() + 2 * (b64 * Wh).sum() + n2 * (b64 ** 2).sum())
    mag = 0.5 * abs(c) * ((aWG * np.abs(W64)).sum() + 2 * (np.abs(b64) * aWh).sum() + abs(n2) * (b64 ** 2).sum())
    return (dW, bdW), (db, bdb), (loss, 2 * U * (2 * k + d + 40) * mag + 2 * U * abs(L0))


def gram_emul(W, b, G, h, n2, c, wrong=None):
    """fp32: WG in 8 K-chunks added in order, then the finish kernel's formulas; wrong: 'no_bh' | 'single_cross'"""
    f = np.float32
    d, k = W.shape
    chunk = -(-k // 8)
    WG = np.zeros((d, k), np.float32)
    for ks in range(8):
        l0, l1 = ks * chunk, min(k, (ks + 1) * chunk)
        part = np.zeros((d, k), np.float32)
        for l in range(l0, l1):
            part = part + W[:, l:l + 1] * G[l:l + 1, :]
        WG = WG + part
    bb = np.zeros(d, np.float32) if b is None else b
    hh = np.zeros(k, np.float32) if h is None else h
    dW = f(c) * (WG + (0 if wrong == "no_bh" else 1) * bb[:, None] * hh[None, :])
    wh = seq_sum_sq(W, np.broadcast_to(hh, W.shape))
    quad = seq_sum_sq(WG, W)
    db = f(c) * (wh + f(n2) * bb)
    two = f(1) if wrong == "single_cross" else f(2)
    loss = (f(0.5) * f(c) * (quad + two * bb * wh + f(n2) * bb * bb)).astype(np.float32)
    acc = f(0)
    for v in loss:
        acc = acc + v
    return dW, db, acc


def gram_inputs(rng, d, k, m=None):
    W = x_values(rng, d, k) / np.float32(math.sqrt(k))
    X = rng.standard_normal((m or k + 3, k))
    G = ((X.T @ X) / X.shape[0]).astype(np.float32)
    G = np.triu(G) + np.triu(G, 1).T                      # exactly symmetric
    return W, x_values(rng, d, 1)[:, 0], G.astype(np.float32), x_values(rng, k, 1)[:, 0]


@pytest.mark.parametrize("d,k", [(7, 1), (1, 7), (20, 65), (63, 9)])
def test_feat_reg_bound_accepts_fp32_and_rejects_wrong_terms(d, k):
    rng = np.random.default_rng(d * 100 + k)
    W, b, G, h = gram_inputs(rng, d, k)
    n2, c = 3.0, 0.7
    (dW, bdW), (db, bdb), (loss, bl) = gram_ref(W, b, G, h, n2, c, 0.0, 0.0, 0.0)
    gw, gb, gl = gram_emul(W, b, G, h, n2, c)
    assert passes(gw, dW, bdW) and passes(gb, db, bdb) and passes(gl, loss, bl)
    assert not passes(gram_emul(W, b, G, h, n2, c, "no_bh")[0], dW, bdW)
    assert not passes(gram_emul(W, b, G, h, n2, c, "single_cross")[2], loss, bl)


@gpu
def test_rank1_add_matches_fp64():
    from llmrec_b200 import ops
    rng = np.random.default_rng(6)
    blocks, refs = [], []
    for n, w in ((0, 5), (1, 1), (1000, 33), (300, 768), (77, 100), (4097, 31)):
        Y0 = x_values(rng, n, w)
        tbl = dev(x_values(rng, n, 3))
        yb = wide(Y0, 4, 4)
        bias = x_values(rng, w, 1)[:, 0]
        blocks.append((yb[1], tbl[:, 1], dev(bias)))        # scale: a strided column
        s = tbl[:, 1].cpu().numpy().astype(np.float64)
        ref = Y0.astype(np.float64) + s[:, None] * bias.astype(np.float64)[None, :]
        refs.append((yb, ref, w))
    ops.rank1_add(blocks)
    for yb, ref, w in refs:
        got = yb[0].cpu().numpy()
        check(got[:, 4:4 + w], ref, U * np.abs(ref), "rank1_add", f"width {w}")
        assert np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + w:]).all()


@gpu
@pytest.mark.parametrize("width", [1, 31, 33, 100, 768])
def test_scaled_colsum_matches_fp64_and_is_deterministic(width):
    from llmrec_b200 import ops
    rng = np.random.default_rng(width)
    ns = [0, 1, 1023, 1024, 4097] + ([200000] if width <= 100 else [])
    configs = [[(0, None)], [(1, "s"), (1023, None), (1024, "s")], [(ns[i % 5], "s" if i % 2 else None) for i in range(32)],
               [(ns[-1], "s"), (ns[-1] // 2 + 1, None)]]
    results = []
    for ci, cfg in enumerate(configs):
        terms_np, terms_dev = [], []
        for n, sc in cfg:
            G = x_values(rng, n, width)
            tbl = x_values(rng, n, 3) if sc else None
            gbuf = wide(G, 4, 4)
            terms_dev.append((gbuf[1], dev(tbl)[:, 2] if sc else None))
            terms_np.append((G, tbl[:, 2] if sc else None))
        for acc in (False, True):
            out0 = x_values(rng, 1, width)[0]
            obuf = wide(out0[None, :], 4, 4)
            ops.scaled_colsum(terms_dev, obuf[1][0], accumulate=acc)
            y, b = colsum_ref(terms_np, out0 if acc else None)
            got = obuf[0].cpu().numpy()
            check(got[0, 4:4 + width], y, b, "scaled_colsum", f"width {width} config {ci} acc={acc}")
            assert np.isnan(got[0, :4]).all() and np.isnan(got[0, 4 + width:]).all()
            if not acc:
                results.append((terms_dev, got[0, 4:4 + width].copy()))
    for terms_dev, first in results[::-1]:                  # again, after calls of other shapes on the same scratch
        o = torch.empty(width, device=cuda)
        ops.scaled_colsum(terms_dev, o)
        assert same_bits(o.cpu().numpy(), first), f"width {width}: scaled_colsum changed bits"


@gpu
@pytest.mark.parametrize("d,k", [(1, 1), (7, 1), (1, 7), (7, 7), (63, 65), (65, 63), (200, 7), (7, 200), (768, 768), (65, 768), (768, 65),
                                 (200, 200)])
def test_feat_reg_gram_matches_fp64_and_is_deterministic(d, k):
    from llmrec_b200 import ops
    rng = np.random.default_rng(d * 1000 + k)
    W, b, G, h = gram_inputs(rng, d, k)
    n2, c = 1234.0, 0.3
    for with_b, with_h in ((True, True), (False, True), (True, False), (False, False)):
        dW0, db0, L0 = x_values(rng, d, k), x_values(rng, d, 1)[:, 0], 0.75
        dWt, dbt, loss = dev(dW0), dev(db0), torch.tensor([L0], device=cuda)
        args = (dev(W), dev(b) if with_b else None, dev(G), dev(h) if with_h else None, n2, c)
        ops.feat_reg_gram(*args, dWt, dbt if with_b else None, loss)
        (rW, bW), (rb, bb), (rl, bl) = gram_ref(W, b if with_b else None, G, h if with_h else None, n2, c, dW0.astype(np.float64),
                                                db0.astype(np.float64), L0)
        what = f"d={d} k={k} b={with_b} h={with_h}"
        check(dWt, rW, bW, "feat_reg_gram", what + " dW")
        if with_b:
            check(dbt, rb, bb, "feat_reg_gram", what + " db")
        else:
            assert same_bits(dbt.cpu().numpy(), db0)
        check(loss.cpu().numpy(), rl, bl, "feat_reg_gram", what + " loss")
        first = (dWt.cpu().numpy(), dbt.cpu().numpy(), loss.cpu().numpy())
        for other in (False, True):                          # the same bits again, also after a call of another shape
            if other:
                W2, b2, G2, h2 = gram_inputs(rng, d + 1, k + 2)
                ops.feat_reg_gram(dev(W2), dev(b2), dev(G2), dev(h2), 1.0, 1.0, torch.zeros(d + 1, k + 2, device=cuda),
                                  torch.zeros(d + 1, device=cuda), torch.zeros(1, device=cuda))
            dWt.copy_(dev(dW0)); dbt.copy_(dev(db0)); loss.fill_(L0)
            ops.feat_reg_gram(*args, dWt, dbt if with_b else None, loss)
            assert all(same_bits(x.cpu().numpy(), y) for x, y in zip((dWt, dbt, loss), first)), what


@gpu
def test_feat_reg_gram_rejects_bad_operands():
    from llmrec_b200 import ops
    d, k = 6, 10
    W, G, dW = torch.zeros(d, k, device=cuda), torch.zeros(k, k, device=cuda), torch.zeros(d, k, device=cuda)
    b, h, db, loss = torch.zeros(d, device=cuda), torch.zeros(k, device=cuda), torch.zeros(d, device=cuda), torch.zeros(1, device=cuda)
    ok = dict(W=W, b=b, G=G, h=h, n2=1.0, c=1.0, dW=dW, db=db, loss=loss)
    ops.feat_reg_gram(**ok)
    bad = {"W": torch.zeros(k, d, device=cuda).t(), "G": torch.zeros(k, k + 1, device=cuda), "dW": torch.zeros(d, 2 * k, device=cuda)[:, :k],
           "b": torch.zeros(d + 1, device=cuda), "h": torch.zeros(2 * k, device=cuda)[::2], "db": torch.zeros(d, dtype=torch.float64, device=cuda),
           "loss": torch.zeros(1)}
    for name, t in bad.items():
        with pytest.raises(ValueError, match=f"{name} must"):
            ops.feat_reg_gram(**(ok | {name: t}))
    with pytest.raises(ValueError):
        ops.feat_reg_gram(**(ok | {"dW": None}))


# =================================================================================================================================
# 5. evaluation
# =================================================================================================================================
def topk_ref(S, masked, K, tie_desc=False):
    """(score desc, id asc) ranking of the candidates; -1 / -inf past the candidate count.  tie_desc: the wrong tie rule"""
    idx = np.full((S.shape[0], K), -1, np.int64)
    val = np.full((S.shape[0], K), -np.inf)
    for b in range(S.shape[0]):
        cand = np.nonzero(~masked[b])[0]
        order = np.lexsort((-cand if tie_desc else cand, -S[b, cand]))[:K]
        idx[b, :order.size], val[b, :order.size] = cand[order], S[b, cand[order]]
    return idx, val


def auc_ref(scores, truth, mask, n_items):
    """exact Mann-Whitney AUC of one user: positives = distinct in-range truth ids not masked, negatives = the other unmasked items"""
    mask = set(int(i) for i in mask)
    tset = set(int(i) for i in truth)
    P = sorted(i for i in tset if 0 <= i < n_items and i not in mask)
    Nn = [i for i in range(n_items) if i not in mask and i not in tset]
    if not P or not Nn:
        return Fraction(0)
    ns = np.sort(scores[Nn])
    less = int(np.searchsorted(ns, scores[P], "left").sum())
    eq = int((np.searchsorted(ns, scores[P], "right") - np.searchsorted(ns, scores[P], "left")).sum())
    return Fraction(2 * less + eq, 2 * len(P) * len(Nn))


def auc_emul(scores, truth, mask, n_items, wrong=None):
    """the kernel's counting: truth in chunks of 128, a duplicate skipped when it equals the entry before it; wrong: 'tie_one' (a tie
    counts 1) | 'chunk_dup' (the duplicate check stops at the chunk start)"""
    mask, tset = set(int(i) for i in mask), set(int(i) for i in truth)
    negs = [i for i in range(n_items) if i not in mask and i not in tset]
    less = eq = npos = 0
    for tb in range(0, max(len(truth), 1), 128):
        for e in range(tb, min(len(truth), tb + 128)):
            i = int(truth[e])
            first = tb if wrong == "chunk_dup" else 0
            if 0 <= i < n_items and i not in mask and (e == first or truth[e - 1] != i):
                npos += 1
                less += sum(scores[j] < scores[i] for j in negs)
                eq += sum(scores[j] == scores[i] for j in negs)
    if npos == 0 or not negs:
        return Fraction(0)
    return Fraction(2 * less + (2 if wrong == "tie_one" else 1) * eq, 2 * npos * len(negs))


def auc_users(rng, n_items):
    """[(truth, mask)]: 129 / 256 / 300 positives, duplicates (one across the 128 boundary), masked truth, out-of-range ids, empty
    truth, no negatives, a plain user"""
    perm = lambda m: np.sort(rng.choice(n_items, m, replace=False))
    rows = []
    for m in (129, 256, 300):
        rows.append((perm(m), perm(40)))
    t = perm(199)
    t = np.sort(np.concatenate([t, [t[126], t[10]]]))
    assert t[127] == t[128]
    rows.append((t, perm(30)))
    t = perm(150)
    rows.append((t, np.union1d(t[::3], perm(20))))          # a third of the truth is also masked
    rows.append((np.concatenate([[-5, -1], perm(60), [n_items, n_items + 9]]), perm(10)))
    rows.append((np.zeros(0, np.int64), perm(50)))
    t = perm(100)
    rows.append((t, np.setdiff1d(np.arange(n_items), t)))   # no negatives
    rows.append((perm(20), np.zeros(0, np.int64)))
    return rows


def test_eval_references_reject_wrong_rules():
    rng = np.random.default_rng(8)
    n_items = 400
    S = rng.integers(-3, 4, n_items).astype(np.float64)      # integer scores: many exact ties
    rows = auc_users(rng, n_items)
    for t, m in rows:
        assert auc_emul(S, t, m, n_items) == auc_ref(S, t, m, n_items)
    assert any(auc_emul(S, t, m, n_items, "tie_one") != auc_ref(S, t, m, n_items) for t, m in rows)
    t, m = rows[3]                                            # the duplicate across the 128 boundary
    assert auc_emul(S, t, m, n_items, "chunk_dup") != auc_ref(S, t, m, n_items)
    masked = np.zeros((1, n_items), bool)
    assert not np.array_equal(topk_ref(S[None], masked, 50)[0], topk_ref(S[None], masked, 50, tie_desc=True)[0])


def csr(rows):
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    col = np.concatenate([np.asarray(r, np.int32) for r in rows] + [np.zeros(0, np.int32)])
    return i32(rp), i32(col if col.size else np.zeros(1, np.int32))


@gpu
@pytest.mark.parametrize("n_items", [1, 255, 256, 257])
@pytest.mark.parametrize("d", [20, 64, 300])
def test_score_topk_simt_is_exact_on_integer_scores(d, n_items):
    from llmrec_b200 import ops
    from llmrec_b200 import _native as N
    rng = np.random.default_rng(d + n_items)
    n_users = 40
    Uh = rng.integers(-2, 3, (n_users, d)).astype(np.float32)
    Ih = rng.integers(-2, 3, (n_items, d)).astype(np.float32)
    masks = [np.sort(rng.choice(n_items, rng.integers(0, n_items // 4 + 1), replace=False)) for _ in range(n_users)]
    masks[3] = np.arange(max(0, n_items - 10))                # fewer candidates than K: a -1 tail
    mrp, mcol = csr(masks)
    users = rng.integers(0, n_users, 37).astype(np.int32)
    users[:2] = (3, 3)
    S = Uh[users].astype(np.float64) @ Ih.T.astype(np.float64)
    masked = np.zeros((users.size, n_items), bool)
    for b, u in enumerate(users):
        masked[b, masks[u]] = True
    Ub, Ib = wide(Uh), wide(Ih)
    for K in sorted({1, min(17, n_items), min(64, n_items)}):
        ridx, rval = topk_ref(S, masked, K)
        for mode in ((2, 0) if d != 64 else (2,)):             # mode 0 falls back to the SIMT kernel where wgmma has no tile
            idx, val = ops.score_topk(Ub[1], Ib[1], i32(users), mrp, mcol, K, mode=mode, want_vals=True)
            assert np.array_equal(idx.cpu().numpy(), ridx), f"d={d} n_items={n_items} K={K} mode={mode}"
            assert np.array_equal(val.cpu().numpy().astype(np.float64), rval)
        # users in chunks: scratch for 3 users at a time
        sc = torch.empty(3 * n_items + 1, device=cuda)
        idx = torch.empty((users.size, K), dtype=torch.int32, device=cuda)
        ut = i32(users)
        N.check(N.lib().llmrec_score_topk_f32(ops._p(Ub[1]), ops._ld(Ub[1]), ops._p(Ib[1]), ops._ld(Ib[1]), ops._p(ut), users.size,
                                              n_items, d, ops._p(mrp), ops._p(mcol), K, ops._p(idx), None, 2, ops._p(sc), sc.numel(),
                                              ops._stream()), "score_topk")
        assert np.array_equal(idx.cpu().numpy(), ridx), f"chunked users, d={d} n_items={n_items} K={K}"
    for K in (65, 100, 1000):                                 # the C ABI takes K <= 64
        if K <= n_items:
            with pytest.raises(RuntimeError, match="K="):
                ops.score_topk(Ub[1], Ib[1], i32(users), mrp, mcol, K, mode=2)


@gpu
@pytest.mark.parametrize("d", [20, 300])
def test_score_topk_simt_random_fp32_swaps_only_within_the_bound(d):
    from llmrec_b200 import ops
    rng = np.random.default_rng(d)
    n_items, K = 3000, 64
    Uh, Ih = rng.standard_normal((50, d)).astype(np.float32), rng.standard_normal((n_items, d)).astype(np.float32)
    users = np.arange(50, dtype=np.int32)
    mrp, mcol = csr([np.sort(rng.choice(n_items, 100, replace=False)) for _ in range(50)])
    idx, val = ops.score_topk(dev(Uh), dev(Ih), i32(users), mrp, mcol, K, mode=2, want_vals=True)
    idx, val = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64)
    S = Uh.astype(np.float64) @ Ih.T.astype(np.float64)
    Bd = 2 * U * d * (np.abs(Uh.astype(np.float64)) @ np.abs(Ih.T.astype(np.float64)))
    mask_np = [mcol.cpu().numpy()[a:b] for a, b in zip(mrp.cpu().numpy()[:-1], mrp.cpu().numpy()[1:])]
    for b in range(50):
        sel = idx[b]
        assert (sel >= 0).all() and np.unique(sel).size == K and not np.isin(sel, mask_np[b]).any()
        check(val[b], S[b, sel], Bd[b, sel], "topk scores", f"d={d} user {b}")
        lo = (S[b, sel] + Bd[b, sel]).min()
        rest = np.setdiff1d(np.setdiff1d(np.arange(n_items), sel), mask_np[b])
        assert (S[b, rest] - Bd[b, rest]).max() <= lo, f"d={d} user {b}: an item outside the top-K scores clearly higher"
        hi = S[b, sel] + Bd[b, sel]
        assert (S[b, sel][1:] - Bd[b, sel][1:] <= hi[:-1]).all(), f"d={d} user {b}: the list is out of order beyond the bound"


@gpu
@pytest.mark.parametrize("d", [7, 300])
@pytest.mark.parametrize("with_mask", [True, False])
def test_user_auc_matches_exact_mann_whitney(d, with_mask):
    from llmrec_b200 import ops
    rng = np.random.default_rng(d + with_mask)
    n_items = 700
    rows = auc_users(rng, n_items)
    if not with_mask:
        rows = [(t, np.zeros(0, np.int64)) for t, _ in rows]
    n_users = len(rows)
    Uh = rng.integers(-2, 3, (n_users, d)).astype(np.float32)
    Ih = rng.integers(-2, 3, (n_items, d)).astype(np.float32)
    trp, tcol = csr([t for t, _ in rows])
    mrp, mcol = csr([m for _, m in rows]) if with_mask else (None, None)
    users = np.concatenate([np.arange(n_users), [2, 3]]).astype(np.int32)
    got = ops.user_auc(wide(Uh)[1], wide(Ih)[1], i32(users), mrp, mcol, trp, tcol).cpu().numpy()
    for b, u in enumerate(users):
        S = Ih.astype(np.float64) @ Uh[u].astype(np.float64)
        ref = auc_ref(S, rows[u][0], rows[u][1], n_items)
        want = np.float32(float(ref))
        assert abs(float(got[b]) - float(want)) <= float(np.spacing(np.abs(want))), f"d={d} mask={with_mask} user {u}: {got[b]} vs {ref}"
        if u == 6 or (u == 7 and with_mask):
            assert got[b] == 0.0, f"user {u}: an empty class gives AUC 0"


@gpu
def test_topk_hits_matches_membership():
    from llmrec_b200 import ops
    rng = np.random.default_rng(2)
    n_items, n_users, K = 500, 30, 40
    truth = [np.sort(rng.choice(n_items, rng.integers(0, 60), replace=False)) for _ in range(n_users)]
    truth[4] = np.zeros(0, np.int64)
    trp, tcol = csr(truth)
    users = rng.integers(0, n_users, 25).astype(np.int32)
    users[0] = 4
    idx = rng.integers(0, n_items, (25, K)).astype(np.int32)
    for b, u in enumerate(users):
        if truth[u].size:
            idx[b, :5] = truth[u][:5][rng.integers(0, min(5, truth[u].size), 5)]
    idx[:, -3:] = -1
    idx[7, :] = -1
    hits = ops.topk_hits(i32(idx), i32(users), trp, tcol).cpu().numpy()
    ref = np.array([[i >= 0 and i in set(truth[u].tolist()) for i in row] for row, u in zip(idx, users)])
    assert np.array_equal(hits.astype(bool), ref) and set(np.unique(hits)) <= {0, 1}
