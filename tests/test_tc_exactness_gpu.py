"""-m gpu: the tensor-core projection and scoring kernels held to exact references across the space their C ABI accepts.

Projections (proj_tc.cu): every width d = 32 .. 256 in mode 0 (3xTF32) and mode 1 (plain TF32), 128- and 256-wide tiles, n and k
at tile edges, X as a column slice of a wider table, strided Y / dY -- against fp64.  A precision fingerprint tells 3xTF32 from
plain TF32 from the SIMT kernel.  The weight-gradient reduce under accumulate (single and shared outputs) must be exact and
bitwise reproducible, and an empty problem inside a group must change nothing.

Scoring (score_tc.cu): the tensor-core lists must equal the exact SIMT lists bit for bit (ids and values) whenever the true
top-K lies inside each catalog split's candidate heap; the SIMT lists are checked against fp64."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

cuda = torch.device("cuda")
NAN, NINF = float("nan"), float("-inf")
WIDTHS = [32, 64, 96, 128, 160, 192, 224, 256]
TOL = {0: 1e-4, 1: 5e-3}      # mode 0: fp32-class; mode 1: plain TF32 operands (~2^-11 per product); relative to |Y| ~ 1, |dW| ~ sqrt(n)
SMS = 132                     # H100 SXM


def _gen(seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def _ld(t):
    from llmrec_b200 import ops
    return ops._ld(t)


def _table(g, n, k, lead=4, pad=8, positive=False):
    """X[n x k] as a column slice of a wider row-major table (the hoisted side-feature tables): ld = lead + k + pad, a multiple of 4,
    and the slice starts 16 bytes into its row."""
    shape = (n, lead + k + pad)
    T = 1.0 + torch.rand(shape, generator=g, device=cuda) if positive else torch.randn(shape, generator=g, device=cuda)
    return T[:, lead:lead + k]


def _assert_proj_tc(d, X, out):
    """The operands satisfy the tensor-core preconditions (proj_tc_supported and the dispatcher), so no case tests SIMT instead."""
    assert d % 32 == 0 and 32 <= d <= 256
    assert X.shape[1] % 4 == 0 and _ld(X) % 4 == 0 and X.data_ptr() % 16 == 0
    assert _ld(out) % 4 == 0 and out.data_ptr() % 16 == 0


def _rows_per_chunk(n):   # wg_rows_per_chunk in proj_tc.cu
    r = 2048
    while r > 256 and n // r < 4:
        r //= 2
    return r


def _uses_256_wide_tiles(dims):
    """The grouped launches pick 256-row / 256-feature tiles at d <= 128 when those still give every SM a unit (pick_mb)."""
    fwd = sum(-(-n // 256) for n, _ in dims)
    wg = sum(-(-k // 256) * -(-n // _rows_per_chunk(n)) for n, k in dims)
    return fwd >= SMS and wg >= SMS


# ------------------------------------------------------------------------------------------------------------------------------
# projections
# ------------------------------------------------------------------------------------------------------------------------------
SMALL = [(n, k) for n in (1, 63, 65, 257) for k in (4, 36, 100, 1536)]          # 16 problems: two grouped launches, 128-wide tiles
BIG = [(9000, 1536)] * 4 + [(8001, 100), (9001, 36), (7777, 4)]                 # >= 132 units at 256 wide


def _projection_case(dims, d, mode, seed):
    from llmrec_b200 import ops
    g = _gen(seed)
    Xs = [_table(g, n, k) for n, k in dims]
    Ws = [torch.randn(d, k, generator=g, device=cuda) / k ** 0.5 for _, k in dims]
    bs = [torch.randn(d, generator=g, device=cuda) for _ in dims]
    wides = [torch.full((n, 3 * d), NAN, device=cuda) for n, _ in dims]
    Ys = [w[:, d:2 * d] for w in wides]                                                 # strided output views, NaN until written
    for X, Y in zip(Xs, Ys):
        _assert_proj_tc(d, X, Y)
    ops.proj_fwd_group(list(zip(Xs, Ws, bs, Ys)), d, mode)
    tol = TOL[mode]
    for (n, k), X, W, b, Y, wide in zip(dims, Xs, Ws, bs, Ys, wides):
        torch.testing.assert_close(Y.double(), X.double() @ W.double().t() + b.double(), rtol=tol, atol=tol, msg=lambda m: f"fwd n={n} k={k}: {m}")
        assert bool(wide[:, :d].isnan().all() and wide[:, 2 * d:].isnan().all()), f"fwd n={n} k={k} wrote outside its view"
    dYs = [torch.randn(n, 3 * d, generator=g, device=cuda)[:, d:2 * d] for n, _ in dims]   # strided dY views
    dWs = [torch.full((d, k), NAN, device=cuda) for _, k in dims]                       # every element must be written
    dbs = [torch.full((d,), NAN, device=cuda) for _ in dims]
    for X, dY in zip(Xs, dYs):
        _assert_proj_tc(d, X, dY)
    ops.proj_wgrad_group(list(zip(Xs, dYs, dWs, dbs, [False] * len(dims))), d, mode)
    for (n, k), X, dY, dW, db in zip(dims, Xs, dYs, dWs, dbs):
        torch.testing.assert_close(dW.double(), dY.double().t() @ X.double(), rtol=tol, atol=tol * n ** 0.5, msg=lambda m: f"wgrad n={n} k={k}: {m}")
        torch.testing.assert_close(db.double(), dY.double().sum(0), rtol=1e-4, atol=1e-4 * n ** 0.5, msg=lambda m: f"db n={n} k={k}: {m}")


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("d", WIDTHS)
def test_projection_every_width_mode_and_tile(d, mode):
    """128-wide tiles on small problems (n at 1, 63, 65, 257 around the 64-row blocks, k = 4 .. 1536 including k % 32 != 0), then a
    group large enough for 256-wide tiles at d <= 128 (many tiles per CTA above), forward and weight gradient against fp64."""
    _projection_case(SMALL[:8], d, mode, seed=10 * d + mode)
    _projection_case(SMALL[8:], d, mode, seed=10 * d + mode + 1)
    assert _uses_256_wide_tiles(BIG)
    _projection_case(BIG, d, mode, seed=10 * d + mode + 2)


def _max_rel(got, ref):
    return float(((got.double() - ref) / ref).abs().max())


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("d", WIDTHS)
def test_precision_fingerprint(d, mode):
    """All operands in [1, 2): TF32 truncation leaves a low part of up to 2^-10 relative and nothing cancels, so the dropped
    products show.  3xTF32 keeps lo*hi + hi*lo (a missing or swapped one costs ~2^-11 ~ 5e-4 relative): within 5e-5.  Plain TF32
    must show its ~1e-3 error (above 1e-4 proves the tensor cores ran, not the SIMT kernel) and stay below 4e-3.  The reduction
    length is 256 (k forward, n in the weight gradient), so fp32 accumulation stays near 1e-5."""
    from llmrec_b200 import ops
    g = _gen(d + mode)
    n, k = 256, 256
    X = _table(g, n, k, positive=True)
    W = 1.0 + torch.rand(d, k, generator=g, device=cuda)
    dY = (1.0 + torch.rand(n, 3 * d, generator=g, device=cuda))[:, d:2 * d]
    Y = torch.empty(n, d, device=cuda)
    _assert_proj_tc(d, X, Y)
    _assert_proj_tc(d, X, dY)
    ops.proj_fwd_group([(X, W, None, Y)], d, mode)
    dW, db = torch.empty(d, k, device=cuda), torch.empty(d, device=cuda)
    ops.proj_wgrad_group([(X, dY, dW, db, False)], d, mode)
    fwd = _max_rel(Y, X.double() @ W.double().t())
    wg = _max_rel(dW, dY.double().t() @ X.double())
    assert _max_rel(db, dY.double().sum(0)) < 5e-5
    if mode == 0:
        assert fwd < 5e-5 and wg < 5e-5, (fwd, wg)
        Y2, dW2 = torch.empty_like(Y), torch.empty_like(dW)                            # the exact SIMT kernels sum in another order
        ops.proj_fwd_group([(X, W, None, Y2)], d, 2)
        ops.proj_wgrad_group([(X, dY, dW2, None, False)], d, 2)
        assert not torch.equal(Y, Y2) and not torch.equal(dW, dW2)
    else:
        assert 1e-4 < fwd < 4e-3 and 1e-4 < wg < 4e-3, (fwd, wg)


ACC_CASES = {
    "single": ([(9000, 1536)], [True], True, False),                                   # (dims, accumulate flags, with db, shared)
    "item_trans": ([(9000, 1536), (8000, 1536), (7001, 1536), (9000, 1536), (6000, 1536)], [False, True, True, True, True], True, True),
    "hoisted": ([(3000, 1536), (9001, 1536)], [True, True], False, True),
}


@pytest.mark.parametrize("case", list(ACC_CASES))
@pytest.mark.parametrize("d", WIDTHS)
def test_wgrad_accumulate_and_shared_outputs(d, case):
    """The ordered reduce under accumulate on a random prior: one problem, the 5 attribute tables sharing item_trans's dW / db
    (flags F,T,T,T,T), and the hoisted image / text pair sharing a dW already holding the feat_reg term (T,T; bias elsewhere).
    k = 1536 gives hundreds of reduce blocks in flight.  Against fp64, and bitwise equal across two runs from the same prior:
    the reduce has no atomics, so any difference is a race between blocks writing the same element."""
    from llmrec_b200 import ops
    dims, flags, with_db, shared = ACC_CASES[case]
    g = _gen(d)
    k = dims[0][1]
    Xs = [_table(g, n, k) for n, _ in dims]
    dYs = [torch.randn(n, 2 * d, generator=g, device=cuda)[:, d:] for n, _ in dims]
    n_out = 1 if shared else len(dims)
    priors = [(torch.randn(d, k, generator=g, device=cuda), torch.randn(d, generator=g, device=cuda)) for _ in range(n_out)]
    runs = []
    for _ in range(2):
        outs = [(W.clone(), b.clone()) for W, b in priors]
        probs = []
        for p, (X, dY, acc) in enumerate(zip(Xs, dYs, flags)):
            dW, db = outs[0 if shared else p]
            _assert_proj_tc(d, X, dY)
            probs.append((X, dY, dW, db if with_db else None, acc))
        ops.proj_wgrad_group(probs, d, 0)
        runs.append(outs)
    for (W1, b1), (W2, b2) in zip(*runs):
        assert torch.equal(W1, W2) and torch.equal(b1, b2), "weight-gradient reduce is not reproducible"
    for o, (W, b) in enumerate(runs[0]):
        members = range(len(dims)) if shared else [o]
        first = min(members)
        refW = sum(dYs[p].double().t() @ Xs[p].double() for p in members)
        refb = sum(dYs[p].double().sum(0) for p in members)
        if flags[first]:
            refW, refb = refW + priors[o][0].double(), refb + priors[o][1].double()
        n = sum(dims[p][0] for p in members)
        torch.testing.assert_close(W.double(), refW, rtol=1e-4, atol=1e-4 * n ** 0.5)
        if with_db:
            torch.testing.assert_close(b.double(), refb, rtol=1e-4, atol=1e-4 * n ** 0.5)
        else:
            assert torch.equal(b, priors[o][1])                                          # no db passed: untouched


@pytest.mark.parametrize("d,mode", [(64, 0), (96, 0), (128, 1), (192, 0), (256, 1)])
def test_empty_problem_in_a_group_changes_nothing(d, mode):
    """A problem with n = 0 inside a grouped call gives the same bits as the group without it, in both directions: it has no
    tiles; as a source of a shared dW / db it adds nothing; with its own dW / db it writes zeros (or keeps the prior under
    accumulate), as the SIMT path does.  A group of empty problems alone behaves the same."""
    from llmrec_b200 import ops
    g = _gen(d + mode)
    A, B, C = _table(g, 700, 100), _table(g, 1300, 1536), _table(g, 257, 4)
    E, Z = _table(g, 300, 1536)[:0], _table(g, 300, 36)[:0]                         # empty column slices of wider tables
    W = {name: torch.randn(d, X.shape[1], generator=g, device=cuda) for name, X in (("A", A), ("B", B), ("C", C), ("E", E))}
    b = torch.randn(d, generator=g, device=cuda)
    outs = {name: torch.full((n, 3 * d), NAN, device=cuda)[:, d:2 * d] for name, n in (("A", 700), ("B", 1300), ("C", 257), ("E", 0))}
    ops.proj_fwd_group([(A, W["A"], b, outs["A"]), (E, W["E"], b, outs["E"]), (B, W["B"], None, outs["B"]), (C, W["C"], b, outs["C"])], d, mode)
    plain = {name: torch.empty(n, d, device=cuda) for name, n in (("A", 700), ("B", 1300), ("C", 257))}
    ops.proj_fwd_group([(A, W["A"], b, plain["A"]), (B, W["B"], None, plain["B"]), (C, W["C"], b, plain["C"])], d, mode)
    for name in plain:
        assert torch.equal(outs[name], plain[name]), name
    ops.proj_fwd_group([(E, W["E"], b, outs["E"])], d, mode)                           # nothing but an empty problem

    dY = {name: torch.randn(n, 2 * d, generator=g, device=cuda)[:, d:] for name, n in (("A", 700), ("B", 1300), ("C", 257), ("E", 0), ("Z", 0))}
    prior = (torch.randn(d, 36, generator=g, device=cuda), torch.randn(d, generator=g, device=cuda))

    def grads(with_empty):
        o = {name: (torch.full((d, k), NAN, device=cuda), torch.full((d,), NAN, device=cuda)) for name, k in (("A", 100), ("S", 1536), ("C", 4), ("Z", 36))}
        o["Zacc"] = (prior[0].clone(), prior[1].clone())
        probs = [(A, dY["A"], *o["A"], False), (B, dY["B"], *o["S"], False)]
        if with_empty:
            probs += [(E, dY["E"], *o["S"], True), (Z, dY["Z"], *o["Z"], False), (Z, dY["Z"], *o["Zacc"], True)]
        probs += [(C, dY["C"], *o["C"], False)]
        ops.proj_wgrad_group(probs, d, mode)
        return o

    got, want = grads(True), grads(False)
    for name in ("A", "S", "C"):
        assert torch.equal(got[name][0], want[name][0]) and torch.equal(got[name][1], want[name][1]), name
    assert bool((got["Z"][0] == 0).all() and (got["Z"][1] == 0).all())
    assert torch.equal(got["Zacc"][0], prior[0]) and torch.equal(got["Zacc"][1], prior[1])
    alone = (torch.full((d, 36), NAN, device=cuda), torch.full((d,), NAN, device=cuda))
    kept = (prior[0].clone(), prior[1].clone())
    ops.proj_wgrad_group([(Z, dY["Z"], *alone, False), (Z, dY["Z"], *kept, True)], d, mode)
    assert bool((alone[0] == 0).all() and (alone[1] == 0).all())
    assert torch.equal(kept[0], prior[0]) and torch.equal(kept[1], prior[1])


# ------------------------------------------------------------------------------------------------------------------------------
# scoring
# ------------------------------------------------------------------------------------------------------------------------------
def _assert_score_tc(U, I, K):
    """The operands satisfy score_tc_supported, so mode 0 runs the tensor-core kernel and no case compares SIMT with SIMT."""
    assert U.shape[1] in (32, 64, 96, 128) and K <= 64
    assert _ld(U) % 4 == 0 and _ld(I) % 4 == 0 and U.data_ptr() % 16 == 0 and I.data_ptr() % 16 == 0


def _score_plan(n_batch, n_items):
    """(splits, tiles per split) of the catalog (score_plan in score_tc.cu): 128-item tiles, at most 6 splits of >= 32 tiles."""
    utiles, itiles = -(-n_batch // 64), -(-n_items // 128)
    s = 1 if utiles >= SMS // 2 else -(-SMS // utiles)
    s = max(1, min(s, itiles // 32 if itiles >= 32 else 1, 6))
    tps = -(-itiles // s)
    return -(-itiles // tps), tps


def _csr(rows, n_users):
    rowptr = np.zeros(n_users + 1, np.int32)
    rowptr[1:] = np.cumsum([len(r) for r in rows])
    col = np.concatenate([np.asarray(sorted(r), np.int32) for r in rows]) if rowptr[-1] else np.zeros(1, np.int32)
    return torch.from_numpy(rowptr).to(cuda), torch.from_numpy(col).to(cuda)


def _dense_mask(rows, n_items):
    m = torch.zeros(len(rows), n_items, dtype=torch.bool)
    for u, r in enumerate(rows):
        if r:
            m[u, torch.tensor(sorted(r))] = True
    return m.to(cuda)


def _fp64_scores(U, I, users, mask):
    """fp64 scores (train items -inf) and, per user, a bound on |fp32 sequential-FMA dot - exact| (d 2^-24 sum |u_j i_j|)."""
    Ub, I64 = U[users.long()].double(), I.double()
    S = Ub @ I64.t()
    bound = (Ub.abs() @ I64.abs().t()).amax(1, keepdim=True) * U.shape[1] * 2.0 ** -24
    if mask is not None:
        S = S.masked_fill(mask[users.long()], NINF)
    return S, bound


def _assert_sorted_distinct(idx, val):
    """(score desc, id asc) order, ids listed once, the -1 / -inf tail last."""
    v, i = val.double(), idx
    assert bool(((v[:, :-1] > v[:, 1:]) | ((v[:, :-1] == v[:, 1:]) & ((i[:, :-1] < i[:, 1:]) | (i[:, 1:] < 0)))).all())
    assert bool(((i[:, 1:] < 0) | (i[:, :-1] >= 0)).all())
    s = i.sort(1).values
    assert not bool(((s[:, 1:] == s[:, :-1]) & (s[:, 1:] >= 0)).any())


def _check_lists_vs_fp64(idx, val, S, bound, K):
    """The exact lists against fp64 (tie-aware): exactly min(K, candidates) entries, no train item, and at every rank the listed
    score equals the fp64 score of that rank up to fp32 rounding -- lists may differ from fp64's only where rounding flips a
    near-tie.  Values are the listed items' scores to fp32 rounding."""
    _assert_sorted_distinct(idx, val)
    n_cand = (S > NINF).sum(1, keepdim=True)
    have = torch.arange(K, device=cuda)[None, :] < n_cand
    assert torch.equal(idx >= 0, have), "list length != min(K, candidates)"
    assert bool((val[~have] == NINF).all())
    got = torch.where(have, S.gather(1, idx.clamp_min(0).long()), torch.full_like(S[:, :K], NINF))
    assert bool(torch.isfinite(got[have]).all()), "a train item was ranked"
    want = S.topk(K, dim=1).values
    err = torch.where(have, (got - want).abs(), torch.zeros_like(got))
    assert bool((err <= 2 * bound).all()), float((err - 2 * bound).max())
    verr = torch.where(have, (val.double() - got).abs(), torch.zeros_like(got))
    assert bool((verr <= bound).all())


def _assert_bitwise_equal(a, b, what):
    (ia, va), (ib, vb) = a, b
    bad = ((ia != ib) | (va.view(torch.int32) != vb.view(torch.int32))).any(1)
    assert not bool(bad.any()), f"{what}: tensor-core and SIMT lists differ on {int(bad.sum())} rows, first {int(bad.nonzero()[0])}"


SCORE_ITEMS = [70, 1000, 4097, 8193, 12289, 17366, 20481, 40000]   # 1, 1, 1, 2, 3, 4, 5, 6 catalog splits; ragged last tiles
SCORE_KS = [1, 20, 50, 64]
SCORE_BATCHES = [1, 64, 65, 300]


def _scoring_catalog(d, ni, seed):
    """U / I as column slices of wider buffers; 400 users with random train rows plus special ones: two users whose train row
    holds their top K + 24 items (spread over tiles and splits), one with every item in it, one with all but 5; a batch order
    that starts with the special users and repeats users inside and across 64-user tiles."""
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    nu = 400
    Uw, Iw = torch.randn(nu, d + 8, generator=g), torch.randn(ni, d + 12, generator=g)
    U, I = Uw[:, 4:4 + d], Iw[:, 8:8 + d]
    rows = [set(rng.choice(ni, size=int(rng.integers(0, 8)), replace=False).tolist()) for _ in range(nu)]
    for u in (0, 3):
        top = np.argsort(-(I.double() @ U[u].double()).numpy(), kind="stable")
        rows[u] |= set(top[:min(64 + 24, ni // 2)].tolist())
    rows[1] = set(range(ni))
    rows[2] = set(range(ni)) - set(rng.choice(ni, size=5, replace=False).tolist())
    seq = torch.randperm(nu, generator=g)[:300]
    seq[:4] = torch.tensor([0, 1, 2, 3])
    seq[5], seq[64], seq[299] = 0, 3, 2
    Uw, Iw = Uw.to(cuda), Iw.to(cuda)
    return Uw[:, 4:4 + d], Iw[:, 8:8 + d], rows, seq.to(torch.int32).to(cuda)


@pytest.mark.parametrize("ni", SCORE_ITEMS)
@pytest.mark.parametrize("d", [32, 64, 96, 128])
def test_scoring_tensor_core_lists_equal_exact_lists(d, ni):
    """Tensor-core scoring (mode 0) against the exact SIMT kernel (mode 2), bit for bit in ids and values, for K in 1 .. 64 and
    batches of 1, 64, 65, 300 users (ragged user tiles, duplicates, masked top items, users with fewer than K candidates), with
    and without a mask; the SIMT lists against fp64."""
    from llmrec_b200 import ops
    U, I, rows, seq = _scoring_catalog(d, ni, seed=d * 100003 + ni)
    rowptr, col = _csr(rows, U.shape[0])
    mask = _dense_mask(rows, ni)
    for K in SCORE_KS:
        _assert_score_tc(U, I, K)
        for nb in SCORE_BATCHES:
            users = seq[:nb].contiguous()
            for masked in ((True, False) if K == 64 or nb == 65 else (True,)):
                rp, cl = (rowptr, col) if masked else (None, None)
                tc = ops.score_topk(U, I, users, rp, cl, K, mode=0, want_vals=True)
                ex = ops.score_topk(U, I, users, rp, cl, K, mode=2, want_vals=True)
                what = f"K={K} nb={nb} masked={masked}"
                S, bound = _fp64_scores(U, I, users, mask if masked else None)
                try:
                    _check_lists_vs_fp64(*ex, S, bound, K)
                except AssertionError as e:
                    raise AssertionError(f"SIMT vs fp64, {what}: {e}") from None
                _assert_bitwise_equal(tc, ex, what)


BAND_BASE, BAND_NOISE = 6.0, 1e-6


def _banded_catalog(d, ni, nb, band, lo, hi, seed):
    """nb users along orthonormal directions u_b; each owns a band of `band` items base*u_b + 1e-6*noise (random directions: the
    band's scores sit within a few ulps of each other, so 3xTF32 orders them differently from fp32), ids drawn from [lo, hi)
    disjoint between users.  Every other item scores ~0.01.  Each user's train row masks 3 band items and 5 others."""
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    Q, _ = torch.linalg.qr(torch.randn(d, d, generator=g, dtype=torch.float64))
    Uw = torch.zeros(nb, d + 8)
    Uw[:, 4:4 + d] = Q[:, :nb].t().float()
    Iw = torch.zeros(ni, d + 4)
    Iw[:, :d] = 0.01 * torch.randn(ni, d, generator=g)
    ids = rng.choice(np.arange(lo, hi), size=(nb, band), replace=False)
    for b in range(nb):
        Iw[torch.from_numpy(ids[b]), :d] = BAND_BASE * Uw[b, 4:4 + d] + BAND_NOISE * torch.randn(band, d, generator=g)
    rows = []
    for b in range(nb):
        rows.append(set(rng.choice(ids[b], size=3, replace=False).tolist()) | set(rng.choice(ni, size=5, replace=False).tolist()))
    U, I = Uw.to(cuda)[:, 4:4 + d], Iw.to(cuda)[:, :d]
    return U, I, [set(x.tolist()) for x in ids], rows


@pytest.mark.parametrize("case", ["fits", "overflows_one_of_6_splits", "overflows_the_only_split"])
@pytest.mark.parametrize("d", [32, 64, 128])
def test_scoring_near_tied_band_and_candidate_slack(d, case):
    """Each user's top items form a band of near-ties whose 3xTF32 order differs from the exact fp32 order.  When the band (K + 8
    items, ids over all 6 splits) fits every split's candidate heap (K + 16 rounded up to 8), the rescored lists must equal the
    SIMT lists bit for bit.  A band of K + 40 inside ONE split's range overflows that heap: then the lists must still be sorted,
    drawn from the band, and free of train items."""
    from llmrec_b200 import ops
    nb = 32
    ni = 4000 if case == "overflows_the_only_split" else 40000
    splits, tps = _score_plan(nb, ni)
    for K in SCORE_KS:
        if case == "fits":
            band, lo, hi = K + 8, 0, ni
        else:
            s = splits // 2
            band, lo, hi = K + 40, s * tps * 128, min(ni, (s + 1) * tps * 128)
        U, I, bands, rows = _banded_catalog(d, ni, nb, band, lo, hi, seed=d * 1000 + K + len(case))
        rowptr, col = _csr(rows, nb)
        users = torch.arange(nb, dtype=torch.int32, device=cuda)
        _assert_score_tc(U, I, K)
        tc = ops.score_topk(U, I, users, rowptr, col, K, mode=0, want_vals=True)
        ex = ops.score_topk(U, I, users, rowptr, col, K, mode=2, want_vals=True)
        S, bound = _fp64_scores(U, I, users, _dense_mask(rows, ni))
        _check_lists_vs_fp64(*ex, S, bound, K)
        for idx in (tc[0], ex[0]):
            for b, r in enumerate(idx.cpu().tolist()):
                assert set(r) <= bands[b] - rows[b], (case, K, b)
        if case == "fits":
            _assert_bitwise_equal(tc, ex, f"K={K}")
        else:
            _assert_sorted_distinct(*tc)
            assert bool((tc[0] >= 0).all())
