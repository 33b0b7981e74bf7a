"""-m gpu: explanations on the real kernels (llmrec_explain_f32, recommend.explain, Trainer.explain).

1. Exact outputs: every contrib / own / last is bit-identical to a host restatement of the arithmetic contract (fmaf chains by the
   round-to-odd float64 restatement of tests/test_rerank_gpu.py, every other operation one fp32 operation in order), at every width,
   odd and multiple-of-4 leading dimensions, L = 1..3, histories of 1 and of more than 1,000 items, P = 1 and 64 with padding; top_ids /
   top_vals equal a host lexsort of the restated totals.
2. Independence: a (query, target, history item) gets the same bits alone, in a batch, with its targets permuted, beside other queries
   and on a second call.
3. The identity own + last + sum contrib = <U[u], I[i]> on netflix-shaped engines, for every user's recommend top-10.
4. Fold-ins: a trained user's own row as a history, an unknown user, an edgeless history item, new-item targets, the ID-only engine.
5. No side effects between --deterministic 1 steps.
6. Rejections before any launch."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import test_checkpoint_gpu as C  # noqa: E402
import test_deterministic_gpu as D  # noqa: E402
from test_rerank_gpu import _fma_chain  # noqa: E402

cuda = torch.device("cuda")
F32 = np.float32


def _padded(g, n, d, pad):
    return torch.randn(n, d + pad, device=cuda, generator=g)[:, :d]


def _operands(d, L, pad, n_side, seed=0, nu=40, ni=1500, n_cat=1700):
    """Synthetic operands of one explanation call: user-side rows, item-side sources (side blocks of one buffer, as Pi), catalog."""
    g = torch.Generator(device=cuda).manual_seed(seed)
    Fu = _padded(g, nu, n_side * d, pad)
    Pi = _padded(g, ni, n_side * d, pad)
    o = dict(own_src=_padded(g, nu, d, pad), last_src=_padded(g, nu, d, pad + 2),
             side_usr=[Fu[:, t * d:(t + 1) * d] for t in range(n_side)], side_src=[Pi[:, t * d:(t + 1) * d] for t in range(n_side)],
             coefs=[0.02, 2.8, 0.005, 0.7][:n_side], id_src=[_padded(g, ni, d, pad) for _ in range(L - 1)], I=_padded(g, n_cat, d, pad + 1),
             n_layers=L + 1)
    o["side_usr"][0][3] = 0.0                                        # a zero side row: the 1e-12 clamp
    return o


def _queries(rng, ni, n_cat, P, sizes, nu=40):
    m = len(sizes)
    hist = [np.sort(rng.choice(ni, s, replace=False)) for s in sizes]
    targets = rng.integers(0, n_cat, (m, P))
    targets[rng.random((m, P)) < 0.2] = -1                            # padding slots
    targets[0, 0] = -1
    qrow = rng.integers(0, nu, m)
    su = (rng.random(m) + 0.05).astype(F32)
    return qrow, su, hist, targets


def _call(o, qrow, su, hist, targets, top=0):
    from llmrec_b200 import ops
    rp = np.concatenate([[0], np.cumsum([h.size for h in hist])])
    col = np.concatenate(hist) if hist else np.zeros(0, np.int64)
    i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a).astype(np.int32)).to(cuda)
    return ops.explain(o["own_src"], o["last_src"], o["side_usr"], o["side_src"], o["coefs"], o["id_src"], o["I"], i32(qrow),
                       torch.from_numpy(np.asarray(su, F32)).to(cuda), i32(rp), i32(col), i32(targets), o["n_layers"], top)


def _restate(o, qrow, su, hist, targets):
    """The contract on the host -> (contrib [P * nnz x C], own [m x P], last [m x P]) as float32 numpy."""
    m, P = targets.shape
    n_side, n_id = len(o["side_usr"]), len(o["id_src"])
    Cn = 1 + n_side
    inv = F32(1.0) / F32(o["n_layers"])
    I = o["I"]
    # own / last
    q_rep = torch.from_numpy(np.repeat(qrow, P)).to(cuda)
    t_flat = targets.reshape(-1)
    t_ok = torch.from_numpy(np.maximum(t_flat, 0)).to(cuda)
    own = _fma_chain(o["own_src"], I, q_rep, t_ok).cpu().numpy() * inv
    last = _fma_chain(o["last_src"], I, q_rep, t_ok).cpu().numpy() * inv
    own[t_flat < 0] = 0
    last[t_flat < 0] = 0
    # side weights
    w = np.zeros((m, max(n_side, 1)), F32)
    q = torch.from_numpy(qrow).to(cuda)
    for t in range(n_side):
        ss = _fma_chain(o["side_usr"][t], o["side_usr"][t], q, q).cpu().numpy()
        w[:, t] = (F32(o["coefs"][t]) / np.maximum(np.sqrt(ss), F32(1e-12))) * su
    # every (query, target, history item)
    bq, bp, bh = [], [], []
    for b in range(m):
        H = hist[b].size
        bq.append(np.full(P * H, b)); bp.append(np.repeat(np.arange(P), H)); bh.append(np.tile(hist[b], P))
    bq, bp, bh = (np.concatenate(x).astype(np.int64) for x in (bq, bp, bh))
    tgt = targets[bq, bp]
    ti, hi = torch.from_numpy(np.maximum(tgt, 0)).to(cuda), torch.from_numpy(bh).to(cuda)
    contrib = np.zeros((bq.size, Cn), F32)
    s = np.zeros(bq.size, F32)
    for l in range(n_id):
        s = s + _fma_chain(o["id_src"][l], I, hi, ti).cpu().numpy()
    contrib[:, 0] = (s * su[bq]) * inv
    for t in range(n_side):
        contrib[:, 1 + t] = _fma_chain(o["side_src"][t], I, hi, ti).cpu().numpy() * w[bq, t]
    contrib[tgt < 0] = 0
    return contrib, own.reshape(m, P), last.reshape(m, P)


def _host_top(contrib, hist, targets, N):
    m, P = targets.shape
    ids = np.full((m, P, N), -1, np.int64)
    vals = np.full((m, P, N), -np.inf, F32)
    off = 0
    for b in range(m):
        H = hist[b].size
        for p in range(P):
            if targets[b, p] < 0:
                vals[b, p] = 0
                continue
            rows = contrib[P * off + p * H:P * off + (p + 1) * H]
            tot = np.zeros(H, F32)
            for c in range(rows.shape[1]):
                tot = tot + rows[:, c]
            o = np.lexsort((hist[b], -tot.astype(np.float64)))[:N]
            ids[b, p, :o.size] = hist[b][o]
            vals[b, p, :o.size] = tot[o]
        off += H
    return ids, vals


def _same(a, b):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


@pytest.mark.parametrize("pad", [5, 8], ids=["ld-odd", "ld-x4"])
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("d", [20, 32, 64, 128, 256, 300])
def test_outputs_are_the_contract(d, L, pad):
    n_side = 4 if L != 1 else 3
    o = _operands(d, L, pad, n_side, seed=d + L)
    rng = np.random.default_rng(d * 10 + L)
    for P, sizes in ((1, [1, 1200, 0, 7]), (64, [1, 1100, 33, 0, 65])):
        qrow, su, hist, targets = _queries(rng, 1500, 1700, P, sizes)
        qrow[-1] = 3                                                   # the zero side row
        contrib, own, last, tids, tvals = _call(o, qrow, su, hist, targets, top=0)
        want_c, want_o, want_l = _restate(o, qrow, su, hist, targets)
        assert _same(contrib.cpu().numpy(), want_c), (P, int((contrib.cpu().numpy() != want_c).sum()))
        assert _same(own.cpu().numpy(), want_o) and _same(last.cpu().numpy(), want_l), P
        assert tids is None and tvals is None
        if L == 1:
            assert not contrib[:, 0].any()
        for N in (1, 10, 64):
            c2, _, _, tids, tvals = _call(o, qrow, su, hist, targets, top=N)
            assert _same(c2.cpu().numpy(), want_c)
            want_i, want_v = _host_top(want_c, hist, targets, N)
            assert np.array_equal(tids.cpu().numpy(), want_i), (P, N)
            assert _same(tvals.cpu().numpy(), want_v), (P, N)


def test_outputs_do_not_depend_on_the_batch():
    o = _operands(64, 2, 5, 4, seed=3)
    rng = np.random.default_rng(3)
    qrow, su, hist, targets = _queries(rng, 1500, 1700, 20, [5, 300, 1, 40, 9, 70])
    full = [x.cpu().numpy() for x in _call(o, qrow, su, hist, targets, top=5)]
    again = [x.cpu().numpy() for x in _call(o, qrow, su, hist, targets, top=5)]
    assert all(_same(a, b) if a.dtype == F32 else np.array_equal(a, b) for a, b in zip(full, again))     # a second call
    P, rp = targets.shape[1], np.concatenate([[0], np.cumsum([h.size for h in hist])])
    blk = lambda c, b: c[P * rp[b]:P * rp[b + 1]].reshape(P, hist[b].size, -1)
    for b in range(len(hist)):
        perm = rng.permutation(P)
        one = [x.cpu().numpy() for x in _call(o, qrow[b:b + 1], su[b:b + 1], hist[b:b + 1], targets[b:b + 1, perm], top=5)]
        assert _same(one[0].reshape(P, hist[b].size, -1), blk(full[0], b)[perm]), b      # alone, targets permuted
        assert _same(one[1][0], full[1][b][perm]) and _same(one[2][0], full[2][b][perm])
        assert np.array_equal(one[3][0], full[3][b][perm]) and _same(one[4][0], full[4][b][perm])
    # other queries added in front
    q2, s2, h2, t2 = _queries(rng, 1500, 1700, 20, [2, 500, 17])
    more = [x.cpu().numpy() for x in _call(o, np.concatenate([q2, qrow]), np.concatenate([s2, su]), h2 + hist,
                                           np.concatenate([t2, targets]), top=5)]
    off = P * sum(h.size for h in h2)
    assert _same(more[0][off:], full[0]) and _same(more[1][3:], full[1]) and np.array_equal(more[3][3:], full[3])


def _decomposition_fp64(hp, users, targets, res):
    """own, last and every contrib in float64 from the engine's own tensors (the fold-in's formulas without fp32 rounding)."""
    L, d = hp.L, hp.d
    inv = 1.0 / (L + 1)
    rp = hp.ui.rowptr.long().cpu()
    col = hp.ui.col.long()
    I = hp.I.double()
    tot = torch.zeros(targets.shape, dtype=torch.float64, device=cuda)
    mag = torch.zeros(targets.shape, dtype=torch.float64, device=cuda)
    srcs = [hp.Il[l].double() for l in range(L - 1)]
    sides = list(zip(hp.sides.fused(hp.Fu, hp.prof_u), hp.sides.fused(hp.Pi, hp.prof_i), hp._side_coefs())) if hp.has_feats else []
    su = hp.ui.rs.double()
    for b, u in enumerate(users.tolist()):
        h = col[rp[u]:rp[u + 1]]
        Ii = I[targets[b].clamp(min=0)]                                       # [P x d]
        terms = [hp.Ul[0][u].double() @ Ii.T * inv, hp.Ul[L][u].double() @ Ii.T * inv]
        for X in srcs:
            terms.append((X[h] @ Ii.T) * su[u] * inv)                         # [H x P]
        for x_u, X, c in sides:
            wt = c / max(float(x_u[u].double().norm()), 1e-12) * su[u]
            terms.append((X[h].double() @ Ii.T) * wt)
        tot[b] = sum(t.sum(0) if t.dim() == 2 else t for t in terms)
        mag[b] = sum(t.abs().sum(0) if t.dim() == 2 else t.abs() for t in terms)
    return tot, mag


def _sums(res):
    """own + last + sum contrib per (query, target) in float64, and the sum of the magnitudes"""
    m, P = res.own.shape
    rp = res.hist_rowptr.cpu().tolist()
    tot = res.own.double() + res.last.double()
    mag = res.own.double().abs() + res.last.double().abs()
    for b in range(m):
        blk = res.contrib[P * rp[b]:P * rp[b + 1]].double().view(P, rp[b + 1] - rp[b], len(res.channels))
        tot[b] += blk.sum((1, 2))
        mag[b] += blk.abs().sum((1, 2))
    return tot, mag


C_BOUND = 4     # c of the identity's bound c * (d + H + C) * 2^-24 * (|own| + |last| + sum |contrib|)


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_identity_on_a_netflix_shaped_engine(hoisted):
    from llmrec_b200 import ops, recommend
    hp = D._engine(False, hoisted)
    rng = np.random.default_rng(2)
    for _ in range(2):
        B = 1024
        u = torch.from_numpy(rng.integers(0, hp.nu, B).astype(np.int32)).to(cuda)
        p, n = (torch.from_numpy(rng.integers(0, hp.ni, B).astype(np.int32)).to(cuda) for _ in range(2))
        hp.train_step_graphed(u, p, n)
    hp.forward()
    rp, col = hp.ui.rowptr, hp.ui.col
    ids, _ = recommend.top_k(hp, rp, col, K=10, exclude="train")
    res = recommend.explain(hp, rp, col, ids)
    assert res.channels == ["id", "image", "text", "profile"] + D.KEYS and res.contrib.shape[1] == 9
    users = torch.arange(hp.nu, device=cuda)
    score = ops.score_pairs(hp.U, hp.I, users.to(torch.int32).repeat_interleave(10), ids.reshape(-1).to(torch.int32)).view(-1, 10).double()
    tot, mag = _sums(res)
    H = (hp.ui.rowptr[1:] - hp.ui.rowptr[:-1]).double()[:, None]
    if hoisted:
        assert bool(((tot - score).abs() <= 1e-4 * mag).all()), float(((tot - score).abs() / mag).max())
        return
    bound = C_BOUND * (hp.d + H + 9) * 2.0 ** -24 * mag
    err = (tot - score).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    sample = torch.from_numpy(np.sort(rng.choice(hp.nu, 600, replace=False))).to(cuda)
    t64, m64 = _decomposition_fp64(hp, sample.cpu(), ids[sample], res)
    assert bool(((tot[sample] - t64).abs() <= bound[sample]).all()), float(((tot[sample] - t64).abs() / bound[sample]).max())
    assert bool(((score[sample] - t64).abs() <= bound[sample]).all())


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1"]], ids=["default", "hoisted"])
def test_fold_ins_tiny(tiny_root, extra):
    from llmrec_b200 import ops
    with C._flags(tiny_root, ["--cuda_graph", "0"] + extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        nu, ni = hp.nu, hp.ni
        rng = np.random.default_rng(5)
        users = rng.choice(nu, 12, replace=False)
        items = rng.integers(-1, ni, (12, 7))
        trained = tr.explain(items, users=users, top=3)
        rp, col = hp.ui.rowptr.cpu().numpy(), hp.ui.col.cpu().numpy()
        hists = [col[rp[u]:rp[u + 1]].tolist() for u in users]
        folded = tr.explain(items, users=users, histories=hists, top=3)
        assert torch.equal(trained.hist_rowptr, folded.hist_rowptr) and torch.equal(trained.hist, folded.hist)
        for name in ("contrib", "own", "last"):                          # the bound of the fold-in against the trained rows
            a, b = getattr(trained, name), getattr(folded, name)
            scale = a.abs().amax() if a.numel() else 0
            assert bool(((a - b).abs() <= (1e-4 if extra else 2e-6) * scale).all()), name
        # unknown users: no ID layer; an edgeless item in a history; the identity against the fold-in's own scores
        deg = np.bincount(col, minlength=ni)
        dead = np.flatnonzero(deg == 0)
        hist = [[1, 5, 9], [2, 2, 7], [int(dead[0]) if dead.size else 3, 4], []]
        known = [-1, int(users[0]), -1, -1]
        tg = [[0, 1, 2], [3], [4, 5], [6, 7]]
        res = tr.explain(tg, users=known, histories=hist)
        assert res.hist_rowptr.tolist() == [0, 3, 5, 7, 7] and res.hist[3:5].tolist() == [2, 7]          # repeats collapse
        assert not res.own[0].any() and not res.own[2].any() and res.own[1, 0] != 0
        assert res.of(3)["contrib"].shape == (3, 0, len(res.channels))
        Uf = tr.fold_in(hist, known=known)
        q = torch.tensor([b for b, t in enumerate(tg) for _ in t], dtype=torch.int32, device=cuda)
        i = torch.tensor([x for t in tg for x in t], dtype=torch.int32, device=cuda)
        s = ops.score_pairs(Uf, hp.I, q, i)
        tot, mag = _sums(res)
        got = torch.cat([tot[b, :len(t)] for b, t in enumerate(tg)])
        mg = torch.cat([mag[b, :len(t)] for b, t in enumerate(tg)])
        lim = (1e-4 if extra else C_BOUND * (hp.d + 3 + len(res.channels)) * 2.0 ** -24) * mg
        assert bool(((got - s.double()).abs() <= lim).all())
        # new-item targets against score(..., new_items=...)
        lists = [[0, 1, 2], list(range(0, nu, 5))]
        u2 = [int(users[1]), int(users[2])]
        res = tr.explain([[ni, ni + 1, 3], [ni + 1]], users=u2, new_items=lists)
        s = tr.score([u2[0]] * 3 + [u2[1]], [ni, ni + 1, 3, ni + 1], new_items=lists).double()
        tot, mag = _sums(res)
        got, mg = torch.cat([tot[0], tot[1, :1]]), torch.cat([mag[0], mag[1, :1]])
        H = max(len(col[rp[u]:rp[u + 1]]) for u in u2)
        lim = (1e-4 if extra else C_BOUND * (hp.d + H + len(res.channels)) * 2.0 ** -24) * mg
        assert bool(((got - s).abs() <= lim).all())
        assert res.targets[1].tolist() == [ni + 1, -1, -1] and res.own[1, 1] == 0 and not res.of(1)["contrib"][1].any()


def test_id_only_engine_has_one_channel():
    import scipy.sparse as sp
    from llmrec_b200 import ops, recommend
    from llmrec_b200.engine import HotPath, HotPathConfig
    from llmrec_b200.graph import BipartiteGraph
    rng = np.random.default_rng(0)
    nu, ni, d, L = 500, 800, 128, 2
    R = sp.csr_matrix((np.ones(6000, F32), (rng.integers(0, nu, 6000), rng.integers(0, ni, 6000))), shape=(nu, ni))
    R.sum_duplicates(); R.data[:] = 1.0
    g = BipartiteGraph(R, cuda)
    params = {"user_id_embedding.weight": torch.randn(nu, d, device=cuda) * 0.1, "item_id_embedding.weight": torch.randn(ni, d, device=cuda) * 0.1}
    hp = HotPath((g.ui, g.iu, g.uiT, g.iuT), params, None, HotPathConfig(embed_size=d, n_layers=L))
    hp.forward()
    ids, _ = recommend.top_k(hp, g.rowptr_u, g.col_u, K=10, exclude="train")
    res = recommend.explain(hp, g.rowptr_u, g.col_u, ids, top=4)
    assert res.channels == ["id"] and res.contrib.shape[1] == 1 and res.top_ids.shape == (nu, 10, 4)
    score = ops.score_pairs(hp.U, hp.I, torch.arange(nu, device=cuda, dtype=torch.int32).repeat_interleave(10),
                            ids.reshape(-1).to(torch.int32)).view(nu, 10).double()
    tot, mag = _sums(res)
    H = (g.ui.rowptr[1:] - g.ui.rowptr[:-1]).double()[:, None]
    assert bool(((tot - score).abs() <= C_BOUND * (d + H + 1) * 2.0 ** -24 * mag).all())


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1", "--cuda_graph", "0"]], ids=["default-graph", "hoisted-eager"])
def test_explain_changes_no_run_state(tiny_root, extra):
    N, k = 8, 3
    with C._flags(tiny_root, ["--deterministic", "1"] + extra) as build:
        a, ba = build(), []
        C._steps(a, N, ba)
        sa = C._state(a)
        b, bb = build(), []
        C._steps(b, k, bb)
        lists = [[1, 2, 3], list(range(0, b.n_users, 2))]
        b.explain(np.tile(np.arange(10), (b.n_users, 1)), top=3)
        b.explain([[1, 2, b.n_items + 1]], users=[3], histories=[[4, 5]], new_items=lists)
        C._steps(b, N - k, bb)
        sb = C._state(b)
    C._same_batches(ba, bb)
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_rejections(tiny_root):
    from llmrec_b200 import ops, recommend
    from llmrec_b200.dist import ShardedGraph, ShardedHotPath, synthetic_shard
    from llmrec_b200.engine import HotPathConfig
    with C._flags(tiny_root, []) as build:
        tr = build()
        nu, ni = tr.n_users, tr.n_items
        launches = ops.STATS["launches"]
        for items in ([[0, ni]], [[-2, 3]], [[1.5]], np.full((nu, 3), ni)):
            with pytest.raises(ValueError, match="candidates|integers"):
                tr.explain(items, users=None if hasattr(items, "shape") else [0])
        for top in (0, 65, 2.0, True):
            with pytest.raises(ValueError, match="1..64"):
                tr.explain([[1, 2]], users=[0], top=top)
        with pytest.raises(ValueError, match="rows"):
            tr.explain([[1, 2]])
        with pytest.raises(ValueError, match="rows"):
            tr.explain([[1, 2]], histories=[[1], [2]])
        with pytest.raises(ValueError, match="known"):
            tr.explain([[1]], users=[nu], histories=[[1]])
        with pytest.raises(ValueError, match="outside"):
            tr.explain([[1]], histories=[[ni]])
        with pytest.raises(ValueError, match="users"):
            tr.explain([[1]], users=[nu])
        assert ops.STATS["launches"] == launches, "a rejected call launched a kernel"
    for flag in (["--mask_rate", "0.1"], ["--drop_rate", "0.1"]):
        with C._flags(tiny_root, flag) as build:
            tr = build()
            with pytest.raises(ValueError, match="fixed model"):
                tr.explain([[1, 2]], users=[0])
    ul, it, _, _ = synthetic_shard(64, 48, 400, 0, 1, cuda, seed=0)
    g = ShardedGraph(ul, it, 64, 48, solo=True)
    hp = ShardedHotPath(g, torch.randn(64, 32, device=cuda), torch.randn(48, 32, device=cuda), HotPathConfig(embed_size=32, n_layers=2), 0, solo=True)
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.explain(hp, g.rowptr_u, g.col_u, [[1]], users=[0])
