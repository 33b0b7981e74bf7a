"""-m gpu: diversified recommendations on the real kernel (llmrec_diversify_f32, ops.diversify, recommend.top_k / rerank with
diversity=, Trainer.recommend / Trainer.rerank, --candidates_diversity).

1. Exactness: ids, scores and sims are bit-identical to the host restatement (tests/diversify_model.mmr_select) fed with cosines from the
   round-to-odd float64 restatement of the fmaf chain, at d in {20, 32, 64, 128, 200, 256}, odd and multiple-of-4 leading dimensions,
   P in {1, 7, 64, 65, 257, 1024}, K in {1, 10, P}, lambda in {0, 0.25, 0.5, 0.7, 1}, with padding, repeated ids, equal scores,
   identical rows, NaN and -inf scores, on both the shared-memory and the streamed pool-row paths.
2. Batch independence: the same bits when queries are split across launches or permuted.
3. lambda = 1 at the netflix shape: the first K of the pool (modes 0 and 2), `recommend(K)` itself in mode 2, and `rerank`.
4. Trainer paths equal ops.diversify of their own pools (histories, new items, among, exclude_items), and each pick's sim is the
   cosine `similar_items` returns for that pair.
5. No side effects between --deterministic 1 steps; the --candidates_diversity file of an eval-only run; rejections."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import test_checkpoint_gpu as C  # noqa: E402
import test_deterministic_gpu as D  # noqa: E402
from diversify_model import mmr_select  # noqa: E402
from test_rerank_gpu import _fma_chain  # noqa: E402

cuda = torch.device("cuda")
LAMBDAS = (0.0, 0.25, 0.5, 0.7, 1.0)
POOL_BUDGET = 110 * 1024          # llmrec_diversify_f32 keeps the pool rows in shared memory up to this many bytes


def _gram(X, pool, chunk=1 << 16):
    """fp32 [m x P x P]: G[b, p, q] = the fmaf chain of X[pool[b, p]] and X[pool[b, q]] (padding reads row 0; it is never used)"""
    m, P = pool.shape
    ids = pool.clamp(min=0).to(cuda)
    a = ids[:, :, None].expand(m, P, P).reshape(-1)
    b = ids[:, None, :].expand(m, P, P).reshape(-1)
    out = torch.empty(a.numel(), dtype=torch.float32, device=cuda)
    for s in range(0, a.numel(), chunk):
        out[s:s + chunk] = _fma_chain(X, X, a[s:s + chunk], b[s:s + chunk])
    return out.reshape(m, P, P).cpu().numpy()


def _same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    return bool(((a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))).all())


def _catalog(d, pad, n=3000, seed=0):
    from llmrec_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(seed)
    X0 = torch.randn(n, d + 3, device=cuda, generator=g)[:, :d]
    src, dst = torch.randint(0, n, (2, 300), device=cuda, generator=g)
    X0[dst] = X0[src]                                                          # identical rows: cosine ties
    X = torch.empty(n, d + pad, device=cuda)[:, :d]                            # the leading dimension under test
    ops.row_normalize(X0, out=X)
    return X


def _pools(m, P, n, seed):
    """ids int64 [m x P] with repeats, -1 padding and out-of-range ids anywhere; scores fp32 with ties, NaN and -inf"""
    g = np.random.default_rng(seed)
    ids = g.integers(0, n, (m, P))
    if P > 1:
        r = g.integers(0, P, (m, P // 5 + 1))
        ids[np.arange(m)[:, None], r] = ids[np.arange(m)[:, None], g.integers(0, P, r.shape)]       # repeated ids
    ids[g.random((m, P)) < 0.1] = -1
    ids[g.random((m, P)) < 0.02] = n + 7                                       # outside the catalog: padding
    s = np.round(g.standard_normal((m, P)), 1).astype(np.float32)             # equal scores
    s[g.random((m, P)) < 0.05] = np.nan
    s[g.random((m, P)) < 0.05] = -np.inf
    return ids, s


def _check(X, ids, s, K, lam, got, G):
    n = X.shape[0]
    gi, gv, gs = (t.cpu().numpy() for t in got)
    for b in range(ids.shape[0]):
        r = np.where((ids[b] >= 0) & (ids[b] < n), ids[b], -1)
        wi, wv, ws = mmr_select(r, s[b], G[b], K, lam)
        assert np.array_equal(gi[b], wi), (b, K, lam, gi[b][:12], wi[:12])
        assert _same_bits(gv[b], wv) and _same_bits(gs[b], ws), (b, K, lam)


@pytest.mark.parametrize("pad", [5, 8], ids=["ld-odd", "ld-x4"])
@pytest.mark.parametrize("d", [20, 32, 64, 128, 200, 256])
def test_selection_is_the_host_restatement(d, pad):
    from llmrec_b200 import ops
    X = _catalog(d, pad)
    n = X.shape[0]
    paths = set()
    for P in (1, 7, 64, 65, 257, 1024):
        m = 2 if P == 1024 else 8
        ids, s = _pools(m, P, n, seed=P + d)
        G = _gram(X, torch.from_numpy(np.where((ids >= 0) & (ids < n), ids, -1)))
        paths.add(P * (d | 1) * 4 <= POOL_BUDGET)
        pid, ps = torch.from_numpy(ids).to(cuda), torch.from_numpy(s).to(cuda)
        for K in sorted({1, min(10, P), P}):
            for lam in LAMBDAS:
                _check(X, ids, s, K, lam, ops.diversify(X, pid, ps, K, lam), G)
    assert paths == ({True} if d < 32 else {True, False})                      # from d = 32 on, P = 1024 streams its rows


@pytest.mark.parametrize("P", [64, 1024], ids=["shared", "streamed"])
def test_outputs_do_not_depend_on_the_batch(P):
    from llmrec_b200 import ops
    X = _catalog(64, 8)
    ids, s = _pools(24, P, X.shape[0], seed=3)
    pid, ps = torch.from_numpy(ids).to(cuda), torch.from_numpy(s).to(cuda)
    K = 20
    whole = ops.diversify(X, pid, ps, K, 0.5)
    parts = [ops.diversify(X, pid[a:b], ps[a:b], K, 0.5) for a, b in ((0, 1), (1, 13), (13, 24))]
    perm = torch.randperm(24, device=cuda)
    shuffled = ops.diversify(X, pid[perm], ps[perm], K, 0.5)
    bits = lambda t: t.view(torch.int32) if t.is_floating_point() else t
    for j in range(3):
        assert torch.equal(bits(torch.cat([p[j] for p in parts])), bits(whole[j])), j
        assert torch.equal(bits(shuffled[j]), bits(whole[j][perm])), j


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_lambda_one_is_the_pool_netflix_shape(hoisted):
    from llmrec_b200 import recommend
    hp = D._engine(False, hoisted)
    hp.forward()
    g = np.random.default_rng(4)
    users = np.sort(g.choice(hp.nu, 512, replace=False))
    rp, col = hp.ui.rowptr, hp.ui.col
    for mode in (0, 2):
        p_ids, p_vals = recommend.top_k(hp, rp, col, users=users, K=64, mode=mode)
        for K, P in ((10, 64), (10, 10), (1, 30)):
            ids, vals = recommend.top_k(hp, rp, col, users=users, K=K, mode=mode, diversity=1, pool=P)
            if P == 64:
                assert torch.equal(ids, p_ids[:, :K]) and torch.equal(vals.view(torch.int32), p_vals[:, :K].view(torch.int32)), (mode, K)
            if mode == 2:
                t_ids, t_vals = recommend.top_k(hp, rp, col, users=users, K=K, mode=2)
                assert torch.equal(ids, t_ids) and torch.equal(vals.view(torch.int32), t_vals.view(torch.int32)), K
    cand = p_ids[:, torch.randperm(64, device=cuda)]
    for K in (10, 64):
        r_ids, r_vals = recommend.rerank(hp, rp, col, cand, users=users, K=K)
        d_ids, d_vals = recommend.rerank(hp, rp, col, cand, users=users, K=K, diversity=1)
        assert torch.equal(d_ids, r_ids) and torch.equal(d_vals.view(torch.int32), r_vals.view(torch.int32)), K
    # lambda < 1 changes lists but keeps each row's best item first
    ids, _ = recommend.top_k(hp, rp, col, users=users, K=10, mode=2, diversity=0.5)
    p_ids, _ = recommend.top_k(hp, rp, col, users=users, K=64, mode=2)
    assert torch.equal(ids[:, 0], p_ids[:, 0]) and not torch.equal(ids, p_ids[:, :10])


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1"]], ids=["default", "hoisted"])
def test_trainer_paths_are_diversify_of_their_pools_tiny(tiny_root, extra):
    from llmrec_b200 import ops, recommend
    with C._flags(tiny_root, extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        ni, nu = hp.ni, hp.nu
        g = np.random.default_rng(6)
        lists = [list(range(0, nu, 3)), [1, 4, 7], [1, 4, 7], [], list(range(1, nu, 2))]
        n = ni + len(lists)
        Rn = recommend.new_items_csr(lists, nu)
        X = ops.row_normalize(torch.cat([hp.I, tr.fold_in_items(lists)]))
        hist = [g.integers(0, ni, int(g.integers(0, 30))).tolist() for _ in range(12)] + [[]]
        known = [int(g.integers(-1, nu)) for _ in hist]
        S = np.sort(g.choice(n, n // 2, replace=False))
        ex = [g.integers(-1, n, 6).tolist() for _ in hist]
        calls = [dict(), dict(users=list(range(0, nu, 5))), dict(users=known, histories=hist, new_items=lists),
                 dict(users=known, histories=hist, new_items=lists, among=S, exclude_items=ex, exclude="none")]
        for kw in calls:
            for K, P, lam in ((5, 20, 0.5), (10, None, 0.0), (3, 3, 0.7)):
                ids, vals = tr.recommend(K=K, diversity=lam, pool=P, **kw)
                pool = P or min(64, S.size if "among" in kw else n if "new_items" in kw else ni)
                p_ids, p_vals = tr.recommend(K=pool, **kw)
                w_ids, w_vals, _ = ops.diversify(X if "new_items" in kw else X[:ni], p_ids, p_vals, K, lam)
                assert torch.equal(ids, w_ids) and torch.equal(vals.view(torch.int32), w_vals.view(torch.int32)), (kw.keys(), K, P, lam)
        cand = [g.integers(-1, n, int(g.integers(0, 80))).tolist() for _ in hist]
        for K, P, lam in ((5, 30, 0.5), (None, 12, 0.25), (4, None, 0.7)):
            ids, vals = tr.rerank(cand, users=known, histories=hist, new_items=lists, K=K, diversity=lam, pool=P)
            pool = P or max(min(1024, max(len({c for c in r if c >= 0}) for r in cand)), K or 1)
            p_ids, p_vals = tr.rerank(cand, users=known, histories=hist, new_items=lists, K=pool)
            w_ids, w_vals, _ = ops.diversify(X, p_ids, p_vals, K or pool, lam)
            assert torch.equal(ids, w_ids) and torch.equal(vals.view(torch.int32), w_vals.view(torch.int32)), (K, P, lam)
        # each pick's sim is its largest cosine to an earlier pick, with the bits similar_items returns
        p_ids, p_vals = tr.recommend(K=30, users=list(range(0, nu, 9)), new_items=lists)
        ids, _, sims = recommend.diversify(hp, Rn, p_ids, p_vals, 8, 0.3)
        assert bool(torch.isneginf(sims[:, 0]).all())
        for b in range(ids.shape[0]):
            for t in range(1, 8):
                if int(ids[b, t]) < 0:
                    continue
                _, c = recommend.similar_items(hp, [int(ids[b, t])], K=1, new_items=Rn, among=ids[b, :t], mode=2)
                assert c[0, 0].view(torch.int32) == sims[b, t].view(torch.int32), (b, t)


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1", "--cuda_graph", "0"]], ids=["default-graph", "hoisted-eager"])
def test_diversified_calls_change_no_run_state(tiny_root, extra):
    N, k = 8, 3
    with C._flags(tiny_root, ["--deterministic", "1"] + extra) as build:
        a, ba = build(), []
        C._steps(a, N, ba)
        sa = C._state(a)
        b, bb = build(), []
        C._steps(b, k, bb)
        lists = [[1, 2, 3], list(range(0, b.n_users, 2))]
        b.recommend(K=5, diversity=0.5, new_items=lists)
        b.recommend(K=3, users=[1], histories=[[4, 5]], diversity=0.2, pool=9, among=list(range(40)))
        b.rerank(np.tile(np.arange(20), (b.n_users, 1)), K=5, diversity=0.7)
        C._steps(b, N - k, bb)
        sb = C._state(b)
    C._same_batches(ba, bb)
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_candidates_diversity_file_of_an_eval_only_run(tiny_root, tmp_path):
    save = str(tmp_path / "ck")
    F = str(tmp_path / "data" / "candidate_indices")
    base = [sys.executable, os.path.join(REPO, "main.py"), "--data_path", tiny_root, "--dataset", "netflix", "--batch_size", "128",
            "--debug", "--lr", "0.001", "--verbose", "1"]
    env = dict(os.environ, PYTHONPATH=REPO)
    subprocess.run(base + ["--epoch", "2", "--save_dir", save], check=True, cwd=str(tmp_path), env=env)
    best = os.path.join(save, "best.pt")
    subprocess.run(base + ["--resume", best, "--eval_only", "1", "--candidates_out", F, "--candidates_k", "10",
                           "--candidates_diversity", "0.5", "--candidates_pool", "30"], check=True, cwd=str(tmp_path), env=env)
    assert sorted(os.listdir(tmp_path / "data")) == ["candidate_indices"]
    f = pickle.load(open(F, "rb"))
    with C._flags(tiny_root, ["--resume", best, "--eval_only", "1"]) as build:
        tr = build()
        ids, _ = tr.recommend(K=10, exclude="none", diversity=0.5, pool=30)
        plain, _ = tr.recommend(K=10, exclude="none")
    assert isinstance(f, torch.Tensor) and f.dtype == torch.int64 and torch.equal(f, ids.cpu())
    assert not torch.equal(f, plain.cpu())


def test_rejections(tiny_root):
    from llmrec_b200 import ops, recommend
    from llmrec_b200.dist import ShardedGraph, ShardedHotPath, synthetic_shard
    from llmrec_b200.engine import HotPathConfig
    with C._flags(tiny_root, []) as build:
        tr = build()
        ni = tr.n_items
        launches = ops.STATS["launches"]
        for lam in (float("nan"), -0.5, 1.5, "0.5", True):
            with pytest.raises(ValueError, match="diversity"):
                tr.recommend(K=5, diversity=lam)
            with pytest.raises(ValueError, match="diversity"):
                tr.rerank([[1, 2]], users=[0], diversity=lam)
        for pool in (4, 65, 5.0):
            with pytest.raises(ValueError, match="pool"):
                tr.recommend(K=5, diversity=0.5, pool=pool)
        with pytest.raises(ValueError, match="pool"):
            tr.recommend(K=5, diversity=0.5, pool=11, among=list(range(10)))
        for pool in (4, 1025):
            with pytest.raises(ValueError, match="pool"):
                tr.rerank([[1, 2]], users=[0], K=5, diversity=0.5, pool=pool)
        with pytest.raises(ValueError, match="give diversity"):
            tr.recommend(K=5, pool=20)
        with pytest.raises(ValueError, match="outside"):
            tr.recommend(K=5, diversity=0.5, among=[ni])
        assert ops.STATS["launches"] == launches, "a rejected call launched a kernel"
        X = ops.row_normalize(tr.hot.I)
        pid = torch.zeros((2, 8), dtype=torch.int64, device=cuda)
        ps = torch.zeros((2, 8), dtype=torch.float32, device=cuda)
        for K, lam in ((9, 0.5), (0, 0.5), (4, float("nan")), (4, 1.5), (4, -0.1)):
            with pytest.raises(RuntimeError, match="diversify"):
                ops.diversify(X, pid, ps, K, lam)
        with pytest.raises(RuntimeError, match="diversify"):
            ops.diversify(X, torch.zeros((1, 1025), dtype=torch.int64, device=cuda), torch.zeros((1, 1025), device=cuda), 4, 0.5)
    for flag in (["--mask_rate", "0.1"], ["--drop_rate", "0.1"]):
        with C._flags(tiny_root, flag) as build:
            tr = build()
            with pytest.raises(ValueError, match="fixed model"):
                tr.recommend(K=5, diversity=0.5)
            with pytest.raises(ValueError, match="fixed model"):
                tr.rerank([[1, 2]], users=[0], diversity=0.5)
    ul, it, _, _ = synthetic_shard(64, 48, 400, 0, 1, cuda, seed=0)
    g = ShardedGraph(ul, it, 64, 48, solo=True)
    hp = ShardedHotPath(g, torch.randn(64, 32, device=cuda), torch.randn(48, 32, device=cuda), HotPathConfig(embed_size=32, n_layers=2), 0, solo=True)
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.top_k(hp, g.rowptr_u, g.col_u, users=[0], K=5, diversity=0.5)
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.rerank(hp, g.rowptr_u, g.col_u, [[1]], users=[0], diversity=0.5)
