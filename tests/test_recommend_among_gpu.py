"""-m gpu: top-K over a catalog given by ids and per-query exclusions on the real kernels (llmrec_score_topk_among_f32,
recommend.top_k(among=, exclude_items=), recommend.similar_items(among=), Trainer.recommend / similar_items, --candidates_among).

1. ABI: score_topk_among equals one reference call -- llmrec_score_topk_f32 over the whole catalog with every id outside `among`
   appended to each mask row: mode 2 gives the same ids and bit-identical scores; mode 0 the same, but for near-tie swaps at the
   boundary.  d in {32, 64, 96, 128, 200} (tensor-core and SIMT paths), K in {1, 10, 64}, |among| in {K, 127, 128, 129, 10 %, all},
   sets holding item 0 and item n - 1, masked ids outside the set, rows whose whole set is masked, duplicated I rows (ties).
   among = arange(n) is bit-identical to the plain call in both modes.
2. API (netflix-shaped engine, default and hoisted): recommend(among=S, exclude="train") in mode 2 is rerank([S] * m) bit for bit;
   exclude_items (with histories, new items and new ids inside `among`) is a host lexsort of score_pairs scores with the merged mask.
3. similar_items(among=S) returns only ids of S, never the query, and meets the float64 cosine restatement of the neighbour test.
4. No side effects between --deterministic 1 steps; the --candidates_among file; rejections before any launch."""
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
import test_recommend_gpu as R  # noqa: E402

cuda = torch.device("cuda")


def _csr(rows):
    rp = torch.tensor(np.concatenate([[0], np.cumsum([len(r) for r in rows])]), dtype=torch.int32, device=cuda)
    col = torch.tensor(np.concatenate([np.asarray(r, dtype=np.int64) for r in rows] + [np.zeros(0, np.int64)]), dtype=torch.int32, device=cuda)
    return rp, col


def _reference(U, I, users, S, mask, K, mode):
    """llmrec_score_topk_f32 on the whole catalog, every id outside S appended to each mask row"""
    from llmrec_b200 import ops
    outside = np.setdiff1d(np.arange(I.shape[0]), S)
    rp, col = _csr([np.union1d(m, outside) for m in mask])
    return ops.score_topk(U, I, users, rp, col, K, mode=mode, want_vals=True)


def _near_tie_check(ids, vals, ref_ids, ref_vals, S64, K):
    """mode 0 against the exact reference: rows may differ only by swaps of scores within 1e-5 of the row's scale at the boundary"""
    for b in range(ids.shape[0]):
        if torch.equal(ids[b], ref_ids[b]) and torch.equal(vals[b].view(torch.int32), ref_vals[b].view(torch.int32)):
            continue
        got, want = ids[b][ids[b] >= 0], ref_ids[b][ref_ids[b] >= 0]
        assert got.numel() == want.numel(), b
        tol = 1e-5 * float(S64[b].abs().max())
        s_got, s_want = S64[b, got.long()], S64[b, want.long()]
        assert bool((s_got >= float(s_want.min()) - tol).all()), b
        missing = want[~torch.isin(want, got)]
        assert bool((S64[b, missing.long()] <= float(s_got.min()) + tol).all()), b


@pytest.mark.parametrize("d", [32, 64, 96, 128, 200])
def test_among_is_the_masked_full_catalog_call(d):
    from llmrec_b200 import ops
    nu, n = 150, 3000
    gen = torch.Generator(device=cuda).manual_seed(d)
    U = torch.randn(nu, d, device=cuda, generator=gen)
    I = torch.randn(n, d, device=cuda, generator=gen)
    g = np.random.default_rng(d)
    src, dst = g.integers(0, n, 400), g.integers(0, n, 400)
    I[torch.from_numpy(dst).to(cuda)] = I[torch.from_numpy(src).to(cuda)]            # exact ties: duplicated rows
    users = torch.from_numpy(g.integers(0, nu, 100)).to(cuda, torch.int32)
    S64 = U.double()[users.long()] @ I.double().t()
    for K in (1, 10, 64):
        for size in (K, 127, 128, 129, n // 10, n):
            if size == 1:
                S = np.array([n - 1])                                                    # the last column of the last tile
            else:                                                                        # item 0 and item n - 1 are in every set
                S = np.arange(n) if size == n else np.union1d([0, n - 1], g.choice(np.arange(1, n - 1), size - 2, replace=False))
                assert S[0] == 0 and S[-1] == n - 1
            assert S.size == size
            mask = [np.sort(g.choice(n, int(g.integers(0, 300)), replace=False)) for _ in range(nu)]   # ids in and outside S
            full = int(users[0])
            mask[full] = np.union1d(mask[full], S)                                       # the whole set masked: a padded row
            mrp, mcol = _csr(mask)
            among = torch.from_numpy(S).to(cuda, torch.int32)
            for mode in (2, 0):
                ids, vals = ops.score_topk_among(U, I, users, among, mrp, mcol, K, mode=mode, want_vals=True)
                ref_ids, ref_vals = _reference(U, I, users, S, mask, K, mode)
                assert bool((ids[0] == -1).all()) and bool(torch.isneginf(vals[0]).all())
                live = ids >= 0
                assert bool(torch.isin(ids[live], among).all())
                if mode == 2:
                    assert torch.equal(ids, ref_ids), (K, size, int((ids != ref_ids).any(1).sum()))
                    assert torch.equal(vals.view(torch.int32), ref_vals.view(torch.int32)), (K, size)
                else:
                    exact_ids, exact_vals = _reference(U, I, users, S, mask, K, 2)
                    _near_tie_check(ids, vals, exact_ids, exact_vals, S64, K)
                    _near_tie_check(ids, vals, ref_ids, ref_vals, S64, K)
                    got = ops.score_pairs(U, I, users.repeat_interleave(K)[live.reshape(-1)], ids[live].contiguous())
                    assert torch.equal(got.view(torch.int32), vals[live].view(torch.int32))    # returned scores are the exact chain
            if size == n:                                                                 # the identity map is the plain call
                for mode in (2, 0):
                    a = ops.score_topk_among(U, I, users, among, mrp, mcol, K, mode=mode, want_vals=True)
                    b = ops.score_topk(U, I, users, mrp, mcol, K, mode=mode, want_vals=True)
                    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32)), (K, mode)


def _lexsort_topk(s, cand, K):
    o = np.lexsort((cand, -s.astype(np.float64)))[:K]
    ids = np.full(K, -1, np.int64)
    ids[:o.size] = cand[o]
    return ids


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_among_and_exclude_items_netflix_shape(hoisted):
    from llmrec_b200 import ops, recommend
    hp = D._engine(False, hoisted)
    hp.forward()
    g = np.random.default_rng(7)
    rp, col = hp.ui.rowptr, hp.ui.col
    users = np.sort(g.choice(hp.nu, 400, replace=False))
    S = g.choice(hp.ni, hp.ni // 10, replace=False)
    S_list = np.unique(S)
    S = np.concatenate([S, S[:10]])                                                  # unsorted, with repeats
    every = (torch.arange(len(users) + 1, dtype=torch.int64) * S_list.size, torch.from_numpy(S_list).repeat(len(users)))
    for K in (1, 10, 64):
        t_ids, t_vals = recommend.top_k(hp, rp, col, users=users, K=K, exclude="train", mode=2, among=S)       # unsorted, repeats
        r_ids, r_vals = recommend.rerank(hp, rp, col, every, users=users, K=K, exclude="train")
        assert torch.equal(t_ids, r_ids) and torch.equal(t_vals.view(torch.int32), r_vals.view(torch.int32)), K
    # exclude_items with histories, new items and new ids inside `among`
    lists = [list(range(0, hp.nu, 5)), [1, 4, 7], [], list(range(3, hp.nu, 11))]
    n = hp.ni + len(lists)
    cat = recommend._catalog(hp, recommend.new_items_csr(lists, hp.nu))
    hist = [g.integers(0, hp.ni, int(g.integers(0, 40))).tolist() for _ in range(30)] + [[]]
    known = [int(g.integers(-1, hp.nu)) for _ in hist]
    among = np.concatenate([g.choice(hp.ni, 3000, replace=False), [hp.ni, hp.ni + 1, hp.ni + 3]])
    extra = [g.integers(0, n, int(g.integers(0, 300))).tolist() for _ in hist]
    extra[0] += list(among[:50]) + [hp.ni + 1]
    extra[1] = list(among)                                                           # the whole set hidden
    Hr, _, _, _, kn = recommend._queries(hp, rp, col, known, hist)
    Uf = recommend._query_rows(hp, Hr, kn)
    K = 20
    for exclude in ("train", "none"):
        for mode in (2, 0):
            ids, vals = recommend.top_k(hp, rp, col, users=known, K=K, exclude=exclude, histories=hist, mode=mode, new_items=lists,
                                        among=among, exclude_items=extra)
            want = np.full((len(hist), K), -1, np.int64)
            S64 = torch.zeros(len(hist), n, dtype=torch.float64, device=cuda)
            masked = torch.ones(len(hist), n, dtype=torch.bool, device=cuda)
            for b, h in enumerate(hist):
                m = set(extra[b])
                if exclude == "train":
                    m |= set(h) | ({hp.ni + j for j, l in enumerate(lists) if known[b] in l} if known[b] >= 0 else set())
                cand = np.array(sorted(set(among.tolist()) - m), dtype=np.int64)
                q = torch.full((cand.size,), b, dtype=torch.int32, device=cuda)
                s = ops.score_pairs(Uf, cat, q, torch.from_numpy(cand).to(cuda, torch.int32)).cpu().numpy()
                want[b] = _lexsort_topk(s, cand, K)
                S64[b] = Uf[b].double() @ cat.double().t()
                masked[b, torch.from_numpy(cand).to(cuda)] = False
            if mode == 2:
                assert np.array_equal(ids.cpu().numpy(), want), exclude
            else:
                R._check_topk(ids, vals, S64, masked, K)
            assert bool((ids[1] == -1).all())
    # trained users with exclude_items, including a repeated user with different rows
    u2 = [5, 9, 5]
    extra2 = [[1, 2, 3], [-1, -1, -1], list(range(0, hp.ni, 2))]
    ids, _ = recommend.top_k(hp, rp, col, users=u2, K=10, exclude="train", mode=2, exclude_items=np.array([e[:3] for e in extra2]))
    for b, u in enumerate(u2):
        cand = np.setdiff1d(np.arange(hp.ni), np.union1d(col[rp[u]:rp[u + 1]].cpu().numpy(), [x for x in extra2[b][:3] if x >= 0]))
        s = ops.score_pairs(hp.U, hp.I, torch.full((cand.size,), u, dtype=torch.int32, device=cuda),
                            torch.from_numpy(cand).to(cuda, torch.int32)).cpu().numpy()
        assert ids[b].tolist() == _lexsort_topk(s, cand, 10).tolist(), b


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1"]], ids=["default", "hoisted"])
def test_similar_items_among_against_fp64_cosine(tiny_root, extra):
    K = 15
    with C._flags(tiny_root, extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        ni = hp.ni
        lists = [list(range(0, hp.nu, 3)), [1, 4, 7], [1, 4, 7], [2]]
        cat = torch.cat([hp.I, tr.fold_in_items(lists)]).double()
        Xn = cat / cat.norm(dim=1, keepdim=True).clamp_min(1e-12)
        g = np.random.default_rng(11)
        S = np.union1d(g.choice(ni, 120, replace=False), [ni + 1, ni + 2])
        q = list(range(0, ni, 7)) + [ni, ni + 1, ni + 2, ni + 3] + [int(S[0]), int(S[5])]      # queries in and outside S
        ids, vals = tr.similar_items(q, K=K, new_items=lists, among=torch.from_numpy(S))
        assert ids.dtype == torch.int64 and tuple(ids.shape) == (len(q), K)
        assert bool(torch.isin(ids[ids >= 0].cpu(), torch.from_numpy(S)).all())
        assert not bool((ids == torch.tensor(q, device=cuda)[:, None]).any())
        Sc = Xn[q] @ Xn.t()
        masked = torch.ones_like(Sc, dtype=torch.bool)
        masked[:, torch.from_numpy(S).to(cuda)] = False
        masked[torch.arange(len(q)), torch.tensor(q)] = True                     # never the query itself
        R._check_topk(ids, vals, Sc, masked, K)
        b1 = q.index(ni + 1)
        assert ni + 2 in ids[b1].tolist()                                          # identical lists are each other's nearest


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1", "--cuda_graph", "0"]], ids=["default-graph", "hoisted-eager"])
def test_among_and_exclude_items_change_no_run_state(tiny_root, extra):
    N, k = 8, 3
    with C._flags(tiny_root, ["--deterministic", "1"] + extra) as build:
        a, ba = build(), []
        C._steps(a, N, ba)
        sa = C._state(a)
        b, bb = build(), []
        C._steps(b, k, bb)
        lists = [[1, 2, 3], list(range(0, b.n_users, 2))]
        b.recommend(K=10, among=list(range(0, b.n_items, 3)))
        b.recommend(users=[1, 2], K=5, exclude="train", histories=[[1, 2, 3], []], new_items=lists, among=[1, 5, 9, b.n_items + 1, 300],
                    exclude_items=[[5], [b.n_items + 1]])
        b.similar_items([0, 7], K=5, among=np.arange(50))
        C._steps(b, N - k, bb)
        sb = C._state(b)
    C._same_batches(ba, bb)
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_candidates_among_file_of_an_eval_only_run(tiny_root, tmp_path):
    save, out, S_path = str(tmp_path / "ck"), str(tmp_path / "data" / "candidate_indices"), str(tmp_path / "among.pkl")
    base = [sys.executable, os.path.join(REPO, "main.py"), "--data_path", tiny_root, "--dataset", "netflix", "--batch_size", "128",
            "--debug", "--lr", "0.001", "--verbose", "1"]
    env = dict(os.environ, PYTHONPATH=REPO)
    subprocess.run(base + ["--epoch", "2", "--save_dir", save], check=True, cwd=str(tmp_path), env=env)
    best = os.path.join(save, "best.pt")
    S = np.random.default_rng(3).choice(400, 60, replace=False)
    pickle.dump(torch.from_numpy(S), open(S_path, "wb"))
    run = base + ["--resume", best, "--eval_only", "1"]
    subprocess.run(run + ["--candidates_out", out, "--candidates_k", "10", "--candidates_among", S_path], check=True, cwd=str(tmp_path),
                   env=env)
    assert sorted(os.listdir(tmp_path / "data")) == ["candidate_indices"]
    cand = pickle.load(open(out, "rb"))
    assert isinstance(cand, torch.Tensor) and cand.dtype == torch.int64 and cand.device.type == "cpu" and tuple(cand.shape) == (300, 10)
    with C._flags(tiny_root, ["--resume", best, "--eval_only", "1"]) as build:
        tr = build()
        ids, _ = tr.recommend(K=10, exclude="none", among=S)
        assert torch.equal(ids.cpu(), cand)
    # bad flags and bad files fail before the first step: nothing is trained, nothing is written
    pickle.dump(np.array([[1, 2]]), open(str(tmp_path / "bad.pkl"), "wb"))
    for flags, msg in ((["--candidates_among", S_path], "--candidates_out"),
                       (["--candidates_out", str(tmp_path / "x"), "--candidates_among", str(tmp_path / "bad.pkl")], "1-D"),
                       (["--candidates_out", str(tmp_path / "x"), "--candidates_among", str(tmp_path / "missing")], "cannot read"),
                       (["--candidates_out", str(tmp_path / "x"), "--candidates_k", "61", "--candidates_among", S_path], "1..60")):
        r = subprocess.run(base + ["--epoch", "1"] + flags, cwd=str(tmp_path), env=env, capture_output=True, text=True)
        assert r.returncode != 0 and msg in r.stderr, (flags, r.stderr[-2000:])
        assert "Epoch" not in r.stdout + r.stderr
    assert not os.path.exists(tmp_path / "x")


def test_rejections_before_any_launch(tiny_root):
    from llmrec_b200 import ops
    with C._flags(tiny_root, []) as build:
        tr = build()
        nu, ni = tr.n_users, tr.n_items
        launches = ops.STATS["launches"]
        for among, msg in (([0, ni], "outside"), ([-1, 3], "outside"), ([1.5, 2.0], "integers"), (np.zeros(3), "integers"),
                           (torch.ones(3, dtype=torch.bool), "integers"), ([], "empty"), (np.zeros(0, np.int64), "empty")):
            with pytest.raises(ValueError, match=msg):
                tr.recommend(K=1, among=among)
            with pytest.raises(ValueError, match=msg):
                tr.similar_items([0], K=1, among=among)
        with pytest.raises(ValueError, match="outside"):
            tr.recommend(K=1, among=[ni + 2], new_items=[[1], [2]])
        with pytest.raises(ValueError, match="1..3"):
            tr.recommend(K=4, among=[1, 2, 3, 3])                                  # K counts distinct ids
        with pytest.raises(ValueError, match="1..2"):
            tr.similar_items([0], K=3, among=[1, 2])
        with pytest.raises(ValueError, match="rows"):
            tr.recommend(users=[0, 1], K=5, exclude_items=[[1]])
        with pytest.raises(ValueError, match="rows"):
            tr.recommend(K=5, exclude_items=[[1]] * (nu - 1))
        with pytest.raises(ValueError, match="rows"):
            tr.recommend(K=5, histories=[[1], [2]], exclude_items=[[1]])
        for bad in ([[ni]], [[-2]], [[0.5]]):
            with pytest.raises(ValueError, match="outside|integers"):
                tr.recommend(users=[0], K=5, exclude_items=bad)
        assert ops.STATS["launches"] == launches, "a rejected call launched a kernel"
