"""-m gpu: pair scores and re-ranking of given candidates on the real kernels (llmrec_score_pairs_f32, llmrec_rerank_f32, Trainer.score,
Trainer.rerank, --rerank_in / --rerank_out).

1. Pair scores are exact: bit-identical to a sequential-fmaf restatement of the chain (round-to-odd float64, so every fmaf is rounded
   once), to the scores score_topk returns for the same (user, item) in modes 0 and 2, and within the fp32 chain's bound of float64.
2. Selection is exact at every edge: the kernel's (ids, scores) equal a host lexsort on (-score, id) of its own pair scores.
3. Re-ranking the whole catalog with exclude="train" returns `recommend`'s lists bit for bit (mode 2); in mode 0 every shared id carries
   the same score bits; re-ranking recommend's own top-64 returns it unchanged.
4. Histories and new items on the tiny data set, default and hoisted engines.
5. No side effects between --deterministic 1 steps.
6. The --rerank_out file of an eval-only run.
7. Rejections."""
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

cuda = torch.device("cuda")


def _fma_chain(U, I, u, i):
    """a = 0; a = fmaf(U[u, j], I[i, j], a) for j = 0..d-1, exactly: the float64 product is exact, the float64 sum is made round-to-odd
    (its exact error breaks an even result toward the error's side), and round-to-odd at 53 bits then rounds to fp32 as fmaf does."""
    Ud, Id = U.double()[u], I.double()[i]
    a = torch.zeros(u.numel(), dtype=torch.float64, device=U.device)
    for j in range(U.shape[1]):
        p = Ud[:, j] * Id[:, j]
        s = p + a
        bp = s - a
        e = (p - bp) + (a - (s - bp))                     # TwoSum: s + e == p + a exactly
        even = (s.view(torch.int64) & 1) == 0
        fix = (e != 0) & even & torch.isfinite(s)
        s = torch.where(fix, torch.nextafter(s, torch.where(e > 0, torch.full_like(s, float("inf")), torch.full_like(s, float("-inf")))), s)
        a = s.float().double()
    return a.float()


def _mats(d, nu=300, ni=2000, seed=0, pad=5):
    g = torch.Generator(device=cuda).manual_seed(seed)
    U = torch.randn(nu, d + pad, device=cuda, generator=g)[:, :d]
    I = torch.randn(ni, d + pad + 3, device=cuda, generator=g)[:, :d]
    return U, I


@pytest.mark.parametrize("pad", [5, 8], ids=["ld-odd", "ld-x4"])
@pytest.mark.parametrize("d", [32, 64, 96, 128, 200])
def test_pair_scores_are_the_fmaf_chain(d, pad):
    from llmrec_b200 import ops
    U, I = _mats(d, pad=pad)
    if pad == 8:
        I = torch.randn(2000, d + 8, device=cuda)[:, :d]
    g = torch.Generator(device=cuda).manual_seed(d)
    n = 5000
    u = torch.randint(0, U.shape[0], (n,), device=cuda, generator=g, dtype=torch.int32)
    i = torch.randint(0, I.shape[0], (n,), device=cuda, generator=g, dtype=torch.int32)
    s = ops.score_pairs(U, I, u, i)
    want = _fma_chain(U, I, u.long(), i.long())
    assert torch.equal(s.view(torch.int32), want.view(torch.int32)), int((s != want).sum())
    ex = (U.double()[u.long()] * I.double()[i.long()])
    bound = d * 2.0 ** -24 / (1 - d * 2.0 ** -24) * ex.abs().sum(1)
    assert bool(((s.double() - ex.sum(1)).abs() <= bound).all())
    # the scores score_topk returns for the same (user, item), in both modes
    users = torch.arange(64, device=cuda, dtype=torch.int32)
    no_rp = torch.zeros(U.shape[0] + 1, dtype=torch.int32, device=cuda)
    no_col = torch.zeros(0, dtype=torch.int32, device=cuda)
    for mode in (0, 2):
        ids, vals = ops.score_topk(U, I, users, no_rp, no_col, 64, mode=mode, want_vals=True)
        got = ops.score_pairs(U, I, users.repeat_interleave(64), ids.reshape(-1).contiguous())
        assert torch.equal(got.view(torch.int32), vals.reshape(-1).view(torch.int32)), mode


def _host_rerank(S, rows, mask, K):
    """rows: list of candidate id arrays; S: dict-free scorer -> per row the lexsort on (-score, id) of the kernel's own pair scores"""
    ids = np.full((len(rows), K), -1, dtype=np.int64)
    vals = np.full((len(rows), K), -np.inf, dtype=np.float32)
    for r, c in enumerate(rows):
        c = np.unique(c[c >= 0])
        c = c[~np.isin(c, mask[r])]
        s = S(r, c)
        o = np.lexsort((c, -s.astype(np.float64)))[:K]        # NaN (-NaN) sorts last, ties by id
        ids[r, :o.size] = c[o]
        vals[r, :o.size] = s[o]
    return ids, vals


@pytest.mark.parametrize("d", [64, 50], ids=["d64-vec", "d50-scalar"])
def test_selection_is_exact_at_every_edge(d):
    from llmrec_b200 import ops
    n_cat = 6000
    gen = torch.Generator(device=cuda).manual_seed(1)
    if d == 64:                                                                      # 16-byte loads
        U, I = torch.randn(40, d, device=cuda, generator=gen), torch.randn(n_cat, d, device=cuda, generator=gen)
    else:                                                                            # odd leading dimensions: 4-byte loads
        U, I = torch.randn(40, d + 3, device=cuda, generator=gen)[:, :d], torch.randn(n_cat, d + 5, device=cuda, generator=gen)[:, :d]
    g = np.random.default_rng(2)
    src = g.integers(0, n_cat, 300)
    dst = g.integers(0, n_cat, 300)
    I[torch.from_numpy(dst).to(cuda)] = I[torch.from_numpy(src).to(cuda)]       # exact ties: duplicated rows
    U[:, 0] = -2.0
    ninf, nan = g.choice(n_cat, 40, replace=False).reshape(2, 20)
    I[torch.from_numpy(ninf).to(cuda), 0] = 3e38                                     # -2 * 3e38 = -inf, and stays -inf
    I[torch.from_numpy(nan).to(cuda), 1] = float("nan")                             # NaN from its second term on
    lengths = [0, 1, 31, 32, 33, 1023, 1024, 1025, 5000, n_cat]
    rows, q = [], []
    for L in lengths:
        for variant in range(3):
            c = (g.integers(0, n_cat, L) if variant == 1 else np.arange(n_cat) if L == n_cat else g.choice(n_cat, L, replace=False)).astype(np.int64)
            if variant == 2:                                                             # repeats, -inf / NaN scores, padding
                c = np.concatenate([c, c[: L // 3], ninf[:3], nan[:3]])
                c[g.integers(0, c.size, max(1, c.size // 7))] = -1
            rows.append(c)
            q.append(int(g.integers(0, U.shape[0])))
    rows.append(np.concatenate([ninf, nan, [-1, -1]]))                                   # only -inf / NaN candidates
    q.append(0)
    mask = [np.sort(g.choice(n_cat, int(g.integers(0, 200)), replace=False)) for _ in range(U.shape[0])]
    mrp = torch.tensor(np.concatenate([[0], np.cumsum([x.size for x in mask])]), dtype=torch.int32, device=cuda)
    mcol = torch.tensor(np.concatenate(mask), dtype=torch.int32, device=cuda)
    rp = torch.tensor(np.concatenate([[0], np.cumsum([x.size for x in rows])]), dtype=torch.int32, device=cuda)
    col = torch.tensor(np.concatenate(rows), dtype=torch.int32, device=cuda)
    qrow = torch.tensor(q, dtype=torch.int32, device=cuda)
    pair_u = torch.arange(U.shape[0], device=cuda, dtype=torch.int32).repeat_interleave(n_cat)
    pair_i = torch.arange(n_cat, device=cuda, dtype=torch.int32).repeat(U.shape[0])
    S_all = ops.score_pairs(U, I, pair_u, pair_i).reshape(U.shape[0], n_cat).cpu().numpy()
    assert np.isnan(S_all[:, nan]).all() and np.isneginf(S_all[:, ninf]).all()
    for masked in (False, True):
        for K in (1, 10, 64, 1000, 1024):
            ids, vals = ops.rerank(U, I, qrow, rp, col, mrp if masked else None, mcol if masked else None, K)
            want_i, want_v = _host_rerank(lambda r, c: S_all[q[r], c], rows,
                                          [mask[x] if masked else np.zeros(0, np.int64) for x in q], K)
            got_i, got_v = ids.cpu().numpy(), vals.cpu().numpy()
            assert np.array_equal(got_i, want_i), (masked, K, int(np.argmax((got_i != want_i).any(1))))
            same = (got_v.view(np.int32) == want_v.view(np.int32)) | (np.isnan(got_v) & np.isnan(want_v))
            assert same.all(), (masked, K)
    # the only -inf / NaN row: every real candidate before the padding, -inf before NaN
    ids, vals = ops.rerank(U, I, qrow[-1:], torch.tensor([0, rows[-1].size], dtype=torch.int32, device=cuda),
                           torch.from_numpy(rows[-1]).to(cuda, torch.int32), None, None, 64)
    assert ids[0, :20].tolist() == sorted(ninf.tolist()) and ids[0, 20:40].tolist() == sorted(nan.tolist())
    assert bool((ids[0, 40:] == -1).all()) and bool(torch.isnan(vals[0, 20:40]).all())


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_rerank_of_the_whole_catalog_is_recommend_netflix_shape(hoisted):
    from llmrec_b200 import recommend
    hp = D._engine(False, hoisted)
    hp.forward()
    g = np.random.default_rng(4)
    users = np.sort(g.choice(hp.nu, 512, replace=False))
    rp, col = hp.ui.rowptr, hp.ui.col
    every = (torch.arange(len(users) + 1, dtype=torch.int64) * hp.ni, torch.arange(hp.ni).repeat(len(users)))
    for K in (1, 10, 64):
        r_ids, r_vals = recommend.rerank(hp, rp, col, every, users=users, K=K, exclude="train")
        for mode in (2, 0):
            t_ids, t_vals = recommend.top_k(hp, rp, col, users=users, K=K, exclude="train", mode=mode)
            if mode == 2:
                assert torch.equal(r_ids, t_ids) and torch.equal(r_vals.view(torch.int32), t_vals.view(torch.int32)), K
            else:
                both = (r_ids[:, :, None] == t_ids[:, None, :]) & (t_ids[:, None, :] >= 0)
                rr, jr, jt = both.nonzero(as_tuple=True)
                assert rr.numel() >= 0.9 * len(users) * K
                assert torch.equal(r_vals[rr, jr].view(torch.int32), t_vals[rr, jt].view(torch.int32)), K
    ids, vals = recommend.top_k(hp, rp, col, users=users, K=64, exclude="train", mode=0)
    for exclude in ("train", "none"):
        again, v2 = recommend.rerank(hp, rp, col, ids, users=users, K=64, exclude=exclude)
        assert torch.equal(again, ids) and torch.equal(v2.view(torch.int32), vals.view(torch.int32))


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1"]], ids=["default", "hoisted"])
def test_histories_and_new_items_tiny(tiny_root, extra):
    from llmrec_b200 import ops
    with C._flags(tiny_root, extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        ni, nu = hp.ni, hp.nu
        g = np.random.default_rng(6)
        lists = [list(range(0, nu, 3)), [1, 4, 7], [1, 4, 7], [], list(range(1, nu, 2))]
        n = ni + len(lists)
        cat = torch.cat([hp.I, tr.fold_in_items(lists)])
        hist = [g.integers(0, ni, int(g.integers(0, 30))).tolist() for _ in range(20)] + [[]]
        known = [int(g.integers(-1, nu)) for _ in hist]
        Uf = tr.fold_in(hist, known=known)
        cand = [g.integers(-1, n, int(g.integers(0, 80))).tolist() for _ in hist]
        cand[0] += [ni, ni + 1, ni + 2, ni + 4]
        ids, vals = tr.rerank(cand, users=known, K=100, histories=hist, new_items=lists)
        for r, c in enumerate(cand):
            c = np.unique(np.array([x for x in c if x >= 0], dtype=np.int64))
            q = torch.full((c.size,), r, dtype=torch.int32, device=cuda)
            s = ops.score_pairs(Uf, cat, q, torch.from_numpy(c).to(cuda, torch.int32)).cpu().numpy()
            o = np.lexsort((c, -s.astype(np.float64)))
            assert ids[r, :c.size].tolist() == c[o].tolist() and bool((ids[r, c.size:] == -1).all())
            assert np.array_equal(vals[r, :c.size].cpu().numpy().view(np.int32), s[o].view(np.int32))
        # exclude="train": exactly what recommend masks, for trained users and for histories
        users = list(range(0, nu, 7))
        every = [list(range(n))] * len(users)
        ids, _ = tr.rerank(every, users=users, K=1024, exclude="train", new_items=lists)
        rp, col = hp.ui.rowptr.cpu(), hp.ui.col.cpu()
        for b, u in enumerate(users):
            masked = set(col[rp[u]:rp[u + 1]].tolist()) | {ni + j for j, l in enumerate(lists) if u in l}
            assert set(ids[b][ids[b] >= 0].tolist()) == set(range(n)) - masked
        every = [list(range(n))] * len(hist)
        ids, _ = tr.rerank(every, users=known, K=1024, exclude="train", histories=hist, new_items=lists)
        for b, (h, k) in enumerate(zip(hist, known)):
            masked = set(h) | ({ni + j for j, l in enumerate(lists) if k in l} if k >= 0 else set())
            assert set(ids[b][ids[b] >= 0].tolist()) == set(range(n)) - masked
        # Trainer.score: trained and new items, the bits of the chain
        u = g.integers(0, nu, 500)
        i = g.integers(0, n, 500)
        s = tr.score(u, i, new_items=lists)
        want = ops.score_pairs(hp.U, cat, torch.from_numpy(u).to(cuda, torch.int32), torch.from_numpy(i).to(cuda, torch.int32))
        assert s.dtype == torch.float32 and torch.equal(s.view(torch.int32), want.view(torch.int32))
        # K=None: the longest surviving row
        ids, _ = tr.rerank([[1, 2, 2, -1], [3]], users=[0, 1])
        assert tuple(ids.shape) == (2, 2) and sorted(ids[0].tolist()) == [1, 2] and ids[1].tolist()[1] == -1


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1", "--cuda_graph", "0"]], ids=["default-graph", "hoisted-eager"])
def test_score_and_rerank_change_no_run_state(tiny_root, extra):
    N, k = 8, 3
    with C._flags(tiny_root, ["--deterministic", "1"] + extra) as build:
        a, ba = build(), []
        C._steps(a, N, ba)
        sa = C._state(a)
        b, bb = build(), []
        C._steps(b, k, bb)
        lists = [[1, 2, 3], list(range(0, b.n_users, 2))]
        b.score([0, 1, 2], [5, b.n_items, 7], new_items=lists)
        b.rerank(np.tile(np.arange(20), (b.n_users, 1)), K=5)
        b.rerank([[1, 2, b.n_items + 1]], users=[3], exclude="train", histories=[[4, 5]], new_items=lists)
        C._steps(b, N - k, bb)
        sb = C._state(b)
    C._same_batches(ba, bb)
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_rerank_file_of_an_eval_only_run(tiny_root, tmp_path):
    save = str(tmp_path / "ck")
    F, G = str(tmp_path / "data" / "candidate_indices"), str(tmp_path / "data" / "reranked")
    base = [sys.executable, os.path.join(REPO, "main.py"), "--data_path", tiny_root, "--dataset", "netflix", "--batch_size", "128",
            "--debug", "--lr", "0.001", "--verbose", "1"]
    env = dict(os.environ, PYTHONPATH=REPO)
    subprocess.run(base + ["--epoch", "2", "--save_dir", save], check=True, cwd=str(tmp_path), env=env)
    best = os.path.join(save, "best.pt")
    run = base + ["--resume", best, "--eval_only", "1"]
    subprocess.run(run + ["--candidates_out", F, "--candidates_k", "10"], check=True, cwd=str(tmp_path), env=env)
    subprocess.run(run + ["--rerank_in", F, "--rerank_out", G], check=True, cwd=str(tmp_path), env=env)
    assert sorted(os.listdir(tmp_path / "data")) == ["candidate_indices", "reranked"]      # no .tmp left behind
    f, out = pickle.load(open(F, "rb")), pickle.load(open(G, "rb"))
    assert isinstance(out, torch.Tensor) and out.dtype == torch.int64 and out.device.type == "cpu"
    assert torch.equal(out, f)                                                            # the model's own list comes back unchanged
    shuffled = f[:, torch.randperm(f.shape[1])]
    with C._flags(tiny_root, ["--resume", best, "--eval_only", "1"]) as build:
        tr = build()
        ids, _ = tr.rerank(shuffled)
        assert torch.equal(ids.cpu(), out)


def test_rejections(tiny_root, tmp_path):
    from llmrec_b200 import ops, recommend
    from llmrec_b200.dist import ShardedGraph, ShardedHotPath, synthetic_shard
    from llmrec_b200.engine import HotPathConfig
    with C._flags(tiny_root, []) as build:
        tr = build()
        nu, ni = tr.n_users, tr.n_items
        launches = ops.STATS["launches"]
        for cand in ([[0, ni]], [[-2, 3]], [[1.5]], np.full((nu, 3), ni), np.zeros((nu, 2)), torch.zeros(nu, 2, dtype=torch.bool)):
            with pytest.raises(ValueError, match="candidates|integers"):
                tr.rerank(cand, users=None if hasattr(cand, "shape") else [0])
        for K in (0, 1025, 2.0, True):
            with pytest.raises(ValueError, match="1..1024"):
                tr.rerank([[1, 2]], users=[0], K=K)
        with pytest.raises(ValueError, match="K = None"):
            tr.rerank([list(range(ni + 700))] * 2 + [[1]], users=[0, 1, 2], new_items=[[1]] * 700)
        with pytest.raises(ValueError, match="rows"):
            tr.rerank([[1, 2]])                                                           # 1 row, no users: one row per user needed
        with pytest.raises(ValueError, match="rows"):
            tr.rerank([[1, 2]], users=[0, 1])
        with pytest.raises(ValueError, match="exclude"):
            tr.rerank([[1, 2]], users=[0], exclude="all")
        with pytest.raises(ValueError, match="one pair"):
            tr.score([0, 1], [2])
        for u, i in (([nu], [0]), ([0], [ni]), ([-1], [0]), ([0.5], [0])):
            with pytest.raises(ValueError, match="outside|integers"):
                tr.score(u, i)
        with pytest.raises(ValueError, match="outside"):
            tr.score([0], [ni + 2], new_items=[[1], [2]])
        with pytest.raises(ValueError, match="known"):
            tr.rerank([[1]], users=[nu], histories=[[1]])
        assert ops.STATS["launches"] == launches, "a rejected call launched a kernel"
    for flag in (["--mask_rate", "0.1"], ["--drop_rate", "0.1"]):
        with C._flags(tiny_root, flag) as build:
            tr = build()
            with pytest.raises(ValueError, match="fixed model"):
                tr.rerank([[1, 2]], users=[0])
            with pytest.raises(ValueError, match="fixed model"):
                tr.score([0], [1])
    ul, it, _, _ = synthetic_shard(64, 48, 400, 0, 1, cuda, seed=0)
    g = ShardedGraph(ul, it, 64, 48, solo=True)
    hp = ShardedHotPath(g, torch.randn(64, 32, device=cuda), torch.randn(48, 32, device=cuda), HotPathConfig(embed_size=32, n_layers=2), 0, solo=True)
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.rerank(hp, g.rowptr_u, g.col_u, [[1]], users=[0])
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.score_pairs(hp, [0], [1])
