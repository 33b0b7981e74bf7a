"""-m gpu: items added after training on the real kernels (HotPath.fold_in_items, Trainer.recommend(new_items=...),
Trainer.similar_items, llmrec_row_normalize_f32).

1. Folding in a trained item's own column of R reproduces the eval forward's I row: bit for bit where the iu tile plan keeps the row
   whole, within 2e-6 of the row's scale where it cuts the row into pieces (default engine); within 1e-4 on the hoisted engine (its Fi
   is (iu.ui.X)W^T + ci b, fold-in's is iu.(ui.(X W^T + b))).
2. New items (repeated user ids, an empty list, unknown items, a hub list longer than tile_nnz) against a float64 restatement of the item
   side of Models.py:152-197 on the engine's user side and the tables' exact values.
3. Top-K over the grown catalog against float64 U.[I; I_new]^T; item-to-item neighbours against float64 cosine.
4. No side effects: calls between deterministic steps leave the run bit-identical to an uninterrupted one.
5. Rejections."""
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
import test_recommend_gpu as R  # noqa: E402

cuda = torch.device("cuda")


def _split_items(hp):
    k = hp.iu.plan
    rows = torch.zeros(hp.ni, dtype=torch.bool, device=cuda)
    if k.n_split:
        rows[k.split_row[:k.n_split].long()] = True
    return rows


def _check_trained_items(hp, hoisted, tf32=False):
    hp.forward()
    If = hp.fold_in_items(hp.iu.rowptr, hp.iu.col, known=torch.arange(hp.ni))
    I = hp.I
    torch.cuda.synchronize()
    assert torch.isfinite(If).all()
    scale = I.abs().amax(1, keepdim=True)
    if hoisted:
        tol = 1e-3 if tf32 else 1e-4                      # TF32 rounds the two association orders' operands differently
        err = float(((If - I).abs() / scale).max())
        assert err <= tol, err
        return
    split = _split_items(hp)
    whole = ~split
    assert torch.equal(If[whole], I[whole]), int((If[whole] != I[whole]).any(1).sum())
    assert bool(((If - I).abs() <= 2e-6 * scale).all())
    return int(split.sum())


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_fold_in_items_reproduces_trained_items_netflix_shape(hoisted):
    hp = D._engine(False, hoisted)
    rng = np.random.default_rng(1)
    for _ in range(3):
        B = 1024
        u = torch.from_numpy(rng.integers(0, hp.nu, B).astype(np.int32)).to(cuda)
        p, n = (torch.from_numpy(rng.integers(0, hp.ni, B).astype(np.int32)).to(cuda) for _ in range(2))
        hp.train_step_graphed(u, p, n)
    n_split = _check_trained_items(hp, hoisted)
    if not hoisted:
        assert n_split > 0, "the power-law item degrees give the netflix shape split item rows"


@pytest.mark.parametrize("extra", R.TINY)
def test_fold_in_items_reproduces_trained_items_tiny(tiny_root, extra):
    with C._flags(tiny_root, ["--cuda_graph", "0"] + extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        _check_trained_items(tr.hot, tr.hoisted, tf32="tf32" in extra)


def _fold_in_item_fp64(hp, users, known):
    """The item side of Models.py:152-197 for one item row in float64: the engine's user side (Fu, Ul), P_usr from the user table's
    exact values."""
    p, d, L = hp.p, hp.d, hp.L
    us = torch.tensor(sorted(set(users)), dtype=torch.long, device=cuda)
    rs = (us.numel() + 1e-8) ** -0.5
    zero = torch.zeros(d, dtype=torch.float64, device=cuda)
    row = lambda T: rs * T.double()[us].sum(0) if us.numel() else zero
    Xu = R._dense_table(hp.feats["user"], p["user_trans.weight"].shape[1])
    P_usr = Xu @ p["user_trans.weight"].double().t() + p["user_trans.bias"].double()
    sides = [row(hp.blk(hp.Fu, s)) for s in range(hp.S)]
    sides = sides[:2] + [row(P_usr)] + sides[2:]
    layers = [hp.E_i[known].double() if known >= 0 else zero]
    for l in range(1, L + 1):
        x = row(hp.Ul[l])
        layers.append(torch.softmax(x, 0) if l == L else x)
    I = sum(layers) / (L + 1)
    for x, c in zip(sides, hp._side_coefs()):
        I = I + c * x / x.norm().clamp_min(1e-12)
    return I


def test_fold_in_of_new_items_against_fp64(tiny_root):
    with C._flags(tiny_root, ["--cuda_graph", "0"]) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        tile = hp.iu.plan.tile_nnz
        rp, col = hp.iu.rowptr.cpu(), hp.iu.col.cpu()
        column = lambda i: col[rp[i]:rp[i + 1]].tolist()
        hub = list(range(0, hp.nu, 2))
        assert len(hub) > tile, (len(hub), tile)
        cases = [(column(3) + [17], 3), ([8, 1, 8, 1, 1, 40], -1), ([], -1), ([], 5), (column(9), -1), (hub, -1), (hub, 12),
                 ([hp.nu - 1], -1)]
        I = tr.fold_in_items([u for u, _ in cases], known=[k for _, k in cases])
        for b, (u, k) in enumerate(cases):
            want = _fold_in_item_fp64(hp, u, k)
            err = float((I[b].double() - want).abs().max() / want.abs().max())
            assert err <= 1e-5, (b, err)
        d, L = hp.d, hp.L
        assert float((I[2] - 1.0 / d / (L + 1)).abs().max()) <= 1e-9            # empty: last layer softmax(0) = 1/d, all else 0
        assert torch.allclose(I[6] - I[5], hp.E_i[12] / (L + 1), rtol=1e-4, atol=1e-6)   # the same hub, with and without layer 0


def _grown(hp, lists):
    n, nu = hp.ni + len(lists), hp.nu
    Rt = torch.zeros(nu, len(lists), dtype=torch.bool, device=cuda)             # user u named by new item j
    for j, l in enumerate(lists):
        Rt[l, j] = True
    return n, Rt


@pytest.mark.parametrize("extra", [[], ["--proj_mode", "fp32"], ["--hoist_side", "1"]], ids=["3xtf32", "fp32", "hoisted"])
def test_topk_over_the_grown_catalog_against_fp64(tiny_root, extra):
    K = 20
    with C._flags(tiny_root, extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        ni, nu = hp.ni, hp.nu
        g = np.random.default_rng(5)
        # new items: hubs that score high for many users, two identical lists (exact ties), an empty list
        lists = [list(range(0, nu, 3)), g.integers(0, nu, 40).tolist(), [1, 4, 7], [1, 4, 7], [], list(range(1, nu, 2))]
        n, Rt = _grown(hp, lists)
        cat = torch.cat([hp.I, tr.fold_in_items(lists)]).double()
        Rm = torch.zeros(nu, ni, dtype=torch.bool, device=cuda)
        urp, ucol = hp.ui.rowptr.long(), hp.ui.col.long()
        Rm[torch.repeat_interleave(torch.arange(nu, device=cuda), urp[1:] - urp[:-1]), ucol] = True
        users = list(range(0, nu, 2))
        seen_new = False
        for exclude in ("train", "none"):
            ids, vals = tr.recommend(users=users, K=K, exclude=exclude, new_items=lists)
            assert ids.dtype == torch.int64 and tuple(ids.shape) == (len(users), K)
            masked = torch.cat([Rm, Rt], 1)[users] if exclude == "train" else torch.zeros(len(users), n, dtype=torch.bool, device=cuda)
            R._check_topk(ids, vals, hp.U[users].double() @ cat.t(), masked, K)
            seen_new |= bool((ids >= ni).any())
            for row in ids.tolist():                                                # identical new items 2 and 3: the lower id first
                if ni + 3 in row:
                    assert ni + 2 in row and row.index(ni + 2) < row.index(ni + 3)
        assert seen_new, "no new item was recommended"
        # folded-in histories: the history and the new items naming its trained id are masked; a near-full history pads with -1 / -inf
        hist = [g.integers(0, ni, int(g.integers(0, 30))).tolist() for _ in range(30)] + [list(range(ni - 5))]
        known = [int(g.integers(-1, nu)) for _ in hist[:-1]] + [0]
        Uf = tr.fold_in(hist, known=known)
        H = torch.zeros(len(hist), n, dtype=torch.bool, device=cuda)
        for b, (h, k) in enumerate(zip(hist, known)):
            H[b, h] = True
            if k >= 0:
                H[b, ni:] = Rt[k]
        ids, vals = tr.recommend(users=known, K=K, histories=hist, new_items=lists)
        R._check_topk(ids, vals, Uf.double() @ cat.t(), H, K)
        n_left = n - int(H[-1].sum())
        assert n_left < K and bool((ids[-1, n_left:] == -1).all()) and bool(torch.isinf(vals[-1, n_left:]).all())


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1"]], ids=["default", "hoisted"])
def test_similar_items_against_fp64_cosine(tiny_root, extra):
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
        q = list(range(0, ni, 7)) + [ni, ni + 1, ni + 2, ni + 3]
        ids, vals = tr.similar_items(q, K=K, new_items=lists)
        assert ids.dtype == torch.int64 and tuple(ids.shape) == (len(q), K)
        S = Xn[q] @ Xn.t()
        masked = torch.zeros_like(S, dtype=torch.bool)
        masked[torch.arange(len(q)), torch.tensor(q)] = True                  # never the query itself
        R._check_topk(ids, vals, S, masked, K)
        b1, b2 = q.index(ni + 1), q.index(ni + 2)
        assert ni + 2 in ids[b1].tolist() and ni + 1 in ids[b2].tolist()       # identical lists are each other's nearest
        assert abs(float(vals[b1, 0]) - 1.0) <= 1e-5
        ids0, _ = tr.similar_items(list(range(0, ni, 7)), K=K)                 # trained catalog only
        assert bool((ids0 < ni).all())


@pytest.mark.parametrize("d", [32, 64, 96, 128, 200])
def test_row_normalize_kernel(d):
    from llmrec_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(d)
    X = torch.randn(1000, d + 8, device=cuda, generator=g)[:, :d]              # a column slice: leading dimension d + 8
    X[3] = 0.0
    Y = ops.row_normalize(X)
    want = torch.nn.functional.normalize(X.double(), dim=1)
    assert float((Y.double() - want).abs().max()) <= 1e-6
    assert torch.equal(Y[3], torch.zeros(d, device=cuda))
    Z = X.clone()
    ops.row_normalize(Z, out=Z)                                                  # in place
    assert torch.equal(Z, Y)


@pytest.mark.parametrize("extra", [[], ["--cuda_graph", "0"], ["--hoist_side", "1"], ["--hoist_side", "1", "--cuda_graph", "0"]],
                         ids=["default-graph", "default-eager", "hoisted-graph", "hoisted-eager"])
def test_item_calls_change_no_run_state(tiny_root, extra):
    N, k = 8, 3
    with C._flags(tiny_root, ["--deterministic", "1"] + extra) as build:
        a, ba = build(), []
        C._steps(a, N, ba)
        sa = C._state(a)
        b, bb = build(), []
        C._steps(b, k, bb)
        ni, lists = b.n_items, [[1, 2, 3], [], list(range(0, b.n_users, 2))]
        b.fold_in_items(lists, known=[4, -1, -1])
        b.recommend(K=10, new_items=lists)
        b.recommend(users=[1, 2], K=5, histories=[[1, 2, 3], []], new_items=lists)
        b.similar_items([0, 5, ni, ni + 2], K=10, new_items=lists)
        C._steps(b, N - k, bb)
        sb = C._state(b)
    C._same_batches(ba, bb)
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_rejections(tiny_root):
    from llmrec_b200 import recommend
    from llmrec_b200.dist import ShardedGraph, ShardedHotPath, synthetic_shard
    from llmrec_b200.engine import HotPathConfig
    with C._flags(tiny_root, []) as build:
        tr = build()
        nu, ni = tr.n_users, tr.n_items
        for lists in ([[0, nu]], [[-1, 3]]):
            with pytest.raises(ValueError, match="user id .* outside"):
                tr.fold_in_items(lists)
            with pytest.raises(ValueError, match="user id .* outside"):
                tr.recommend(K=10, new_items=lists)
            with pytest.raises(ValueError, match="user id .* outside"):
                tr.similar_items([0], new_items=lists)
        with pytest.raises(ValueError, match="known"):
            tr.fold_in_items([[1], [2]], known=[ni, -1])
        with pytest.raises(ValueError, match="known"):
            tr.fold_in_items([[1], [2]], known=[0])
        with pytest.raises(ValueError, match="outside"):                      # histories take trained item ids only
            tr.recommend(histories=[[1, ni]], new_items=[[3]])
        for q in ([ni + 1], [-1], [1.5]):
            with pytest.raises(ValueError, match="query ids"):
                tr.similar_items(q, new_items=[[3]])
        for K in (0, 65):
            with pytest.raises(ValueError, match="1..64"):
                tr.recommend(K=K, new_items=[[3]])
            with pytest.raises(ValueError, match="1..64"):
                tr.similar_items([0], K=K)
        with pytest.raises(ValueError, match="user-id list"):
            tr.fold_in_items(None)
    for flag in (["--mask_rate", "0.1"], ["--drop_rate", "0.1"]):
        with C._flags(tiny_root, flag) as build:
            tr = build()
            for call in (lambda: tr.fold_in_items([[1, 2]]), lambda: tr.recommend(K=10, new_items=[[1]]), lambda: tr.similar_items([0])):
                with pytest.raises(ValueError, match="fixed model"):
                    call()
    ul, it, _, _ = synthetic_shard(64, 48, 400, 0, 1, cuda, seed=0)
    g = ShardedGraph(ul, it, 64, 48, solo=True)
    hp = ShardedHotPath(g, torch.randn(64, 32, device=cuda), torch.randn(48, 32, device=cuda), HotPathConfig(embed_size=32, n_layers=2), 0, solo=True)
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.top_k(hp, g.rowptr_u, g.col_u, K=10, new_items=[[1]])
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.similar_items(hp, [0], K=10)
