"""-m gpu: recommendations on the real kernels (HotPath.fold_in, Trainer.recommend, --candidates_out).

1. Folding in a training user's own training row reproduces the eval forward's U row: bit for bit where the tile plan keeps the row
   whole, within 2e-6 of the row's scale where it cuts the row into pieces (default engine); within the hoisted engine's reassociation
   tolerance there (its Fu is (ui.X)W^T + cu b, fold-in's is ui.(X W^T + b)).
2. New histories (an edgeless item, repeated ids, an empty history, unknown users) against a float64 restatement of Models.py:152-197
   on the engine's item side and the tables' exact values.
3. Top-K of trained and folded-in users against float64 U.I^T with lowest-id ties, both exclusion modes.
4. No side effects: recommend / fold_in between deterministic steps leave the run bit-identical to an uninterrupted one.
5. The candidate file of a `--resume best.pt --eval_only 1 --candidates_out F` run.
6. Rejections."""
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


def _split_rows(hp):
    k = hp.ui.plan
    rows = torch.zeros(hp.nu, dtype=torch.bool, device=cuda)
    if k.n_split:
        rows[k.split_row[:k.n_split].long()] = True
    return rows


def _check_training_rows(hp, hoisted, tf32=False):
    hp.forward()
    Uf = hp.fold_in(hp.ui.rowptr, hp.ui.col, known=torch.arange(hp.nu))
    U = hp.U
    torch.cuda.synchronize()
    assert torch.isfinite(Uf).all()
    if hoisted:
        tol = 1e-3 if tf32 else 1e-5                      # TF32 rounds the two association orders' operands differently
        torch.testing.assert_close(Uf, U, rtol=100 * tol, atol=tol)
        return
    split = _split_rows(hp)
    whole = ~split
    assert torch.equal(Uf[whole], U[whole]), int((Uf[whole] != U[whole]).any(1).sum())
    scale = U.abs().amax(1, keepdim=True)
    assert bool(((Uf - U).abs() <= 2e-6 * scale).all())


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_fold_in_reproduces_training_users_netflix_shape(hoisted):
    hp = D._engine(False, hoisted)
    rng = np.random.default_rng(1)
    for _ in range(3):
        B = 1024
        u = torch.from_numpy(rng.integers(0, hp.nu, B).astype(np.int32)).to(cuda)
        p, n = (torch.from_numpy(rng.integers(0, hp.ni, B).astype(np.int32)).to(cuda) for _ in range(2))
        hp.train_step_graphed(u, p, n)
    _check_training_rows(hp, hoisted)


TINY = [pytest.param(["--feat_dtype", f, "--proj_mode", m], id=f"default-{f}-{m}") for f, m in
        (("fp32", "3xtf32"), ("fp32", "tf32"), ("fp32", "fp32"), ("bf16", "3xtf32"), ("int8", "3xtf32"), ("bf16", "tf32"), ("int8", "tf32"))]
TINY += [pytest.param(["--hoist_side", "1", "--feat_dtype", f, "--proj_mode", m], id=f"hoisted-{f}-{m}") for f, m in
         (("fp32", "3xtf32"), ("fp32", "tf32"), ("bf16", "3xtf32"), ("int8", "3xtf32"))]


@pytest.mark.parametrize("extra", TINY)
def test_fold_in_reproduces_training_users_tiny(tiny_root, extra):
    with C._flags(tiny_root, ["--cuda_graph", "0"] + extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        _check_training_rows(tr.hot, tr.hoisted, tf32="tf32" in extra)


def _dense_table(X, k):
    from llmrec_b200 import feat_int8
    return (feat_int8.dequantize(X, k) if X.dtype == torch.int8 else X).double()


def _fold_in_fp64(hp, hist, known):
    """Models.py:152-197 for one user row in float64: the engine's item side (Il, prof_i), Pi from the tables' exact values."""
    p, d, L = hp.p, hp.d, hp.L
    items = torch.tensor(sorted(set(hist)), dtype=torch.long, device=cuda)
    rs = (items.numel() + 1e-8) ** -0.5
    row = lambda T: rs * T.double()[items].sum(0) if items.numel() else torch.zeros(T.shape[1], dtype=torch.float64, device=cuda)
    proj = lambda X, w: _dense_table(X, p[w + ".weight"].shape[1])[items] @ p[w + ".weight"].double().t() + p[w + ".bias"].double()
    f = hp.feats
    tabs = [(f["image"], "image_trans"), (f["text"], "text_trans")] + [(f["item"][k], "item_trans") for k in hp.keys]
    sides = [rs * proj(X, w).sum(0) if items.numel() else torch.zeros(d, dtype=torch.float64, device=cuda) for X, w in tabs]
    sides = sides[:2] + [row(hp.prof_i)] + sides[2:]
    layers = [hp.E_u[known].double() if known >= 0 else torch.zeros(d, dtype=torch.float64, device=cuda)]
    for l in range(1, L + 1):
        x = row(hp.Il[l - 1])
        layers.append(torch.softmax(x, 0) if l == L else x)
    U = sum(layers) / (L + 1)
    for x, c in zip(sides, hp._side_coefs()):
        U = U + c * x / x.norm().clamp_min(1e-12)
    return U


def test_fold_in_of_new_histories_against_fp64(tiny_root):
    with C._flags(tiny_root, ["--cuda_graph", "0"]) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        dead = torch.nonzero(hp._live_pos < 0).flatten().tolist()
        assert dead, "the tiny data set has edgeless items"
        rp, col = hp.ui.rowptr.cpu(), hp.ui.col.cpu()
        train = lambda u: col[rp[u]:rp[u + 1]].tolist()
        cases = [(train(3) + [dead[0]], 3), ([dead[1], 7, dead[1], 7, 7, 11], -1), ([], -1), ([], 5), (train(9), -1),
                 (train(12)[:1] + dead[2:5], 12), (list(range(0, 400, 37)), -1)]
        U = tr.fold_in([h for h, _ in cases], known=[k for _, k in cases])
        for b, (h, k) in enumerate(cases):
            want = _fold_in_fp64(hp, h, k)
            err = float((U[b].double() - want).abs().max() / want.abs().max())
            assert err <= 1e-5, (b, err)
        d, L = hp.d, hp.L
        assert torch.equal(U[2], torch.full((d,), 1.0 / d / (L + 1), device=cuda)) or \
            float((U[2] - 1.0 / d / (L + 1)).abs().max()) <= 1e-9             # empty: last layer softmax(0) = 1/d, all else 0


def _check_topk(ids, vals, S64, masked, K):
    """ids / vals [m x K] against float64 scores S64 [m x n] with the masked (row, item) pairs excluded"""
    S = S64.clone()
    S[masked] = float("-inf")
    ref_v, ref_i = torch.sort(S, dim=1, descending=True, stable=True)            # stable: ties -> lowest id
    for b in range(ids.shape[0]):
        got = ids[b][ids[b] >= 0]
        n_cand = int(torch.isfinite(S[b]).sum())
        assert got.numel() == min(K, n_cand)
        assert not masked[b, got].any(), "an excluded item was returned"
        assert bool(torch.isinf(vals[b][ids[b] < 0]).all())
        scale = float(S64[b].abs().max())
        tol = 1e-5 * scale
        s_got = S64[b, got]
        assert got.numel() == 0 or float((vals[b][: got.numel()].double() - s_got).abs().max()) <= tol
        want = ref_i[b, : got.numel()]
        if not torch.equal(got, want):                                            # only near-ties at the boundary may swap
            kth = float(ref_v[b, got.numel() - 1])
            assert bool((s_got >= kth - tol).all())
            missing = want[~torch.isin(want, got)]
            assert bool((S64[b, missing] <= float(s_got.min()) + tol).all())


@pytest.mark.parametrize("extra", [[], ["--proj_mode", "fp32"], ["--hoist_side", "1"]], ids=["3xtf32", "fp32", "hoisted"])
def test_topk_against_fp64(tiny_root, extra):
    K = 20
    with C._flags(tiny_root, extra) as build:
        tr = build()
        for _ in range(3):
            tr.train_next_batch()
        hp = tr._current_model()
        n, nu = hp.ni, hp.nu
        I64 = hp.I.double()
        R = torch.zeros(nu, n, dtype=torch.bool, device=cuda)
        rp, col = hp.ui.rowptr.long(), hp.ui.col.long()
        R[torch.repeat_interleave(torch.arange(nu, device=cuda), rp[1:] - rp[:-1]), col] = True
        users = list(range(0, nu, 3))
        for exclude in ("train", "none"):
            ids, vals = tr.recommend(users=users, K=K, exclude=exclude)
            assert ids.dtype == torch.int64 and vals.dtype == torch.float32 and tuple(ids.shape) == (len(users), K)
            S = hp.U[users].double() @ I64.t()
            _check_topk(ids, vals, S, R[users] if exclude == "train" else torch.zeros_like(R[users]), K)
        g = np.random.default_rng(3)
        hist = [g.integers(0, n, int(g.integers(0, 30))).tolist() for _ in range(40)] + [list(range(n - 5))]
        known = [int(g.integers(-1, nu)) for _ in hist]
        Uf = tr.fold_in(hist, known=known)
        H = torch.zeros(len(hist), n, dtype=torch.bool, device=cuda)
        for b, h in enumerate(hist):
            H[b, h] = True
        for exclude in ("train", "none"):
            ids, vals = tr.recommend(users=known, K=K, exclude=exclude, histories=hist)
            _check_topk(ids, vals, Uf.double() @ hp.I.double().t(), H if exclude == "train" else torch.zeros_like(H), K)


@pytest.mark.parametrize("extra", [[], ["--cuda_graph", "0"], ["--hoist_side", "1"], ["--hoist_side", "1", "--cuda_graph", "0"]],
                         ids=["default-graph", "default-eager", "hoisted-graph", "hoisted-eager"])
def test_recommend_changes_no_run_state(tiny_root, extra):
    N, k = 8, 3
    with C._flags(tiny_root, ["--deterministic", "1"] + extra) as build:
        a, ba = build(), []
        C._steps(a, N, ba)
        sa = C._state(a)
        b, bb = build(), []
        C._steps(b, k, bb)
        b.recommend(K=10)
        b.recommend(users=[1, 2], K=5, exclude="none", histories=[[1, 2, 3], []])
        b.fold_in([[4, 5, 399]], known=[7])
        C._steps(b, N - k, bb)
        sb = C._state(b)
    C._same_batches(ba, bb)
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_candidate_file_of_an_eval_only_run(tiny_root, tmp_path):
    save, out = str(tmp_path / "ck"), str(tmp_path / "data" / "candidate_indices")
    base = [sys.executable, os.path.join(REPO, "main.py"), "--data_path", tiny_root, "--dataset", "netflix", "--batch_size", "128",
            "--debug", "--lr", "0.001", "--verbose", "1"]
    env = dict(os.environ, PYTHONPATH=REPO)
    subprocess.run(base + ["--epoch", "2", "--save_dir", save], check=True, cwd=str(tmp_path), env=env)
    best = os.path.join(save, "best.pt")
    assert os.path.exists(best)
    subprocess.run(base + ["--resume", best, "--eval_only", "1", "--candidates_out", out, "--candidates_k", "10"], check=True,
                   cwd=str(tmp_path), env=env)
    assert sorted(os.listdir(tmp_path / "data")) == ["candidate_indices"]        # no .tmp left behind
    cand = pickle.load(open(out, "rb"))                                           # gpt_ui_aug.py:85
    assert isinstance(cand, torch.Tensor) and cand.dtype == torch.int64 and cand.device.type == "cpu"
    with C._flags(tiny_root, ["--resume", best, "--eval_only", "1"]) as build:
        tr = build()
        hp = tr._current_model()
        assert tuple(cand.shape) == (hp.nu, 10)
        S = hp.U.double() @ hp.I.double().t()
        vals = S.gather(1, cand.to(cuda)).float()
        _check_topk(cand.to(cuda), vals, S, torch.zeros_like(S, dtype=torch.bool), 10)


def test_rejections(tiny_root):
    from llmrec_b200 import recommend
    from llmrec_b200.dist import ShardedGraph, ShardedHotPath, synthetic_shard
    from llmrec_b200.engine import HotPathConfig
    with C._flags(tiny_root, []) as build:
        tr = build()
        for h in ([[0, 400]], [[-1, 3]]):
            with pytest.raises(ValueError, match="outside"):
                tr.recommend(histories=h)
        for K in (0, 65):
            with pytest.raises(ValueError, match="1..64"):
                tr.recommend(K=K)
    with pytest.raises(ValueError, match="n_items"):
        recommend.check_k(12, 10)
    with C._flags(tiny_root, ["--mask_rate", "0.1"]) as build:
        with pytest.raises(ValueError, match="fixed model"):
            build().recommend(K=10)
    with C._flags(tiny_root, ["--drop_rate", "0.1"]) as build:
        with pytest.raises(ValueError, match="fixed model"):
            build().fold_in([[1, 2]])
    ul, it, _, _ = synthetic_shard(64, 48, 400, 0, 1, cuda, seed=0)
    g = ShardedGraph(ul, it, 64, 48, solo=True)
    hp = ShardedHotPath(g, torch.randn(64, 32, device=cuda), torch.randn(48, 32, device=cuda), HotPathConfig(embed_size=32, n_layers=2), 0, solo=True)
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.top_k(hp, g.rowptr_u, g.col_u, K=10)
