"""-m gpu: group recommendations on the real kernels (llmrec_score_topk_group_f32, recommend.top_k_groups, Trainer.recommend_groups,
--groups_in / --groups_out).

1. Exactness: member scores from the round-to-odd float64 restatement of the fmaf chain (test_rerank_gpu._fma_chain), aggregated in
   numpy float32 by the group rule (tests/group_model.py), masked and ranked on the host: the kernel's ids and score bits are identical,
   in modes 0 and 2, for d in {20, 32, 64, 96, 128, 200}: at d in {32, 64, 96, 128} with aligned operands (mode 0 then runs the
   tensor-core selection and rescoring, checked from what that path leaves in its scratch) and with odd leading dimensions (the SIMT fallback),
   K in {1, 10, 64}, every agg, groups of 1..64 members packed unevenly across tiles (64 singletons in one tile, one 64-member group),
   duplicated item rows (exact ties), item rows one ulp apart (near ties), a NaN member row, a member whose scores reach exactly -inf
   by overflow (exact -inf group scores under mean and min), `among` and group mask rows.
2. Singleton groups are `top_k` bit for bit at the netflix shape, for every user, every agg and both modes.
3. Mode 0 equals mode 2 at the netflix shape; the same rows when the groups are permuted or split across calls.
4. No side effects between --deterministic 1 steps; the --groups_out file of an eval-only run is Trainer.recommend_groups; rejections
   launch nothing."""
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
import group_model as GM  # noqa: E402
import test_checkpoint_gpu as C  # noqa: E402
import test_deterministic_gpu as D  # noqa: E402
from test_rerank_gpu import _fma_chain  # noqa: E402

cuda = torch.device("cuda")
AGGS = ("mean", "min", "max")


def _csr(rows, dev=cuda):
    rp = torch.tensor(np.concatenate([[0], np.cumsum([len(r) for r in rows])]), dtype=torch.int32)
    col = torch.tensor(np.concatenate([np.asarray(r, dtype=np.int64) for r in rows] + [np.zeros(0, np.int64)]), dtype=torch.int32)
    return rp.to(dev), col.to(dev)


def _groups(g, nu):
    """groups of 1, 2, 3, 17, 63 and 64 members, in an order that packs them unevenly across 64-row tiles, with 64 singletons in a
    row (one whole tile) -> list of ascending member lists"""
    sizes = [3, 63, 1, 17, 2, 64] + [1] * 64 + [17, 2, 63, 3, 1, 2, 1, 17]
    pool = np.setdiff1d(np.arange(nu), [7, 11])                                          # the NaN / -inf rows join groups 0 and 4 only
    return [sorted(g.choice(pool, s, replace=False).tolist()) for s in sizes]


def _want(Sm, rows, groups, cat, masks, agg, K):
    """host restatement: member scores Sm (fp32 [rows x n]) -> ids / score bits per group"""
    pos = {u: r for r, u in enumerate(rows)}
    ids, vals = [], []
    for grp, m in zip(groups, masks):
        keep = ~np.isin(cat, m)
        s = GM.aggregate(Sm[[pos[u] for u in grp]][:, cat], agg)
        i, v = GM.rank(s[keep], cat[keep], K)
        ids.append(i); vals.append(v)
    return np.stack(ids), np.stack(vals)


def _ran_tensor_cores(call, I, cat):
    """Whether `call` (one ops.score_topk_group) took the tensor-core path: that path leaves the TF32 hi parts of the catalog rows
    (the mantissa cut to 10 bits) at the start of the op's scratch; the SIMT path starts it with the member CSR and score rows."""
    from llmrec_b200 import ops
    call()
    torch.cuda.synchronize()
    scratch = ops._score_scratch[I.device.index]
    rows = I[torch.from_numpy(cat).to(I.device)]
    hi = (rows.contiguous().view(torch.int32) & ~0x1fff).view(torch.float32)
    got = scratch[:hi.numel()].view_as(hi)
    same = bool(torch.equal(got.view(torch.int32), hi.view(torch.int32)))
    scratch.zero_()                                                                      # no stale copy for the next check
    return same


TC_WIDTHS = (32, 64, 96, 128)


@pytest.mark.parametrize("d,layout", [(20, "ld-odd")] + [(d, lay) for d in TC_WIDTHS for lay in ("ld-odd", "ld-x4")] + [(200, "ld-odd")])
def test_group_topk_is_the_host_restatement(d, layout):
    """ld-x4: leading dimensions a multiple of 4 floats on 16-byte aligned bases, so mode 0 at d in {32, 64, 96, 128} runs the
    tensor-core selection and rescoring (checked from what that path leaves in its scratch); ld-odd: every mode takes the SIMT path"""
    from llmrec_b200 import ops
    nu, n = 300, 3000
    pad_u, pad_i = (3, 5) if layout == "ld-odd" else (4, 8)
    gen = torch.Generator(device=cuda).manual_seed(d)
    U = torch.randn(nu, d + pad_u, device=cuda, generator=gen)[:, :d]
    I = torch.randn(n, d + pad_i, device=cuda, generator=gen)[:, :d]
    g = np.random.default_rng(d)
    src, dst = g.integers(0, n, 300), g.integers(0, n, 300)
    I[torch.from_numpy(dst).to(cuda)] = I[torch.from_numpy(src).to(cuda)]              # exact ties: duplicated rows
    near = torch.from_numpy(g.integers(0, n - 1, 100)).to(cuda)
    I[near + 1] = I[near]
    col0 = I[near + 1, 1]
    I[near + 1, 1] = torch.nextafter(col0, torch.full_like(col0, float("inf")))        # near ties: one ulp apart in one entry
    # member 11 reaches an exact -inf score by overflow on the `big` items (2^100 * -2^100 in the first step of the chain; both
    # TF32-exact, so the 3xTF32 products agree) and scores every other item finitely; column 0 is zero for every other member
    big = torch.from_numpy(g.choice(n, 20, replace=False)).to(cuda)
    U[:, 0] = 0.0
    U[11, 0] = 2.0 ** 100
    I[big, 0] = -(2.0 ** 100)
    U[7] = float("nan")
    groups = _groups(g, nu)
    groups[0] = sorted(set(groups[0]) | {7})                                            # a NaN member
    groups[4] = sorted(set(groups[4]) | {11})                                           # a member with -inf scores
    rows = np.arange(nu)
    Sm = np.stack([_fma_chain(U, I, torch.full((n,), u, device=cuda, dtype=torch.long), torch.arange(n, device=cuda)).cpu().numpy()
                   for u in rows])
    big_np = big.cpu().numpy()
    assert np.isneginf(Sm[11, big_np]).all() and np.isfinite(np.delete(Sm[11], big_np)).all()
    for agg in ("mean", "min"):                                                          # exact -inf group scores, not NaN
        assert np.isneginf(GM.aggregate(Sm[groups[4]][:, big_np], agg)).all(), agg
    assert np.isfinite(GM.aggregate(Sm[groups[4]][:, big_np], "max")).all()
    rp, members = _csr(groups, "cpu")
    members = members.to(cuda)
    tc = d in TC_WIDTHS and layout == "ld-x4"
    if tc:
        assert U.stride(0) % 4 == 0 and I.stride(0) % 4 == 0 and U.data_ptr() % 16 == 0 and I.data_ptr() % 16 == 0
    for sub in ("all", "among"):
        cat = np.arange(n) if sub == "all" else np.union1d([0, n - 1], g.choice(n, 700, replace=False))
        among = None if sub == "all" else torch.from_numpy(cat).to(cuda, torch.int32)
        masks = [np.sort(g.choice(n, int(g.integers(0, 300)), replace=False)) for _ in groups]
        masks[5] = cat[: cat.size - 3]                                                    # only three items left
        mrp, mcol = _csr(masks)
        for mode in (2, 0):                                                               # which path each mode takes
            ran = _ran_tensor_cores(lambda: ops.score_topk_group(U, I, rp, members, among, mrp, mcol, 10, agg="mean", mode=mode), I, cat)
            assert ran == (mode == 0 and tc), (mode, layout)
        for agg in AGGS:
            for K in (1, 10, 64):
                want_i, want_v = _want(Sm, rows, groups, cat, masks, agg, K)
                for mode in (2, 0):
                    ids, vals = ops.score_topk_group(U, I, rp, members, among, mrp, mcol, K, agg=agg, mode=mode, want_vals=True)
                    got_i, got_v = ids.cpu().numpy(), vals.cpu().numpy()
                    bad = np.flatnonzero((got_i != want_i).any(1) | (got_v.view(np.int32) != want_v.view(np.int32)).any(1))
                    assert bad.size == 0, (sub, agg, K, mode, bad[:5], got_i[bad[:1]], want_i[bad[:1]])
                assert (want_i[0] == -1).all()                                                # the NaN member's group: nothing
                assert (want_i[5][:3] >= 0).all() and (K <= 3 or (want_i[5][3:] == -1).all())
                if agg != "max":                                                              # -inf group scores never returned
                    assert not np.isin(want_i[4], big_np).any()


def _netflix():
    hp = D._engine(False, False)
    hp.forward()
    return hp


def test_singletons_are_recommend_and_modes_agree_netflix_shape():
    from llmrec_b200 import recommend
    hp = _netflix()
    rp, col = hp.ui.rowptr, hp.ui.col
    users = np.arange(hp.nu)
    for mode in (0, 2):
        t_ids, t_vals = recommend.top_k(hp, rp, col, users=users, K=10, mode=mode)
        for agg in AGGS:
            ids, vals = recommend.top_k_groups(hp, rp, col, [[u] for u in users], K=10, agg=agg, mode=mode)
            assert torch.equal(ids, t_ids) and torch.equal(vals.view(torch.int32), t_vals.view(torch.int32)), (mode, agg)
    g = np.random.default_rng(1)
    perm = g.permutation(hp.nu)
    groups = [perm[i:i + 4].tolist() for i in range(0, hp.nu, 4)]                       # every user, in groups of 4
    for agg in AGGS:
        a = recommend.top_k_groups(hp, rp, col, groups, K=10, agg=agg, mode=0)
        b = recommend.top_k_groups(hp, rp, col, groups, K=10, agg=agg, mode=2)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32)), agg
        # batch independence: permuted groups, and the groups split across calls
        p = g.permutation(len(groups))
        c = recommend.top_k_groups(hp, rp, col, [groups[i] for i in p], K=10, agg=agg, mode=0)
        assert torch.equal(c[0], a[0][torch.from_numpy(p).to(cuda)]) and torch.equal(c[1], a[1][torch.from_numpy(p).to(cuda)]), agg
        h = len(groups) // 3
        parts = [recommend.top_k_groups(hp, rp, col, groups[s:e], K=10, agg=agg, mode=0) for s, e in ((0, h), (h, len(groups)))]
        assert torch.equal(torch.cat([x[0] for x in parts]), a[0]) and torch.equal(torch.cat([x[1] for x in parts]), a[1]), agg
        # each returned score is the rule over score_pairs of the members
        sc = recommend.score_pairs(hp, np.repeat(np.asarray(groups[0]), 10), np.tile(a[0][0].cpu().numpy(), len(groups[0])))
        want = GM.aggregate(sc.view(len(groups[0]), 10).cpu().numpy()[np.argsort(groups[0])], agg)
        assert np.array_equal(a[1][0].cpu().numpy().view(np.int32), want.view(np.int32)), agg


@pytest.mark.parametrize("extra", [[], ["--hoist_side", "1", "--cuda_graph", "0"]], ids=["default-graph", "hoisted-eager"])
def test_recommend_groups_changes_no_run_state(tiny_root, extra):
    N, k = 8, 3
    with C._flags(tiny_root, ["--deterministic", "1"] + extra) as build:
        a, ba = build(), []
        C._steps(a, N, ba)
        sa = C._state(a)
        b, bb = build(), []
        C._steps(b, k, bb)
        b.recommend_groups([[1, 2, 3], [4], list(range(64))], K=10, agg="min")
        b.recommend_groups([[5, 6]], K=3, agg="mean", new_items=[[5], [7]], among=[1, 5, 9, b.n_items + 1], exclude_items=[[5]])
        C._steps(b, N - k, bb)
        sb = C._state(b)
    C._same_batches(ba, bb)
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_groups_file_of_an_eval_only_run(tiny_root, tmp_path):
    from llmrec_b200 import ops
    save, out, F = str(tmp_path / "ck"), str(tmp_path / "groups_out"), str(tmp_path / "groups.pkl")
    base = [sys.executable, os.path.join(REPO, "main.py"), "--data_path", tiny_root, "--dataset", "netflix", "--batch_size", "128",
            "--debug", "--lr", "0.001", "--verbose", "1"]
    env = dict(os.environ, PYTHONPATH=REPO)
    subprocess.run(base + ["--epoch", "2", "--save_dir", save], check=True, cwd=str(tmp_path), env=env)
    best = os.path.join(save, "best.pt")
    g = np.random.default_rng(4)
    groups = [g.choice(300, int(s), replace=True).tolist() for s in g.integers(1, 9, 50)] + [[299, 0, 0]]
    pickle.dump(groups, open(F, "wb"))
    subprocess.run(base + ["--resume", best, "--eval_only", "1", "--groups_in", F, "--groups_out", out, "--groups_k", "12",
                           "--groups_agg", "min"], check=True, cwd=str(tmp_path), env=env)
    got = pickle.load(open(out, "rb"))
    assert isinstance(got, torch.Tensor) and got.dtype == torch.int64 and got.device.type == "cpu" and tuple(got.shape) == (51, 12)
    with C._flags(tiny_root, ["--resume", best, "--eval_only", "1"]) as build:
        tr = build()
        ids, _ = tr.recommend_groups(groups, K=12, agg="min", exclude="train")
        assert torch.equal(ids.cpu(), got)
        launches = ops.STATS["launches"]
        for bad, msg in (([[1], []], "empty"), ([[300]], "outside"), ([list(range(65))], "65 distinct")):
            with pytest.raises(ValueError, match=msg):
                tr.recommend_groups(bad, K=5)
        for kw, msg in ((dict(K=0), "K = "), (dict(K=401), "K = "), (dict(agg="median"), "agg"), (dict(exclude_items=[[1]]), "rows"),
                        (dict(among=[1, 2], K=3), "1..2")):
            with pytest.raises(ValueError, match=msg):
                tr.recommend_groups([[1, 2], [3]], **kw)
        assert ops.STATS["launches"] == launches, "a rejected call launched a kernel"
    # bad flags and files fail before the first step
    pickle.dump([[1], []], open(str(tmp_path / "bad.pkl"), "wb"))
    for flags, msg in ((["--groups_in", F], "go together"), (["--groups_in", str(tmp_path / "bad.pkl"), "--groups_out", out], "empty"),
                       (["--groups_in", str(tmp_path / "missing"), "--groups_out", out], "cannot read"),
                       (["--groups_in", F, "--groups_out", str(tmp_path / "x"), "--groups_k", "65"], "K = ")):
        r = subprocess.run(base + ["--epoch", "1"] + flags, cwd=str(tmp_path), env=env, capture_output=True, text=True)
        assert r.returncode != 0 and msg in r.stderr, (flags, r.stderr[-2000:])
        assert "Epoch" not in r.stdout + r.stderr
    assert not os.path.exists(tmp_path / "x")
