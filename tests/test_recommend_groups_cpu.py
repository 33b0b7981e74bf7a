"""Group recommendations without a GPU: canonical groups and their rejections, the group mask rows (the union of the members' rows and
the new items naming any member), `among` / `exclude_items` rows, every rejection of `top_k_groups` / `Trainer.recommend_groups`
before anything runs, the --groups_in / --groups_out flags and file, and `top_k_groups` end to end on kernel stand-ins
(tests/ops_emulator.py plus the stand-ins of tests/group_model.py, in a child process)."""
import os
import pickle
import sys
import types

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import group_model as GM  # noqa: E402


def _bare_engine(nu=100, ni=12):
    from llmrec_b200.engine import HotPath
    hp = HotPath.__new__(HotPath)
    hp.nu, hp.ni, hp.E_u = nu, ni, torch.zeros(1)
    return hp


def _train(nu=100, ni=12, seed=0):
    g = np.random.default_rng(seed)
    rows = [np.unique(g.integers(0, ni, int(g.integers(0, 5)))) for _ in range(nu)]
    rp = torch.tensor(np.concatenate([[0], np.cumsum([r.size for r in rows])]), dtype=torch.int32)
    return rows, rp, torch.tensor(np.concatenate(rows), dtype=torch.int32)


def _rows(rp, col):
    rp = rp.tolist()
    return [col[rp[r]:rp[r + 1]].tolist() for r in range(len(rp) - 1)]


def test_groups_csr_is_canonical():
    from llmrec_b200 import recommend
    rp, col = recommend.groups_csr([[5, 1, 5], [3], np.array([9, 0, 9, 0], dtype=np.int16), torch.tensor([7, 2])], 10)
    assert rp.dtype == col.dtype == torch.int64
    assert _rows(rp, col) == [[1, 5], [3], [0, 9], [2, 7]]
    rp2, col2 = recommend.groups_csr((np.array([0, 3, 4]), torch.tensor([5, 5, 1, 3])), 10)
    assert _rows(rp2, col2) == [[1, 5], [3]]
    assert recommend.groups_csr([list(range(64))], 64)[1].numel() == 64
    assert recommend.groups_csr([[3] * 200], 10)[1].tolist() == [3]                     # repeats collapse before the size check
    rp, col = recommend.groups_csr([], 10)
    assert rp.tolist() == [0] and col.numel() == 0


def test_groups_csr_rejections():
    from llmrec_b200 import recommend
    for bad, msg in (([[1], []], "group 1 is empty"), ([[0, 10]], "user id 10 is outside \\[0, 10\\)"), ([[-1]], "outside"),
                     ([list(range(65))], "group 0 has 65 distinct members; at most 64"), ([[0.5]], "integers"),
                     ([torch.ones(2, dtype=torch.bool)], "integers"), ((np.array([0, 2]), np.array([1])), "rowptr"), (5, "sequence"),
                     (["ab"], "list of user ids"), ([3, 4], "list of user ids")):
        with pytest.raises(ValueError, match=msg):
            recommend.groups_csr(bad, 10 if "65" not in msg else 100)


def test_check_agg():
    from llmrec_b200 import recommend
    assert [recommend.check_agg(a) for a in ("mean", "min", "max")] == ["mean", "min", "max"]
    for bad in ("avg", None, 0, "MEAN"):
        with pytest.raises(ValueError, match="agg"):
            recommend.check_agg(bad)


def test_group_mask_rows_are_the_union_of_the_members_rows():
    from llmrec_b200 import recommend
    hp = _bare_engine()
    train, rp, col = _train()
    groups = [[4, 2, 9], [7], [2, 4], [50, 51, 52, 53]]
    new_items = [[9], [1, 2], [], [52, 3]]                                              # new items 12..15 and the users naming them
    job = recommend.prepare_group_top_k(hp, rp, col, groups, K=3, new_items=new_items)
    named = {u: [12 + j for j, us in enumerate(new_items) if u in us] for u in range(hp.nu)}
    want = [sorted(set().union(*[set(train[u].tolist()) | set(named[u]) for u in g])) for g in groups]
    assert _rows(job["mask_rowptr"], job["mask_col"]) == want
    assert job["mask_rowptr"].dtype == job["mask_col"].dtype == torch.int32
    assert _rows(job["member_rowptr"], job["members"]) == [[2, 4, 9], [7], [2, 4], [50, 51, 52, 53]]
    job = recommend.prepare_group_top_k(hp, rp, col, groups, K=3, exclude="none", new_items=new_items)
    assert _rows(job["mask_rowptr"], job["mask_col"]) == [[]] * 4
    # exclude_items: one row per group, merged (sorted union, padding dropped)
    extra = np.array([[11, -1], [0, 0], [5, 1], [-1, -1]])
    job = recommend.prepare_group_top_k(hp, rp, col, groups, K=3, exclude_items=extra, among=[11, 0, 5, 5, 3])
    want2 = [sorted(set(w) | {x for x in e.tolist() if x >= 0}) for w, e in zip([sorted(set().union(*[set(train[u].tolist()) for u in g]))
                                                                                  for g in groups], extra)]
    assert _rows(job["mask_rowptr"], job["mask_col"]) == want2
    assert job["among"].tolist() == [0, 3, 5, 11]


def test_rejections_before_anything_runs():
    from llmrec_b200 import recommend
    hp = _bare_engine()
    _, rp, col = _train()
    top = lambda groups=([1, 2], [3]), **kw: recommend.prepare_group_top_k(hp, rp, col, groups, **{"K": 2, **kw})
    for groups, msg in (([[1], []], "empty"), ([[100]], "outside \\[0, 100\\)"), ([list(range(65))], "65 distinct members")):
        with pytest.raises(ValueError, match=msg):
            top(groups)
    with pytest.raises(ValueError, match="agg"):
        top(agg="median")
    for K in (0, 13, 65, True, 2.0):
        with pytest.raises(ValueError, match="K = "):
            top(K=K)
    with pytest.raises(ValueError, match="1..2 .*\\|among\\| = 2"):
        top(K=3, among=[4, 4, 7])
    with pytest.raises(ValueError, match="exclude_items: 1 rows for 2 groups"):
        top(exclude_items=[[1]])
    with pytest.raises(ValueError, match="exclude"):
        top(exclude="all")
    with pytest.raises(ValueError, match="outside"):
        top(among=[12])
    with pytest.raises(ValueError, match="single-GPU engines"):
        recommend.prepare_group_top_k(types.SimpleNamespace(nu=100, ni=12), rp, col, [[1]], K=2)   # a sharded engine
    top(K=14, new_items=[[0], [1]])                                                     # new items grow the catalog


def _fake_trainer(masked=False, hot=None):
    from llmrec_b200 import main as M
    tr = types.SimpleNamespace(hot=hot or _bare_engine(), masked_mode=masked, n_users=100, n_items=12, args=types.SimpleNamespace())
    _, rp, col = _train()
    tr.graph = types.SimpleNamespace(rowptr_u=rp, col_u=col)
    tr._current_model = lambda: M.Trainer._current_model(tr)
    return tr


def test_trainer_refuses_the_mask_branch_and_sharded_engines():
    from llmrec_b200 import main as M
    with pytest.raises(ValueError, match="fixed model"):
        M.Trainer.recommend_groups(_fake_trainer(masked=True), [[1, 2]], K=2)
    with pytest.raises(ValueError, match="single-GPU engines"):
        M.Trainer.recommend_groups(_fake_trainer(hot=types.SimpleNamespace(nu=100, ni=12)), [[1, 2]], K=2)
    with pytest.raises(ValueError, match="empty"):                                     # the arguments before the model
        M.Trainer.recommend_groups(_fake_trainer(masked=True), [[]], K=2)


def test_flags(tmp_path):
    from llmrec_b200 import main as M
    from llmrec_b200.utility.parser import build_parser, parse_args
    a = parse_args([])
    assert a.groups_in is None and a.groups_out is None and a.groups_k == 10 and a.groups_agg == "mean"
    a = parse_args(["--groups_in", "F", "--groups_out", "G", "--groups_k", "5", "--groups_agg", "min"])
    assert (a.groups_in, a.groups_out, a.groups_k, a.groups_agg) == ("F", "G", 5, "min")
    assert "--groups_in" in build_parser().format_help()
    with pytest.raises(SystemExit):
        parse_args(["--groups_agg", "median"])
    F, G = str(tmp_path / "F"), str(tmp_path / "G")
    args = lambda **kw: types.SimpleNamespace(**{**dict(groups_in=None, groups_out=None, groups_k=10, groups_agg="mean"), **kw})
    tr = _fake_trainer()
    assert M.check_groups_flags(args(), tr) is None
    for kw in (dict(groups_in=F), dict(groups_out=G)):
        with pytest.raises(ValueError, match="go together"):
            M.check_groups_flags(args(**kw), tr)
    with pytest.raises(ValueError, match="cannot read"):
        M.check_groups_flags(args(groups_in=F, groups_out=G), tr)
    pickle.dump([[3, 1, 1], [7], np.array([2, 9])], open(F, "wb"))
    rp, col = M.check_groups_flags(args(groups_in=F, groups_out=G), tr)
    assert _rows(rp, col) == [[1, 3], [7], [2, 9]]
    with pytest.raises(ValueError, match="fixed model"):
        M.check_groups_flags(args(groups_in=F, groups_out=G), _fake_trainer(masked=True))
    for K in (0, 13):
        with pytest.raises(ValueError, match="K = "):
            M.check_groups_flags(args(groups_in=F, groups_out=G, groups_k=K), tr)
    with pytest.raises(ValueError, match="agg"):
        M.check_groups_flags(args(groups_in=F, groups_out=G, groups_agg="median"), tr)
    for bad, msg in (([[1], []], "empty"), ([[100]], "outside"), ([list(range(65))], "65 distinct"), ({1: 2}, "list"),
                     (([0, 1], [1]), "list"), ([[0.5]], "integers")):
        pickle.dump(bad, open(F, "wb"))
        with pytest.raises(ValueError, match=msg):
            M.check_groups_flags(args(groups_in=F, groups_out=G), tr)


def test_groups_out_file(tmp_path):
    from llmrec_b200 import main as M
    G = str(tmp_path / "sub" / "G")
    calls = []
    ids = torch.tensor([[4, 2, -1], [0, 1, 3]], dtype=torch.int64)
    tr = types.SimpleNamespace(recommend_groups=lambda groups, **kw: calls.append((groups, kw)) or (ids, None))
    assert M.Trainer.write_groups(tr, G, [[1, 2], [3]], K=3, agg="max") == G
    assert calls == [([[1, 2], [3]], dict(K=3, agg="max", exclude="train"))]
    got = pickle.load(open(G, "rb"))
    assert isinstance(got, torch.Tensor) and got.dtype == torch.int64 and got.device.type == "cpu" and torch.equal(got, ids)
    assert not os.path.exists(G + ".tmp")


def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    ops_emulator.install()
    import group_model as GM
    from llmrec_b200 import ops, recommend
    ops.score_topk = GM.score_topk_standin
    ops.score_topk_group = GM.score_topk_group_standin
    from llmrec_b200.engine import HotPath, HotPathConfig, PARAM_ORDER
    from llmrec_b200.graph import BipartiteGraph
    from oracle import llmrec_oracle as O
    data = O.load_dataset(ddir)
    O.set_seed(2022)
    otr = O.OracleTrainer(data, O.OracleConfig(batch_size=128))
    params = {k: otr.params[k].detach().clone() for k in PARAM_ORDER}
    feats = dict(image=otr.feats["image"].clone(), text=otr.feats["text"].clone(), user=otr.feats["user"].clone(),
                 item={k: v.clone() for k, v in otr.feats["item"].items()})
    g = BipartiteGraph(data.train_mat, "cpu")
    hp = HotPath((g.ui, g.iu, g.uiT, g.iuT), params, feats, HotPathConfig(batch_size=128))
    U, I = hp.forward()
    rp, col = g.rowptr_u, g.col_u
    res = {}
    rng = np.random.default_rng(3)
    groups = [sorted(rng.choice(hp.nu, int(s), replace=False).tolist()) for s in rng.integers(1, 8, 40)]
    S = GM.member_scores(U, I, np.arange(hp.nu)).numpy()
    for agg in ("mean", "min", "max"):
        ids, vals = recommend.top_k_groups(hp, rp, col, groups, K=10, agg=agg)
        ok = True
        for b, grp in enumerate(groups):                                                  # the host restatement
            masked = np.unique(np.concatenate([col[rp[u]:rp[u + 1]].numpy() for u in grp]))
            cand = np.setdiff1d(np.arange(hp.ni), masked)
            want_i, want_v = GM.rank(GM.aggregate(S[grp][:, cand], agg), cand, 10)
            ok &= ids[b].tolist() == want_i.tolist() and np.array_equal(vals[b].numpy().view(np.int32), want_v.view(np.int32))
        res[f"restatement_{agg}"] = ok
        # repeats and member order do not change a row
        shuffled = [list(reversed(grp)) + grp[:1] for grp in groups]
        ids2, vals2 = recommend.top_k_groups(hp, rp, col, shuffled, K=10, agg=agg)
        res[f"canonical_{agg}"] = bool(torch.equal(ids, ids2)) and bool(torch.equal(vals, vals2))
        # singletons are `top_k`
        users = list(range(0, hp.nu, 7))
        a = recommend.top_k_groups(hp, rp, col, [[u] for u in users], K=10, agg=agg)
        b = recommend.top_k(hp, rp, col, users=users, K=10)
        res[f"singleton_{agg}"] = bool(torch.equal(a[0], b[0])) and bool(torch.equal(a[1].view(torch.int32), b[1].view(torch.int32)))
    # among, exclude_items and new items naming a member
    among = rng.choice(hp.ni, 60, replace=False)
    extra = [rng.integers(0, hp.ni, 5).tolist() for _ in groups]
    ids, _ = recommend.top_k_groups(hp, rp, col, groups, K=10, agg="min", among=among, exclude_items=extra)
    ok = True
    for b, grp in enumerate(groups):
        masked = np.union1d(np.concatenate([col[rp[u]:rp[u + 1]].numpy() for u in grp]), extra[b])
        cand = np.setdiff1d(np.sort(among), masked)
        ok &= ids[b].tolist() == GM.rank(GM.aggregate(S[grp][:, cand], "min"), cand, 10)[0].tolist()
    res["among_exclude_items"] = ok
    out[0] = res


def test_top_k_groups_on_the_stand_ins(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    res = dict(out)[0]
    assert all(res.values()), {k: v for k, v in res.items() if not v}
