"""Restricted catalogs and per-query exclusions without a GPU: the id checks of `among`, the merge of exclusion rows, the rejections of
`top_k` / `similar_items` before anything runs, the --candidates_among flag and file, and `top_k(among=, exclude_items=)` end to end on
kernel stand-ins (tests/ops_emulator.py plus the score_topk_among stand-in below, in a child process)."""
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


def score_topk_among_standin(U, I, users, among, mask_rowptr, mask_col, K, mode=0, want_vals=False):   # llmrec_score_topk_among_f32
    """the catalog I[among]: exact fp32 scores, masked global ids dropped, ties -> lowest id, -1 / -inf past the last survivor"""
    a = among.long()
    S = U[users.long()] @ I[a].t()
    for b, u in enumerate(users.long().tolist()):
        S[b, torch.isin(a, mask_col[mask_rowptr[u]:mask_rowptr[u + 1]].long())] = float("-inf")
    val, pos = torch.sort(S, dim=1, descending=True, stable=True)
    val, idx = val[:, :K], a[pos[:, :K]].to(torch.int32)
    idx = torch.where(torch.isinf(val), torch.full_like(idx, -1), idx)
    return (idx, val) if want_vals else idx


def test_catalog_ids_sort_collapse_and_reject():
    from llmrec_b200 import recommend
    for a in ([5, 1, 5, 0], np.array([5, 1, 5, 0], dtype=np.int16), torch.tensor([[5, 1], [5, 0]])):
        got = recommend.catalog_ids(a, 6, "cpu")
        assert got.dtype == torch.int32 and got.tolist() == [0, 1, 5]
    for bad, msg in (([0, 6], "item id 6 is outside \\[0, 6\\)"), ([-1], "item id -1 is outside"), ([1.0], "integers"),
                     (np.zeros(2, dtype=np.float32), "integers"), (torch.ones(2, dtype=torch.bool), "integers"), ([], "empty"),
                     (torch.zeros(0, dtype=torch.int64), "empty")):
        with pytest.raises(ValueError, match=msg):
            recommend.catalog_ids(bad, 6, "cpu")


def test_merge_rows_is_the_sorted_union():
    from llmrec_b200 import recommend
    g = np.random.default_rng(0)
    n, m = 40, 9
    a = [np.unique(g.integers(0, n, int(g.integers(0, 8)))) for _ in range(m)]
    b = [g.integers(-1, n, int(g.integers(0, 8))) for _ in range(m)]                     # unsorted, repeats, -1 padding
    a_rp = torch.tensor(np.concatenate([[0], np.cumsum([x.size for x in a])]), dtype=torch.int32)
    b_rp = torch.tensor(np.concatenate([[0], np.cumsum([x.size for x in b])]), dtype=torch.int64)
    rp, col = recommend.merge_rows(a_rp, torch.tensor(np.concatenate(a), dtype=torch.int32), b_rp, torch.tensor(np.concatenate(b)), n)
    assert rp.dtype == col.dtype == torch.int32
    for r in range(m):
        want = sorted(set(a[r].tolist()) | {x for x in b[r].tolist() if x >= 0})
        assert col[rp[r]:rp[r + 1]].tolist() == want, r
    rp, col = recommend.merge_rows(torch.zeros(3, dtype=torch.int32), torch.zeros(0, dtype=torch.int32), torch.zeros(3, dtype=torch.int64),
                                   torch.zeros(0, dtype=torch.int64), n)
    assert rp.tolist() == [0, 0, 0] and col.numel() == 0


def _bare_engine(nu=5, ni=12):
    from llmrec_b200.engine import HotPath
    hp = HotPath.__new__(HotPath)
    hp.nu, hp.ni, hp.E_u = nu, ni, torch.zeros(1)
    return hp


def test_rejections_before_anything_runs():
    from llmrec_b200 import recommend
    hp = _bare_engine()
    rp, col = torch.zeros(6, dtype=torch.int32), torch.zeros(0, dtype=torch.int32)
    top = lambda **kw: recommend.prepare_top_k(hp, rp, col, **{"K": 2, **kw})
    for among, msg in (([0, 12], "outside"), ([-3], "outside"), ([0.5], "integers"), ([], "empty")):
        with pytest.raises(ValueError, match=msg):
            top(among=among)
        with pytest.raises(ValueError, match=msg):
            recommend.similar_items(hp, [0], K=1, among=among)
    with pytest.raises(ValueError, match="1..2 .*\\|among\\| = 2"):
        top(K=3, among=[4, 4, 7])
    with pytest.raises(ValueError, match="1..1 "):
        recommend.similar_items(hp, [0], K=2, among=[3])
    top(among=[12, 13], new_items=[[0], [1]])                                           # new ids are catalog ids n_items + j
    with pytest.raises(ValueError, match="outside"):
        top(among=[14], new_items=[[0], [1]])
    with pytest.raises(ValueError, match="exclude_items: 2 rows for 5 users"):
        top(exclude_items=[[1], [2]])
    with pytest.raises(ValueError, match="exclude_items: 1 rows for 2 histories"):
        top(histories=[[1], [2]], exclude_items=[[1]])
    for bad, msg in (([[12]] * 5, "outside"), ([[-2]] * 5, "outside"), ([[0.5]] * 5, "integers")):
        with pytest.raises(ValueError, match=msg):
            top(exclude_items=bad)
    job = top(users=[3, 3], exclude_items=np.array([[1, -1], [2, 5]]), among=[9, 1, 2, 5])
    assert job["per_query"] and job["among"].tolist() == [1, 2, 5, 9]
    assert [job["mask_col"][job["mask_rowptr"][r]:job["mask_rowptr"][r + 1]].tolist() for r in range(2)] == [[1], [2, 5]]


def test_flags(tmp_path):
    from llmrec_b200 import main as M
    from llmrec_b200.utility.parser import build_parser, parse_args
    assert parse_args([]).candidates_among is None
    assert parse_args(["--candidates_out", "F", "--candidates_among", "S"]).candidates_among == "S"
    assert "--candidates_among" in build_parser().format_help()
    args = lambda **kw: types.SimpleNamespace(**{**dict(candidates_out=None, candidates_k=10, candidates_among=None), **kw})
    S = str(tmp_path / "S")
    assert M.check_candidates_flags(args(), 20) is None
    assert M.check_candidates_flags(args(candidates_out="F"), 20) is None
    with pytest.raises(ValueError, match="1..20"):
        M.check_candidates_flags(args(candidates_out="F", candidates_k=21), 20)
    with pytest.raises(ValueError, match="give --candidates_out"):
        M.check_candidates_flags(args(candidates_among=S), 20)
    with pytest.raises(ValueError, match="cannot read"):
        M.check_candidates_flags(args(candidates_out="F", candidates_among=S), 20)
    for good in (torch.tensor([7, 3, 3, 19]), np.array([7, 3, 3, 19]), [7, 3, 3, 19]):
        pickle.dump(good, open(S, "wb"))
        got = M.check_candidates_flags(args(candidates_out="F", candidates_k=3, candidates_among=S), 20)
        assert got.dtype == torch.int64 and got.tolist() == [3, 7, 19]
    with pytest.raises(ValueError, match="1..3 "):
        M.check_candidates_flags(args(candidates_out="F", candidates_k=4, candidates_among=S), 20)
    for bad, msg in ((np.array([[1, 2]]), "1-D"), ([[1, 2], [3]], "1-D"), ({1, 2}, "1-D"), (np.array([1.5]), "integers"),
                     (np.array([20]), "outside"), ([], "empty")):
        pickle.dump(bad, open(S, "wb"))
        with pytest.raises(ValueError, match=msg):
            M.check_candidates_flags(args(candidates_out="F", candidates_among=S), 20)


def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    ops_emulator.install()
    from llmrec_b200 import ops, recommend
    ops.score_topk_among = score_topk_among_standin
    ops.row_normalize = lambda X, out=None: torch.nn.functional.normalize(X, dim=1)          # llmrec_row_normalize_f32
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
    rng = np.random.default_rng(5)
    S = rng.choice(hp.ni, 50, replace=False)
    users = list(range(0, hp.nu, 9))
    # among: the full-catalog call with every id outside S masked
    ids, _ = recommend.top_k(hp, rp, col, users=users, K=10, exclude="train", among=S)
    outside = [list(np.setdiff1d(np.arange(hp.ni), S))] * len(users)
    want, _ = recommend.top_k(hp, rp, col, users=users, K=10, exclude="train", exclude_items=outside)
    res["among"] = bool(torch.equal(ids, want)) and bool(torch.isin(ids[ids >= 0], torch.from_numpy(S)).all())
    # exclude_items: a host lexsort over the full catalog with the merged mask
    extra = [rng.integers(0, hp.ni, 30).tolist() for _ in users]
    ids, _ = recommend.top_k(hp, rp, col, users=users, K=10, exclude="train", exclude_items=extra)
    ok = True
    for b, u in enumerate(users):
        cand = np.setdiff1d(np.arange(hp.ni), np.union1d(col[rp[u]:rp[u + 1]].numpy(), extra[b]))
        s = (U[u] @ I[torch.from_numpy(cand)].t()).numpy()
        ok &= ids[b].tolist() == cand[np.lexsort((cand, -s.astype(np.float64)))[:10]].tolist()
    res["exclude_items"] = ok
    # the default path is the unrestricted call
    a, _ = recommend.top_k(hp, rp, col, users=users, K=10)
    b, _ = recommend.top_k(hp, rp, col, users=users, K=10, among=np.arange(hp.ni))
    res["identity"] = bool(torch.equal(a, b))
    # similar_items: neighbours only from S, never the query
    q = [int(S[0]), int(S[1]), 0, 3]
    ids, _ = recommend.similar_items(hp, q, K=10, among=S)
    res["similar"] = bool(torch.isin(ids[ids >= 0], torch.from_numpy(S)).all()) and not bool((ids == torch.tensor(q)[:, None]).any())
    out[0] = res


def test_top_k_among_on_the_stand_ins(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    res = dict(out)[0]
    assert all(res.values()), {k: v for k, v in res.items() if not v}
