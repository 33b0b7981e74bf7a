"""Pair scores and re-ranking without a GPU: candidate parsing in its three forms, padding and the validation messages, the shared
exclusion mask against the masks `top_k` built before it was shared, the --rerank_in / --rerank_out / --rerank_k flags, and the
--rerank_out file of `Trainer.rerank` on kernel stand-ins (tests/ops_emulator.py plus the two below, in a child process)."""
import os
import pickle
import sys
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def score_pairs_standin(U, I, qrow, item):                      # llmrec_score_pairs_f32
    return (U[qrow.long()] * I[item.long()]).sum(1)


def rerank_standin(U, I, qrow, rp, col, mask_rowptr, mask_col, K):   # llmrec_rerank_f32
    ids = torch.full((qrow.numel(), K), -1, dtype=torch.int32)
    vals = torch.full((qrow.numel(), K), float("-inf"))
    for r, q in enumerate(qrow.long().tolist()):
        c = col[rp[r]:rp[r + 1]].long()
        c = torch.unique(c[(c >= 0) & (c < I.shape[0])])
        if mask_rowptr is not None:
            c = c[~torch.isin(c, mask_col[mask_rowptr[q]:mask_rowptr[q + 1]].long())]
        s = (U[q] * I[c]).sum(1)
        key = np.lexsort((c.numpy(), -s.double().numpy()))[:K]
        ids[r, :key.size] = c[key].to(torch.int32)
        vals[r, :key.size] = s[key]
    return ids, vals


def test_candidates_in_three_forms_and_padding():
    from llmrec_b200 import recommend
    want_rp, want_col = [0, 3, 3, 5], [4, -1, 2, 0, 0]
    for cand in ([[4, -1, 2], [], [0, 0]], [np.array([4, -1, 2]), (), torch.tensor([0, 0])],
                 (np.array(want_rp), torch.tensor(want_col, dtype=torch.int32))):
        rp, col = recommend.candidates_csr(cand, 5)
        assert rp.tolist() == want_rp and col.tolist() == want_col and rp.dtype == col.dtype == torch.int64
    for dense in (np.array([[3, 1, -1], [0, 0, 4]]), torch.tensor([[3, 1, -1], [0, 0, 4]], dtype=torch.int32)):
        rp, col = recommend.candidates_csr(dense, 5)
        assert rp.tolist() == [0, 3, 6] and col.tolist() == [3, 1, -1, 0, 0, 4]
    rp, col = recommend.candidates_csr(np.zeros((0, 4), dtype=np.int64), 5)
    assert rp.tolist() == [0] and col.numel() == 0


def test_candidate_validation_messages():
    from llmrec_b200 import recommend
    for bad, msg in (([[0, 5]], "item id 5 is outside \\[0, 5\\) \\(-1 = padding\\)"), ([[-2]], "item id -2 is outside"),
                     ([[1.5]], "must be integers"), (np.zeros((2, 2)), "must be integers"), (torch.ones(2, 2, dtype=torch.bool), "must be integers"),
                     (np.zeros(3, dtype=np.int64), "2-D"), ((np.array([0, 2]), np.array([1])), "rowptr"),
                     ((np.array([1, 1]), np.array([1])), "rowptr"), ((np.array([0, 2, 1]), np.array([1])), "rowptr")):
        with pytest.raises(ValueError, match=msg):
            recommend.candidates_csr(bad, 5)
    assert recommend.check_rerank_k(None) is None and recommend.check_rerank_k(1024) == 1024 and recommend.check_rerank_k(np.int64(3)) == 3
    for K in (0, 1025, 2.0, True, "3"):
        with pytest.raises(ValueError, match="1..1024"):
            recommend.check_rerank_k(K)
    u, i = recommend.check_pairs([0, 2], torch.tensor([4, 1]), 3, 5)
    assert u.tolist() == [0, 2] and i.tolist() == [4, 1]
    for users, items, msg in (([0], [1, 2], "one pair"), ([3], [0], "user id 3 is outside \\[0, 3\\)"), ([0], [-1], "item id -1"),
                              ([0.0], [1], "integers")):
        with pytest.raises(ValueError, match=msg):
            recommend.check_pairs(users, items, 3, 5)


def test_query_blocks_bound_the_candidates_per_launch():
    from llmrec_b200 import recommend
    rp = torch.tensor([0, 3, 3, 10, 11, 20, 21])
    blocks = list(recommend._blocks(rp, 5))
    assert blocks[0][0] == 0 and blocks[-1][1] == 6 and all(a[1] == b[0] for a, b in zip(blocks, blocks[1:]))
    for s, e in blocks:
        assert e > s and (int(rp[e] - rp[s]) <= 5 or e == s + 1)
    assert list(recommend._blocks(torch.tensor([0]), 5)) == []


def _old_top_k_mask(ni, rp, col, exclude, Rn, users, histories_csr_m):
    """the mask construction of recommend.top_k before it moved into exclusion_mask (kept here as the yardstick)"""
    from llmrec_b200.recommend import _i32, append_rows, select_rows
    dev = col.device
    if exclude == "none":
        return torch.zeros(rp.numel(), dtype=torch.int32, device=dev), col[:0]
    if Rn is not None and Rn.nnz:
        Rt = sp.csr_matrix(Rn.T)
        Rt.sort_indices()
        nrp, ncol = _i32(Rt.indptr, dev), _i32(Rt.indices, dev)
        if histories_csr_m is not None:
            m = histories_csr_m
            kn = np.full(m, -1) if users is None else np.asarray(users)
            nrp, ncol = select_rows(nrp, ncol, torch.from_numpy(kn.astype(np.int64).reshape(-1)))
        rp, col = append_rows(rp, col, nrp, ncol, ni)
    return rp, col


def test_exclusion_mask_is_the_old_top_k_mask():
    from llmrec_b200 import recommend
    from llmrec_b200.graph import histories_csr
    g = np.random.default_rng(0)
    nu, ni = 30, 50
    train = histories_csr([g.integers(0, ni, int(g.integers(0, 9))).tolist() for _ in range(nu)], ni)
    trp, tcol = recommend._i32(train.indptr, "cpu"), recommend._i32(train.indices, "cpu")
    eng = types.SimpleNamespace(ni=ni)
    hist = histories_csr([g.integers(0, ni, 5).tolist() for _ in range(7)], ni)
    hrp, hcol = recommend._i32(hist.indptr, "cpu"), recommend._i32(hist.indices, "cpu")
    for new_items in (None, [[]], [[1, 2, 29], [], list(range(0, nu, 4))]):
        Rn = recommend.new_items_csr(new_items, nu)
        for exclude in ("train", "none"):
            got = recommend.exclusion_mask(eng, trp, tcol, exclude, Rn)
            want = _old_top_k_mask(ni, trp, tcol, exclude, Rn, None, None)
            assert all(torch.equal(a, b) for a, b in zip(got, want))
            for users in (None, [2, -1, 29, 0, 0, 5, -1]):
                kn = np.full(7, -1) if users is None else np.asarray(users)
                got = recommend.exclusion_mask(eng, hrp, hcol, exclude, Rn, kn.astype(np.int64))
                want = _old_top_k_mask(ni, hrp, hcol, exclude, Rn, users, 7)
                assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_flags(tmp_path):
    from llmrec_b200 import main as M
    from llmrec_b200.engine import HotPath
    from llmrec_b200.utility.parser import build_parser, parse_args
    a = parse_args([])
    assert a.rerank_in is None and a.rerank_out is None and a.rerank_k is None
    a = parse_args(["--rerank_in", "F", "--rerank_out", "G", "--rerank_k", "20"])
    assert (a.rerank_in, a.rerank_out, a.rerank_k) == ("F", "G", 20)
    text = build_parser().format_help()
    assert "--rerank_in" in text and "--rerank_out" in text and "--rerank_k" in text
    tr = types.SimpleNamespace(masked_mode=False, hot=HotPath.__new__(HotPath), n_users=3, n_items=10)
    F = str(tmp_path / "F")
    pickle.dump(torch.tensor([[1, 2], [3, -1], [9, 9]]), open(F, "wb"))
    args = lambda **kw: types.SimpleNamespace(**{**dict(rerank_in=None, rerank_out=None, rerank_k=None), **kw})
    assert M.check_rerank_flags(args(), tr) == (None, None)
    cand, K = M.check_rerank_flags(args(rerank_in=F, rerank_out="G"), tr)
    assert K == 2 and torch.equal(torch.as_tensor(cand), torch.tensor([[1, 2], [3, -1], [9, 9]]))
    assert M.check_rerank_flags(args(rerank_in=F, rerank_out="G", rerank_k=5), tr)[1] == 5
    with pytest.raises(ValueError, match="go together"):
        M.check_rerank_flags(args(rerank_in=F), tr)
    with pytest.raises(ValueError, match="1..1024"):
        M.check_rerank_flags(args(rerank_in=F, rerank_out="G", rerank_k=0), tr)
    with pytest.raises(ValueError, match="fixed model"):
        M.check_rerank_flags(args(rerank_in=F, rerank_out="G"), types.SimpleNamespace(**{**vars(tr), "masked_mode": True}))
    with pytest.raises(ValueError, match="single-GPU"):
        M.check_rerank_flags(args(rerank_in=F, rerank_out="G"), types.SimpleNamespace(**{**vars(tr), "hot": object()}))
    with pytest.raises(ValueError, match="cannot read"):
        M.check_rerank_flags(args(rerank_in=str(tmp_path / "missing"), rerank_out="G"), tr)
    for bad, msg in ((np.zeros((2, 2), dtype=np.int64), "n_users = 3"), (np.zeros(3, dtype=np.int64), "2-D"),
                     (np.full((3, 2), 10), "outside"), ([[1]] * 3, "2-D")):
        pickle.dump(bad, open(F, "wb"))
        with pytest.raises(ValueError, match=msg):
            M.check_rerank_flags(args(rerank_in=F, rerank_out="G"), tr)


def _worker(rank, ddir, out_dir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    ops_emulator.install()
    from llmrec_b200 import ops, recommend
    ops.score_pairs, ops.rerank = score_pairs_standin, rerank_standin
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
    # the candidate_indices round trip: top-10 of every user, re-ranked after a shuffle, written and read back
    cand, _ = recommend.top_k(hp, rp, col, K=10, exclude="none")
    shuffled = cand[:, torch.randperm(10)]
    ids, vals = recommend.rerank(hp, rp, col, shuffled.numpy())
    path = recommend.write_candidates(os.path.join(out_dir, "reranked"), ids)
    back = pickle.load(open(path, "rb"))
    res["round trip"] = bool(torch.equal(back, cand)) and back.dtype == torch.int64 and sorted(os.listdir(out_dir)) == ["reranked"]
    # query blocks: the same lists however the candidates are cut into launches
    recommend.CAND_BLOCK = 7
    again, v2 = recommend.rerank(hp, rp, col, shuffled.numpy())
    res["blocks"] = bool(torch.equal(again, ids) and torch.equal(v2, vals))
    # exclude="train" over every item is the top-K of the same queries
    users = [0, 5, 7, 11]
    every = [list(range(hp.ni))] * len(users)
    r_ids, _ = recommend.rerank(hp, rp, col, every, users=users, K=10, exclude="train")
    t_ids, _ = recommend.top_k(hp, rp, col, users=users, K=10, exclude="train")
    res["top-k"] = bool(torch.equal(r_ids, t_ids))
    # pair scores: the stand-in's U . I
    s = recommend.score_pairs(hp, [0, 3], [5, 9])
    res["pairs"] = bool(torch.allclose(s, torch.stack([U[0] @ I[5], U[3] @ I[9]])))
    out[0] = res


def test_rerank_file_round_trip_on_the_stand_ins(tiny_root, tmp_path):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), str(tmp_path), out), nprocs=1, join=True)
    res = dict(out)[0]
    assert all(res.values()), {k: v for k, v in res.items() if not v}
