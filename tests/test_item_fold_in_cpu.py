"""Items added after training, without a GPU: the CSR of user lists, the grown mask CSR, and on the kernel stand-ins
(tests/ops_emulator.py, installed in a child process, plus a stand-in for llmrec_row_normalize_f32 defined here) the one item fold-in
launch and its segments, layer 0, top-K over the grown catalog and item-to-item neighbours."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def test_user_lists_collapse_repeats_sort_rows_and_reject_bad_user_ids():
    from llmrec_b200.recommend import new_items_csr
    R = new_items_csr([[4, 0, 4, 2], [], [1, 1]], 5)
    assert R.shape == (3, 5) and R.indptr.tolist() == [0, 3, 3, 4] and R.indices.tolist() == [0, 2, 4, 1] and np.all(R.data == 1)
    same = new_items_csr((torch.tensor([0, 4, 4, 6]), np.array([4, 0, 4, 2, 1, 1])), 5)
    assert (same != R).nnz == 0
    assert (new_items_csr(R, 5) != R).nnz == 0 and new_items_csr(None, 5) is None
    for bad in ([[0, 5]], [[-1]]):
        with pytest.raises(ValueError, match="new_items: user id"):
            new_items_csr(bad, 5)
    with pytest.raises(ValueError, match="new_items: rowptr"):
        new_items_csr((np.array([0, 3]), np.array([1, 2])), 5)


def test_grown_mask_csr():
    from llmrec_b200.recommend import append_rows, select_rows
    i32 = lambda a: torch.tensor(a, dtype=torch.int32)
    # the new items' transpose: row u = the new items naming user u
    nrp, ncol = i32([0, 2, 2, 3, 5]), i32([0, 3, 1, 0, 2])
    rp, col = select_rows(nrp, ncol, torch.tensor([3, -1, 0, 3, 1]))
    assert rp.dtype == col.dtype == torch.int32
    assert rp.tolist() == [0, 2, 2, 4, 6, 6] and col.tolist() == [0, 2, 0, 3, 0, 2]
    rp, col = select_rows(nrp, ncol, torch.tensor([], dtype=torch.long))
    assert rp.tolist() == [0] and col.numel() == 0
    # training rows (4 users over 10 items) followed by the new items at ids 10 + j: every row stays sorted
    trp, tcol = i32([0, 3, 3, 4, 6]), i32([1, 5, 9, 0, 2, 7])
    rp, col = append_rows(trp, tcol, nrp, ncol, 10)
    assert rp.tolist() == [0, 5, 5, 7, 11]
    rows = [col[rp[u]:rp[u + 1]].tolist() for u in range(4)]
    assert rows == [[1, 5, 9, 10, 13], [], [0, 11], [2, 7, 10, 12]]
    rp, col = append_rows(trp, tcol, torch.zeros(5, dtype=torch.int32), i32([]), 10)
    assert torch.equal(rp, trp) and torch.equal(col, tcol)


def _row_normalize(X, out=None):                                     # llmrec_row_normalize_f32
    y = X / X.norm(dim=1, keepdim=True).clamp_min(1e-12)
    if out is None:
        return y
    out.copy_(y)
    return out


def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    ops_emulator.install()
    from llmrec_b200 import ops, recommend
    ops.row_normalize = _row_normalize
    from llmrec_b200.engine import HotPath, HotPathConfig, PARAM_ORDER
    from llmrec_b200.graph import BipartiteGraph
    from llmrec_b200.hoist import HoistedHotPath
    from oracle import llmrec_oracle as O
    data = O.load_dataset(ddir)
    res = {}
    for hoisted in (False, True):
        O.set_seed(2022)
        otr = O.OracleTrainer(data, O.OracleConfig(batch_size=128))
        params = {k: otr.params[k].detach().clone() for k in PARAM_ORDER}
        feats = dict(image=otr.feats["image"].clone(), text=otr.feats["text"].clone(), user=otr.feats["user"].clone(),
                     item={k: v.clone() for k, v in otr.feats["item"].items()})
        g = BipartiteGraph(data.train_mat, "cpu")
        cfg = HotPathConfig(batch_size=128)
        hp = HoistedHotPath((g.ui, g.iu, g.uiT, g.iuT), params, feats, cfg, g.ones_propagated()) if hoisted else \
            HotPath((g.ui, g.iu, g.uiT, g.iuT), params, feats, cfg)
        U, I = hp.forward()
        ni, nu, L, d = hp.ni, hp.nu, hp.L, hp.d
        if hoisted:
            hp.P_usr.fill_(float("nan"))                              # the hoisted forward never writes P_usr: item fold-in projects it
        # the one launch: its segments, in order
        seen = []
        real = ops.CsrOperator.apply
        ops.CsrOperator.apply = lambda self, segs, src_mask=None: (seen.append((self.n_rows, self.n_cols, [(X.data_ptr(), Y.shape, sm) for X, Y, _, sm in segs])), real(self, segs))[1]
        try:
            rp, col = g.rowptr_i, g.col_i
            If = hp.fold_in_items(rp, col, known=torch.arange(ni))
        finally:
            ops.CsrOperator.apply = real
        want = [hp.blk(hp.Fu, s).data_ptr() for s in range(hp.S)] + [hp.P_usr.data_ptr()] + [hp.Ul[l].data_ptr() for l in range(1, L + 1)]
        res[hoisted, "one launch"] = len(seen) == 1 and seen[0][:2] == (ni, nu) and [s[0] for s in seen[0][2]] == want and \
            [s[2] for s in seen[0][2]] == [False] * (hp.S + L) + [True] and all(s[1] == (ni, d) for s in seen[0][2])
        p = hp.p
        res[hoisted, "P_usr"] = bool(torch.allclose(hp.P_usr, feats["user"] @ p["user_trans.weight"].t() + p["user_trans.bias"], rtol=1e-5, atol=1e-6))
        tol = 2e-4 if hoisted else 1e-5                               # the hoisted engine's Fi is (iu.ui.X)W^T + ci b, reassociated
        res[hoisted, "trained items"] = bool(torch.allclose(If, I, rtol=tol, atol=tol * 1e-2))
        # layer 0: E_i[known] for a trained item, a zero row for a new one; everything else equal
        Iz = hp.fold_in_items(rp, col)
        res[hoisted, "layer 0"] = bool(torch.allclose(If - Iz, hp.E_i / (L + 1), rtol=1e-4, atol=1e-7))
        Ie = hp.fold_in_items(torch.tensor([0, 0]), torch.zeros(0, dtype=torch.int64))
        res[hoisted, "empty"] = bool(torch.allclose(Ie, torch.full((1, d), 1.0 / d / (L + 1)), rtol=1e-6, atol=0))
        with_rep = hp.fold_in_items(torch.tensor([0, 5]), torch.tensor([3, 3, 8, 3, 8]))
        res[hoisted, "repeats collapse"] = bool(torch.equal(with_rep, hp.fold_in_items(torch.tensor([0, 2]), torch.tensor([3, 8]))))
        # top-K over the grown catalog: three new items; trained users exclude their training rows and the new items naming them
        lists = [[0, 5], [5], [7, 0, 9]]
        urp, ucol = g.rowptr_u, g.col_u
        users = [0, 5, 7, 9, 11]
        ids, vals = recommend.top_k(hp, urp, ucol, users=users, K=20, new_items=lists)
        cat = torch.cat([I, hp.fold_in_items(torch.tensor([0, 2, 3, 6]), torch.tensor([0, 5, 5, 7, 0, 9]))])
        ok = tuple(ids.shape) == (5, 20) and ids.dtype == torch.int64
        for b, u in enumerate(users):
            masked = set(ucol[urp[u]:urp[u + 1]].tolist()) | {ni + j for j, l in enumerate(lists) if u in l}
            S = (U[u] @ cat.t()).clone()
            S[list(masked)] = float("-inf")
            ok &= not set(ids[b].tolist()) & masked
            ok &= ids[b].tolist() == torch.sort(S, descending=True, stable=True)[1][:20].tolist()
        n_ids, _ = recommend.top_k(hp, urp, ucol, users=[0], K=64, exclude="none", new_items=lists)
        ok &= n_ids[0].tolist() == torch.sort(U[0] @ cat.t(), descending=True, stable=True)[1][:64].tolist()
        # folded-in histories: the history and the new items naming its trained id are masked
        hist = [[1, 2, 3], [4], []]
        fid, _ = recommend.top_k(hp, urp, ucol, users=[5, -1, 0], K=30, histories=hist, new_items=lists)
        for b, (h, k) in enumerate(zip(hist, [5, -1, 0])):
            masked = set(h) | {ni + j for j, l in enumerate(lists) if k in l}
            ok &= not set(fid[b].tolist()) & masked
        res[hoisted, "grown top-k"] = bool(ok)
        # neighbours: cosine over the grown catalog, never the query itself
        q = [0, 3, ni, ni + 2]
        sid, sval = recommend.similar_items(hp, q, K=15, new_items=lists)
        Xn = cat / cat.norm(dim=1, keepdim=True)
        ok = tuple(sid.shape) == (4, 15)
        for b, i in enumerate(q):
            S = (Xn[i] @ Xn.t()).clone()
            S[i] = float("-inf")
            ok &= i not in sid[b].tolist() and sid[b].tolist() == torch.sort(S, descending=True, stable=True)[1][:15].tolist()
            ok &= bool(torch.allclose(sval[b], S[sid[b]], rtol=1e-5, atol=1e-6))
        res[hoisted, "similar"] = bool(ok)
    out[0] = res


def test_item_fold_in_on_the_stand_ins(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    res = dict(out)[0]
    assert all(res.values()), {k: v for k, v in res.items() if not v}


def test_k_limits_of_neighbours():
    from llmrec_b200 import recommend
    assert recommend.check_k(4, 4, "the catalog size - 1") == 4
    with pytest.raises(ValueError, match="at most the catalog size - 1 = 4"):
        recommend.check_k(5, 4, "the catalog size - 1")
