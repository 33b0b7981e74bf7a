"""Explanations without a GPU: the channel names, the `top` check, and -- on kernel stand-ins (tests/ops_emulator.py plus the
llmrec_explain_f32 stand-in below, in a child process) -- the result layout, `Explanation.of`, padding, repeated history ids, the
identity against U . I, the selection, fold-ins, new items and the rejections before any launch."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def explain_standin(own_src, last_src, side_usr, side_src, coefs, id_src, I, qrow, su, hist_rowptr, hist_col, targets, n_layers, top=0):
    """llmrec_explain_f32 in plain torch (fp32, not the kernel's chain order)."""
    m, P = targets.shape
    inv = 1.0 / n_layers
    C = 1 + len(side_usr)
    contrib = torch.zeros(P * int(hist_col.numel()), C)
    own, last = torch.zeros(m, P), torch.zeros(m, P)
    tids = torch.full((m, P, top), -1, dtype=torch.int32) if top else None
    tvals = torch.full((m, P, top), float("-inf")) if top else None
    rp = hist_rowptr.long()
    for b in range(m):
        u, h = int(qrow[b]), hist_col[rp[b]:rp[b + 1]].long()
        w = [c / max(float(x[u].norm()), 1e-12) * float(su[b]) for x, c in zip(side_usr, coefs)]
        for p in range(P):
            i = int(targets[b, p])
            if i < 0 or i >= I.shape[0]:
                if top:
                    tvals[b, p] = 0
                continue
            own[b, p], last[b, p] = own_src[u] @ I[i] * inv, last_src[u] @ I[i] * inv
            blk = torch.zeros(h.numel(), C)
            for X in id_src:
                blk[:, 0] += X[h] @ I[i] * float(su[b]) * inv
            for t, X in enumerate(side_src):
                blk[:, 1 + t] = X[h] @ I[i] * w[t]
            contrib[P * rp[b] + p * h.numel():P * rp[b] + (p + 1) * h.numel()] = blk
            if top:
                tot = blk.sum(1)
                o = np.lexsort((h.numpy(), -tot.double().numpy()))[:top]
                tids[b, p, :o.size] = h[o].to(torch.int32)
                tvals[b, p, :o.size] = tot[o]
    explain_standin.calls += 1
    return contrib, own, last, tids, tvals


explain_standin.calls = 0


def test_channels_and_top():
    from llmrec_b200 import recommend
    assert recommend.channels(types.SimpleNamespace(has_feats=True, keys=["a", "b"])) == ["id", "image", "text", "profile", "a", "b"]
    assert recommend.channels(types.SimpleNamespace(has_feats=False, keys=[])) == ["id"]
    assert recommend.check_top(None) is None and recommend.check_top(64) == 64 and recommend.check_top(np.int32(1)) == 1
    for top in (0, 65, 2.0, True, "3"):
        with pytest.raises(ValueError, match="1..64"):
            recommend.check_top(top)


def test_explanation_of():
    from llmrec_b200 import recommend
    rp = torch.tensor([0, 2, 2, 5])
    hist = torch.tensor([4, 7, 1, 2, 3])
    P, C = 3, 2
    contrib = torch.arange(P * 5 * C, dtype=torch.float32).view(P * 5, C)
    own, last = torch.arange(9.0).view(3, P), -torch.arange(9.0).view(3, P)
    res = recommend.Explanation(["id", "x"], rp, hist, contrib, own, last, None, None, torch.zeros(3, P, dtype=torch.int64))
    assert len(res) == 3
    q = res.of(2)
    assert q["hist"].tolist() == [1, 2, 3] and q["contrib"].shape == (P, 3, C) and q["own"].tolist() == [6, 7, 8]
    assert torch.equal(q["contrib"].reshape(-1, C), contrib[P * 2:P * 5]) and q["top_ids"] is None
    assert res.of(1)["contrib"].shape == (P, 0, C)
    with pytest.raises(IndexError):
        res.of(3)


def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    ops_emulator.install()
    from llmrec_b200 import ops, recommend
    ops.explain = explain_standin
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
    ids, _ = recommend.top_k(hp, rp, col, K=10, exclude="train")
    e = recommend.explain(hp, rp, col, ids, top=3)
    nnz, C = int(col.numel()), len(e.channels)
    res["layout"] = (e.contrib.shape == (10 * nnz, C) and e.own.shape == (hp.nu, 10) and e.top_ids.shape == (hp.nu, 10, 3)
                     and torch.equal(e.hist_rowptr, rp.long()) and torch.equal(e.hist, col.long()) and C == 4 + len(hp.keys))
    ok = True
    for u in (0, 5, hp.nu - 1):
        q = e.of(u)
        tot = q["own"] + q["last"] + q["contrib"].sum((1, 2))
        want = U[u] @ I[ids[u]].T
        ok &= bool(torch.allclose(tot, want, rtol=1e-4, atol=1e-5))
        best = torch.sort(q["contrib"].sum(2), dim=1, descending=True, stable=True)[1][:, :3]
        n = best.shape[1]                                                   # fewer history items than `top`: padded with -1
        ok &= bool(torch.equal(q["top_ids"][:, :n], q["hist"][best])) and bool((q["top_ids"][:, n:] == -1).all())
    res["identity"] = ok
    # histories: repeats collapse, an unknown user has own = 0, ragged targets are padded, padding gives zeros
    ni = hp.ni
    lists = [[0, 1, 2]]
    e = recommend.explain(hp, rp, col, [[1, 2, ni], [3]], users=[-1, 4], histories=[[5, 5, 2], [7]], new_items=lists)
    q0, q1 = e.of(0), e.of(1)
    Uf = hp.fold_in(torch.tensor([0, 2, 3]), torch.tensor([5, 2, 7]), known=[-1, 4])
    cat = torch.cat([I, hp.fold_in_items(torch.tensor([0, 3]), torch.tensor(lists[0]))])
    tot0 = q0["own"] + q0["last"] + q0["contrib"].sum((1, 2))
    res["histories"] = (q0["hist"].tolist() == [2, 5] and not q0["own"].any() and q1["targets"].tolist() == [3, -1, -1]
                        and not q1["contrib"][1:].any() and q1["own"][1] == 0
                        and bool(torch.allclose(tot0, Uf[0] @ cat[[1, 2, ni]].T, rtol=1e-4, atol=1e-5)))
    # rejections: nothing reaches the kernel
    calls = explain_standin.calls
    bad = 0
    for kw in (dict(items=[[ni]], users=[0]), dict(items=[[1]], users=[0], top=0), dict(items=[[1]]), dict(items=[[1]], users=[hp.nu]),
               dict(items=[[1]], histories=[[1], [2]]), dict(items=[[1]], histories=[[ni]]), dict(items=[[1.5]], users=[0])):
        try:
            recommend.explain(hp, rp, col, **kw)
        except ValueError:
            bad += 1
    res["rejections"] = bad == 7 and explain_standin.calls == calls
    out[0] = res


def test_layout_and_fold_ins_on_the_stand_ins(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    res = dict(out)[0]
    assert all(res.values()), {k: v for k, v in res.items() if not v}
