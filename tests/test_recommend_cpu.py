"""Recommendations without a GPU: the history CSRs, the one fold-in launch and its layer 0 on the kernel stand-ins
(tests/ops_emulator.py, installed in a child process), the --candidates_out / --candidates_k flags and the candidate file."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


def test_history_csr_collapses_repeats_sorts_rows_and_rejects_bad_ids():
    from llmrec_b200.graph import histories_csr, history_matrix, inv_sqrt_degree
    R = histories_csr([[5, 1, 5, 5, 0], [], [3, 3]], 6)
    assert R.shape == (3, 6) and R.indptr.tolist() == [0, 3, 3, 4] and R.indices.tolist() == [0, 1, 5, 3] and np.all(R.data == 1)
    same = histories_csr((np.array([0, 5, 5, 7]), torch.tensor([5, 1, 5, 5, 0, 3, 3])), 6)
    assert (same != R).nnz == 0 and same.indptr.tolist() == R.indptr.tolist()
    s = inv_sqrt_degree(R)                                          # the distinct items count, as su does for R
    assert s[0] == np.power(3 + 1e-8, -0.5) and s[1] == np.power(1e-8, -0.5) and s[2] == 1 / np.sqrt(1 + 1e-8)
    for bad in ([[0, 6]], [[-1]]):
        with pytest.raises(ValueError, match="outside"):
            histories_csr(bad, 6)
    with pytest.raises(ValueError, match="rowptr"):
        history_matrix([0, 3], [1, 2], 6)
    assert histories_csr([], 6).shape == (0, 6)


def test_flags():
    from llmrec_b200.utility.parser import build_parser, parse_args
    a = parse_args([])
    assert a.candidates_out is None and a.candidates_k == 10
    a = parse_args(["--candidates_out", "x/candidate_indices", "--candidates_k", "20"])
    assert a.candidates_out == "x/candidate_indices" and a.candidates_k == 20
    text = build_parser().format_help()
    assert "--candidates_out" in text and "--candidates_k" in text


def test_k_limits():
    from llmrec_b200 import recommend
    assert recommend.check_k(64, 100) == 64 and recommend.check_k(5, 5) == 5
    for K, n in ((0, 100), (65, 100), (11, 10), (True, 10), (2.0, 10)):
        with pytest.raises(ValueError, match="K = "):
            recommend.check_k(K, n)
    with pytest.raises(ValueError, match="single-GPU"):
        recommend.check_engine(object())


def test_candidate_file_is_the_pickled_int64_tensor_and_written_atomically(tmp_path):
    from llmrec_b200 import recommend
    path = str(tmp_path / "data" / "candidate_indices")
    ids = torch.tensor([[3, 1, 2], [0, 2, -1]], dtype=torch.int32)
    assert recommend.write_candidates(path, ids) == path
    got = pickle.load(open(path, "rb"))                             # how the augmentation stage reads it
    assert isinstance(got, torch.Tensor) and got.dtype == torch.int64 and got.device.type == "cpu" and torch.equal(got, ids.long())
    assert sorted(os.listdir(tmp_path / "data")) == ["candidate_indices"]

    class Boom:                                                     # a failed write keeps the previous file and leaves no .tmp
        def __reduce__(self):
            raise RuntimeError("boom")

    real = pickle.dump
    try:
        pickle.dump = lambda obj, f: real(Boom(), f)
        with pytest.raises(RuntimeError, match="boom"):
            recommend.write_candidates(path, ids + 1)
    finally:
        pickle.dump = real
    assert torch.equal(pickle.load(open(path, "rb")), ids.long()) and sorted(os.listdir(tmp_path / "data")) == ["candidate_indices"]


def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    ops_emulator.install()
    from llmrec_b200 import ops, recommend
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
        nu, L, d = hp.nu, hp.L, hp.d
        # the one launch: its segments, in order
        seen = []
        real = ops.CsrOperator.apply
        ops.CsrOperator.apply = lambda self, segs, src_mask=None: (seen.append((self.n_rows, [(X.data_ptr(), Y.shape, sm) for X, Y, _, sm in segs])), real(self, segs))[1]
        try:
            rp, col = g.rowptr_u, g.col_u
            Uf = hp.fold_in(rp, col, known=torch.arange(nu))
        finally:
            ops.CsrOperator.apply = real
        want = [hp.blk(hp.Pi, s).data_ptr() for s in range(hp.S)] + [hp.prof_i.data_ptr()] + [hp.Il[l].data_ptr() for l in range(L)]
        res[hoisted, "one launch"] = len(seen) == 1 and seen[0][0] == nu and [s[0] for s in seen[0][1]] == want and \
            [s[2] for s in seen[0][1]] == [False] * (hp.S + L) + [True]
        tol = 2e-4 if hoisted else 1e-5                               # the hoisted engine's Fu is (ui.X)W^T + cu b, reassociated
        res[hoisted, "training rows"] = bool(torch.allclose(Uf, U, rtol=tol, atol=tol * 1e-2))
        # layer 0: E_u[known] for a trained user, a zero row for an unknown one; everything else equal
        Uz = hp.fold_in(rp, col)
        res[hoisted, "layer 0"] = bool(torch.allclose(Uf - Uz, hp.E_u / (L + 1), rtol=1e-4, atol=1e-7))
        # an empty history: every layer 1..L-1 and every side term 0, the last layer softmax(0) = 1/d
        Ue = hp.fold_in(torch.tensor([0, 0]), torch.zeros(0, dtype=torch.int64))
        res[hoisted, "empty"] = bool(torch.allclose(Ue, torch.full((1, d), 1.0 / d / (L + 1)), rtol=1e-6, atol=0))
        # top-K on the stand-in scorer: trained users with their training rows masked, and the same rows folded in
        ids, vals = recommend.top_k(hp, rp, col, users=[0, 5, 7], K=10)
        hist = [col[rp[u]:rp[u + 1]].tolist() for u in (0, 5, 7)]
        fid, fvals = recommend.top_k(hp, rp, col, users=[0, 5, 7], K=10, histories=hist)
        ok = ids.dtype == torch.int64 and vals.dtype == torch.float32 and tuple(ids.shape) == (3, 10)
        for b, u in enumerate((0, 5, 7)):
            ok &= not set(ids[b].tolist()) & set(hist[b]) and not set(fid[b].tolist()) & set(hist[b])
        n_ids, _ = recommend.top_k(hp, rp, col, users=[0], K=10, exclude="none")
        s = (U[0:1] @ I.t())[0]
        ok &= n_ids[0].tolist() == torch.sort(s, descending=True, stable=True)[1][:10].tolist()
        res[hoisted, "top-k"] = bool(ok)
    out[0] = res


def test_fold_in_on_the_stand_ins(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    res = dict(out)[0]
    assert all(res.values()), {k: v for k, v in res.items() if not v}
