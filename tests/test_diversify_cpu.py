"""Diversified recommendations without a GPU: the checks of `diversity` and `pool`, their defaults, the --candidates_diversity /
--candidates_pool flags, rejections before anything runs, the selection rule of the host restatement (tests/diversify_model.mmr_select),
and a diversified candidate file end to end on kernel stand-ins (tests/ops_emulator.py and tests/diversify_model.diversify, in a child
process)."""
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
from diversify_model import mmr_select  # noqa: E402


def test_check_diversity_and_pool():
    from llmrec_b200 import recommend
    assert recommend.check_diversity(None) is None
    for good in (0, 1, 0.5, np.float32(0.7), np.int64(1)):
        assert recommend.check_diversity(good) == float(good)
    for bad in (float("nan"), -0.01, 1.01, -1, 2, "0.5", True, np.bool_(False), [0.5], torch.tensor(0.5)):
        with pytest.raises(ValueError, match="diversity = "):
            recommend.check_diversity(bad)
    assert recommend.check_pool(10, 10, 64, "") == 10 and recommend.check_pool(np.int32(64), 1, 64, "") == 64
    for bad in (9, 65, 10.0, True, "20"):
        with pytest.raises(ValueError, match=f"pool = .*P in 10..64"):
            recommend.check_pool(bad, 10, 64, "")


def test_selection_rule():
    # four items: 0 and 1 are the same direction, 2 is orthogonal to both, 3 is between
    X = np.array([[1, 0], [1, 0], [0, 1], [0.6, 0.8]], dtype=np.float32)
    G = X @ X.T
    ids, s = np.array([0, 1, 2, 3]), np.array([4, 3, 1, 2], dtype=np.float32)
    assert mmr_select(ids, s, G, 4, 1.0)[0].tolist() == [0, 1, 3, 2]                  # lambda = 1: by score
    i, v, c = mmr_select(ids, s, G, 4, 0.0)                                            # lambda = 0: least similar first, ties to the id
    assert i.tolist() == [0, 2, 3, 1] and v.tolist() == [4, 1, 2, 3]
    assert c[0] == -np.inf and c[1] == 0 and c[2] == np.float32(0.8) and c[3] == 1
    # padding anywhere, a repeated id picked once, fewer than K left: -1 / -inf / -inf
    i, v, c = mmr_select(np.array([-1, 2, 2, -1, 0]), np.array([9, 1, 5, 9, 0], dtype=np.float32), G[[0, 2, 2, 0, 0]][:, [0, 2, 2, 0, 0]], 4,
                         0.5)
    assert i.tolist() == [2, 0, -1, -1] and v.tolist()[:2] == [5, 0] and np.isneginf(v[2:]).all() and np.isneginf(c[2:]).all()
    # a NaN score ranks last; a repeated id retires with its pick
    i, v, _ = mmr_select(np.array([5, 4, 5]), np.array([np.nan, 1, 2], dtype=np.float32), np.ones((3, 3), np.float32), 2, 1.0)
    assert i.tolist() == [5, 4] and v[0] == 2


def _bare_engine(nu=5, ni=12):
    from llmrec_b200.engine import HotPath
    hp = HotPath.__new__(HotPath)
    hp.nu, hp.ni, hp.E_u = nu, ni, torch.zeros(1)
    return hp


def test_defaults_and_rejections_before_anything_runs():
    from llmrec_b200 import ops, recommend
    hp = _bare_engine(ni=100)
    rp, col = torch.zeros(6, dtype=torch.int32), torch.zeros(0, dtype=torch.int32)
    top = lambda **kw: recommend.prepare_top_k(hp, rp, col, **{"K": 5, **kw})
    job = top()
    assert job["K"] == 5 and job["diversify"] is None
    job = top(diversity=0.5)
    assert job["K"] == 64 and job["diversify"] == (5, 0.5)                              # the pool: min(64, rankable ids)
    assert top(diversity=1, pool=20)["K"] == 20
    assert top(diversity=0, among=[3, 9, 9, 40, 41, 42])["K"] == 5 and top(diversity=0, among=list(range(30)))["K"] == 30
    assert top(diversity=0, pool=5)["K"] == 5
    for kw, msg in ((dict(diversity=float("nan")), "diversity"), (dict(diversity=-0.1), "diversity"), (dict(diversity=1.5), "diversity"),
                    (dict(diversity="a"), "diversity"), (dict(diversity=0.5, pool=4), "P in 5..64"),
                    (dict(diversity=0.5, pool=65), "P in 5..64"), (dict(diversity=0.5, pool=31, among=list(range(30))), "P in 5..30"),
                    (dict(pool=10), "give diversity")):
        with pytest.raises(ValueError, match=msg):
            top(**kw)
    cand = [[1, 2, 2, -1, 7], [3]] + [[4]] * 3
    rr = lambda **kw: recommend.prepare_rerank(hp, rp, col, cand, **kw)
    job = rr(diversity=0.5)
    assert job["K"] == 3 and job["diversify"] == (3, 0.5)                               # P = the longest surviving row, K = P
    job = rr(diversity=0.5, K=2)
    assert job["K"] == 3 and job["diversify"] == (2, 0.5)
    job = rr(diversity=0.5, K=8)
    assert job["K"] == 8 and job["diversify"] == (8, 0.5)                               # never below K: padded as rerank pads
    job = rr(diversity=0.5, pool=1024)
    assert job["K"] == 1024 and job["diversify"] == (1024, 0.5)
    assert rr()["diversify"] is None and rr()["K"] == 3
    for kw, msg in ((dict(diversity=0.5, pool=ops.RERANK_MAX_K + 1), "P in 1..1024"), (dict(diversity=0.5, K=10, pool=9), "P in 10..1024"),
                    (dict(diversity=2), "diversity"), (dict(pool=5), "give diversity")):
        with pytest.raises(ValueError, match=msg):
            rr(**kw)


def test_flags(tmp_path):
    from llmrec_b200 import main as M
    from llmrec_b200.utility.parser import build_parser, parse_args
    a = parse_args([])
    assert a.candidates_diversity is None and a.candidates_pool is None
    a = parse_args(["--candidates_out", "F", "--candidates_diversity", "0.7", "--candidates_pool", "30"])
    assert a.candidates_diversity == 0.7 and a.candidates_pool == 30
    text = build_parser().format_help()
    assert "--candidates_diversity" in text and "--candidates_pool" in text
    args = lambda **kw: types.SimpleNamespace(**{**dict(candidates_out=None, candidates_k=10, candidates_among=None,
                                                       candidates_diversity=None, candidates_pool=None), **kw})
    assert M.check_candidates_flags(args(candidates_out="F", candidates_diversity=0.5), 100) is None
    assert M.check_candidates_flags(args(candidates_out="F", candidates_diversity=0.5, candidates_pool=64), 100) is None
    for kw, msg in ((dict(candidates_diversity=0.5), "give --candidates_out"), (dict(candidates_pool=20), "give --candidates_out"),
                    (dict(candidates_out="F", candidates_pool=20), "give --candidates_diversity"),
                    (dict(candidates_out="F", candidates_diversity=float("nan")), "diversity"),
                    (dict(candidates_out="F", candidates_diversity=-0.5), "diversity"),
                    (dict(candidates_out="F", candidates_diversity=1.5), "diversity"),
                    (dict(candidates_out="F", candidates_diversity=0.5, candidates_pool=9), "P in 10..64"),
                    (dict(candidates_out="F", candidates_diversity=0.5, candidates_pool=65), "P in 10..64")):
        with pytest.raises(ValueError, match=msg):
            M.check_candidates_flags(args(**kw), 100)
    S = str(tmp_path / "S")
    pickle.dump(list(range(20)), open(S, "wb"))
    got = M.check_candidates_flags(args(candidates_out="F", candidates_among=S, candidates_diversity=0.5, candidates_pool=20), 100)
    assert got.tolist() == list(range(20))
    with pytest.raises(ValueError, match="P in 10..20"):
        M.check_candidates_flags(args(candidates_out="F", candidates_among=S, candidates_diversity=0.5, candidates_pool=21), 100)


def _worker(rank, ddir, path, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import diversify_model
    import ops_emulator
    from test_recommend_among_cpu import score_topk_among_standin
    ops_emulator.install()
    from llmrec_b200 import ops, recommend
    ops.score_topk_among = score_topk_among_standin
    ops.diversify = diversify_model.diversify
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
    # the candidate file: every user's diversified top-10 from a pool of 30, nothing excluded
    ids, vals = recommend.top_k(hp, rp, col, K=10, exclude="none", diversity=0.5, pool=30)
    recommend.write_candidates(path, ids)
    f = pickle.load(open(path, "rb"))
    pool_i, pool_v = recommend.top_k(hp, rp, col, K=30, exclude="none")
    want_i, want_v, _ = diversify_model.diversify(torch.nn.functional.normalize(I, dim=1), pool_i, pool_v, 10, 0.5)
    res["file"] = f.dtype == torch.int64 and tuple(f.shape) == (hp.nu, 10) and torch.equal(f, want_i) and torch.equal(vals, want_v)
    res["from the pool"] = all(set(f[u].tolist()) <= set(pool_i[u].tolist()) for u in range(hp.nu)) and f[:, 0].tolist() == pool_i[:, 0].tolist()
    res["changes lists"] = not torch.equal(f, pool_i[:, :10])
    ids1, vals1 = recommend.top_k(hp, rp, col, K=10, exclude="none", diversity=1, pool=30)
    res["lambda 1"] = torch.equal(ids1, pool_i[:, :10]) and torch.equal(vals1, pool_v[:, :10])
    # the default pool is min(64, rankable ids), and among / exclude="train" reach the pool call
    S = np.arange(0, hp.ni, 2)
    a, _ = recommend.top_k(hp, rp, col, users=[0, 1, 2], K=5, diversity=0.3, among=S)
    p_i, p_v = recommend.top_k(hp, rp, col, users=[0, 1, 2], K=min(64, S.size), among=S)
    res["among"] = torch.equal(a, diversify_model.diversify(torch.nn.functional.normalize(I, dim=1), p_i, p_v, 5, 0.3)[0])
    out[0] = res


def test_candidate_file_on_the_stand_ins(tiny_root, tmp_path):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), str(tmp_path / "candidate_indices"), out), nprocs=1, join=True)
    res = dict(out)[0]
    assert all(res.values()), {k: v for k, v in res.items() if not v}
