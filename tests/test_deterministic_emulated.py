"""Deterministic steps (`--deterministic 1`, HotPathConfig.deterministic) without a GPU: the torch stand-ins of the ordered ops implement the
order definition of include/llmrec_b200.h literally (tests/ops_emulator_ordered.py); the default and the hoisted engine with the option set still track the CPU oracle
within the tolerances of test_engine_emulated.py / test_hoist_emulated.py (eager and capacity form); the parser takes the flag and
leaves the reference's 42 alone; the combinations the option does not cover raise."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)

F = np.float32


def _order_fixture(seed=0, B=40, nu=6, ni=7, d=5):
    """Heads whose per-triplet contributions are exact in fp32 (power-of-two values, one product per contribution non-zero) but
    whose sums depend on the order: magnitudes spread over 40 binades."""
    rng = np.random.default_rng(seed)
    p2 = lambda *s: (2.0 ** rng.integers(-20, 20, s) * rng.choice([-1.0, 1.0], s)).astype(F)
    users, pos, neg = rng.integers(0, nu, B), rng.integers(0, ni, B), rng.integers(0, ni, B)
    neg[3] = pos[3]
    return p2(nu, d), p2(ni, d), users.astype(np.int32), pos.astype(np.int32), neg.astype(np.int32)


def test_emulated_ordered_scatter_is_the_definition():
    import ops_emulator_ordered as E
    rng = np.random.default_rng(1)
    G = (2.0 ** rng.integers(-30, 30, (50, 4))).astype(F) * rng.choice([-1, 1], (50, 4)).astype(F)
    idx = rng.integers(-1, 5, 50).astype(np.int32)
    Y0 = (2.0 ** rng.integers(-30, 30, (5, 4))).astype(F)
    want = Y0.copy()
    for b in range(50):
        if idx[b] >= 0:
            want[idx[b]] = want[idx[b]] + G[b]
    Y = torch.from_numpy(Y0.copy())
    E.scatter_add_rows_ordered(torch.from_numpy(G), torch.from_numpy(idx), Y)
    assert np.array_equal(Y.numpy().view(np.uint32), want.view(np.uint32))
    rev = Y0.copy()
    for b in reversed(range(50)):
        if idx[b] >= 0:
            rev[idx[b]] = rev[idx[b]] + G[b]
    assert not np.array_equal(rev.view(np.uint32), want.view(np.uint32)), "the fixture cannot tell one order from another"


def test_emulated_slot_plan_sorts_by_row_then_slot():
    import ops_emulator_ordered as E
    _, _, users, pos, neg = _order_fixture()
    B = users.size
    for live in (B, 7, 1):
        meta = None if live == B else torch.tensor([live, 0], dtype=torch.int32)
        plan = E.bpr_slot_plan(torch.from_numpy(users), torch.from_numpy(pos), torch.from_numpy(neg), meta=meta).numpy()
        su, ru = plan[:live], plan[B:B + live]
        assert sorted(zip(users[:live].tolist(), range(live))) == list(zip(ru.tolist(), su.tolist()))
        items = np.stack([pos[:live], neg[:live]], 1).reshape(-1)
        si, ri = plan[2 * B:2 * B + 2 * live], plan[4 * B:4 * B + 2 * live]
        assert sorted(zip(items.tolist(), range(2 * live))) == list(zip(ri.tolist(), si.tolist()))


def test_emulated_ordered_heads_follow_the_definition():
    """Two heads sharing GU and GI: the ordered stand-in equals a numpy loop over (head, b, pos before neg) on the per-triplet
    gradients, which differs from the same loop run backwards."""
    import ops_emulator_ordered as E
    XU, XI, users, pos, neg = _order_fixture(seed=2)
    t = torch.from_numpy
    B, nk = users.size, 11
    GU0, GI0 = np.ones_like(XU), np.ones_like(XI) * F(0.5)
    heads_of = lambda GU, GI: [(t(XU), t(XI), GU, GI, 1.0, 1.0), (t(XU * F(2)), t(XI), GU, GI, 0.5, 0.0)]
    GU, GI = t(GU0.copy()), t(GI0.copy())
    out, loss = torch.zeros(8), torch.zeros(1)
    plan = E.bpr_slot_plan(t(users), t(pos), t(neg))
    E.bpr_heads(heads_of(GU, GI), t(users), t(pos), t(neg), nk, 0.01, out, loss, None, ordered=plan)
    # per-triplet gradients of each head alone, from the unordered stand-in on a batch of one row per triplet
    wu, wi = GU0.copy(), GI0.copy()
    ru, ri = GU0.copy(), GI0.copy()
    contrib = []
    for h in range(2):
        a = t(heads_of(None, None)[h][0].numpy()[users]); q = t(XI[pos]); r = t(XI[neg])
        gu, gi = torch.zeros(B, XU.shape[1]), torch.zeros(2 * B, XU.shape[1])
        ar = torch.arange(B, dtype=torch.int32)
        E.bpr_heads([(a, torch.cat([q, r]), gu, gi, heads_of(None, None)[h][4], heads_of(None, None)[h][5])], ar, ar, ar + B, nk, 0.01,
                    torch.zeros(4), torch.zeros(1), None)
        contrib.append((gu.numpy(), gi.numpy()))
    for h in range(2):
        gu, gi = contrib[h]
        for b in range(B):
            wu[users[b]] = wu[users[b]] + gu[b]
            wi[pos[b]] = wi[pos[b]] + gi[b]
            wi[neg[b]] = wi[neg[b]] + gi[B + b]
    for h in (1, 0):
        gu, gi = contrib[h]
        for b in reversed(range(B)):
            ru[users[b]] = ru[users[b]] + gu[b]
            ri[neg[b]] = ri[neg[b]] + gi[B + b]
            ri[pos[b]] = ri[pos[b]] + gi[b]
    assert np.array_equal(GU.numpy().view(np.uint32), wu.view(np.uint32))
    assert np.array_equal(GI.numpy().view(np.uint32), wi.view(np.uint32))
    assert not np.array_equal(ru.view(np.uint32), wu.view(np.uint32)) or not np.array_equal(ri.view(np.uint32), wi.view(np.uint32))


def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator_ordered
    ops_emulator_ordered.install()
    from llmrec_b200 import ops
    from llmrec_b200.engine import HotPath, HotPathConfig, PARAM_ORDER
    from llmrec_b200.graph import BipartiteGraph
    from llmrec_b200.hoist import HoistedHotPath
    from oracle import llmrec_oracle as O
    data = O.load_dataset(ddir)
    ok, calls = True, {"plan": 0, "ordered": 0, "scatter": 0, "atomic_scatter": 0}
    plan0, heads0, sc0, sa0 = ops.bpr_slot_plan, ops.bpr_heads, ops.scatter_add_rows_ordered, ops.scatter_add_rows

    def count(name, fn, key=None):
        def f(*a, **kw):
            if key is None or kw.get(key) is not None:
                calls[name] += 1
            return fn(*a, **kw)
        return f

    ops.bpr_slot_plan, ops.bpr_heads = count("plan", plan0), count("ordered", heads0, "ordered")
    ops.scatter_add_rows_ordered, ops.scatter_add_rows = count("scatter", sc0), count("atomic_scatter", sa0)
    for hoisted, weight_size, d, capacity, split in ((False, "[64, 64]", 64, False, False), (False, "[32,32,32]", 32, True, True),
                                                     (True, "[64, 64]", 64, False, False), (True, "[32,32,32]", 32, True, False)):
        ocfg = O.OracleConfig(batch_size=128, embed_size=d, weight_size=eval(weight_size), lr=1e-3)
        O.set_seed(2022)
        otr = O.OracleTrainer(data, ocfg)
        params = {k: otr.params[k].detach().clone() for k in PARAM_ORDER}
        feats = dict(image=otr.feats["image"].clone(), text=otr.feats["text"].clone(), user=otr.feats["user"].clone(),
                     item={k: v.clone() for k, v in otr.feats["item"].items()})
        g = BipartiteGraph(data.train_mat, "cpu")
        cfg = HotPathConfig(embed_size=d, n_layers=len(eval(weight_size)), batch_size=128, deterministic=True)
        ops_ = (g.ui, g.iu, g.uiT, g.iuT)
        hp = HoistedHotPath(ops_, params, feats, cfg, g.ones_propagated()) if hoisted else HotPath(ops_, params, feats, cfg)
        hp.set_optimizer(lr=1e-3)
        hp.force_split = split
        O.set_seed(7)
        for step in range(3):
            users, pos, neg = O.sample_batch(data, ocfg)
            B = len(users)
            t = lambda x: torch.tensor(x, dtype=torch.int32)
            if capacity:
                gi = hp.index_buffer(B)
                gi.zero_()
                gi[0, :B], gi[1, :B], gi[2, :B] = t(users), t(pos), t(neg)
                gi[3, 0], gi[3, 1] = hp.meta_row(B)
                got = float(hp.train_step(gi[0], gi[1], gi[2], gi[3]))
            else:
                got = float(hp.train_step(t(users), t(pos), t(neg)))
            want, _ = otr.step(users, pos, neg)
            ok &= abs(got - want) < 2e-5 * max(1.0, abs(want))
        for k in PARAM_ORDER:
            ok &= bool(torch.allclose(params[k], otr.params[k].detach(), rtol=2e-4, atol=2e-6))
    # every step planned its slots once and ran the ordered heads; the hoisted steps scattered dU and dI in order, never with atomics
    ok &= calls == {"plan": 12, "ordered": 12, "scatter": 12, "atomic_scatter": 0}
    out[0] = bool(ok)
    out[1] = dict(calls)


def test_deterministic_engines_track_the_oracle(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    assert out[0] is True, dict(out)


def test_parser_takes_the_flag_and_keeps_the_reference_flags():
    from llmrec_b200.utility.parser import parse_args
    ref = json.load(open(os.path.join(HERE, "golden", "reference_parser.json")))
    a, b = vars(parse_args([])), vars(parse_args(["--deterministic", "1"]))
    assert a["deterministic"] == 0 and b["deterministic"] == 1 and type(b["deterministic"]) is int
    assert "deterministic" not in ref["defaults"] and len(ref["defaults"]) == 42
    for k, (v, tname) in ref["defaults"].items():
        assert a[k] == v and b[k] == v and type(b[k]).__name__ == tname, k


def test_uncovered_combinations_raise():
    from llmrec_b200.dist import ShardedHotPath
    from llmrec_b200.dist_feat import ShardedFeatureHotPath
    from llmrec_b200.engine import HotPath, HotPathConfig
    E = {"user_id_embedding.weight": torch.zeros(4, 8), "item_id_embedding.weight": torch.zeros(5, 8)}
    with pytest.raises(ValueError, match="tensor-core"):
        HotPath((None,) * 4, E, None, HotPathConfig(embed_size=8, proj_mode=2, deterministic=True))
    cfg = HotPathConfig(embed_size=8, deterministic=True)
    with pytest.raises(ValueError, match="sharded"):
        ShardedHotPath(None, E["user_id_embedding.weight"], E["item_id_embedding.weight"], cfg, 0)
    with pytest.raises(ValueError, match="sharded"):
        ShardedFeatureHotPath(None, E, None, cfg, 0, 0)


def test_product_still_never_imports_the_oracle():
    for root, _, files in os.walk(os.path.join(REPO, "llmrec_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(root, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
    for f in ("bench_deterministic.py",):
        txt = open(os.path.join(REPO, f)).read()
        assert "import oracle" not in txt and "from oracle" not in txt, f
