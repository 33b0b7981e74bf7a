"""The fp64 step model (tests/step_fp64_model.py) on CPU: that its bound accepts legitimate fp32 results, and that it is tight enough
to see every head and every listed mistake of a step.

Calibration: the fp32 oracle (CPU autograd on the same inputs; also with the truncating TF32 / 3xTF32 projection arithmetic at those
modes' tau) and the emulated engines (tests/ops_emulator.py in a child process: HotPath.train_step with and without the split branch
schedule, HoistedHotPath) pass the bound.
Power: in the loud rate configuration (`step_fp64_model.loud`) every head carries a share of some gradient element larger than the
bound, and each mutation of the step below fails it on at least one element.

Data: the seeded tiny netflix set of tests/conftest.py (300 x 400, feature widths 32 / 64 / 96, 5 attribute keys); it has edgeless
items, so feat_reg over n_live differs from feat_reg over n_items.  Batch: the oracle's sampler at seed 7 (B' = 128 + augmented
triplets); its kept-set cuts clear the rounding bound at every head (asserted)."""
import os
import sys

import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import step_fp64_model as SM  # noqa: E402

BATCH_SEED = 7


def _setup(ddir, d=64, L=2):
    """data, fp32 params, fp32 feats, the fp64 operators (from the binary CSR and fp32 scales, as the engine holds them), the loud
    engine config, its OracleConfig and one batch."""
    import ops_emulator
    from llmrec_b200.engine import HotPathConfig, PARAM_ORDER
    from llmrec_b200.graph import inv_sqrt_degree
    from oracle import llmrec_oracle as O
    import numpy as np
    import scipy.sparse as sp
    data = O.load_dataset(ddir)
    R = sp.csr_matrix(data.train_mat); R.sum_duplicates(); R.sort_indices(); R.data[:] = 1.0
    Rt = sp.csr_matrix(R.T); Rt.sort_indices()
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a.astype(dt)))
    ui = ops_emulator.CsrOperator(t(R.indptr, np.int32), t(R.indices, np.int32), *R.shape, rs=t(inv_sqrt_degree(R), np.float32))
    iu = ops_emulator.CsrOperator(t(Rt.indptr, np.int32), t(Rt.indices, np.int32), *Rt.shape, rs=t(inv_sqrt_degree(Rt), np.float32))
    cfg = SM.loud(HotPathConfig(embed_size=d, n_layers=L, batch_size=128))
    ocfg = SM.oracle_config(cfg)
    O.set_seed(2022)
    p0 = O.init_params(ocfg, data)
    params = {k: p0[k].detach().clone() for k in PARAM_ORDER}
    feats = dict(image=torch.tensor(data.image_feats).float(), text=torch.tensor(data.text_feats).float(),
                 user=torch.tensor(data.user_feats).float(), item={k: torch.tensor(v).float() for k, v in data.item_feats.items()})
    O.set_seed(BATCH_SEED)
    batch = O.sample_batch(data, ocfg)
    n_live = int(np.unique(R.indices).size)
    return dict(data=data, params=params, feats=feats, ui=SM.sparse64(ui), iu=SM.sparse64(iu), cfg=cfg, ocfg=ocfg, batch=batch,
                n_items=data.n_items, n_live=n_live)


@pytest.fixture(scope="module")
def tiny(tiny_root):
    torch.set_num_threads(4)
    s = _setup(os.path.join(tiny_root, "netflix_valid_item"))
    s["ref"] = _ref(s)
    return s


def _ref(s, cfg=None, **kw):
    return SM.reference(s["params"], s["feats"], s["ui"], s["iu"], cfg or s["ocfg"], *s["batch"], s["n_items"], **kw)


def test_restatement_is_the_oracle_loss_and_its_kept_sets_are_clear(tiny):
    """The per-head restatement sums to oracle.llmrec_oracle.batch_loss in fp64 (same forward, same heads), and every head's cut
    clears the rounding bound."""
    from oracle import llmrec_oracle as O
    s, ref = tiny, tiny["ref"]
    P = {k: v.double() for k, v in s["params"].items()}
    X = dict(image=s["feats"]["image"].double(), text=s["feats"]["text"].double(), user=s["feats"]["user"].double(),
             item={k: v.double() for k, v in s["feats"]["item"].items()})
    with torch.no_grad():
        out = O.forward(P, X, s["ui"], s["iu"], s["ocfg"])
        total, _ = O.batch_loss(out, *s["batch"], s["n_items"], s["ocfg"])
    assert abs(float(total) - ref.loss) <= 1e-12 * abs(ref.loss)
    B = len(s["batch"][0])
    assert B > s["cfg"].batch_size and ref.n_keep == int((1 - 0.71) * B) >= 1
    assert set(ref.cuts) == {"mf", "img", "txt"} | {"aug:" + k for k in s["feats"]["item"]}
    SM.check_cuts(ref, "fp32", "tiny")


@pytest.mark.parametrize("proj", [None, "3xtf32-rz", "tf32-rz"])
def test_fp32_oracle_passes_the_bound(tiny, proj):
    """The fp32 oracle, with fp32 projections or with the truncating TF32 arithmetic of proj_mode 0 / 1, at that mode's tau."""
    ref32 = _ref(tiny, dtype=torch.float32, proj=proj)
    assert ref32.n_keep == tiny["ref"].n_keep
    SM.check_grads(tiny["ref"], ref32.grads, SM.TAU["fp32" if proj is None else proj[:-3]], what=f"fp32 oracle {proj}")


def test_loud_rates_make_every_head_visible(tiny):
    """Each head's own gradient exceeds the bound on some element: no tolerance hides a head."""
    ref = tiny["ref"]
    for h, g in ref.per_head.items():
        worst = max(float((g[k].abs() / SM.allowed(ref, k, SM.TAU["fp32"])).max()) for k in g)
        assert worst > 10, (h, worst)


def _mutations(s):
    B = len(s["batch"][0])
    keep = s["ref"].n_keep
    cfg, ocfg = s["cfg"], s["ocfg"]
    import dataclasses
    out = [("drop " + h, dict(drop_heads=(h,))) for h in s["ref"].parts]
    out += [("user_cat_rate +1%", dict(cfg=dataclasses.replace(ocfg, user_cat_rate=ocfg.user_cat_rate * 1.01))),
            ("item_cat_rate +1%", dict(cfg=dataclasses.replace(ocfg, item_cat_rate=ocfg.item_cat_rate * 1.01))),
            ("regulariser / B'", dict(reg_div=B)),
            ("n_keep from the sampled B", dict(n_keep=int((1 - ocfg.prune_loss_drop_rate) * cfg.batch_size))),
            ("n_keep + 1", dict(n_keep=keep + 1)), ("n_keep - 1", dict(n_keep=keep - 1)),
            ("last triplet's row gradient dropped", dict(detach_last=True)),
            ("feat_reg over n_live", dict(feat_div=s["n_live"])),
            ("softmax Jacobian -> identity", dict(softmax_identity=True))]
    return out


def test_every_mutation_of_the_step_is_rejected(tiny):
    s = tiny
    assert s["n_live"] < s["n_items"]
    assert int((1 - 0.71) * s["cfg"].batch_size) != s["ref"].n_keep
    missed = []
    for what, kw in _mutations(s):
        g = _ref(s, **kw).grads
        for mode, tau in SM.TAU.items():                  # rejected at every mode's tau, the loosest (plain TF32) included
            res = SM.grad_excess(s["ref"], g, tau)
            if not any(v[1] for v in res.values()):
                missed.append((what, mode, {k: v[0] for k, v in res.items()}))
    assert not missed, missed


# ---- the emulated engines -------------------------------------------------------------------------------------------------------
def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    ops_emulator.install()
    from llmrec_b200.engine import HotPath
    from llmrec_b200.graph import BipartiteGraph
    from llmrec_b200.hoist import HoistedHotPath
    s = _setup(ddir)
    ref = _ref(s)
    res = {}
    for name in ("train_step", "train_step split", "hoisted", "hoisted capacity"):
        params = {k: v.clone() for k, v in s["params"].items()}
        feats = dict(image=s["feats"]["image"].clone(), text=s["feats"]["text"].clone(), user=s["feats"]["user"].clone(),
                     item={k: v.clone() for k, v in s["feats"]["item"].items()})
        g = BipartiteGraph(s["data"].train_mat, "cpu")
        ops = (g.ui, g.iu, g.uiT, g.iuT)
        hp = HoistedHotPath(ops, params, feats, s["cfg"], g.ones_propagated()) if name.startswith("hoisted") else HotPath(ops, params, feats, s["cfg"])
        hp.set_optimizer(lr=1e-3)
        hp.force_split = name.endswith("split")
        users, pos, neg = (torch.tensor(x, dtype=torch.int32) for x in s["batch"])
        B = int(users.numel())
        if name.endswith("capacity"):
            gi = hp.index_buffer(B)
            gi.zero_()
            gi[0, :B], gi[1, :B], gi[2, :B] = users, pos, neg
            gi[3, 0], gi[3, 1] = hp.meta_row(B)
            hp.train_step(gi[0], gi[1], gi[2], gi[3])
        else:
            hp.train_step(users, pos, neg)
        try:
            SM.check_grads(ref, hp.grads, SM.TAU["fp32"], what=name)
            SM.check_loss(ref, hp.loss, hp.head_out, SM.engine_heads(hp.keys), SM.TAU["fp32"], what=name)
            res[name] = "ok"
        except AssertionError as e:
            res[name] = str(e)
    out[0] = res


def test_emulated_engines_pass_the_bound(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    assert all(v == "ok" for v in out[0].values()), dict(out[0])
