"""The sharded engines' steps against the fp64 step model on CPU (tests/dist_fp64.py): dist.ShardedHotPath and
dist_feat.ShardedFeatureHotPath on the emulated kernels (tests/ops_emulator.py) under gloo at world sizes 1 and 2, every case of
dist_fp64.CASES_W1 / CASES_W2 over the five-step SEQUENCE, gradients, losses and every AdamW update (p, m, v) checked per step.

The netflix shape runs one demand case per world size here (the -m gpu tests run it in every form); the odd shapes run every case.

Power: each mutation of the sharded step in dist_fp64.MUTATIONS (an exchange dropped or all-reduced twice, a user gradient
scattered by a non-owner too, a gradient scaled by the world size, the demand row sets left uncleared) must exceed the bound by 10^2
or more on some gradient element (a nonzero where fp64 is exactly zero counts as infinitely over).  Of the engine-equality checks
of tests/dist_gpu_check.py / tests/test_dist_emulated.py, the per-step loss comparison accepts the item gradient divided by the
world size at every step (the loss is formed before the backward chain).  Their allclose on the parameters after AdamW does see it
on this graph: AdamW normalises the step to about lr * sign(g), but a few percent of the item-table elements have gradients near
its eps, where the scale still shows."""
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import dist_fp64 as DF  # noqa: E402
import step_fp64_model as SM  # noqa: E402

MUTATION_WORLD, MUTATION_SHAPE, MUTATION_STEPS = 2, "odd", 2
CASES_W1 = [c for c in DF.CASES_W1 if c["shape"] != "netflix"] + [dict(shape="netflix", demand=True, d=64)]
CASES_W2 = [c for c in DF.CASES_W2 if c["shape"] != "netflix"] + [dict(shape="netflix", demand=True, d=64)]


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _loss_check_after_steps(mutate, dev, n=3):
    """n steps of a clean and a mutated dense engine on the same batches -> (whether every step's losses pass the comparison of
    tests/dist_gpu_check.py, whether the parameters after the run pass its allclose, rtol 1e-4 and atol 1e-6)"""
    clean, bad = DF.build(dict(shape=MUTATION_SHAPE), dev), DF.build(dict(shape=MUTATION_SHAPE), dev)
    mutate(bad.sh)
    ok, prev = True, None
    for k in range(n):
        prev = DF.batches_for(clean, DF.ref_params(clean), k, prev)
        l1, l2 = (float(r.sh.train_step(*(torch.from_numpy(x) for x in prev))) for r in (clean, bad))
        ok &= abs(l1 - l2) < 1e-5 * max(1.0, abs(l1))
    tol = dict(rtol=1e-4, atol=1e-6)
    return ok, torch.allclose(clean.sh.E_u, bad.sh.E_u, **tol) and torch.allclose(clean.sh.E_i, bad.sh.E_i, **tol)


def _worker(rank, world, port, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(max(1, 4 // world))
    import ops_emulator
    ops_emulator.install()
    import dist_fp64 as D
    dev = torch.device("cpu")
    res = {}
    for c in (CASES_W1 if world == 1 else CASES_W2):
        res["case " + D.case_id(c)] = D.run_case(c, dev)
    if world == MUTATION_WORLD:
        for name, (extra, mutate) in D.MUTATIONS.items():
            run = D.build(dict(shape=MUTATION_SHAPE, **extra), dev)
            mutate(run.sh)
            res["mutation " + name] = D.run_steps(run, MUTATION_STEPS, strict=False)
        res["equality checks on item gradient / world"] = _loss_check_after_steps(D.MUTATIONS["item gradient divided by world size"][1], dev)
    out[rank] = res
    dist.destroy_process_group()


_RESULTS = {}


def _results(world):
    if world not in _RESULTS:
        mgr = mp.Manager()
        out = mgr.dict()
        mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
        per_rank = [out[r] for r in range(world)]
        _RESULTS[world] = {k: (DF.merge_ranks([p[k] for p in per_rank]) if isinstance(per_rank[0][k], dict) else
                               tuple(all(p[k][i] for p in per_rank) for i in range(len(per_rank[0][k])))) for k in per_rank[0]}
    return _RESULTS[world]


def test_id_only_reference_is_the_oracle_without_side_terms():
    """step_fp64_model.reference(feats=None) is the oracle's ID head on the oracle's forward with every side term's rate at zero:
    same mf and emb losses, same gradients of both ID tables, to fp64 rounding."""
    import dataclasses
    from llmrec_b200.engine import HotPathConfig
    from oracle import llmrec_oracle as O
    run_R = DF.graph("odd")
    nu, ni = run_R.shape
    coo = run_R.tocoo()
    su = torch.pow(torch.from_numpy(run_R.sum(1).A1).double() + 1e-8, -0.5)
    si = torch.pow(torch.from_numpy(run_R.sum(0).A1).double() + 1e-8, -0.5)
    r, c = torch.from_numpy(coo.row).long(), torch.from_numpy(coo.col).long()
    ui = torch.sparse_coo_tensor(torch.stack([r, c]), su[r], (nu, ni)).coalesce()
    iu = torch.sparse_coo_tensor(torch.stack([c, r]), si[c], (ni, nu)).coalesce()
    cfg = SM.oracle_config(SM.loud(HotPathConfig(embed_size=32, n_layers=2, batch_size=1024)))
    gen = torch.Generator().manual_seed(1)
    P = {DF.UID: torch.randn(nu, 32, generator=gen, dtype=torch.float64) * 0.1,
         DF.IID: torch.randn(ni, 32, generator=gen, dtype=torch.float64) * 0.1}
    import step_fp64_cases as SC
    users, pos, neg = (torch.from_numpy(x).long() for x in SC.draw(nu, ni, 1024, 102, 11))
    ref = SM.reference(P, None, ui, iu, cfg, users, pos, neg, ni)
    # the oracle: its full forward with zero side rates (tiny side tables), its ID head, autograd
    Q = {k: v.clone().requires_grad_(True) for k, v in P.items()}
    for k in ("image", "text", "user", "item"):
        Q[k + "_trans.weight"] = torch.randn(32, 8, generator=gen, dtype=torch.float64)
        Q[k + "_trans.bias"] = torch.randn(32, generator=gen, dtype=torch.float64)
    X = dict(image=torch.randn(ni, 8, generator=gen, dtype=torch.float64), text=torch.randn(ni, 8, generator=gen, dtype=torch.float64),
             user=torch.randn(nu, 8, generator=gen, dtype=torch.float64), item={"a": torch.randn(ni, 8, generator=gen, dtype=torch.float64)})
    out = O.forward(Q, X, ui, iu, dataclasses.replace(cfg, model_cat_rate=0.0, user_cat_rate=0.0, item_cat_rate=0.0))
    mf, emb = O.bpr_head(out["U"][users], out["I"][pos], out["I"][neg], cfg)
    g = torch.autograd.grad(mf + emb, [Q[DF.UID], Q[DF.IID]])
    assert abs(float(mf) - ref.parts["mf"]) <= 1e-12 * abs(ref.parts["mf"])
    assert abs(float(emb) - ref.parts["emb"]) <= 1e-12 * abs(ref.parts["emb"])
    assert set(ref.grads) == {DF.UID, DF.IID} and set(ref.parts) == {"mf", "emb"} and set(ref.cuts) == {"mf"}
    for k, gg in zip((DF.UID, DF.IID), g):
        assert torch.allclose(ref.grads[k], gg, rtol=1e-12, atol=1e-12 * float(gg.abs().max()))
        assert torch.equal(ref.grads[k] == 0, gg == 0)


@pytest.mark.parametrize("world,case", [(1, c) for c in CASES_W1] + [(2, c) for c in CASES_W2],
                         ids=lambda x: DF.case_id(x) if isinstance(x, dict) else f"world{x}")
def test_emulated_sharded_step_matches_the_fp64_model(world, case):
    res = _results(world)["case " + DF.case_id(case)]
    print(f"\nworld {world} {DF.case_id(case)}: grads {res['grads']:.3g}, adamw {res['adamw']:.3g} of the bound; {res['forms']}")
    assert not res["errors"], "\n".join(res["errors"][:6])
    if world == 2 and case.get("item_sharded"):
        assert res["forms"]["item_sharded"] == (case["shape"] != "odd-uneven")
    if world == 2 and case.get("demand"):
        assert res["forms"]["item_opt_sharded"] == (case["shape"] != "odd-uneven")
    if world == 2 and case.get("engine") == "feat":
        assert res["forms"]["even_items"] == (case["shape"] != "odd-uneven")


@pytest.mark.parametrize("name", list(DF.MUTATIONS))
def test_mutation_of_the_sharded_step_fails_the_bound(name):
    res = _results(MUTATION_WORLD)["mutation " + name]
    print(f"\n{name}: worst gradient error {res['grads']:.3g} x the bound")
    assert res["grads"] >= 1e2, f"{name}: only {res['grads']:.3g} x the bound"


def test_loss_comparison_accepts_a_scaled_item_gradient():
    """The gap the fp64 checks close: the per-step loss comparison of the engine-equality checks passes a step whose item gradient
    is divided by the world size; only the parameters after AdamW show it there."""
    loss_ok, params_ok = _results(MUTATION_WORLD)["equality checks on item gradient / world"]
    print(f"\nitem gradient / world: loss comparison passes {loss_ok}, parameter allclose passes {params_ok}")
    assert loss_ok
