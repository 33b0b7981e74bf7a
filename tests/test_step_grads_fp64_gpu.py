"""-m gpu: whole training steps of every engine held to the fp64 step model (tests/step_fp64_model.py): after one step, hp.grads,
hp.loss and every head's head_out slots against the fp64 gradients and losses at the parameters the step started from.

Rates: the loud configuration of `step_fp64_model.loud` (regs0 1e4, mm / aug / feat_reg rates near 1), where every head carries a
share of some gradient element far above the bound (tests/test_step_grads_fp64_cpu.py shows each listed mutation of a step fails
it by 10^3 or more).  Bound: TAU["fp32"] = 2e-5 for fp32 SIMT, TAU["3xtf32"] = 4e-4 for 3xTF32 and bf16 / int8 tables,
TAU["tf32"] = 2e-2 for plain TF32; RHO = 0.1 (the docstring of step_fp64_model gives the reasoning and the calibration).

Shapes, graphs, tables, batches and engines: tests/step_fp64_cases.py (netflix, movielens and the odd shape; B' = 1126, 1128 and 8).
Each reference asserts first that every head's kept-set cut clears the rounding bound (step_fp64_model.check_cuts); the seeds in
step_fp64_cases.SEEDS were chosen for that margin.

The fp64 reference runs on the GPU in float64 and is computed once per (shape, table dtype, batch) and shared by the engine cases
that start from the same parameters."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import step_fp64_model as SM  # noqa: E402
from step_fp64_cases import _batch, _engine  # noqa: E402

pytestmark = pytest.mark.gpu

_REFS = {}


def _reference(hp, key, batch):
    """The fp64 step model at hp's current parameters, once per key = (shape, table dtype, batch)."""
    if key not in _REFS:
        p, f, ui, iu = SM.engine_inputs(hp)
        ref = SM.reference(p, f, ui, iu, SM.oracle_config(hp.cfg), *(torch.from_numpy(x).long() for x in batch), hp.ni)
        del ref.per_head
        _REFS[key] = ref
    return _REFS[key]


def _dev(batch):
    return tuple(torch.from_numpy(x).cuda() for x in batch)


def _run(hp, how, batch, name):
    """One step of `how` on `batch`; hp.grads / hp.loss / hp.head_out then hold its results."""
    u, p, n = _dev(batch)
    if how == "train_step":
        hp.train_step(u, p, n)
    elif how == "pieces":
        hp.forward()
        hp.loss_and_output_grads(u, p, n)
        hp.backward()
    elif how == "graphed":
        # capture on a throwaway batch, put the starting state back in place (the graph holds these addresses), replay the test batch
        snap = hp._snapshot_state()
        hp.train_step_graphed(*_dev(_batch(name, "small")))
        hp.load_state(snap)
        hp.train_step_graphed(u, p, n)
    else:
        raise ValueError(how)
    torch.cuda.synchronize()


def _case(name, batch_name="B1126", dtype="fp32", hoisted=False, mode=0, det=False, how="train_step", branches=True):
    hp = _engine(name, dtype, hoisted, mode, det)
    hp.branches = hp.branches and branches
    batch = _batch(name, batch_name)
    ref = _reference(hp, (name, dtype, batch_name), batch)
    tau = ("3xtf32", "tf32", "fp32")[mode]
    what = f"{name} {batch_name} {dtype} {'hoisted' if hoisted else 'default'} mode={mode} det={det} {how} branches={hp.branches}"
    SM.check_cuts(ref, tau, what)
    _run(hp, how, batch, name)
    tau = SM.TAU[tau]
    res = SM.check_grads(ref, hp.grads, tau, what=what)
    SM.check_loss(ref, hp.loss, hp.head_out, SM.engine_heads(hp.keys), tau, what=what)
    return hp, res


CASES = [
    # default engine: schedules and projection modes
    dict(name="netflix"), dict(name="netflix", branches=False), dict(name="netflix", how="graphed"), dict(name="netflix", how="pieces"),
    dict(name="netflix", mode=1, batch_name="small"), dict(name="netflix", mode=2), dict(name="netflix", det=True),
    dict(name="netflix", batch_name="B1128"), dict(name="netflix", batch_name="small"), dict(name="netflix", batch_name="small", how="graphed"),
    # hoisted engine
    dict(name="netflix", hoisted=True), dict(name="netflix", hoisted=True, how="graphed"), dict(name="netflix", hoisted=True, mode=1, batch_name="small"),
    dict(name="netflix", hoisted=True, det=True), dict(name="netflix", hoisted=True, batch_name="B1128"),
    dict(name="netflix", hoisted=True, batch_name="small"),
    # bf16 / int8 tables
    dict(name="netflix", dtype="bf16"), dict(name="netflix", dtype="int8"), dict(name="netflix", dtype="bf16", hoisted=True),
    dict(name="netflix", dtype="int8", hoisted=True, how="graphed"),
    # movielens and the odd shape
    dict(name="movielens"), dict(name="movielens", hoisted=True, how="graphed"), dict(name="movielens", det=True, how="graphed"),
    dict(name="odd"), dict(name="odd", mode=2), dict(name="odd", mode=1, batch_name="small"), dict(name="odd", hoisted=True),
    dict(name="odd", batch_name="small", how="graphed"),
]


def _id(c):
    return "-".join(f"{k}={v}" for k, v in c.items())


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_step_gradients_match_the_fp64_model(case):
    hp, _ = _case(**case)
    if case["name"] == "odd" and not case.get("hoisted"):
        assert hp.live_i is not None and hp.n_live < hp.ni


def test_step_without_the_live_item_set(monkeypatch):
    """LLMREC_LIVE_ITEMS=0: the full-table projections pass the same bound (the default case above runs with the live set)."""
    monkeypatch.setenv("LLMREC_LIVE_ITEMS", "0")
    hp, _ = _case("netflix")
    assert hp.live_i is None


# ---- through Trainer, built from CLI flags ----------------------------------------------------------------------------------------
LOUD_FLAGS = ["--regs", "[10000.0]", "--aug_mf_rate", "0.9", "--mm_mf_rate", "0.7", "--feat_reg_decay", "0.8", "--model_cat_rate", "0.4",
              "--user_cat_rate", "1.3", "--item_cat_rate", "0.3", "--prune_loss_drop_rate", "0.6", "--batch_size", "200"]


def _oracle_cfg(args):
    from oracle import llmrec_oracle as O
    ws = eval(args.weight_size)
    return O.OracleConfig(embed_size=args.embed_size, weight_size=tuple(ws), batch_size=args.batch_size, regs0=eval(args.regs)[0],
                          model_cat_rate=args.model_cat_rate, user_cat_rate=args.user_cat_rate, item_cat_rate=args.item_cat_rate,
                          aug_mf_rate=args.aug_mf_rate, mm_mf_rate=args.mm_mf_rate, prune_loss_drop_rate=args.prune_loss_drop_rate,
                          feat_reg_decay=args.feat_reg_decay)


def _trainer(tmp_path, extra=()):
    import pickle
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.synth import make_dataset
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir
    root = str(tmp_path) + "/"
    ddir = make_dataset(root, dataset="netflix", n_users=900, n_items=1200, n_inter=6000, dims=(64, 96, 128), seed=4)
    with open(os.path.join(ddir, "augmented_sample_dict"), "rb") as f:
        aug = pickle.load(f)
    for u in range(0, 900, 2):                            # negative ids pass the reference's `< n_items` filter and wrap
        aug[u][0] = -1 - (u % 5)
    with open(os.path.join(ddir, "augmented_sample_dict"), "wb") as f:
        pickle.dump(aug, f)
    args = set_args(parse_args(["--data_path", root, "--dataset", "netflix", "--debug", "--seed", "3", "--embed_size", "64",
                                "--weight_size", "[64, 64]", "--aug_sample_rate", "0.2"] + LOUD_FLAGS + list(extra)))
    M.set_seed(args.seed)
    gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size)
    batch_test.init(gen, args)
    return M.Trainer(data_config={}, data_generator=gen), args, aug


def test_trainer_step_from_flags_matches_the_fp64_model(tmp_path):
    """Non-default rate flags reach HotPathConfig (Models.hot_path): the graphed step of a Trainer against an OracleConfig built
    from the same flags.  A negative augmented id lands in the batch as Python indexing wraps it (main.py:332)."""
    tr, args, aug = _trainer(tmp_path)
    hp = tr.hot
    assert (hp.cfg.regs0, hp.cfg.batch_size, hp.cfg.prune_loss_drop_rate) == (1e4, 200, 0.6)
    from llmrec_b200 import main as M
    M.set_seed(8)
    users, pos, neg = tr.sample_batch()
    B, ni = len(users), tr.n_items
    wrapped = {aug[u][0] % ni for u in users[200:] if aug[u][0] < 0}
    assert B > 200 and wrapped and wrapped <= set(pos[200:])
    p, f, ui, iu = SM.engine_inputs(hp)
    ref = SM.reference(p, f, ui, iu, _oracle_cfg(args), torch.tensor(users), torch.tensor(pos), torch.tensor(neg), ni)
    SM.check_cuts(ref, "3xtf32", "trainer")
    tr.train_batch(users, pos, neg)
    torch.cuda.synchronize()
    SM.check_grads(ref, hp.grads, SM.TAU["3xtf32"], what="trainer")
    SM.check_loss(ref, hp.loss, hp.head_out, SM.engine_heads(hp.keys), SM.TAU["3xtf32"], what="trainer")


def test_trainer_mask_dropout_restoration_step_matches_the_fp64_model(tmp_path):
    """One --drop_rate 0.2 --mask 1 --mask_rate 0.1 --att_re_rate 0.5 step (Trainer._train_batch_masked): the dropout masks it drew,
    the permutations from a copy of the CPU generator state, the masked feature tables it left behind, and the restoration head."""
    tr, args, aug = _trainer(tmp_path, ["--drop_rate", "0.2", "--mask", "1", "--mask_rate", "0.1", "--att_re_rate", "0.5"])
    hp = tr.hot
    assert tr.masked_mode
    from llmrec_b200 import main as M
    M.set_seed(12)                                        # seed 9: two attribute heads' cuts fall inside the rounding bound
    users, pos, neg = tr.sample_batch()
    p, _, ui, iu = SM.engine_inputs(hp)
    state = torch.get_rng_state()
    tr.train_batch(users, pos, neg)
    torch.cuda.synchronize()
    torch.set_rng_state(state)                            # the same permutations, in the engine's order: items, then users
    i_mask = torch.randperm(tr.n_items)[:int(0.1 * tr.n_items)]
    u_mask = torch.randperm(tr.n_users)[:int(0.1 * tr.n_users)]
    _, f, _, _ = SM.engine_inputs(hp)                     # the tables the step projected: masked at its start, in place
    drop = [m.double() for m in tr._last_dropout_masks]
    d = tr.decoder
    restore = dict(rate=0.5, dec=dict(u_w=d.u_net[0].weight.detach(), u_b=d.u_net[0].bias.detach(), i_w=d.i_net[0].weight.detach(),
                                      i_b=d.i_net[0].bias.detach()),
                   raw_user=torch.tensor(tr.user_init_embedding), raw_items={k: torch.tensor(v) for k, v in tr.item_attribute_embedding.items()},
                   i_mask=i_mask, u_mask=u_mask, alpha=args.alpha_l, kind=args.feat_loss_type)
    ref = SM.reference(p, f, ui, iu, _oracle_cfg(args), torch.tensor(users), torch.tensor(pos), torch.tensor(neg), tr.n_items,
                       drop=drop, restore=restore)
    SM.check_cuts(ref, "3xtf32", "masked")
    assert ref.parts["restore"] != 0
    SM.check_grads(ref, hp.grads, SM.TAU["3xtf32"], what="masked")
    SM.check_loss(ref, hp.loss, hp.head_out, SM.engine_heads(hp.keys), SM.TAU["3xtf32"], what="masked")
