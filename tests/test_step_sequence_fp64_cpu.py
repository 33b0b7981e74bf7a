"""Runs of consecutive training steps (tests/step_sequence.py) on the emulated engines: that the sequence checks accept legitimate
fp32 runs, and that they see what a single-step check cannot.

Data: the seeded tiny netflix set and loud configuration of tests/test_step_grads_fp64_cpu.py (300 x 400, batch_size 128, so the
batch capacity is 144).  Batches: 144 (the full capacity), 8, 140, 8, 144, consecutive ones sharing users and items
(`step_fp64_cases._sequence`); every head's kept-set cut clears TAU_CUT["fp32"] at every step (asserted by each step's check).
The emulated default engine fuses the batch's rows as the CUDA engine does (its row sets and the row-list fusion of
tests/ops_emulator.py); the runs other than "default" go through the index buffer and its meta row, as a captured step does, so a
small batch follows stale slots of a larger one.

(a) Calibration: the emulated default engine (eager, and the split branch schedule), the deterministic one and the hoisted one pass
every check of the run at TAU["fp32"]: gradients and losses, the AdamW update, the row sets and the forward after the run.
(b) Power: each mutation below passes step 1 and is rejected at a later step (each one is injected into the child process by a
monkeypatch):
  * `_grad_init` stops zeroing dUl / dIl after its first call;
  * `RowSet.clear` is a no-op after step 1;
  * `_batch_rows` ignores `meta` and reads the whole index buffer;
  * the optimizer's step count stops at 1 (the bias corrections freeze);
  * `forward()` returns the last step's U / I without the full fusion."""
import dataclasses
import os
import sys
import unittest.mock

import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import step_fp64_model as SM  # noqa: E402
from step_fp64_cases import _sequence, draw  # noqa: E402

KINDS = ("cap", "small", "B140", "small", "cap")
SIZES = {"cap": (128, 16), "B140": (128, 12), "small": (6, 2)}              # sampled, augmented
SEEDS = (13, 12, 11, 12, 11)                                             # cuts clear 5 x TAU_CUT["fp32"]


def tiny_batches(nu, ni):
    return _sequence("tiny", SEEDS, KINDS, batch=lambda kind, seed: draw(nu, ni, *SIZES[kind], seed))


def _engine(s, hoisted=False, det=False):
    from llmrec_b200 import ops
    from llmrec_b200.engine import HotPath
    from llmrec_b200.graph import BipartiteGraph
    from llmrec_b200.hoist import HoistedHotPath
    params = {k: v.clone() for k, v in s["params"].items()}
    feats = dict(image=s["feats"]["image"].clone(), text=s["feats"]["text"].clone(), user=s["feats"]["user"].clone(),
                 item={k: v.clone() for k, v in s["feats"]["item"].items()})
    g = BipartiteGraph(s["data"].train_mat, "cpu")
    ops_ = (g.ui, g.iu, g.uiT, g.iuT)
    cfg = dataclasses.replace(s["cfg"], deterministic=det)
    hp = HoistedHotPath(ops_, params, feats, cfg, g.ones_propagated()) if hoisted else HotPath(ops_, params, feats, cfg)
    hp.set_optimizer(lr=1e-3)
    if not hoisted:               # the batch-row fusion of the CUDA engine (HotPath.__init__ turns it on for CUDA devices only)
        hp.demand_fuse = True
        hp.batch_u, hp.batch_i, hp._batch_max = ops.RowSet(hp.nu, "cpu"), ops.RowSet(hp.ni, "cpu"), (0, 0)
    return hp


RUNS = {"default": dict(how="train_step"), "default split": dict(how="buffer", split=True),
        "deterministic": dict(how="buffer", det=True), "hoisted": dict(how="buffer", hoisted=True)}


def _mutations(done):
    """name -> patch context; `done` counts the steps of the run that passed (a patch armed 'after step 1' reads it)."""
    import ops_emulator
    from llmrec_b200 import ops
    from llmrec_b200.engine import HotPath
    grad_init, clear, batch_rows, adam_step = HotPath._grad_init, ops.RowSet.clear, HotPath._batch_rows, ops_emulator.AdamW.step
    calls = []

    def first_touch(self, id_grads=False):
        calls.append(id_grads)
        return grad_init(self, id_grads=id_grads and len(calls) == 1)

    def frozen_count(self, grads, row_masks=None):
        self.t = min(self.t, 0)
        return adam_step(self, grads, row_masks)

    P = unittest.mock.patch.object
    return {
        "_grad_init zeroes dUl / dIl on its first call only": P(HotPath, "_grad_init", first_touch),
        "RowSet.clear is a no-op after step 1": P(ops.RowSet, "clear", lambda self: None if done else clear(self)),
        "_batch_rows ignores meta": P(HotPath, "_batch_rows", lambda self, u, p, n, meta=None: batch_rows(self, u, p, n)),
        "AdamW step count stops at 1": P(ops_emulator.AdamW, "step", frozen_count),
        "forward() keeps the last step's U / I": P(HotPath, "forward", lambda self: (self.U, self.I)),
    }


def _worker(rank, ddir, out):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(4)
    import ops_emulator_ordered
    ops_emulator_ordered.install()
    import step_sequence as SQ
    from test_step_grads_fp64_cpu import _setup
    s = _setup(ddir)
    batches = tiny_batches(s["data"].n_users, s["data"].n_items)
    res = {}
    for name, r in RUNS.items():
        hp = _engine(s, r.get("hoisted", False), r.get("det", False))
        hp.force_split = r.get("split", False)
        try:
            res[name] = ("ok", SQ.run_sequence(hp, batches, "fp32", r["how"], name))
        except AssertionError as e:
            res[name] = ("failed", str(e)[:2000])
    for name in MUTATIONS:
        done = []
        hp = _engine(s)
        with _mutations(done)[name]:
            try:
                SQ.run_sequence(hp, batches, "fp32", "buffer", name, done=done)
                res[name] = ("passed every check", None)
            except AssertionError as e:
                res[name] = ("rejected after %d passing steps" % len(done), str(e)[:400])
    out[0] = res


@pytest.fixture(scope="module")
def runs(tiny_root):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(os.path.join(tiny_root, "netflix_valid_item"), out), nprocs=1, join=True)
    return dict(out[0])


@pytest.mark.parametrize("name", list(RUNS))
def test_emulated_runs_pass_every_check(runs, name):
    status, worst = runs[name]
    assert status == "ok", worst
    print(f"\n{name}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


# mutation -> the number of steps it passes: it is rejected by the checks of the next step (5: by the forward after the run)
MUTATIONS = {"_grad_init zeroes dUl / dIl on its first call only": 1, "RowSet.clear is a no-op after step 1": 1,
             "_batch_rows ignores meta": 1, "AdamW step count stops at 1": 1, "forward() keeps the last step's U / I": 5}


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_mutation_passes_step_1_and_is_rejected_later(runs, name):
    status, msg = runs[name]
    print(f"\n{name}: {status}: {msg}")
    assert status == f"rejected after {MUTATIONS[name]} passing steps", (status, msg)


def test_tiny_batches_share_rows_and_leave_stale_slots():
    """The run's batches: consecutive ones share users and items, and each large -> small change leaves live ids past B'."""
    import numpy as np
    b = tiny_batches(300, 400)
    assert [x[0].size for x in b] == [144, 8, 140, 8, 144]
    for (u0, p0, n0), (u1, p1, n1) in zip(b, b[1:]):
        assert np.intersect1d(u0, u1).size and np.intersect1d(np.r_[p0, n0], np.r_[p1, n1]).size
        assert np.setdiff1d(u0, u1).size and np.setdiff1d(u1, u0).size
