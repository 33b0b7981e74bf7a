"""-m gpu: runs of K = 5 consecutive training steps of one engine held to the fp64 step model (tests/step_fp64_model.py) at every
step, every AdamW update held to its fp64 restatement, and the full forward after the run held to `oracle.llmrec_oracle.forward`.

What one step hands to the next is what these runs check, and a single step cannot: the first touch of dUl / dIl (the batch-row
fusion backward writes the batch's rows only, so a row written by step k and not by step k + 1 must read zero in step k + 1), the
batch row sets (cleared and rebuilt every step; on the graph path from an index buffer whose slots past B' hold earlier batches' ids),
the self-resetting scratch (SpMM long-row tickets, the colsum ticket, the scaled_colsum and feat_reg_gram scratch, the BPR work block
and slot plan), AdamW's device-side step block with m and v, the graph warm-up and its undo, and the rows of U / I that evaluation and
recommendations read after training.

Before step k the fp64 reference is computed at the engine's own parameters (`SM.engine_inputs`), so the fp32 drift of the run does
not enter the bound.  After step k:
  * gradients and losses: `SM.check_cuts`, `SM.check_grads` (with the exact-zero structure rule) and `SM.check_loss` at the case's TAU,
    as tests/test_step_grads_fp64_gpu.py applies them to one step;
  * the update: one fp64 AdamW step (tests/fp64_bounds.adamw_ref) from the pre-step fp32 p, m, v at step count k, with the engine's own
    fp32 gradient, against the new p, m and v; the device step block holds k and its bias corrections (`state_ok`);
  * the row sets of the default engine: exactly the distinct users, and the distinct pos | neg items, of the step's B' live triplets.
After the run, `hp.forward()` and every row of U and I against the fp64 forward at the final parameters, per element:

    |U^_e - U_e| <= tau * (|U_e| + RHO * (max_row |U| + sum_t |c_t|))

(c_t the fusion weights of the side terms, each multiplying a unit row; an unwritten, non-finite element fails).  Calibration
(tests/test_step_sequence_fp64_cpu.py, the emulated fp32 engines after a five-step run at TAU["fp32"]): the default engines reach
0.022 of it, the hoisted one 0.033; a forward() that keeps the last step's batch-row U / I fails it.

The row-set check is what sees a row set that keeps rows of an earlier step or of the index buffer's stale slots: those rows carry
zero loss gradients, so the fusion writes the same values there and every other check passes (the CPU test shows both mutations).

Batches: step_fp64_cases.SEQUENCE = B1126, small (B' = 8), B1128, small, B1126, consecutive ones sharing users and items
(`step_fp64_cases._sequence`).  The seeds of SEQ_SEEDS are the first from 11 up whose every kept-set cut clears, along the fp64
trajectory of the shape (fp64 gradients, fp64 AdamW), 1.2 x TAU_CUT["3xtf32"] at every step (netflix: with fp32, bf16 and int8
tables alike; twice that for movielens and the odd shape); `check_cuts` asserts TAU_CUT again at the engine's own parameters.

On the H100 (SXM 80 GB) the file runs in about 40 s: each netflix case 3 s (the fp64 reference of a step on the GPU 0.1 - 0.4 s).
Largest error / bound ratios: gradients 0.29 - 0.33 at TAU["3xtf32"] (bf16 tables 0.13), 0.78 at TAU["fp32"] (mode 2), 0.29
movielens, 0.02 odd; AdamW 0.37; the forward after the run 0.04 (0.11 in mode 2).

A `graphed` case replays one captured graph for all five steps: the first `train_step_graphed` warms up, captures and replays."""
import os
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import step_fp64_model as SM  # noqa: E402
from step_fp64_cases import _engine, _sequence  # noqa: E402
from step_sequence import run_sequence  # noqa: E402

pytestmark = pytest.mark.gpu

SEQ_SEEDS = {"netflix": (94, 11, 31, 11, 16), "movielens": (86, 11, 18, 11, 13), "odd": (21, 11, 22, 15, 31)}
REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(REPORT.items()):
        print(f"\n{k}: " + ", ".join(f"{a} {b:.3g}" for a, b in v.items()), end="")
    print()


CASES = [
    # default engine
    dict(name="netflix"), dict(name="netflix", branches=False), dict(name="netflix", how="graphed"),
    dict(name="netflix", det=True, how="graphed"), dict(name="netflix", mode=2),
    # hoisted engine
    dict(name="netflix", hoisted=True), dict(name="netflix", hoisted=True, how="graphed"),
    # bf16 / int8 tables
    dict(name="netflix", dtype="bf16"), dict(name="netflix", dtype="int8", hoisted=True, how="graphed"),
    # movielens (L = 3) and the odd shape (edgeless rows, hubs longer than an SpMM tile, a SIMT projection group)
    dict(name="movielens", how="graphed"), dict(name="odd"),
]


def _id(c):
    return "-".join(f"{k}={v}" for k, v in c.items())


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_step_sequence_matches_the_fp64_model(case):
    name, dtype, hoisted, mode = case["name"], case.get("dtype", "fp32"), case.get("hoisted", False), case.get("mode", 0)
    det, how = case.get("det", False), case.get("how", "train_step")
    t0 = time.time()
    hp = _engine(name, dtype, hoisted, mode, det)
    hp.branches = hp.branches and case.get("branches", True)
    tau_name = ("3xtf32", "tf32", "fp32")[mode]
    what = f"{name} {dtype} {'hoisted' if hoisted else 'default'} mode={mode} det={det} {how} branches={hp.branches}"
    worst = run_sequence(hp, _sequence(name, SEQ_SEEDS[name]), tau_name, how, what)
    worst["seconds"] = time.time() - t0
    REPORT[_id(case)] = worst
