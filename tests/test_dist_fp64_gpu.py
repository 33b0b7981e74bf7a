"""-m gpu: the sharded engines' training steps held to the fp64 step model (tests/dist_fp64.py): dist.ShardedHotPath (dense,
demand-driven at d = 32 / 64 / 128, item-row pieces, item-sharded) and dist_feat.ShardedFeatureHotPath (proj_mode 0 and 2) over the
five-step SEQUENCE on the netflix-like and the odd graphs, every step's gradients, losses and AdamW update (p, m, v) checked.

World 1 runs in this process (dist_fp64.CASES_W1).  World 2 (dist_fp64.CASES_W2: uneven user ranges, item_sharded, the demand
mode's item_opt_sharded, uneven item ranges taking the all-reduce forms, dist_feat's even and uneven item ranges) runs
tests/dist_fp64_check.py under torch.distributed.run over NCCL once for all its cases, and skips when fewer than two GPUs are
visible.  Each case prints its worst gradient and AdamW error as a fraction of the bound."""
import json
import os
import subprocess
import sys
import time

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dist_fp64 as DF  # noqa: E402

pytestmark = pytest.mark.gpu
_W2 = {}


def _report(world, case, res):
    print(f"\nworld {world} {DF.case_id(case)}: grads {res['grads']:.3g}, adamw {res['adamw']:.3g} of the bound, "
          f"{res.get('seconds', 0):.1f} s; {res['forms']}")


@pytest.mark.parametrize("case", DF.CASES_W1, ids=DF.case_id)
def test_sharded_step_world1_matches_the_fp64_model(case):
    t0 = time.time()
    res = DF.run_case(case, torch.device("cuda"))
    res["seconds"] = time.time() - t0
    _report(1, case, res)
    assert not res["errors"], "\n".join(res["errors"][:6])


def _world2():
    if not _W2:
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                            "127.0.0.1", "--master-port", "29531", os.path.join(HERE, "dist_fp64_check.py")],
                           capture_output=True, text=True, timeout=1800)
        assert "DIST_FP64_DONE" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
        for line in r.stdout.splitlines():
            if line.startswith("DIST_FP64 "):
                res = json.loads(line[len("DIST_FP64 "):])
                _W2[res["case"]] = res
    return _W2


@pytest.mark.parametrize("case", DF.CASES_W2, ids=DF.case_id)
def test_sharded_step_world2_matches_the_fp64_model(case):
    if torch.cuda.device_count() < 2:
        pytest.skip("world 2 needs two visible GPUs")
    res = _world2()[DF.case_id(case)]
    _report(2, case, res)
    assert not res["errors"], "\n".join(res["errors"][:6])
    forms = res["forms"]
    if case.get("item_sharded"):
        assert forms["item_sharded"] == (case["shape"] != "odd-uneven")
    if case.get("demand"):
        assert forms["item_opt_sharded"] == (case["shape"] != "odd-uneven")
    if case.get("engine") == "feat":
        assert forms["even_items"] == (case["shape"] != "odd-uneven")
