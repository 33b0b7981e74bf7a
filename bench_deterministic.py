"""bench_deterministic.py -- what bit-reproducible steps (--deterministic 1) cost on one H100.

    python bench_deterministic.py --steps 50 --blocks 5 --runs 3 [--repro_steps 20]

For the netflix-shaped (d = 64) and movielens-shaped (d = 128, L = 3) workloads of bench.py, the legs --deterministic 0 and 1 run
ALTERNATELY in one process, each on a fresh Trainer with the same seed, so clock and thermal drift hit both alike.  Every leg reports
ms/step (median of --blocks blocks of --steps graph-replayed, device-resident steps between device events with a synchronise on both
sides; min and max) and the loss_heads family time (HotPath.families; on the deterministic leg it includes the slot plan, which a whole
step builds on a side branch).  A reproducibility line per leg: two fresh Trainers run the same --repro_steps seeded batches and the
largest absolute difference between their parameters is printed -- exactly 0 on the deterministic leg, or the script fails; whatever the
float atomics give on the default leg.  One JSON line on stdout; a summary on stderr.  Needs a CUDA device (no fallback).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import types

REPO = os.path.dirname(os.path.abspath(__file__))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import bench  # noqa: E402
from bench_feat_dtype import card  # noqa: E402


def leg(workload, det, a):
    import torch
    tr, gen, args = bench.make_trainer(workload, a, extra=["--deterministic", str(det)])
    t = bench.time_steps(tr, a, a.steps, a.warmup, float("inf"), a.blocks)     # exactly --blocks blocks
    fam = bench.family_times(tr, t["dev_batches"][0])
    out = {"deterministic": det, "ms_per_step": round(t["ms"] / a.steps, 4), "ms_per_step_min": round(t["ms_min"] / a.steps, 4),
           "ms_per_step_max": round(t["ms_max"] / a.steps, 4), "blocks": t["blocks"], "launches_per_block": t["launches"],
           "loss_heads_ms": round(fam["loss_heads"], 4)}
    del tr, gen
    torch.cuda.empty_cache()
    return out


def final_params(workload, det, a, steps):
    import torch
    tr, gen, args = bench.make_trainer(workload, a, extra=["--deterministic", str(det)])
    for _ in range(steps):
        tr.train_next_batch()                     # seeded host sampler -> staging -> graph replay: the loop of Trainer.train()
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in tr.hot.p.items()}


def repro(workload, det, a, steps):
    """max |p_run1 - p_run2| over all parameters after `steps` identical batches on two fresh Trainers"""
    import torch
    x, y = final_params(workload, det, a, steps), final_params(workload, det, a, steps)
    worst = max(float((x[k] - y[k]).abs().max()) for k in x)
    same = all(torch.equal(x[k], y[k]) for k in x)
    del x, y
    torch.cuda.empty_cache()
    return worst, same


def _median(xs):
    s = sorted(xs)
    return s[len(s) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="steps per timed block (>= 50)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=5, help="timed blocks per leg (the median is reported)")
    ap.add_argument("--runs", type=int, default=3, help="alternating runs of the two legs per workload")
    ap.add_argument("--repro_steps", type=int, default=20, help="steps of the reproducibility check")
    ap.add_argument("--workloads", default="netflix,movielens")
    ap.add_argument("--proj_mode", default="3xtf32", choices=["3xtf32", "tf32"])
    c = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic.py needs a CUDA (H100) device")
    a = types.SimpleNamespace(proj_mode=c.proj_mode, host_sampler="native", graph=1, max_blocks=c.blocks,
                              steps=max(c.steps, 50), warmup=max(c.warmup, 3), blocks=c.blocks)
    name, limit = card()
    result = {"metric": "deterministic_ab", "gpu": name, "power_limit": limit, "proj_mode": c.proj_mode, "cuda_graph": True,
              "timing": f"median of {c.blocks} blocks of {a.steps} device-resident steps per leg; legs alternate deterministic 0 / 1", "workloads": {}}
    failed = False
    for wl in c.workloads.split(","):
        runs = {0: [], 1: []}
        for _ in range(c.runs):
            for det in (0, 1):
                runs[det].append(leg(wl, det, a))
        summary = {str(det): {k: _median([r[k] for r in rs]) for k in ("ms_per_step", "loss_heads_ms")} for det, rs in runs.items()}
        summary["slowdown_ms_per_step"] = round(summary["1"]["ms_per_step"] / summary["0"]["ms_per_step"], 4)
        rep = {}
        for det in (0, 1):
            worst, same = repro(wl, det, a, c.repro_steps)
            rep[str(det)] = {"steps": c.repro_steps, "max_abs_param_diff": worst, "bit_identical": same}
            sys.stderr.write(f"{wl:9s} deterministic={det}: two runs of {c.repro_steps} steps differ by at most {worst:.3g} (bit-identical: {same})\n")
        failed |= not rep["1"]["bit_identical"]
        result["workloads"][wl] = {"workload": bench.workload_string(wl), "runs": {str(k): v for k, v in runs.items()}, "median_of_runs": summary,
                                   "reproducibility": rep}
        for det, rs in runs.items():
            for r in rs:
                sys.stderr.write(f"{wl:9s} deterministic={det}: {r['ms_per_step']:.4f} ms/step [{r['ms_per_step_min']:.4f}, {r['ms_per_step_max']:.4f}]  "
                                 f"loss_heads {r['loss_heads_ms']:.4f} ms\n")
    print(json.dumps(result), flush=True)
    if failed:
        raise SystemExit("--deterministic 1: two runs on the same batches gave different parameters")


if __name__ == "__main__":
    main()
