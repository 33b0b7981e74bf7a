"""bench_feat_dtype.py -- fp32 vs bf16 (vs int8) side-feature tables (--feat_dtype) on one H100.

    python bench_feat_dtype.py --steps 50 --blocks 5 --runs 3 [--dtypes fp32,bf16,int8]

For the netflix-shaped (d = 64) and movielens-shaped (d = 128, L = 3) workloads of bench.py, the legs of --dtypes (default fp32,bf16)
run ALTERNATELY in one process (fp32, bf16, fp32, bf16, ...), each on a fresh Trainer with the same seed, so clock and thermal drift
hit all alike.  Every leg reports ms/step (median of --blocks blocks of --steps device-resident steps, min and max), the
proj_fwd / proj_wgrad family times with GB/s from roofline's algorithmic bytes, the resident feature bytes (an int8 table's row
scales and padding included), eval users/s and the leg's Recall@20 / NDCG@20 (bf16 and int8 legs train on rounded tables).  One JSON line on stdout; a summary table on stderr.  Needs a CUDA device (no fallback).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import types

REPO = os.path.dirname(os.path.abspath(__file__))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import bench  # noqa: E402


def card():
    """(name, power limit) of GPU 0 from a query-only nvidia-smi call."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (x.strip() for x in out.split(",")[:2])
        return name, limit
    except Exception as e:
        return None, repr(e)[:100]


def feature_bytes(model):
    bufs = [model.image_feats, model.text_feats, model.user_feats] + list(model.item_feats.values())
    return sum(t.numel() * t.element_size() for t in bufs)


def leg(workload, feat_dtype, a):
    import torch
    from llmrec_b200.roofline import step_bytes
    tr, gen, args = bench.make_trainer(workload, a, extra=["--feat_dtype", feat_dtype])
    t = bench.time_steps(tr, a, a.steps, a.warmup, float("inf"), a.blocks)     # exactly --blocks blocks
    fam = bench.family_times(tr, t["dev_batches"][0])
    by = step_bytes(tr.hot, tr.graph.nnz)
    ev = bench.eval_leg(tr, gen, tr.n_items)
    out = {"feat_dtype": feat_dtype, "ms_per_step": round(t["ms"] / a.steps, 4), "ms_per_step_min": round(t["ms_min"] / a.steps, 4),
           "ms_per_step_max": round(t["ms_max"] / a.steps, 4), "blocks": t["blocks"], "launches_per_block": t["launches"],
           "feature_bytes": feature_bytes(tr.model_mm)}
    for f in ("proj_fwd", "proj_wgrad"):
        out[f + "_ms"] = round(fam[f], 4)
        out[f + "_gbs"] = round(by[f] / (fam[f] * 1e-3) / 1e9, 1)
    out["eval_users_per_sec"] = ev["value"]
    out["recall@20"], out["ndcg@20"] = ev["recall@20"], ev["ndcg@20"]
    del tr, gen
    torch.cuda.empty_cache()
    return out


def _median(xs):
    s = sorted(xs)
    return s[len(s) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="steps per timed block")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=5, help="timed blocks per leg (the median is reported)")
    ap.add_argument("--runs", type=int, default=3, help="alternating runs of the --dtypes legs per workload")
    ap.add_argument("--dtypes", default="fp32,bf16", help="comma-separated --feat_dtype legs, run in this order (fp32 first: speedups are vs fp32)")
    ap.add_argument("--workloads", default="netflix,movielens")
    ap.add_argument("--proj_mode", default="3xtf32")
    ap.add_argument("--graph", type=int, default=1)
    c = ap.parse_args()
    dtypes = c.dtypes.split(",")
    if not dtypes or any(dt not in ("fp32", "bf16", "int8") for dt in dtypes) or len(set(dtypes)) != len(dtypes):
        raise SystemExit(f"--dtypes: a list of distinct fp32 / bf16 / int8, got {c.dtypes!r}")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_feat_dtype.py needs a CUDA (H100) device")
    a = types.SimpleNamespace(proj_mode=c.proj_mode, host_sampler="native", graph=c.graph, max_blocks=c.blocks,
                              steps=c.steps, warmup=max(c.warmup, 3), blocks=c.blocks)
    name, limit = card()
    result = {"metric": "feat_dtype_ab", "gpu": name, "power_limit": limit, "proj_mode": c.proj_mode, "cuda_graph": bool(c.graph),
              "timing": f"median of {c.blocks} blocks of {c.steps} device-resident steps per leg; legs alternate {' / '.join(dtypes)}", "workloads": {}}
    for wl in c.workloads.split(","):
        runs = {dt: [] for dt in dtypes}
        for _ in range(c.runs):
            for dt in dtypes:
                runs[dt].append(leg(wl, dt, a))
        summary = {dt: {k: _median([r[k] for r in rs]) for k in ("ms_per_step", "proj_fwd_ms", "proj_wgrad_ms", "eval_users_per_sec")}
                   for dt, rs in runs.items()}
        if dtypes == ["fp32", "bf16"]:
            summary["speedup_ms_per_step"] = round(summary["fp32"]["ms_per_step"] / summary["bf16"]["ms_per_step"], 3)
        elif len(dtypes) > 1:
            summary["speedup_ms_per_step"] = {dt: round(summary[dtypes[0]]["ms_per_step"] / summary[dt]["ms_per_step"], 3) for dt in dtypes[1:]}
        result["workloads"][wl] = {"workload": bench.workload_string(wl), "runs": runs, "median_of_runs": summary}
        for dt, rs in runs.items():
            for r in rs:
                sys.stderr.write(f"{wl:9s} {dt}: {r['ms_per_step']:.4f} ms/step [{r['ms_per_step_min']:.4f}, {r['ms_per_step_max']:.4f}]  "
                                 f"proj_fwd {r['proj_fwd_ms']:.4f} ms ({r['proj_fwd_gbs']} GB/s)  proj_wgrad {r['proj_wgrad_ms']:.4f} ms "
                                 f"({r['proj_wgrad_gbs']} GB/s)  features {r['feature_bytes'] / 1e6:.1f} MB  eval {r['eval_users_per_sec']} users/s  "
                                 f"R@20 {r['recall@20']:.5f} N@20 {r['ndcg@20']:.5f}\n")
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
