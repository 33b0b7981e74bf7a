"""bench_device_sampler.py -- what drawing the batches on the GPU costs or saves, per sampler mode, on one H100.

    python bench_device_sampler.py --steps 200 --blocks 5 --runs 3

Legs --device_sampler 0 (the reference's batches from the C host sampler, staged through pinned memory), 1 (the GPU's own stream) and 2
(the reference's batches drawn on the GPU) run ALTERNATELY in one process on fresh Trainers with the same seed, netflix shape, default and
hoisted engine, CUDA graph replay.  Each leg times the body of Trainer.train()'s loop (Trainer.train_next_batch: sampling, staging,
replay) between device events: --blocks blocks of --steps steps, the median block is reported per leg, the median over --runs per mode.
Then the sampler kernel alone (llmrec_device_sample_batch_ref, us per batch, events around --kernel_calls launches) at the netflix shape
and on a synthetic graph of 10 M users.  Last, legs 0 and 2 each draw --check_steps batches on fresh Trainers and the batches are compared:
the script fails if any differs.  One JSON line on stdout, a summary on stderr.  Needs a CUDA device (no fallback).
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


def _median(xs):
    s = sorted(xs)
    return s[len(s) // 2]


def _flags(mode, hoisted):
    return ["--device_sampler", str(mode), "--hoist_side", str(int(hoisted))]


def leg(mode, hoisted, a):
    import torch
    tr, gen, _ = bench.make_trainer("netflix", a, extra=_flags(mode, hoisted))
    for _ in range(a.warmup):
        tr.train_next_batch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    blocks = []
    for _ in range(a.blocks):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.steps):
            tr.train_next_batch()
        e1.record()
        torch.cuda.synchronize()
        blocks.append(e0.elapsed_time(e1) / a.steps)
    if tr.ref_sampler:
        tr.device_sampler.check()
    del tr, gen
    torch.cuda.empty_cache()
    return round(_median(blocks), 4)


def batches(mode, a, n):
    import torch
    tr, gen, _ = bench.make_trainer("netflix", a, extra=_flags(mode, False))
    out = []
    for _ in range(n):
        tr.train_next_batch()
        g = tr.hot._gidx
        out.append(g[:3, :int(g[3, 0])].cpu().clone())
    del tr, gen
    torch.cuda.empty_cache()
    return out


def kernel_us(exist, rowptr, col, n_items, batch, aug, calls):
    """us per llmrec_device_sample_batch_ref launch (CUDA events around `calls` launches after 5 warm-up launches)"""
    import torch
    from llmrec_b200.device_sampler import ReferenceDeviceSampler
    import numpy as np
    order = np.concatenate([np.sort(col[rowptr[u]:rowptr[u + 1]]) for u in range(len(rowptr) - 1)]) if len(rowptr) < 100000 else None
    if order is None:                      # sort every row at once: key = row * n_items + item
        rows = np.repeat(np.arange(len(rowptr) - 1, dtype=np.int64), np.diff(rowptr))
        order = col[np.lexsort((col, rows))]
    ds = ReferenceDeviceSampler(exist, rowptr, col, order, n_items, batch, aug[0], aug[1], n_items, 0.1, "cuda")
    cap = 2 * batch + 8
    buf = torch.zeros((4, cap), dtype=torch.int32, device="cuda")
    meta = torch.arange(cap + 1, dtype=torch.int32, device="cuda").repeat_interleave(2).view(-1, 2).contiguous()
    for _ in range(5):
        ds.fill(buf, meta)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        ds.fill(buf, meta)
    e1.record()
    torch.cuda.synchronize()
    ds.check()
    return round(1e3 * e0.elapsed_time(e1) / calls, 2)


def synthetic(n_users, n_items, deg, seed=0):
    import numpy as np
    rng = np.random.default_rng(seed)
    d = rng.integers(1, 2 * deg, n_users)
    rowptr = np.zeros(n_users + 1, dtype=np.int64)
    np.cumsum(d, out=rowptr[1:])
    col = (rng.pareto(1.2, int(rowptr[-1])) * 50).astype(np.int64) % n_items
    aug = (rng.integers(0, n_items + n_items // 10, n_users), rng.integers(0, n_items, n_users))
    return np.arange(n_users), rowptr.astype(np.int32), col.astype(np.int32), aug


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="steps per timed block")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3, help="alternating runs of the three legs")
    ap.add_argument("--kernel_calls", type=int, default=200)
    ap.add_argument("--check_steps", type=int, default=100)
    c = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_sampler.py needs a CUDA (H100) device")
    a = types.SimpleNamespace(proj_mode="3xtf32", host_sampler="native", graph=1, steps=c.steps, warmup=c.warmup, blocks=c.blocks)
    name, limit = card()
    result = {"metric": "device_sampler_ab", "gpu": name, "power_limit": limit, "workload": bench.workload_string("netflix"),
              "timing": f"Trainer.train_next_batch, CUDA graph replay; median of {c.blocks} blocks of {c.steps} steps per leg, "
                        f"median of {c.runs} alternating runs per mode", "engines": {}}
    for hoisted in (False, True):
        runs = {0: [], 1: [], 2: []}
        for _ in range(c.runs):
            for mode in (0, 1, 2):
                runs[mode].append(leg(mode, hoisted, a))
        eng = "hoisted" if hoisted else "default"
        result["engines"][eng] = {"ms_per_step": {str(m): _median(v) for m, v in runs.items()}, "runs": {str(m): v for m, v in runs.items()}}
        for m, v in runs.items():
            sys.stderr.write(f"{eng:8s} --device_sampler {m}: {_median(v):.4f} ms/step  (runs {v})\n")
    # the kernel alone
    tr, gen, _ = bench.make_trainer("netflix", a, extra=_flags(2, False))
    ds = tr.device_sampler
    nf = dict(exist=ds.exist.cpu().numpy(), rowptr=ds.rowptr.cpu().numpy(), col=ds.col.cpu().numpy(), n_items=ds.n_items, batch=ds.batch,
              aug=(ds.aug_pos.cpu().numpy(), ds.aug_neg.cpu().numpy()))
    del tr, gen, ds
    torch.cuda.empty_cache()
    us_nf = kernel_us(**nf, calls=c.kernel_calls)
    ex, rp, col, aug = synthetic(10_000_000, 1_000_000, 5)
    us_10m = kernel_us(ex, rp, col, 1_000_000, nf["batch"], aug, c.kernel_calls)
    result["kernel_us_per_batch"] = {"netflix": us_nf, "10M_users_1M_items": us_10m, "batch": nf["batch"], "aug_sample_rate": 0.1}
    sys.stderr.write(f"sampler kernel: {us_nf} us/batch at the netflix shape, {us_10m} us/batch with 10 M users\n")
    # legs 0 and 2 draw the same batches
    x, y = batches(0, a, c.check_steps), batches(2, a, c.check_steps)
    same = len(x) == len(y) and all(torch.equal(p, q) for p, q in zip(x, y))
    result["identical_batches_0_vs_2"] = {"steps": c.check_steps, "identical": same}
    sys.stderr.write(f"--device_sampler 0 and 2 drew identical batches over {c.check_steps} steps: {same}\n")
    print(json.dumps(result), flush=True)
    if not same:
        raise SystemExit("--device_sampler 2 drew other batches than --device_sampler 0")


if __name__ == "__main__":
    main()
