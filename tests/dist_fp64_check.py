"""The sharded engines' steps against the fp64 step model on GPUs, every case of tests/dist_fp64.CASES_W2 (or CASES_W1 at world 1).
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29531 tests/dist_fp64_check.py
Rank 0 prints one line per case: DIST_FP64 <json> with the case, the worst gradient / AdamW ratios, the exchange forms that ran
and every rank's failures; DIST_FP64_DONE at the end."""
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import dist_fp64 as DF  # noqa: E402


def main():
    world = int(os.environ.get("WORLD_SIZE", 1)); rank = int(os.environ.get("RANK", 0))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    if world > 1:
        dist.init_process_group("nccl")
    dev = torch.device("cuda")
    for case in (DF.CASES_W2 if world > 1 else DF.CASES_W1):
        t0 = time.time()
        try:
            res = DF.run_case(case, dev)
        except Exception as e:                        # a failure outside the checks is reported as the case's error
            res = dict(grads=float("inf"), adamw=float("inf"), errors=[f"{type(e).__name__}: {e}"], forms={})
        res["seconds"] = time.time() - t0
        parts = [None] * world
        if world > 1:
            dist.all_gather_object(parts, res)
        else:
            parts = [res]
        if rank == 0:
            print("DIST_FP64 " + json.dumps(dict(case=DF.case_id(case), **DF.merge_ranks(parts))), flush=True)
    if rank == 0:
        print("DIST_FP64_DONE", flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
