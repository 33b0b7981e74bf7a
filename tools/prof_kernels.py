"""Micro-driver for the hot kernel families.

  prof_kernels.py [all|proj|spmm]   one NF-shaped call of each family (projection fwd / wgrad groups on full tables, SpMM launches)
  prof_kernels.py step [--dump DIR | --compare DIR] [--lib-root TREE]
      the grouped projections at the training step's own shapes: the item tables on the live items, their weight gradient paired
      with column blocks of GPi through the sorted live-row map, the user table in full (netflix d = 64, movielens d = 128), for
      fp32 and bf16 tables and modes 0 and 1.  Each group is replayed from its own CUDA graph between CUDA events (median of
      5 x 50 replays).  --dump writes Y, dW and db of every set, --compare checks them bit for bit against a dump; --lib-root imports
      the package from another tree (e.g. a worktree of an earlier commit, built) so that two builds see the same inputs.
"""
import argparse, os, subprocess, sys

ap = argparse.ArgumentParser()
ap.add_argument("which", nargs="?", default="all", choices=("all", "proj", "spmm", "step"))
ap.add_argument("--dump", metavar="DIR")
ap.add_argument("--compare", metavar="DIR")
ap.add_argument("--lib-root", metavar="TREE", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.lib_root))
import numpy as np
import scipy.sparse as sp
import torch
from llmrec_b200 import ops
from llmrec_b200.graph import BipartiteGraph

torch.manual_seed(0)
dev = "cuda"
nu, ni, d = 13187, 17366, int(os.environ.get("D", 64))
which = args.which
reps = int(os.environ.get("REPS", 3))
mode = int(os.environ.get("MODE", 0))
if which in ("all", "proj"):
    dims = [(ni, 1536)] * 5 + [(nu, 1536), (ni, 768), (ni, 512)]
    Xs = [torch.randn(n, k, device=dev) for n, k in dims]
    Ws = {k: torch.randn(d, k, device=dev) / k ** 0.5 for k in (1536, 768, 512)}
    Wu = torch.randn(d, 1536, device=dev) / 39.0
    b = torch.zeros(d, device=dev)
    outs = [torch.empty(n, d, device=dev) for n, _ in dims]
    fw = [(X, (Wu if i == 5 else Ws[X.shape[1]]), b, o) for i, (X, o) in enumerate(zip(Xs, outs))]
    dWs = [torch.empty(d, X.shape[1], device=dev) for X in Xs]
    dbs = [torch.empty(d, device=dev) for _ in Xs]
    wg = [(X, o, dW, db_, False) for X, o, dW, db_ in zip(Xs, outs, dWs, dbs)]
    for _ in range(reps):
        ops.proj_fwd_group(fw, d, mode)
        ops.proj_wgrad_group(wg, d, mode)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, fn in (("fwd", lambda: ops.proj_fwd_group(fw, d, mode)), ("wgrad", lambda: ops.proj_wgrad_group(wg, d, mode))):
        e0.record()
        for _ in range(10):
            fn()
        e1.record(); torch.cuda.synchronize()
        byts = sum(4 * n * k + 4 * k * d + 4 * n * d for n, k in dims)
        ms = e0.elapsed_time(e1) / 10
        print(f"proj_{name}: {ms:.4f} ms  {byts / ms / 1e6:.1f} GB/s", flush=True)
if which in ("all", "spmm"):
    rng = np.random.default_rng(0)
    w = 1.0 / np.power(np.arange(ni) + 8.0, 0.8); w /= w.sum()
    rows = rng.integers(0, nu, 43000); cols = rng.choice(ni, size=43000, p=w)
    m = sp.csr_matrix((np.ones(43000, np.float32), (rows, cols)), shape=(nu, ni)); m.sum_duplicates(); m.data[:] = 1
    for tile in (0, 8, 16, 32):
        g = BipartiteGraph(m, dev, tile_nnz=tile)
        for S in (8, 1):
            Xi = torch.randn(ni, S * d, device=dev); Yu = torch.empty(nu, S * d, device=dev); Yi = torch.empty(ni, S * d, device=dev)
            su = [(Xi[:, s * d:(s + 1) * d], Yu[:, s * d:(s + 1) * d], None, False) for s in range(S)]
            si = [(Yu[:, s * d:(s + 1) * d], Yi[:, s * d:(s + 1) * d], None, False) for s in range(S)]
            for _ in range(reps):
                g.ui.apply(su); g.iu.apply(si)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for name, op, segs in (("ui", g.ui, su), ("iu", g.iu, si)):
                e0.record()
                for _ in range(20):
                    op.apply(segs)
                e1.record(); torch.cuda.synchronize()
                print(f"spmm tile={tile} S={S} {name}: {e0.elapsed_time(e1) / 20 * 1e3:.1f} us  max_deg={int((op.rowptr[1:] - op.rowptr[:-1]).max())}", flush=True)


# ---- the step's projection groups -------------------------------------------------------------------------------------------
# (users, items, live items, d): netflix is the flagship workload; movielens runs at d = 128.  Tables: 5 attribute tables
# (k = 1536, sharing item_trans), text (768), image (512) on the live items, the user-profile table (1536) on every user.
STEP_SETS = {"netflix": (13187, 17366, 12174, 64), "movielens": (12495, 10322, 8055, 128)}


def gpu_line():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name()
    return f"card, power limit, SM clock, max SM clock: {out}"


def step_problems(name, dtype):
    nu_, ni_, nl, d_ = STEP_SETS[name]
    g = torch.Generator(device=dev).manual_seed(1234 + d_)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    live = torch.sort(torch.randperm(ni_, device=dev, generator=g)[:nl]).values.to(torch.int32).contiguous()
    X = [rnd(nl, 1536) for _ in range(5)] + [rnd(nl, 768), rnd(nl, 512)]
    Xu = rnd(nu_, 1536)
    X, Xu = [x.to(dtype) for x in X], Xu.to(dtype)
    GPi, GPu = rnd(ni_, 7 * d_), rnd(nu_, d_)               # GPi: column block 0 image, 1 text, 2.. attributes (the engine's layout)
    blk = lambda s: GPi[:, s * d_:(s + 1) * d_]
    W = {k: rnd(d_, k) / k ** 0.5 for k in (1536, 768, 512)}
    Wu, b = rnd(d_, 1536) / 39.0, rnd(d_)
    Pi, Pu = torch.zeros(ni_, 7 * d_, device=dev), torch.empty(nu_, d_, device=dev)
    grads = {key: torch.empty(d_, k, device=dev) for key, k in (("item", 1536), ("user", 1536), ("text", 768), ("image", 512))}
    gradb = {key: torch.empty(d_, device=dev) for key in grads}
    fw = [(X[j], W[1536], b, Pi[:, (2 + j) * d_:(3 + j) * d_], live) for j in range(5)]
    fw += [(Xu, Wu, b, Pu), (X[5], W[768], b, Pi[:, d_:2 * d_], live), (X[6], W[512], b, Pi[:, :d_], live)]
    wg = [(X[j], blk(2 + j), grads["item"], gradb["item"], j > 0, live) for j in range(5)]
    wg += [(Xu, GPu, grads["user"], gradb["user"], False), (X[5], blk(1), grads["text"], gradb["text"], False, live),
           (X[6], blk(0), grads["image"], gradb["image"], False, live)]
    return d_, fw, wg, grads, gradb


def graph_ms(fn, rounds=5, replays=50):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        fn()
    gr.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(rounds):
        e0.record()
        for _ in range(replays):
            gr.replay()
        e1.record(); torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / replays)
    return float(np.median(out))


if which == "step":
    print(gpu_line(), flush=True)
    bad = 0
    for name in STEP_SETS:
        for dtype in (torch.float32, torch.bfloat16):
            for m in (0, 1):
                tag = f"{name}_{str(dtype).split('.')[-1]}_mode{m}"
                d_, fw, wg, grads, gradb = step_problems(name, dtype)
                t_fwd = graph_ms(lambda: ops.proj_fwd_group(fw, d_, m))
                t_wg = graph_ms(lambda: ops.proj_wgrad_group(wg, d_, m))
                ops.proj_fwd_group(fw, d_, m); ops.proj_wgrad_group(wg, d_, m); torch.cuda.synchronize()
                res = {f"dW_{k}": v.cpu() for k, v in grads.items()} | {f"db_{k}": v.cpu() for k, v in gradb.items()}
                res |= {f"Y_{j}": f[3].cpu() for j, f in enumerate(fw)}
                line = f"{tag}: proj_fwd {t_fwd:.4f} ms  proj_wgrad {t_wg:.4f} ms"
                if args.dump:
                    os.makedirs(args.dump, exist_ok=True)
                    torch.save(res, os.path.join(args.dump, tag + ".pt"))
                if args.compare:
                    ref = torch.load(os.path.join(args.compare, tag + ".pt"))
                    diff = [k for k in ref if not torch.equal(ref[k].view(torch.int32), res[k].view(torch.int32))]
                    bad += len(diff)
                    line += "  Y/dW/db bit-identical" if not diff else f"  DIFFERENT: {diff}"
                print(line, flush=True)
    if bad:
        sys.exit(1)
