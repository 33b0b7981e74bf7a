"""bench_recommend.py -- recommendation throughput (Trainer.recommend / recommend.top_k, --candidates_out, item fold-in and item-to-item
neighbours) on one H100.

    python bench_recommend.py [--reps 3] [--syn_users 131072] [--syn_histories 8192] [--syn_items 65536] [--syn_scale 1.0]
                              [--pairs 1048576] [--legs rerank,score_pairs,explain,diversify]

Eleven legs per workload, each timed end to end on the host clock between device synchronises (median of --reps calls after one
warm-up call):
  known         trained users scored from U with their training items excluded (exclude="train"), K = 10; users/s
  fold_in       held-out histories folded in (HotPath.fold_in) and scored, exclude="train", K = 10; users/s
  candidates    the --candidates_out file: every user's top-10 over the whole catalog, nothing excluded, pickled to a temporary file;
                users/s
  fold_in_items trained items' user lists folded in as new items (HotPath.fold_in_items, no ID embedding); items/s
  similar       item-to-item neighbours (recommend.similar_items) of trained items over the trained catalog, K = 10; queries/s
  rerank        every user (synthetic: --syn_users users) re-ranks --rerank_c random candidates (netflix 100, synthetic 200), K = 10,
                nothing excluded (Trainer.rerank / recommend.rerank); queries/s and candidates/s
  score_pairs   --pairs random (trained user, trained item) pairs scored (Trainer.score / recommend.score_pairs); pairs/s
  among         the known leg over a catalog of 1 %, 10 % and 100 % of the items (recommend.top_k(among=...)); users/s.  Each size also
                times its kernel alone (llmrec_score_topk_among_f32, all users in one launch, between CUDA events), the plain call
                (llmrec_score_topk_f32 over the whole catalog) and, where the [users x |among|] candidate CSR fits in int32, the same
                question answered by llmrec_rerank_f32 with the set as every user's list
  explain       the known leg's top-10 of every user (synthetic: --syn_users users) explained (Trainer.explain / recommend.explain:
                every (target, history item, channel) contribution, own and last); queries/s.  Also times the kernel alone
                (llmrec_explain_f32, all queries in one launch, between CUDA events, median of 5 windows of 20 launches) and reports
                it as GB/s of gathered rows: per query its 10 target rows, its two user rows and, per history item, the n_id + n_side
                source rows (4*d bytes each)
  diversify     diversified lists, lambda = 0.5, K = 10 (Trainer.recommend / recommend.top_k / recommend.rerank with diversity=):
                every user's (synthetic: --syn_users users') pick from the top-64 pool of `recommend`, and at the synthetic shape also
                from the re-ranked pool of 200 random candidates; queries/s.  Also times the kernel alone on the same pools
                (llmrec_diversify_f32, all queries in one launch, between CUDA events, median of 5 windows of 20 launches) and reports,
                for lambda = 1, 0.7 and 0.5, the lists' mean pairwise cosine of the normalised item rows and their mean score (lambda = 1
                is the plain top-10 of the pool)
  groups        group lists, K = 10, exclude="train" (Trainer.recommend_groups / recommend.top_k_groups): every user (synthetic: the
                first 131,072 = 4 x 32,768) in random groups of 4, agg mean and min; groups/s.  Also times the kernel alone
                (llmrec_score_topk_group_f32, all groups in one launch, between CUDA events) next to llmrec_score_topk_f32 for the same
                members one by one, the known leg's kernel
Every call includes the full eval forward a recommendation starts with.  The rerank and score_pairs legs also time their kernel alone
(llmrec_rerank_f32 / llmrec_score_pairs_f32 between CUDA events, median of 5 windows of 20 launches) and report it as GB/s of gathered
rows: 4*d bytes per candidate row plus 4 per id (pairs: two rows and two ids), against the size of I (L2-resident at netflix,
HBM-resident at the synthetic shape).
Workloads: the netflix shape of bench.py (Trainer with side features, held-out histories = a user's training row plus its test items;
every item's user list and every item as a query), and the 10M x 1M x 200M synthetic of dist_bench (ID-only single-GPU engine,
d = 128, L = 2; histories = a training row plus two random items, folded in as unknown users; the known and candidates legs score the
first --syn_users users; the item legs take --syn_items random items).
One JSON line on stdout with the card's name and power limit; a summary on stderr.  Needs a CUDA device (no fallback).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time
import types

REPO = os.path.dirname(os.path.abspath(__file__))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import bench  # noqa: E402
from bench_feat_dtype import card  # noqa: E402


def _timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2], min(ts), max(ts)


ONLY = set()               # --legs: the legs to run (empty: all)


def _leg(name, n_users, fn, reps, unit="users", label=None):
    if ONLY and name not in ONLY:
        return None
    med, lo, hi = _timed(fn, reps)
    out = {unit: n_users, "s_per_call": round(med, 5), "s_min": round(lo, 5), "s_max": round(hi, 5), unit + "_per_s": round(n_users / med, 1)}
    sys.stderr.write(f"  {label or name:13s} {n_users:9d} {unit:7s}  {med * 1e3:9.2f} ms/call  {n_users / med:12.0f} {unit}/s\n")
    return out


def _kernel(fn, reps=20, windows=5):
    """median seconds per launch of `fn` between CUDA events"""
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3 / reps)
    return sorted(ts)[len(ts) // 2]


def _serving_legs(U, I, e2e_rerank, e2e_pairs, n_q, c, n_pairs, reps, seed=0):
    """The rerank and score_pairs legs: end to end (`e2e_*`, given the candidates / pairs) and the kernel alone on U / I"""
    import torch
    from llmrec_b200 import ops
    dev, d = U.device, int(U.shape[1])
    g = torch.Generator(device=dev).manual_seed(seed)
    cand = torch.randint(0, I.shape[0], (n_q, c), device=dev, generator=g, dtype=torch.int32)
    qrow = torch.arange(n_q, dtype=torch.int32, device=dev)
    rp = torch.arange(n_q + 1, dtype=torch.int32, device=dev) * c
    col = cand.reshape(-1).contiguous()
    pu = torch.randint(0, U.shape[0], (n_pairs,), device=dev, generator=g, dtype=torch.int32)
    pi = torch.randint(0, I.shape[0], (n_pairs,), device=dev, generator=g, dtype=torch.int32)
    i_mb = I.shape[0] * d * 4 / 1e6
    if ONLY and "rerank" not in ONLY and "score_pairs" not in ONLY:
        return {}
    rr = _leg("rerank", n_q, lambda: e2e_rerank(cand), reps, unit="queries")
    if rr is None:
        return {"score_pairs": _pairs_legs(U, I, e2e_pairs, pu, pi, reps)}
    rr["candidates_per_s"] = round(n_q * c / rr["s_per_call"], 1)
    k = _kernel(lambda: ops.rerank(U, I, qrow, rp, col, None, None, 10))
    rr.update(candidates_per_query=c, kernel_s=round(k, 7), kernel_queries_per_s=round(n_q / k, 1),
              kernel_candidates_per_s=round(n_q * c / k, 1), kernel_GB_per_s=round(n_q * c * (4 * d + 4) / k / 1e9, 1), I_MB=round(i_mb, 1))
    sys.stderr.write(f"  {'rerank kernel':13s} {n_q:9d} queries  {k * 1e3:9.3f} ms       {n_q * c / k:12.0f} cand/s  "
                     f"{rr['kernel_GB_per_s']:7.1f} GB/s (I: {i_mb:.1f} MB)\n")
    return {"rerank": rr, "score_pairs": _pairs_legs(U, I, e2e_pairs, pu, pi, reps)}


def _pairs_legs(U, I, e2e_pairs, pu, pi, reps):
    from llmrec_b200 import ops
    n_pairs, d = int(pu.numel()), int(U.shape[1])
    sp_ = _leg("score_pairs", n_pairs, lambda: e2e_pairs(pu, pi), reps, unit="pairs")
    if sp_ is None:
        return None
    k = _kernel(lambda: ops.score_pairs(U, I, pu, pi))
    sp_.update(kernel_s=round(k, 7), kernel_pairs_per_s=round(n_pairs / k, 1), kernel_GB_per_s=round(n_pairs * (8 * d + 8) / k / 1e9, 1))
    sys.stderr.write(f"  {'pairs kernel':13s} {n_pairs:9d} pairs    {k * 1e3:9.3f} ms       {n_pairs / k:12.0f} pairs/s "
                     f"{sp_['kernel_GB_per_s']:7.1f} GB/s\n")
    return sp_


def _among_legs(U, I, mask_rowptr, mask_col, e2e, n_q, mode, reps, seed=0):
    """The among leg at 1 %, 10 % and 100 % of the catalog: end to end (`e2e(ids)`), and the kernels alone for the same users"""
    import torch
    from llmrec_b200 import ops
    if ONLY and "among" not in ONLY:
        return None
    dev, ni = U.device, int(I.shape[0])
    g = torch.Generator(device=dev).manual_seed(seed)
    users = torch.arange(n_q, dtype=torch.int32, device=dev)
    out = {}
    for frac in (0.01, 0.1, 1.0):
        n = max(10, int(round(frac * ni)))
        S = torch.sort(torch.randperm(ni, device=dev, generator=g)[:n])[0].to(torch.int32)
        leg = _leg("among", n_q, lambda: e2e(S), reps, label=f"among {frac:.0%}")
        k = _kernel(lambda: ops.score_topk_among(U, I, users, S, mask_rowptr, mask_col, 10, mode=mode), reps=3, windows=3)
        leg.update(n_among=n, kernel_s=round(k, 7), kernel_users_per_s=round(n_q / k, 1))
        line = f"  {'kernel':13s} {n:9d} among    {k * 1e3:9.3f} ms"
        if frac == 1.0:
            kp = _kernel(lambda: ops.score_topk(U, I, users, mask_rowptr, mask_col, 10, mode=mode), reps=3, windows=3)
            leg["plain_kernel_s"] = round(kp, 7)
            line += f"   plain call {kp * 1e3:9.3f} ms"
        if n_q * n < 2 ** 31:
            rp = torch.arange(n_q + 1, dtype=torch.int64, device=dev).mul_(n).to(torch.int32)
            col = S.repeat(n_q)
            kr = _kernel(lambda: ops.rerank(U, I, users, rp, col, mask_rowptr, mask_col, 10), reps=3, windows=3)
            leg["rerank_kernel_s"] = round(kr, 7)
            line += f"   rerank {kr * 1e3:9.3f} ms"
            del rp, col
        sys.stderr.write(line + "\n")
        out[f"{frac:.0%}"] = leg
    return out


def _groups_leg(U, I, rowptr, col, e2e, n_users, mode, reps, seed=0):
    """The groups leg: n_users users in random groups of 4, end to end (`e2e(groups, agg)`) for agg mean and min, and the kernels alone:
    the group kernel and the per-member score_topk launch of the same users"""
    import numpy as np
    import torch
    from llmrec_b200 import ops, recommend
    if ONLY and "groups" not in ONLY:
        return None
    dev, ni = U.device, int(I.shape[0])
    perm = np.random.default_rng(seed).permutation(n_users)
    groups = [perm[i:i + 4].tolist() for i in range(0, n_users, 4)]
    grp_rp, grp_col = recommend.groups_csr(groups, int(U.shape[0]))
    members = grp_col.to(dev, torch.int32)
    mrp, mcol = recommend.group_rows(rowptr, col, members, grp_rp, ni)
    users = members.clone()
    out = {}
    k_known = _kernel(lambda: ops.score_topk(U, I, users, rowptr, col, 10, mode=mode), reps=3, windows=3)
    for agg in ("mean", "min"):
        leg = _leg("groups", len(groups), lambda: e2e(groups, agg), reps, unit="groups", label=f"groups {agg}")
        k = _kernel(lambda: ops.score_topk_group(U, I, grp_rp, members, None, mrp, mcol, 10, agg=agg, mode=mode), reps=3, windows=3)
        leg.update(members=int(members.numel()), kernel_s=round(k, 7), kernel_groups_per_s=round(len(groups) / k, 1),
                   known_kernel_s=round(k_known, 7))
        sys.stderr.write(f"  {'kernel':13s} {len(groups):9d} groups   {k * 1e3:9.3f} ms   known kernel, same {members.numel()} users "
                         f"{k_known * 1e3:9.3f} ms\n")
        out[agg] = leg
    return out


def _explain_leg(hp, rowptr, col, ids, e2e, users, reps):
    """The explain leg: end to end (`e2e(ids)`, with its eval forward), and the kernel alone on the same queries"""
    import numpy as np
    from llmrec_b200 import ops, recommend
    if ONLY and "explain" not in ONLY:
        return None
    n_q = int(ids.shape[0])
    leg = _leg("explain", n_q, lambda: e2e(ids), reps, unit="queries")
    job = recommend.prepare_explain(hp, rowptr, col, ids, users=users)
    args = recommend.explain_args(hp, job)
    k = _kernel(lambda: ops.explain(*args))
    nnz, d, P = int(job["hist_col"].numel()), hp.d, int(ids.shape[1])
    rows_per_item = len(args[2]) + len(args[5])                  # side terms + id sources
    gb = ((nnz * rows_per_item + n_q * (P + 2)) * 4 * d) / 1e9
    leg.update(targets_per_query=P, history_items=nnz, channels=1 + len(args[2]), kernel_s=round(k, 7),
               kernel_queries_per_s=round(n_q / k, 1), kernel_GB_per_s=round(gb / k, 1),
               outputs_per_s=round(P * nnz * (1 + len(args[2])) / k, 1))
    sys.stderr.write(f"  {'explain kern':13s} {n_q:9d} queries  {k * 1e3:9.3f} ms       {n_q / k:12.0f} queries/s "
                     f"{gb / k:7.1f} GB/s ({nnz} history items, {rows_per_item} rows each)\n")
    del args, job
    return leg


def _list_quality(X, ids, vals, block=8192):
    """mean cosine over the ordered pairs of distinct positions inside each list (rows of the normalised X, fp32 products summed in
    fp64) and mean score of the listed items"""
    import torch
    K = ids.shape[1]
    off = ~torch.eye(K, dtype=torch.bool, device=ids.device)
    cos, pairs = 0.0, 0
    for s in range(0, ids.shape[0], block):
        i = ids[s:s + block]
        ok = i >= 0
        R = X[i.clamp(min=0)].double()
        pair = ok[:, :, None] & ok[:, None, :] & off
        cos += float(torch.bmm(R, R.transpose(1, 2))[pair].sum())
        pairs += int(pair.sum())
    return {"mean_pairwise_cos": round(cos / max(pairs, 1), 4), "mean_score": round(float(vals[ids >= 0].double().mean()), 4)}


def _diversify_leg(X, pool_ids, pool_vals, e2e, reps, label):
    """One diversify measurement: end to end (`e2e()`, with its eval forward), the kernel alone on the same pools (K = 10,
    lambda = 0.5), and the lists' quality at lambda = 1, 0.7 and 0.5"""
    from llmrec_b200 import ops
    n_q, P = (int(x) for x in pool_ids.shape)
    leg = _leg("diversify", n_q, e2e, reps, unit="queries", label=label)
    k = _kernel(lambda: ops.diversify(X, pool_ids, pool_vals, 10, 0.5))
    quality = {str(lam): _list_quality(X, *ops.diversify(X, pool_ids, pool_vals, 10, lam)[:2]) for lam in (1.0, 0.7, 0.5)}
    leg.update(pool=P, K=10, lam=0.5, kernel_s=round(k, 7), kernel_queries_per_s=round(n_q / k, 1),
               kernel_GFMA_per_s=round(n_q * 9 * P * int(X.shape[1]) / k / 1e9, 1), quality=quality)
    sys.stderr.write(f"  {label + ' kern':13s} {n_q:9d} queries  {k * 1e3:9.3f} ms       {n_q / k:12.0f} queries/s  pool {P}\n")
    for lam, q in quality.items():
        sys.stderr.write(f"    lambda {lam}: mean pairwise cos {q['mean_pairwise_cos']:.4f}, mean score {q['mean_score']:.4f}\n")
    return leg


def netflix(a, tmp):
    import numpy as np
    tr, gen, args = bench.make_trainer("netflix", types.SimpleNamespace(proj_mode=a.proj_mode, host_sampler="native", graph=1))
    for _ in range(5):
        tr.train_next_batch()                                     # a model some steps in: U / I stale on all but the last batch's rows
    nu = tr.n_users
    rp, col = tr.graph.rowptr_u.cpu().numpy(), tr.graph.col_u.cpu().numpy()
    users = np.array(sorted(int(u) for u in gen.test_set.keys()))
    hist = [col[rp[u]:rp[u + 1]].tolist() + list(gen.test_set[int(u)]) for u in users]
    path = os.path.join(tmp, "candidate_indices")
    res = {"workload": bench.workload_string("netflix"),
           "known": _leg("known", nu, lambda: tr.recommend(K=10, exclude="train"), a.reps),
           "fold_in": _leg("fold_in", len(hist), lambda: tr.recommend(users=users, K=10, exclude="train", histories=hist), a.reps),
           "candidates": _leg("candidates", nu, lambda: tr.write_candidates(path, 10), a.reps)}
    ni = tr.n_items
    irp, icol = tr.graph.rowptr_i.cpu().numpy(), tr.graph.col_i.cpu().numpy()
    res["fold_in_items"] = _leg("fold_in_items", ni, lambda: tr.fold_in_items((irp, icol)), a.reps, unit="items")
    res["similar"] = _leg("similar", ni, lambda: tr.similar_items(np.arange(ni), K=10), a.reps, unit="queries")
    hp = tr._current_model()
    res.update(_serving_legs(hp.U, hp.I, lambda cand: tr.rerank(cand, K=10), lambda u, i: tr.score(u, i), nu, 100, a.pairs, a.reps))
    res["among"] = _among_legs(hp.U, hp.I, tr.graph.rowptr_u, tr.graph.col_u, lambda S: tr.recommend(K=10, exclude="train", among=S), nu,
                               a.score_mode, a.reps)
    res["groups"] = _groups_leg(hp.U, hp.I, tr.graph.rowptr_u, tr.graph.col_u, lambda gr, agg: tr.recommend_groups(gr, K=10, agg=agg), nu,
                                a.score_mode, a.reps)
    if not ONLY or "explain" in ONLY:
        ids, _ = tr.recommend(K=10, exclude="train")
        res["explain"] = _explain_leg(tr._current_model(), tr.graph.rowptr_u, tr.graph.col_u, ids, lambda t: tr.explain(t), None, a.reps)
    if not ONLY or "diversify" in ONLY:
        from llmrec_b200 import ops
        p_ids, p_vals = tr.recommend(K=64, exclude="train")
        X = ops.row_normalize(tr._current_model().I)
        res["diversify"] = _diversify_leg(X, p_ids, p_vals, lambda: tr.recommend(K=10, exclude="train", diversity=0.5, pool=64), a.reps,
                                          "diversify")
    del tr, gen
    return res


def synthetic(a, tmp):
    import numpy as np
    import torch
    from llmrec_b200 import dist_bench, recommend
    from llmrec_b200.dist import ShardedGraph, synthetic_shard
    from llmrec_b200.engine import HotPath, HotPathConfig
    from llmrec_b200.ops import CsrOperator
    dev = torch.device("cuda", 0)
    nu, ni, ne, d, L = dist_bench.syn_sizes(a.syn_scale)
    ul, it, _, _ = synthetic_shard(nu, ni, ne, 0, 1, dev, seed=0)
    g = ShardedGraph(ul, it, nu, ni, solo=True)
    del ul, it
    iu = CsrOperator(g.rowptr_i, g.col_i, ni, nu, rs=g.si, plan=g.iu_raw.plan)                # iu = diag(si) R^T (one rank: no all-reduce)
    gen = torch.Generator(device=dev).manual_seed(0)
    params = {"user_id_embedding.weight": torch.randn(nu, d, device=dev, generator=gen) * 0.1,
              "item_id_embedding.weight": torch.randn(ni, d, device=dev, generator=gen) * 0.1}
    hp = HotPath((g.ui, iu, g.uiT_raw, g.iuT), params, None, HotPathConfig(embed_size=d, n_layers=L))
    rng = np.random.default_rng(0)
    hu = rng.choice(nu, a.syn_histories, replace=False)
    rp = g.rowptr_u.cpu().numpy()
    col = g.col_u.cpu().numpy()
    hist = [col[rp[u]:rp[u + 1]].tolist() + rng.integers(0, ni, 2).tolist() for u in hu]
    n = min(a.syn_users, nu)
    users = np.arange(n)
    path = os.path.join(tmp, "candidate_indices_synthetic")

    def known():
        hp.forward()
        recommend.top_k(hp, g.rowptr_u, g.col_u, users=users, K=10, exclude="train", mode=a.score_mode)

    def fold():
        hp.forward()
        recommend.top_k(hp, g.rowptr_u, g.col_u, K=10, exclude="train", histories=hist, mode=a.score_mode)

    def cand():
        hp.forward()
        ids, _ = recommend.top_k(hp, g.rowptr_u, g.col_u, users=users, K=10, exclude="none", mode=a.score_mode)
        recommend.write_candidates(path, ids)

    items = np.sort(rng.choice(ni, min(a.syn_items, ni), replace=False))
    irp, icol = g.rowptr_i.cpu().numpy(), g.col_i.cpu().numpy()
    lists = [icol[irp[i]:irp[i + 1]] for i in items]
    item_rp = np.concatenate([[0], np.cumsum([x.size for x in lists])])
    item_col = np.concatenate(lists)

    def fold_items():
        hp.forward()
        hp.fold_in_items(item_rp, item_col)

    def similar():
        hp.forward()
        recommend.similar_items(hp, items, K=10, mode=a.score_mode)

    def rr(cand):
        hp.forward()
        recommend.rerank(hp, g.rowptr_u, g.col_u, cand, users=users, K=10)

    def pairs(u, i):
        hp.forward()
        recommend.score_pairs(hp, u, i)

    res = {"workload": f"synthetic {nu}x{ni}, {g.nnz} training edges, d={d}, L={L}, ID-only engine",
           "known": _leg("known", n, known, a.reps), "fold_in": _leg("fold_in", len(hist), fold, a.reps),
           "candidates": _leg("candidates", n, cand, a.reps),
           "fold_in_items": _leg("fold_in_items", items.size, fold_items, a.reps, unit="items"),
           "similar": _leg("similar", items.size, similar, a.reps, unit="queries")}
    hp.forward()
    res.update(_serving_legs(hp.U, hp.I, rr, pairs, n, 200, a.pairs, a.reps))

    def among(S):
        hp.forward()
        recommend.top_k(hp, g.rowptr_u, g.col_u, users=users, K=10, exclude="train", mode=a.score_mode, among=S)

    hp.forward()
    res["among"] = _among_legs(hp.U, hp.I, g.rowptr_u, g.col_u, among, n, a.score_mode, a.reps)

    def groups(gr, agg):
        hp.forward()
        recommend.top_k_groups(hp, g.rowptr_u, g.col_u, gr, K=10, agg=agg, mode=a.score_mode)

    hp.forward()
    res["groups"] = _groups_leg(hp.U, hp.I, g.rowptr_u, g.col_u, groups, n, a.score_mode, a.reps)

    def explain(ids):
        hp.forward()
        recommend.explain(hp, g.rowptr_u, g.col_u, ids, users=users)

    if not ONLY or "explain" in ONLY:
        hp.forward()
        ids, _ = recommend.top_k(hp, g.rowptr_u, g.col_u, users=users, K=10, exclude="train", mode=a.score_mode)
        res["explain"] = _explain_leg(hp, g.rowptr_u, g.col_u, ids, explain, users, a.reps)
    if not ONLY or "diversify" in ONLY:
        from llmrec_b200 import ops

        def div_known():
            hp.forward()
            recommend.top_k(hp, g.rowptr_u, g.col_u, users=users, K=10, exclude="train", mode=a.score_mode, diversity=0.5, pool=64)

        cand200 = torch.randint(0, ni, (n, 200), device=dev, generator=torch.Generator(device=dev).manual_seed(1))

        def div_rerank():
            hp.forward()
            recommend.rerank(hp, g.rowptr_u, g.col_u, cand200, users=users, K=10, diversity=0.5, pool=200)

        hp.forward()
        X = ops.row_normalize(hp.I)
        p_ids, p_vals = recommend.top_k(hp, g.rowptr_u, g.col_u, users=users, K=64, exclude="train", mode=a.score_mode)
        res["diversify"] = _diversify_leg(X, p_ids, p_vals, div_known, a.reps, "diversify")
        r_ids, r_vals = recommend.rerank(hp, g.rowptr_u, g.col_u, cand200, users=users, K=200)
        res["diversify_rerank"] = _diversify_leg(X, r_ids, r_vals, div_rerank, a.reps, "div rerank")
        del X, p_ids, p_vals, r_ids, r_vals, cand200
    del hp, g, params
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed calls per leg (the median is reported), after one warm-up call")
    ap.add_argument("--proj_mode", default="3xtf32", choices=["3xtf32", "tf32", "fp32"])
    ap.add_argument("--syn_users", type=int, default=131072, help="synthetic workload: users of the known and candidates legs")
    ap.add_argument("--syn_histories", type=int, default=8192, help="synthetic workload: histories of the fold-in leg")
    ap.add_argument("--syn_items", type=int, default=65536, help="synthetic workload: items of the fold_in_items and similar legs")
    ap.add_argument("--syn_scale", type=float, default=1.0, help="size factor of the 10M x 1M x 200M synthetic graph")
    ap.add_argument("--pairs", type=int, default=1 << 20, help="pairs of the score_pairs legs")
    ap.add_argument("--workloads", default="netflix,synthetic")
    ap.add_argument("--legs", default="", help="comma-separated subset of the legs to run (default: all)")
    a = ap.parse_args()
    import torch
    from llmrec_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_recommend.py needs a CUDA (H100) device")
    a.score_mode = ops.SCORE_MODE.get(a.proj_mode, 0)
    ONLY.update(x for x in a.legs.split(",") if x)
    name, limit = card()
    result = {"metric": "recommend_users_per_sec", "gpu": name, "power_limit": limit, "proj_mode": a.proj_mode, "K": 10,
              "timing": f"host clock between device synchronises, median of {a.reps} calls after one warm-up; each call runs the full eval forward",
              "workloads": {}}
    with tempfile.TemporaryDirectory(prefix="llmrec_recommend_") as tmp:
        for wl in a.workloads.split(","):
            sys.stderr.write(f"{wl}:\n")
            result["workloads"][wl] = netflix(a, tmp) if wl == "netflix" else synthetic(a, tmp)
            torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
