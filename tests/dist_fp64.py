"""The sharded engines (dist.ShardedHotPath, dist_feat.ShardedFeatureHotPath) held to the fp64 step model, step by step.  TEST
INFRASTRUCTURE ONLY: tests/test_dist_fp64_gpu.py runs it on the H100 (world 1 in process, world 2 through tests/dist_fp64_check.py
under torch.distributed.run), tests/test_dist_fp64_cpu.py on the emulated kernels (tests/ops_emulator.py) under gloo.

The reference of a step restates what the shards compute: ui from every rank's CSR(R_r) with its own su, iu from every rank's
CSR(R_r^T) (local user columns shifted by the rank's first user) with the all-reduced si, the user table gathered from the ranks'
rows; `step_fp64_model.reference` (feats=None for the ID-only engine) at the parameters the step starts from.  Per step:
  * `check_cuts` (the batch seed is the first from the step's base seed whose every kept-set cut clears twice TAU_CUT in fp64);
  * `check_grads` on this rank's user rows, the item rows it holds the gradient of, and (side-feature engine) every projection
    weight and bias: the bound of step_fp64_model and its exact zeros (the demand step's row-sparse user gradient included);
  * `check_loss` on loss and head_out;
  * `step_sequence.check_adamw`: this rank's p, m and v of every optimized tensor after the update, from the pre-step state and the
    gradient the engine handed to AdamW.
Nothing raises inside a run, so every rank reaches every collective: the failures are collected and returned with the worst ratios.

Shapes: "netflix" (step_fp64_cases, 13187 x 17366, 68933 edges, power-law items); "odd" (step_fp64_cases' odd graph, 700 x 900:
40 edgeless users in the last shard, hub user 1 with 600 edges and hub item 3 under 650 users, both longer than the SpMM tile,
plus item 898 whose 10 edges all come from users 10..19, i.e. from rank 0); "odd-uneven" (its first 699 users and 899 items, so
nu % 2 and ni % 2 are 1 and the item exchanges take the all-reduce forms).  Batches: step_fp64_cases.SEQUENCE (B' = 1126, 8, 1128,
8, 1126) drawn by `step_fp64_cases.draw` over the whole user range (users of both ranks, repeats, pos == neg rows), consecutive
batches sharing ids as in `step_fp64_cases._sequence`.  Rates: `step_fp64_model.loud`."""
import dataclasses
import os
import sys
import types

import numpy as np
import scipy.sparse as sp
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import step_fp64_cases as SC  # noqa: E402
import step_fp64_model as SM  # noqa: E402
from fp64_bounds import RATIOS  # noqa: E402
from step_sequence import check_adamw, opt_tensors  # noqa: E402

UID, IID = "user_id_embedding.weight", "item_id_embedding.weight"
BASE_SEEDS = (11, 31, 51, 71, 91)
LR = 1e-3


def world_rank():
    return (dist.get_world_size(), dist.get_rank()) if dist.is_initialized() else (1, 0)


def _graph(shape):
    if shape == "netflix":
        return SC._graph("netflix")
    R = SC._graph("odd").tocoo()
    j = 898                                                     # an item whose edges all sit on rank 0
    keep = R.col != j
    rows = np.concatenate([R.row[keep], np.arange(10, 20)])
    cols = np.concatenate([R.col[keep], np.full(10, j)])
    R = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=R.shape)
    return R[:699, :899].tocsr() if shape == "odd-uneven" else R


_GRAPHS = {}


def graph(shape):
    if shape not in _GRAPHS:
        _GRAPHS[shape] = _graph(shape)
    return _GRAPHS[shape]


def _gather_rows(t):
    """every rank's rows of `t`, concatenated in rank order (any row counts)"""
    world, _ = world_rank()
    if world == 1:
        return t
    parts = [None] * world
    dist.all_gather_object(parts, t.detach().cpu())
    return torch.cat(parts).to(t.device)


def _coo(rows, cols, vals, shape):
    return torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, shape).coalesce()


def shard_operators(g, lo, nu):
    """fp64 (ui, iu) of the whole graph, assembled from every rank's shard CSRs and scales (see the module docstring)"""
    dev = g.su.device
    rp_u, rp_i = g.rowptr_u.long(), g.rowptr_i.long()
    ru = torch.repeat_interleave(torch.arange(g.nu_local, device=dev), rp_u[1:] - rp_u[:-1])
    ri = torch.repeat_interleave(torch.arange(g.n_items, device=dev), rp_i[1:] - rp_i[:-1])
    u_rows, u_cols, u_vals = _gather_rows(ru + lo), _gather_rows(g.col_u.long()), _gather_rows(g.su.double()[ru])
    i_rows, i_cols, i_vals = _gather_rows(ri), _gather_rows(g.col_i.long() + lo), _gather_rows(g.si.double()[ri])
    return _coo(u_rows, u_cols, u_vals, (nu, g.n_items)), _coo(i_rows, i_cols, i_vals, (g.n_items, nu))


@dataclasses.dataclass
class Run:
    """One engine on this rank and what its steps are checked with."""
    kind: str                   # "id" or "feat"
    sh: object                  # the engine
    shape: str
    lo: int
    hi: int
    nu: int
    ni: int
    ui: torch.Tensor
    iu: torch.Tensor
    feats: dict = None          # full feature tables ("feat")
    tau_name: str = "fp32"


def build(case, dev):
    """case: dict(engine="id" | "feat", shape, d, L (id), demand, pieces, item_sharded (id), mode (feat), loud (id, default True))
    -> Run"""
    from llmrec_b200.dist import ShardedGraph, ShardedHotPath, shard_bounds
    from llmrec_b200.engine import HotPathConfig
    world, rank = world_rank()
    shape, kind = case["shape"], case.get("engine", "id")
    R = graph(shape)
    nu, ni = R.shape
    b = shard_bounds(nu, world)
    lo, hi = b[rank], b[rank + 1]
    Rl = R[lo:hi].tocoo()
    t = lambda a: torch.from_numpy(a.astype(np.int64)).to(dev)
    g = ShardedGraph(t(Rl.row), t(Rl.col), hi - lo, ni, pieces=case.get("pieces", 1))
    ui, iu = shard_operators(g, lo, nu)
    if kind == "id":
        d, L = case.get("d", 64), case.get("L", 2)
        gen = torch.Generator().manual_seed(0)
        Eu, Ei = torch.randn(nu, d, generator=gen) * 0.1, torch.randn(ni, d, generator=gen) * 0.1
        cfg = HotPathConfig(embed_size=d, n_layers=L, batch_size=1024)
        cfg = SM.loud(cfg) if case.get("loud", True) else cfg
        sh = ShardedHotPath(g, Eu[lo:hi].clone().to(dev), Ei.clone().to(dev), cfg, lo, item_sharded=case.get("item_sharded", False),
                            demand=case.get("demand", False))
        assert sh.demand == bool(case.get("demand", False)), "the demand step refused this case"
        sh.set_lr(LR)
        return Run("id", sh, shape, lo, hi, nu, ni, ui, iu)
    from llmrec_b200.dist_feat import ShardedFeatureHotPath
    base = "odd" if shape.startswith("odd") else shape
    _, _, _, d, L = SC.SHAPES[base][:5]
    p, f = SC._tables(base)
    p[UID], p[IID] = p[UID][:nu], p[IID][:ni]
    f = dict(image=f["image"][:ni], text=f["text"][:ni], user=f["user"][:nu], item={k: v[:ni] for k, v in f["item"].items()})
    ib = shard_bounds(ni, world)
    ilo, ihi = ib[rank], ib[rank + 1]
    mode = case.get("mode", 0)
    cfg = SM.loud(HotPathConfig(embed_size=d, n_layers=L, batch_size=1024, proj_mode=mode))
    params = {k: (v[lo:hi] if k == UID else v).clone().to(dev) for k, v in p.items()}
    local = dict(image=f["image"][ilo:ihi].to(dev), text=f["text"][ilo:ihi].to(dev), user=f["user"][lo:hi].to(dev),
                 item={k: v[ilo:ihi].to(dev) for k, v in f["item"].items()})
    sh = ShardedFeatureHotPath(g, params, local, cfg, lo, ilo)
    sh.set_lr(LR)
    full = dict(image=f["image"].to(dev), text=f["text"].to(dev), user=f["user"].to(dev), item={k: v.to(dev) for k, v in f["item"].items()})
    return Run("feat", sh, shape, lo, hi, nu, ni, ui, iu, feats=full, tau_name=("3xtf32", "tf32", "fp32")[mode])


def ref_params(run):
    sh = run.sh
    if run.kind == "id":
        return {UID: _gather_rows(sh.E_u).double(), IID: sh.E_i.detach().double()}
    return {k: (_gather_rows(v) if k == UID else v.detach()).double() for k, v in sh.p.items()}


def _forward64(run, P):
    with torch.no_grad():
        if run.kind == "id":
            return SM.id_forward(P, run.ui, run.iu, SM.oracle_config(run.sh.cfg))
        from oracle import llmrec_oracle as O
        X = dict(image=run.feats["image"].double(), text=run.feats["text"].double(), user=run.feats["user"].double(),
                 item={k: v.double() for k, v in run.feats["item"].items()})
        return O.forward(P, X, run.ui, run.iu, SM.oracle_config(run.sh.cfg))


def _cuts_clear(out, batch, keys, drop_rate, need):
    """every BPR head's kept-set gap of x over `need` x (1 + sum |u| (|p| + |n|)) at the cut (the gap of SM.reference)"""
    u, p, n = (torch.as_tensor(x, dtype=torch.long, device=out["U"].device) for x in batch)
    B = int(u.numel())
    keep = int((1 - drop_rate) * B)
    pairs = [(out["U"], out["I"])]
    if keys is not None:
        pairs += [(out["img_u"], out["img_i"]), (out["txt_u"], out["txt_i"])] + [(out["prof_u"], out["att_i"][k]) for k in keys]
    for XU, XI in pairs:
        a, b, c = XU[u], XI[p], XI[n]
        x = (a * b).sum(1) - (a * c).sum(1) + 1e-8
        order = torch.argsort(x.cpu(), stable=True).to(x.device)
        s = x[order]
        mag = (a.abs() * (b.abs() + c.abs())).sum(1)[order[keep - 1:keep + 1]].max()
        if not float(s[keep] - s[keep - 1]) > need * (1 + float(mag)):
            return False
    return True


def batches_for(run, P, k, prev):
    """step k's batch (kind SEQUENCE[k]): the first seed from BASE_SEEDS[k] whose cuts clear 2 x TAU_CUT at P, ids shared with
    `prev` as step_fp64_cases._sequence does; every rank takes the largest seed any rank chose."""
    kind = SC.SEQUENCE[k]
    out = _forward64(run, P)
    keys = None if run.kind == "id" else run.sh.keys

    def make(seed):
        u, p, n = (x.copy() for x in SC.draw(run.nu, run.ni, *SC.BATCHES[kind], seed))
        if prev is not None:
            pu, pp, pn = prev
            u[0] = u[1] = pu[-1]
            p[0] = p[2] = pp[-1]
            if u.size > 70 and pu.size > 70:
                u[6:70], n[6:70] = pu[6:70], pn[6:70]
        return u, p, n
    seed = BASE_SEEDS[k]
    while not _cuts_clear(out, make(seed), keys, run.sh.cfg.prune_loss_drop_rate, 2 * SM.TAU_CUT[run.tau_name]):
        seed += 1
        assert seed < BASE_SEEDS[k] + 200, "no batch seed with clear kept-set cuts"
    if dist.is_initialized():
        t = torch.tensor([seed], dtype=torch.int64, device=P[UID].device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        seed = int(t)
    return make(seed)


def _sub(ref, rows):
    """ref restricted to the parameters of `rows` (name -> row slice or None for all rows)"""
    pick = lambda d: {k: (d[k] if r is None else d[k][r]) for k, r in rows.items()}
    return dataclasses.replace(ref, grads=pick(ref.grads), mag=pick(ref.mag), per_head={})


def engine_grads(run):
    """(name -> gradient the engine handed to AdamW, name -> row slice of the full gradient it holds)"""
    sh = run.sh
    if run.kind == "id":
        g_u, g_i, ilo = sh.step_grads()
        return {UID: g_u, IID: g_i}, {UID: slice(run.lo, run.hi), IID: slice(ilo, ilo + g_i.shape[0])}
    return dict(sh.grads), {k: (slice(run.lo, run.hi) if k == UID else None) for k in sh.grads}


def _excess(res):
    """worst error / bound of a grad_excess result; a nonzero where fp64 is exactly zero counts as infinitely over"""
    return max((float("inf") if v[2] else v[0]) for v in res.values())


def run_steps(run, n_steps=len(SC.SEQUENCE), strict=True):
    """n_steps steps of SEQUENCE, each checked as the module docstring states.
    -> dict(grads=, adamw=, errors=[...], seeds) with the worst ratios; strict=False skips the loss / AdamW checks (mutations)."""
    sh = run.sh
    tau = SM.TAU[run.tau_name]
    worst = dict(grads=0.0, adamw=0.0, errors=[])
    heads = ["mf"] if run.kind == "id" else SM.engine_heads(sh.keys)
    prev = None
    dev = sh.E_i.device
    for k in range(n_steps):
        what = f"{run.kind} {run.shape} step {k + 1}"
        P = ref_params(run)
        batch = batches_for(run, P, k, prev)
        prev = batch
        ref = SM.reference(P, None if run.kind == "id" else run.feats, run.ui, run.iu, SM.oracle_config(sh.cfg),
                           *(torch.from_numpy(x).long() for x in batch), run.ni)
        try:
            SM.check_cuts(ref, run.tau_name, what)
        except AssertionError as e:
            worst["errors"].append(str(e))
        from llmrec_b200.engine import PARAM_ORDER
        names = [UID, IID] if run.kind == "id" else list(PARAM_ORDER)
        adapter = types.SimpleNamespace(opt=sh.opt, _opt_names=names, grads=None)
        pre = opt_tensors(adapter)
        sh.train_step(*(torch.from_numpy(x).to(dev) for x in batch))
        if dev.type == "cuda":
            torch.cuda.synchronize()
        grads, rows = engine_grads(run)
        res = SM.grad_excess(_sub(ref, rows), grads, tau)
        worst["grads"] = max(worst["grads"], _excess(res))
        bad = {k: v for k, v in res.items() if v[1] or v[2]}
        if bad:
            worst["errors"].append(f"{what}: (worst err / bound, elements over, nonzero where fp64 is exactly zero) {bad}")
        if not strict:
            continue
        try:
            SM.check_loss(ref, sh.loss, sh.head_out, heads, tau, what=what)
        except AssertionError as e:
            worst["errors"].append(str(e))
        adapter.grads = grads
        try:
            worst["adamw"] = max(worst["adamw"], check_adamw(adapter, pre, k + 1, what))
        except AssertionError as e:
            RATIOS.clear()
            worst["errors"].append(str(e))
    return worst


# ---- mutations of dist.ShardedHotPath (tests/test_dist_fp64_cpu.py): each must fail the bound by 10^2 or more ------------------------
def _drop_exchange(sh, hit):
    """the all-reduce of the exchanges `hit(which, src, out)` selects is skipped (those calls run as at world 1)"""
    orig = sh._exchange

    def ex(which, src, out=None, src_mask=None, overlap=None):
        if hit(which, src, out):
            w, sh.world = sh.world, 1
            try:
                return orig(which, src, out, src_mask, overlap)
            finally:
                sh.world = w
        return orig(which, src, out, src_mask, overlap)
    sh._exchange = ex


def _twice_exchange(sh):
    """the forward exchange of layer 1 all-reduced twice"""
    orig = sh._exchange

    def ex(which, src, out=None, src_mask=None, overlap=None):
        r = orig(which, src, out, src_mask, overlap)
        if which == "iu" and src is sh.Ul[1]:
            dist.all_reduce(sh.part if out is None else out)
        return r
    sh._exchange = ex


def _non_owner_scatter(sh):
    """the dense step's user-row gradients: a batch user owned by another rank is also scattered into this rank's table"""
    orig = sh.loss_and_output_grads

    def f(users, pos, neg):
        r = orig(users, pos, neg)
        u = users.long()
        b = int(torch.nonzero((u < sh.lo) | (u >= sh.hi))[0])
        sh.gU[int(u[b]) % sh.nu] += sh.gUb[b]
        return r
    sh.loss_and_output_grads = f


def _item_grad_over_world(sh):
    orig = sh.backward

    def f():
        r = orig()
        sh.g_Ei.div_(sh.world)
        return r
    sh.backward = f


def _user_grad_times_world(sh):
    orig = sh.backward

    def f():
        r = orig()
        sh.g_Eu.mul_(sh.world)
        return r
    sh.backward = f


def _stale_row_sets(sh):
    """the demand step's row sets are cleared before the first step only"""
    orig = sh._train_step_demand

    def f(users, pos, neg):
        r = orig(users, pos, neg)
        for rs in (sh.needU, sh.batchU, sh.batchI):
            rs.clear = lambda: None
        return r
    sh._train_step_demand = f


MUTATIONS = {
    "forward exchange dropped": (dict(), lambda sh: _drop_exchange(sh, lambda which, src, out: which == "iu" and src is sh.Ul[1])),
    "backward exchange dropped": (dict(), lambda sh: _drop_exchange(sh, lambda which, src, out: which == "uiT" and out is sh.parts[sh.L & 1])),
    "forward exchange all-reduced twice": (dict(), _twice_exchange),
    "user gradient also scattered on a non-owner": (dict(), _non_owner_scatter),
    "item gradient divided by world size": (dict(), _item_grad_over_world),
    "user gradient multiplied by world size": (dict(), _user_grad_times_world),
    "demand row sets left uncleared": (dict(demand=True), _stale_row_sets),
}


# ---- the cases ----------------------------------------------------------------------------------------------------------------------
def case_id(c):
    return "-".join(f"{k}={v}" for k, v in c.items())


# world 1: the exchanges are local, so item_sharded / item_opt_sharded / the uneven forms do not arise
CASES_W1 = [
    dict(shape="netflix"), dict(shape="netflix", pieces=3),
    dict(shape="netflix", demand=True, d=32), dict(shape="netflix", demand=True, d=64), dict(shape="netflix", demand=True, d=128),
    dict(shape="odd"), dict(shape="odd", demand=True, d=64),
    dict(engine="feat", shape="netflix", mode=0), dict(engine="feat", shape="netflix", mode=2),
    dict(engine="feat", shape="odd", mode=0), dict(engine="feat", shape="odd", mode=2),
]
# world 2: netflix has an odd user count (uneven user ranges) and an even item count; odd has even counts; odd-uneven odd counts, where
# item_sharded / item_opt_sharded fall back to the all-reduce and dist_feat's item-row gather takes the zero-fill + all-reduce form
CASES_W2 = [
    dict(shape="netflix"), dict(shape="netflix", pieces=3), dict(shape="netflix", item_sharded=True),
    dict(shape="netflix", demand=True, d=64),
    dict(shape="odd"), dict(shape="odd", item_sharded=True), dict(shape="odd", demand=True, d=32), dict(shape="odd", demand=True, d=128),
    dict(shape="odd", pieces=3, demand=True, d=64),
    dict(shape="odd-uneven"), dict(shape="odd-uneven", item_sharded=True), dict(shape="odd-uneven", demand=True, d=64),
    dict(engine="feat", shape="netflix", mode=0), dict(engine="feat", shape="odd", mode=2),
    dict(engine="feat", shape="odd-uneven", mode=0), dict(engine="feat", shape="odd-uneven", mode=2),
]


def run_case(case, dev):
    """build + run_steps, with the engine's sharding facts (which exchange forms ran) -> dict; failures in 'errors'"""
    run = build(case, dev)
    sh = run.sh
    res = run_steps(run)
    res["forms"] = dict(item_sharded=getattr(sh, "item_sharded", False), item_opt_sharded=getattr(sh, "item_opt_sharded", False),
                        even_items=getattr(sh, "even_items", None), demand=getattr(sh, "demand", False), world=world_rank()[0])
    return res


def merge_ranks(parts):
    """per-rank run_case results -> one: the worst ratios, every rank's errors"""
    out = dict(parts[0])
    for p in parts[1:]:
        for k in ("grads", "adamw"):
            out[k] = max(out[k], p[k])
        out["errors"] = out["errors"] + p["errors"]
    return out
