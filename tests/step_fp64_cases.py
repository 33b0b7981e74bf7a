"""The engine cases of the fp64 step tests (tests/test_step_grads_fp64_gpu.py, tests/test_step_sequence_fp64_gpu.py): the seeded graphs,
parameter and feature tables and batches of each shape, and the loud-rate engines built on them.  TEST INFRASTRUCTURE ONLY.

Shapes:
  netflix    13187 x 17366, 68933 edges, d = 64, L = 2, feature widths 512 / 768 / 1536, the netflix attribute keys;
  movielens  12495 x 10322, 57960 edges, d = 128, L = 3, the movielens keys;
  odd        700 x 900, d = 256, L = 1, image width 130 (not a multiple of 4: the tensor-core projections refuse it and that
             problem group runs the fp32 SIMT kernels in every mode), 40 edgeless users, edgeless items, a hub user with 600
             edges and a hub item with 650 (both longer than the SpMM tile).
The graphs follow tests/test_live_items_gpu.py: item popularity falls off as a power law, so many items have no edge and the
default engine's live item set is on.

Batches (seeded, drawn on the host): B' = 1126 (1024 sampled + 102 augmented-style triplets), B' = 1128 (the capacity of
batch_size 1024), and B' = 8 (n_keep = 2).  Every batch repeats users and items, has pos == neg rows and an item that is the
positive of one row and the negative of another."""
import os
import sys

import numpy as np
import scipy.sparse as sp
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import step_fp64_model as SM  # noqa: E402

SHAPES = {  # n_users, n_items, edges, d, L, (image, text, llm) widths, keys
    "netflix": (13187, 17366, 68933, 64, 2, (512, 768, 1536), ("year", "title", "director", "country", "language")),
    "movielens": (12495, 10322, 57960, 128, 3, (512, 768, 1536), ("title", "genre", "director", "country", "language")),
    "odd": (700, 900, 5000, 256, 1, (130, 64, 96), ("title", "genre")),
}
BATCHES = {"B1126": (1024, 102), "B1128": (1024, 104), "small": (6, 2)}     # sampled, augmented
# batch seeds: the first seeds from 11 up whose every kept-set cut clears a margin of 5e-5 (netflix, in fp32, bf16 and int8 tables
# alike) or 1e-4 (B' >= 1126) and 5e-3 (B' = 8, where the TF32 cases run) relative to 1 + sum |u| (|p| + |n|) -- TAU_CUT or more
# (seed 11 of netflix B1126 fails TAU_CUT["fp32"], seed 11 of movielens B1126 leaves 2e-7)
SEEDS = {("netflix", "B1126"): 29, ("netflix", "B1128"): 22, ("netflix", "small"): 11, ("movielens", "B1126"): 86,
         ("movielens", "small"): 11, ("odd", "B1126"): 21, ("odd", "small"): 22}


def _graph(name):
    nu, ni, ne, d, L, dims, keys = SHAPES[name]
    rng = np.random.default_rng(0)
    users_with_edges = nu - 40 if name == "odd" else nu
    rows = np.concatenate([np.arange(users_with_edges), rng.integers(0, users_with_edges, ne - users_with_edges)])
    w = 1.0 / (np.arange(ni) + 8.0) ** 0.8
    cols = rng.choice(ni, size=ne, p=w / w.sum())
    if name == "odd":                                   # hubs: user 1 on 600 items, item 3 under 650 users
        rows = np.concatenate([rows, np.full(600, 1), rng.permutation(users_with_edges)[:650]])
        cols = np.concatenate([cols, rng.permutation(ni)[:600], np.full(650, 3)])
    R = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(nu, ni))
    R.sum_duplicates(); R.data[:] = 1.0
    return R


def _tables(name, seed=0):
    """fp32 params and feature tables (CPU)."""
    nu, ni, ne, d, L, (di, dt, dl), keys = SHAPES[name]
    gen = torch.Generator().manual_seed(seed)
    p = {"user_id_embedding.weight": torch.randn(nu, d, generator=gen) * 0.1, "item_id_embedding.weight": torch.randn(ni, d, generator=gen) * 0.1}
    for k, w in (("image", di), ("text", dt), ("user", dl), ("item", dl)):
        p[k + "_trans.weight"] = torch.randn(d, w, generator=gen) / w ** 0.5
        p[k + "_trans.bias"] = torch.randn(d, generator=gen) * 0.1
    feats = dict(image=torch.randn(ni, di, generator=gen), text=torch.randn(ni, dt, generator=gen), user=torch.randn(nu, dl, generator=gen),
                 item={k: torch.randn(ni, dl, generator=gen) for k in keys})
    return p, feats


def _batch(name, which, seed=None):
    """(users, pos, neg) int32 numpy of shape `name`, kind `which` (BATCHES): `draw`.  seed: SEEDS[(name, which)] unless given."""
    return draw(*SHAPES[name][:2], *BATCHES[which], SEEDS[(name, which)] if seed is None else seed)


def draw(nu, ni, n_s, n_a, seed):
    """(users, pos, neg) int32 numpy: n_s sampled rows, then n_a augmented-style rows of users already in the batch; repeats,
    pos == neg rows, and an item that is both a positive and a negative."""
    rng = np.random.default_rng(seed)
    u = rng.integers(0, nu, n_s); p = rng.integers(0, ni, n_s); n = rng.integers(0, ni, n_s)
    u[1], p[2], n[3] = u[0], p[0], n[0]                   # a repeated user, a repeated positive, a repeated negative
    n[4] = p[4]                                           # pos == neg
    n[5] = p[1]                                           # item p[1] is also a negative
    ua = u[rng.integers(0, n_s, n_a)]
    pa, na = rng.integers(0, ni, n_a), rng.integers(0, ni, n_a)
    if n_a > 2:
        na[0] = pa[0]                                     # pos == neg among the augmented rows
    return tuple(np.concatenate(x).astype(np.int32) for x in ((u, ua), (p, pa), (n, na)))


def _feats_as(feats, dtype, dev):
    from llmrec_b200 import feat_int8
    conv = (lambda X: X.to(dev)) if dtype == "fp32" else (lambda X: X.to(dev, torch.bfloat16)) if dtype == "bf16" else \
        (lambda X: feat_int8.quantize(X.to(dev)).contiguous())
    return dict(image=conv(feats["image"]), text=conv(feats["text"]), user=conv(feats["user"]), item={k: conv(v) for k, v in feats["item"].items()})


_GRAPHS = {}


def _engine(name, dtype="fp32", hoisted=False, mode=0, det=False):
    from llmrec_b200.engine import HotPath, HotPathConfig
    from llmrec_b200.graph import BipartiteGraph
    from llmrec_b200.hoist import HoistedHotPath
    dev = torch.device("cuda")
    if name not in _GRAPHS:
        _GRAPHS[name] = _graph(name)
    g = BipartiteGraph(_GRAPHS[name], dev)
    nu, ni, ne, d, L = SHAPES[name][:5]
    p, feats = _tables(name)
    cfg = SM.loud(HotPathConfig(embed_size=d, n_layers=L, batch_size=1024, proj_mode=mode, deterministic=det))
    ops = (g.ui, g.iu, g.uiT, g.iuT)
    params, fx = {k: v.to(dev) for k, v in p.items()}, _feats_as(feats, dtype, dev)
    hp = HoistedHotPath(ops, params, fx, cfg, g.ones_propagated()) if hoisted else HotPath(ops, params, fx, cfg)
    hp.set_optimizer(lr=1e-3)
    return hp


# ---- runs of steps (tests/test_step_sequence_fp64_gpu.py) -------------------------------------------------------------------------
# Both directions of a size change, with stale index-buffer slots after every large -> small change.
SEQUENCE = ("B1126", "small", "B1128", "small", "B1126")


def _sequence(name, seeds, kinds=SEQUENCE, batch=None):
    """The batches of one run: batch k is `batch(kinds[k], seeds[k])` (default `_batch(name, ...)`) with a few ids taken from batch
    k - 1, so consecutive steps share users and items (the repeated user and repeated positive of slots 0-2, and for B' > 70 the
    users and negatives of slots 6-69) while most rows one step touches are untouched by the next."""
    batch = batch or (lambda kind, seed: _batch(name, kind, seed))
    out = []
    for kind, seed in zip(kinds, seeds):
        u, p, n = (x.copy() for x in batch(kind, seed))
        if out:
            pu, pp, pn = out[-1]
            u[0] = u[1] = pu[-1]
            p[0] = p[2] = pp[-1]
            if u.size > 70 and pu.size > 70:
                u[6:70], n[6:70] = pu[6:70], pn[6:70]
        out.append((u, p, n))
    return out
