"""-m gpu: the row-mapped projections (LLMREC_PROJ_ROW_MAP problems of llmrec_proj_*_group_*, ops.proj_*_group with a per-problem `rows`) and the engine's live
item set (engine.HotPath._build_live_items).

Kernel level, fp32 and bf16 X, modes 3xTF32 / TF32 / SIMT, d in {32, 64, 128, 256}: a compact table holds the listed rows of a full
table.  The forward through the map must give the full-table call's bits on the listed rows and leave every other row untouched (NaN
sentinels); the weight gradient, with dY zero off the list, must meet the fp64 tolerances of the identity form and give the full-table
call's db bit for bit.  Edges: no row listed, one row, counts off the tile, every row listed, a column-slice X.

Engine level, at the netflix and movielens shapes on a graph with edgeless items: the live set is the distinct columns of ui; forward
outputs and loss are bit-identical to the engine without it; whole graphed steps agree with it within the run-to-run spread of the
loss heads' float atomics plus what AdamW makes of the weight gradients' rounding; a graph where every item has an edge builds no
compact tables."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

cuda = torch.device("cuda")
NAN = float("nan")
TOL = {(torch.float32, 0): 1e-4, (torch.float32, 1): 5e-3, (torch.float32, 2): 1e-4,
       (torch.bfloat16, 0): 1e-4, (torch.bfloat16, 1): 3e-2, (torch.bfloat16, 2): 1e-4}


def _gen(seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def _slice(T, dtype, lead=8, pad=8):
    """T [n x k] as a column slice of a wider row-major table of `dtype`: ld = lead + k + pad (a multiple of 8), 16-byte aligned start."""
    n, k = T.shape
    wide = torch.full((n, lead + k + pad), NAN, device=cuda, dtype=dtype)
    wide[:, lead:lead + k] = T.to(dtype)
    return wide[:, lead:lead + k]


# (m rows of the full table, listed rows): none, one, off the 64/128/256-row tiles, every row, several row chunks and tiles
CASES = [(300, "none"), (300, "one"), (1000, 0.7), (257, "all"), (5000, 0.7)]


def _listed(m, how, g):
    if how == "none":
        return torch.zeros(0, dtype=torch.int32, device=cuda)
    if how == "one":
        return torch.tensor([m // 3], dtype=torch.int32, device=cuda)
    if how == "all":
        return torch.arange(m, dtype=torch.int32, device=cuda)
    keep = torch.rand(m, generator=g, device=cuda) < how
    return torch.nonzero(keep).flatten().to(torch.int32)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_row_mapped_projection_matches_the_full_table(d, dtype, mode):
    from llmrec_b200 import ops
    k, k2 = 136, 40
    for ci, (m, how) in enumerate(CASES):
        g = _gen(1000 * d + 10 * mode + ci)
        full = torch.randn(m, k, generator=g, device=cuda)
        rows = _listed(m, how, g)
        n = int(rows.numel())
        X = _slice(full, dtype)                                      # the full table, and the compact table of its listed rows
        Xc = _slice(full[rows.long()], dtype)
        X2 = _slice(torch.randn(m, k2, generator=g, device=cuda), dtype)   # a second problem of the group without a map
        W, W2 = (torch.randn(d, kk, generator=g, device=cuda) / kk ** 0.5 for kk in (k, k2))
        b, b2 = (torch.randn(d, generator=g, device=cuda) for _ in range(2))
        what = f"d={d} {dtype} mode={mode} m={m} listed={how}"

        # forward: listed rows get the full call's bits, the others keep their NaN sentinels (Y a strided view)
        Yf, Y2f = torch.empty(m, d, device=cuda), torch.empty(m, d, device=cuda)
        ops.proj_fwd_group([(X, W, b, Yf), (X2, W2, b2, Y2f)], d, mode)
        wide = torch.full((m, 3 * d), NAN, device=cuda)
        Y, Y2 = wide[:, d:2 * d], torch.full((m, d), NAN, device=cuda)
        ops.proj_fwd_group([(Xc, W, b, Y, rows), (X2, W2, b2, Y2)], d, mode)
        torch.cuda.synchronize()
        on = torch.zeros(m, dtype=torch.bool, device=cuda)
        on[rows.long()] = True
        assert torch.equal(Y[on], Yf[on]), what
        assert bool(Y[~on].isnan().all()), what
        assert bool(wide[:, :d].isnan().all() and wide[:, 2 * d:].isnan().all()), what
        assert torch.equal(Y2, Y2f), what

        # weight gradient: dY zero off the list; db over every row of dY gives the full call's bits
        dY = torch.randn(m, 3 * d, generator=g, device=cuda)[:, d:2 * d]
        dY[~on] = 0.0
        dY2 = torch.randn(m, d, generator=g, device=cuda)
        outs = {}
        for arm in ("full", "map"):
            dW, db = torch.full((d, k), NAN, device=cuda), torch.full((d,), NAN, device=cuda)
            dW2, db2 = torch.full((d, k2), NAN, device=cuda), torch.full((d,), NAN, device=cuda)
            first = (X, dY, dW, db, False) if arm == "full" else (Xc, dY, dW, db, False, rows)
            ops.proj_wgrad_group([first, (X2, dY2, dW2, db2, False)], d, mode)
            outs[arm] = (dW, db, dW2, db2)
        torch.cuda.synchronize()
        dW, db, dW2, db2 = outs["map"]
        tol = TOL[(dtype, mode)]
        Xd = X.double()
        torch.testing.assert_close(dW.double(), dY.double().t() @ Xd, rtol=tol, atol=tol * max(n, 1) ** 0.5, msg=lambda s: f"dW {what}: {s}")
        if mode != 2 or m <= 1024:      # SIMT: one 1024-row chunk is one ordered sum; more chunks add their sums with float atomics
            assert torch.equal(db, outs["full"][1]), what
            assert torch.equal(db2, outs["full"][3]), what
        torch.testing.assert_close(db.double(), dY.double().sum(0), rtol=1e-4, atol=1e-4 * m ** 0.5, msg=lambda s: f"db {what}: {s}")
        torch.testing.assert_close(dW2.double(), dY2.double().t() @ X2.double(), rtol=tol, atol=tol * m ** 0.5, msg=lambda s: f"dW2 {what}: {s}")
        if mode != 2:
            assert torch.equal(dW2, outs["full"][2]), what             # the unmapped problem of the group is unaffected


def test_row_map_must_cover_the_x_rows():
    from llmrec_b200 import ops
    X = torch.randn(10, 32, device=cuda)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(X, torch.randn(32, 32, device=cuda), None, torch.empty(20, 32, device=cuda),
                             torch.arange(9, dtype=torch.int32, device=cuda))], 32, 0)
    with pytest.raises(ValueError):
        ops.proj_wgrad_group([(X, torch.randn(20, 32, device=cuda), torch.empty(32, 32, device=cuda), None, False,
                               torch.arange(10, dtype=torch.int64, device=cuda))], 32, 0)


# ---------------------------------------------------------------------------------------------------------------------------------
# engine
# ---------------------------------------------------------------------------------------------------------------------------------
SHAPES = {"netflix": (13187, 17366, 68933, 64, 2), "movielens": (12495, 10322, 57960, 128, 3)}
KEYS = ["k0", "k1", "k2", "k3", "k4"]
DIMS = dict(image=64, text=96, user=160, item=128)


def _engine(name, every_item=False, seed=0, lr=1e-3):
    """The graph of tests/test_demand_fuse_gpu.py: every user has an edge, item popularity falls off as a power law, so many items have
    none (every_item=True: each item gets one edge more)."""
    from llmrec_b200.engine import HotPath, HotPathConfig
    from llmrec_b200.graph import BipartiteGraph
    nu, ni, ne, d, L = SHAPES[name]
    rng = np.random.default_rng(0)
    rows = np.concatenate([np.arange(nu), rng.integers(0, nu, ne - nu)])
    w = 1.0 / (np.arange(ni) + 8.0) ** 0.8
    cols = rng.choice(ni, size=ne, p=w / w.sum())
    if every_item:
        rows, cols = np.concatenate([rows, rng.integers(0, nu, ni)]), np.concatenate([cols, np.arange(ni)])
    R = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(nu, ni))
    R.sum_duplicates(); R.data[:] = 1.0
    g = BipartiteGraph(R, cuda)
    gen = torch.Generator().manual_seed(seed)
    p = {"user_id_embedding.weight": torch.randn(nu, d, generator=gen) * 0.1, "item_id_embedding.weight": torch.randn(ni, d, generator=gen) * 0.1}
    for k in ("image", "text", "user", "item"):
        p[k + "_trans.weight"] = torch.randn(d, DIMS[k], generator=gen) / DIMS[k] ** 0.5
        p[k + "_trans.bias"] = torch.randn(d, generator=gen) * 0.1
    feats = dict(image=torch.randn(ni, DIMS["image"], generator=gen).to(cuda), text=torch.randn(ni, DIMS["text"], generator=gen).to(cuda),
                 user=torch.randn(nu, DIMS["user"], generator=gen).to(cuda),
                 item={k: torch.randn(ni, DIMS["item"], generator=gen).to(cuda) for k in KEYS})
    hp = HotPath((g.ui, g.iu, g.uiT, g.iuT), {k: v.to(cuda) for k, v in p.items()}, feats, HotPathConfig(embed_size=d, n_layers=L, batch_size=1024))
    hp.set_optimizer(lr=lr)
    return hp, R


def _engine_without_live_set(monkeypatch, name, **kw):
    with monkeypatch.context() as mp:
        mp.setenv("LLMREC_LIVE_ITEMS", "0")
        hp, R = _engine(name, **kw)
    assert hp.live_i is None and hp.fx is hp.feats
    return hp, R


@pytest.mark.parametrize("name", ["netflix", "movielens"])
def test_live_set_is_the_distinct_columns_of_ui(name):
    hp, R = _engine(name)
    want = np.unique(R.tocoo().col)
    assert 0 < want.size < hp.ni
    assert hp.live_i is not None and hp.live_i.dtype == torch.int32 and hp.n_live == want.size
    assert np.array_equal(hp.live_i.cpu().numpy(), want)
    live = hp.live_i.long()
    for k in ("image", "text"):
        assert torch.equal(hp.fx[k], hp.feats[k][live])
    for k in KEYS:
        assert torch.equal(hp.fx["item"][k], hp.feats["item"][k][live])
    assert hp.fx["user"] is hp.feats["user"]


def test_every_item_with_an_edge_builds_no_copies():
    hp, _ = _engine("netflix", every_item=True)
    assert hp.live_i is None and hp.n_live == hp.ni and hp.fx is hp.feats


def _out_grads(hp):
    return {"gU": hp.gU, "gI": hp.gI, "GFu": hp.GFu, "GFi": hp.GFi, "Gprof_u": hp.Gprof_u, "Gprof_i": hp.Gprof_i}


@pytest.mark.parametrize("name", ["netflix", "movielens"])
def test_forward_and_loss_are_bit_identical_to_the_full_tables(name, monkeypatch):
    """Forward (live rows of Pi, P_usr, Fu, Fi, prof_*, U, I), the loss and head_out are bit-identical to the engine without the live
    set, and Pi is zero off the live rows.  From one snapshot of the loss gradients (the heads scatter them with float atomics), the
    backward gives the same bias gradients and ID-embedding gradients bit for bit, the weight gradients to rounding."""
    a, _ = _engine_without_live_set(monkeypatch, name)
    b, _ = _engine(name)
    rng = np.random.default_rng(5)
    B = 1100
    u, p, n = (torch.from_numpy(rng.integers(0, m, B).astype(np.int32)).to(cuda) for m in (a.nu, a.ni, a.ni))
    out, snap = {}, None
    for hp in (a, b):
        hp.forward()
        hp.loss_and_output_grads(u, p, n)
        torch.cuda.synchronize()
        fwd = {k: getattr(hp, k).clone() for k in ("P_usr", "Fu", "Fi", "prof_i", "prof_u", "U", "I", "loss", "head_out")}
        if snap is None:
            snap = {k: v.clone() for k, v in _out_grads(hp).items()}
        else:
            for k, v in _out_grads(hp).items():
                v.copy_(snap[k])
        hp.backward()
        torch.cuda.synchronize()
        out[hp] = fwd, hp.Pi.clone(), {k: v.clone() for k, v in hp.grads.items()}
    (fa, Pa, ga), (fb, Pb, gb) = out[a], out[b]
    for k in fa:
        assert torch.equal(fa[k], fb[k]), (name, k)
    live = b.live_i.long()
    assert torch.equal(Pb[live], Pa[live])
    off = torch.ones(b.ni, dtype=torch.bool, device=cuda); off[live] = False
    assert bool((Pb[off] == 0).all())
    # dW: the two engines sum the same products in another order; bound the difference elementwise by 1e-5 * sum |dY| |X| (3xTF32
    # products carry ~2^-21, fp32 sums ~2^-24 per term) -- a dropped or misplaced row would break it
    G, f = b.GPi.double().abs(), b.feats
    blocks = {"image_trans.weight": [(0, f["image"])], "text_trans.weight": [(1, f["text"])],
              "item_trans.weight": [(2 + j, f["item"][k]) for j, k in enumerate(KEYS)]}
    for k, terms in blocks.items():
        mag = sum(G[:, s * b.d:(s + 1) * b.d].t() @ X.double().abs() for s, X in terms)
        err = (gb[k].double() - ga[k].double()).abs()
        assert bool((err <= 1e-5 * mag).all()), (name, k, float((err / mag.clamp_min(1e-30)).max()))
    for k in ga:
        if not k.endswith("_trans.weight") or k == "user_trans.weight":
            assert torch.equal(ga[k], gb[k]), (name, k)


@pytest.mark.parametrize("name,branches", [("netflix", True), ("movielens", True), ("netflix", False)])
def test_whole_steps_match_the_full_tables(name, branches, monkeypatch):
    """Graphed whole steps on varying B', with and without the live set.  Each step's gradients agree to rounding (1e-4 of the
    tensor's largest gradient; the weight gradients sum their products in another order).  AdamW turns a gradient difference dg into
    an update difference of at most lr * |dg| / eps (its first update is lr * g / (|g| + eps)), which is large where |g| ~ eps: a
    rounding difference of 6e-10 on a gradient of 2e-9 moves a netflix projection weight by 4e-5.  So each parameter element must lie
    within max(2 * spread of two full-table runs, 1e-5) + 2 lr / eps * sum_t |dg_t| of the full-table run; the losses within twice
    their spread."""
    lr, eps = 1e-3, 1e-8

    def run(live):
        hp, _ = _engine(name, lr=lr) if live else _engine_without_live_set(monkeypatch, name)
        assert (hp.live_i is not None) == live
        hp.branches = branches
        rng = np.random.default_rng(4)
        losses, grads = [], []
        for B in (1126, 1030, 1, 1100, 1128, 513):
            u, p, n = (torch.from_numpy(rng.integers(0, m, B).astype(np.int32)).to(cuda) for m in (hp.nu, hp.ni, hp.ni))
            losses.append(float(hp.train_step_graphed(u, p, n)))
            grads.append({k: v.clone() for k, v in hp.grads.items()})
        torch.cuda.synchronize()
        return losses, {k: v.clone() for k, v in hp.p.items()}, grads

    la, pa, ga = run(False)
    lb, pb, _ = run(False)
    ln, pn, gn = run(True)
    for k in pa:
        slack = torch.zeros_like(pa[k])
        for t, (x, y) in enumerate(zip(ga, gn)):
            dg = (y[k] - x[k]).abs()
            assert float(dg.max()) <= 1e-4 * float(x[k].abs().max()), (name, k, t, float(dg.max()), float(x[k].abs().max()))
            slack += dg
        spread = float((pa[k] - pb[k]).abs().max())
        bound = max(2 * spread, 1e-5) + 2 * lr / eps * slack
        assert bool(((pn[k] - pa[k]).abs() <= bound).all()), (name, k, spread, float((pn[k] - pa[k]).abs().max()))
    spread = max(abs(x - y) for x, y in zip(la, lb))
    assert max(abs(x - y) for x, y in zip(ln, la)) <= max(2 * spread, 1e-5 * max(1.0, abs(la[0]))), (la, lb, ln)


def test_refresh_item_feats_follows_in_place_rewrites():
    """The --mask branch overwrites rows of the full attribute tables in place; refresh_item_feats copies the live ones into the
    compact tables."""
    hp, _ = _engine("netflix")
    rows = torch.arange(0, hp.ni, 7, device=cuda)
    for v in hp.feats["item"].values():
        v[rows] = v.mean(0)
    hp.refresh_item_feats(rows)
    live = hp.live_i.long()
    for k in KEYS:
        assert torch.equal(hp.fx["item"][k], hp.feats["item"][k][live])
