"""-m gpu: deterministic steps (`--deterministic 1`): the ordered row gradients of the loss heads (llmrec_bpr_slot_plan +
llmrec_bpr_heads_ordered_f32), the ordered row scatter (llmrec_scatter_add_rows_ordered_f32) and the engines that use them.

Kernel level.  The order is held bit for bit: with every X entry a signed power of two the products e*a, e*q, e*r are exact, so a float32
numpy loop over the definition (heads ascending, batch positions ascending, pos before neg, one add per contribution, coefficients read
back from the kernel's work block) gives the kernel's bits, and the same loop run in another order does not.  Batches without a repeated
row give the atomic form's bits; random batches meet the fp64 bound tests/test_step_tail_exactness_gpu.py states for the row gradients
and leave rows, columns and padding they do not own untouched; a capacity-sized call with a device-side length equals the host-length
call and never reads past B'.

Engine level.  Two fresh engines on the same batches end with bit-identical parameters and AdamW moments -- graph or eager, with or
without branches, default or hoisted engine, fp32 or bf16 tables, host or device sampler -- each run executed once; the deterministic engine stays within the
run-to-run spread of the default one and within the oracle tolerances of the smoke run; the combinations it does not cover raise."""
import math
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

cuda = torch.device("cuda")
F = np.float32
U = 2.0 ** -24


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def wide(a, off=4, gap=5):
    """fp32 block `a` as a column view of a NaN-filled device buffer (leading dimension > d) -> (buffer, view)"""
    a = np.asarray(a, F)
    n, d = a.shape
    buf = np.full((n, off + d + gap), np.nan, F)
    buf[:, off:off + d] = a
    t = dev(buf)
    return t, t[:, off:off + d]


def bits(a):
    return np.ascontiguousarray(a, dtype=F).view(np.uint32)


def pow2(rng, lo, hi, *shape):
    return (2.0 ** rng.integers(lo, hi + 1, shape) * rng.choice([-1.0, 1.0], shape)).astype(F)


def ftz(x):
    return np.where(np.abs(x) < F(2.0 ** -126), F(0), x).astype(F)


def work_of(work, h, cap):
    base = 32 + h * (7 * cap + 8)
    return work[base + 5 * cap: base + 6 * cap], work[base + 7 * cap: base + 7 * cap + 3]


class Heads:
    """n_heads heads over wide, NaN-padded buffers; buf_u / buf_i: which gradient buffer each head adds into (None = no gradient)."""

    def __init__(self, XU, XI, GU0, GI0, buf_u, buf_i, wmf, wemb):
        self.XU, self.XI, self.GU0, self.GI0, self.buf_u, self.buf_i, self.wmf, self.wemb = XU, XI, GU0, GI0, buf_u, buf_i, wmf, wemb
        self.xu = [wide(t)[1] for t in XU]
        self.xi = [wide(t)[1] for t in XI]

    def run(self, users, pos, neg, n_keep, ordered, meta=None, c=0.05):
        from llmrec_b200 import ops
        gu, gi = [wide(t) for t in self.GU0], [wide(t) for t in self.GI0]
        hs = [(self.xu[h], self.xi[h], None if self.buf_u[h] is None else gu[self.buf_u[h]][1], None if self.buf_i[h] is None else gi[self.buf_i[h]][1],
               float(self.wmf[h]), float(self.wemb[h])) for h in range(len(self.xu))]
        cap = int(users.numel())
        work = ops.bpr_work(len(hs), cap, cuda)
        out, loss = torch.zeros(4 * len(hs), device=cuda), torch.full((1,), 1.25, device=cuda)
        plan = ops.bpr_slot_plan(users, pos, neg, meta=meta) if ordered else None
        ops.bpr_heads(hs, users, pos, neg, n_keep, c, out, loss, work, meta=meta, ordered=plan)
        torch.cuda.synchronize()
        return dict(gu=[t[0].cpu().numpy() for t in gu], gi=[t[0].cpu().numpy() for t in gi], out=out.cpu().numpy(), loss=loss.cpu().numpy(),
                    work=work.cpu().numpy(), cap=cap)

    def loop(self, res, users, pos, neg, Bl, reverse=False):
        """float32 loop over the definition -> (GU, GI) lists; reverse: batch positions descending, neg before pos (a wrong order)"""
        GU, GI = [t.copy() for t in self.GU0], [t.copy() for t in self.GI0]
        order = range(Bl - 1, -1, -1) if reverse else range(Bl)
        for h in range(len(self.xu)):
            g, e = work_of(res["work"], h, res["cap"])
            eu, ep, en = (F(x) for x in e)
            if self.buf_u[h] is None and self.buf_i[h] is None:
                continue
            for b in order:
                if g[b] == 0 and self.wemb[h] == 0:
                    continue
                a, q, r = self.XU[h][users[b]], self.XI[h][pos[b]], self.XI[h][neg[b]]
                ga = F(g[b]) * a
                if self.buf_u[h] is not None:
                    G = GU[self.buf_u[h]]
                    G[users[b]] = ftz(ftz(G[users[b]]) + ftz(F(g[b]) * (q - r) + eu * a))
                if self.buf_i[h] is not None:
                    G = GI[self.buf_i[h]]
                    for row, cb in ((neg[b], -ga + en * r), (pos[b], ga + ep * q))[::1 if reverse else -1]:
                        G[row] = ftz(ftz(G[row]) + ftz(cb))
        return GU, GI


def order_case(d, seed):
    """700 triplets over 12 users and 14 items: repeated users, item 0 a hub (>= 300 occurrences, as pos and as neg), pos == neg at
    b = 5, non-zero initial buffers, heads 0 and 2 sharing one GU, heads 1 and 2 one GI; one head without a GU, one without w_emb."""
    rng = np.random.default_rng(seed)
    B, nu, ni, H = 700, 12, 14, 4
    users, pos, neg = rng.integers(0, nu, B), rng.integers(1, ni, B), rng.integers(1, ni, B)
    pos[rng.choice(B, 200, replace=False)] = 0
    neg[rng.choice(np.nonzero(pos != 0)[0], 180, replace=False)] = 0
    neg[5] = pos[5]
    assert (pos == 0).sum() + (neg == 0).sum() >= 300
    XU = [pow2(rng, -14, -10, nu, d) for _ in range(H)]
    XI = [pow2(rng, -13, 11, ni, d) for _ in range(H)]
    GU0 = [pow2(rng, -30, 0, nu, d) for _ in range(2)]
    GI0 = [pow2(rng, -30, 0, ni, d) for _ in range(3)]
    hd = Heads(XU, XI, GU0, GI0, buf_u=[0, 1, 0, None], buf_i=[0, 1, 1, 2], wmf=F([1.0, 0.5, 0.25, 2.0]), wemb=F([1.0, 0.0, 0.5, 0.0]))
    return hd, users, pos, neg


def i32(a):
    return dev(np.asarray(a, np.int32))


@pytest.mark.parametrize("d", [20, 32, 64, 128, 300])
def test_ordered_heads_follow_the_definition_bit_for_bit(d):
    hd, users, pos, neg = order_case(d, seed=d)
    B = users.size
    res = hd.run(i32(users), i32(pos), i32(neg), int(0.6 * B), ordered=True)
    GU, GI = hd.loop(res, users, pos, neg, B)
    for k, want in enumerate(GU):
        got = res["gu"][k]
        assert np.array_equal(bits(got[:, 4:4 + d]), bits(want)), f"d={d}: user gradient buffer {k}"
        assert np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + d:]).all()
    for k, want in enumerate(GI):
        got = res["gi"][k]
        assert np.array_equal(bits(got[:, 4:4 + d]), bits(want)), f"d={d}: item gradient buffer {k}"
        assert np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + d:]).all()
    RU, RI = hd.loop(res, users, pos, neg, B, reverse=True)
    assert not np.array_equal(bits(RU[0]), bits(GU[0])) and not np.array_equal(bits(RI[1]), bits(GI[1])), "the fixture cannot tell a wrong order"
    again = hd.run(i32(users), i32(pos), i32(neg), int(0.6 * B), ordered=True)
    for k in ("gu", "gi"):
        for x, y in zip(res[k], again[k]):
            assert np.array_equal(bits(np.nan_to_num(x)), bits(np.nan_to_num(y)))
    # the forward is shared with the atomic form
    atomic = hd.run(i32(users), i32(pos), i32(neg), int(0.6 * B), ordered=False)
    assert np.array_equal(bits(atomic["out"]), bits(res["out"])) and np.array_equal(bits(atomic["loss"]), bits(res["loss"]))


def random_case(rng, B, nu, ni, d, H=3, distinct=False):
    if distinct:
        users, items = rng.permutation(nu)[:B], rng.permutation(ni)[:2 * B]
        pos, neg = items[:B], items[B:]
    else:
        users, pos, neg = rng.integers(0, nu, B), rng.integers(0, ni, B), rng.integers(0, ni, B)
        neg[0] = pos[0]
    s = F(1 / math.sqrt(d))
    xv = lambda n: (rng.uniform(0.5, 2.0, (n, d)) * rng.choice([-1.0, 1.0], (n, d))).astype(F)
    hd = Heads([xv(nu) * s for _ in range(H)], [xv(ni) * s for _ in range(H)], [xv(nu) for _ in range(2)], [xv(ni) for _ in range(H)],
               buf_u=[0, 1, 1][:H], buf_i=list(range(H)), wmf=F([1.0, 0.7, 0.3][:H]), wemb=F([1.0, 0.0, 0.4][:H]))
    return hd, users, pos, neg


@pytest.mark.parametrize("d", [20, 64, 300])
def test_batches_without_repeated_rows_get_the_atomic_bits(d):
    rng = np.random.default_rng(100 + d)
    B = 257
    hd, users, pos, neg = random_case(rng, B, 400, 600, d, distinct=True)
    hd.buf_u = [0, 1, None]                  # no two heads share a buffer either: every element gets one contribution
    a = hd.run(i32(users), i32(pos), i32(neg), 74, ordered=False)
    o = hd.run(i32(users), i32(pos), i32(neg), 74, ordered=True)
    for k in ("gu", "gi"):
        for x, y in zip(a[k], o[k]):
            assert np.array_equal(bits(np.nan_to_num(x, nan=7.0)), bits(np.nan_to_num(y, nan=7.0))), (d, k)
    assert np.array_equal(bits(a["out"]), bits(o["out"])) and np.array_equal(bits(a["loss"]), bits(o["loss"]))


@pytest.mark.parametrize("d,B", [(20, 255), (64, 1126), (300, 257)])
def test_ordered_gradients_meet_the_fp64_bound_and_touch_nothing_else(d, B):
    rng = np.random.default_rng(7 * d + B)
    nu, ni = B // 3 + 6, B // 2 + 8
    hd, users, pos, neg = random_case(rng, B, nu, ni, d)
    nk = int(0.29 * B)
    res = hd.run(i32(users), i32(pos), i32(neg), nk, ordered=True)
    nb = math.ceil(B / 256)
    refs = {("u", k): [np.zeros((nu, d)), np.zeros((nu, d)), np.zeros((nu, 1))] for k in range(2)}
    refs.update({("i", k): [np.zeros((ni, d)), np.zeros((ni, d)), np.zeros((ni, 1))] for k in range(3)})
    S = lambda idx, n: sp.csr_matrix((np.ones(B), (idx, np.arange(B))), shape=(n, B))
    Su, Sp, Sn, one = S(users, nu), S(pos, ni), S(neg, ni), np.ones((B, 1))
    for h in range(3):
        g, e = work_of(res["work"], h, B)
        gc, (eu, ep, en) = g.astype(np.float64)[:, None], e.astype(np.float64)
        a, q, r = (t.astype(np.float64) for t in (hd.XU[h][users], hd.XI[h][pos], hd.XI[h][neg]))
        live = ((g != 0) | (hd.wemb[h] != 0)).astype(np.float64)[:, None]
        ru, ri = refs[("u", hd.buf_u[h])], refs[("i", hd.buf_i[h])]
        ru[0] += Su @ (live * (gc * (q - r) + eu * a)); ru[1] += Su @ (np.abs(gc) * (np.abs(q) + np.abs(r)) + abs(eu) * np.abs(a)); ru[2] += Su @ one
        ri[0] += Sp @ (live * (gc * a + ep * q)) + Sn @ (live * (-gc * a + en * r))
        ri[1] += Sp @ (np.abs(gc * a) + abs(ep) * np.abs(q)) + Sn @ (np.abs(gc * a) + abs(en) * np.abs(r)); ri[2] += (Sp + Sn) @ one
    for (side, k), (ref, mag, cnt) in refs.items():
        got, G0 = (res["gu"][k], hd.GU0[k]) if side == "u" else (res["gi"][k], hd.GI0[k])
        v, touched = got[:, 4:4 + d], cnt[:, 0] > 0
        assert np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + d:]).all(), "padding written"
        assert np.array_equal(bits(v[~touched]), bits(G0[~touched])), "an untouched gradient row changed"
        g0 = G0[touched].astype(np.float64)
        bound = 2 * U * (cnt[touched] + 2 * d + 2 * nb + 60) * (mag[touched] + np.abs(g0))
        err = np.abs(v[touched].astype(np.float64) - (g0 + ref[touched]))
        assert (err <= bound).all(), (side, k, float((err / bound).max()))


def test_device_side_length_equals_the_host_length_call():
    rng = np.random.default_rng(11)
    cap, d = 264, 64
    hd, users, pos, neg = random_case(rng, cap, 60, 80, d)
    for Bl in (1, 2, 7, cap - 1, cap):
        nk = max(1, int(0.29 * Bl))
        host = hd.run(i32(users[:Bl]), i32(pos[:Bl]), i32(neg[:Bl]), nk, ordered=True)
        u, p, n = users.copy(), pos.copy(), neg.copy()
        u[Bl:], p[Bl:], n[Bl:] = 2 ** 30, 2 ** 30, -(2 ** 30)          # stale slots: reading one faults or lands far outside
        got = hd.run(i32(u), i32(p), i32(n), -1, ordered=True, meta=i32([Bl, nk]))
        for k in ("gu", "gi"):
            for x, y in zip(host[k], got[k]):
                assert np.array_equal(bits(np.nan_to_num(x, nan=7.0)), bits(np.nan_to_num(y, nan=7.0))), (Bl, k)
        assert np.array_equal(bits(host["out"]), bits(got["out"])) and np.array_equal(bits(host["loss"]), bits(got["loss"]))


@pytest.mark.parametrize("d", [20, 64, 300])
def test_ordered_scatter_add_rows_follows_ascending_positions(d):
    from llmrec_b200 import ops
    rng = np.random.default_rng(d)
    n, rows = 1000, 9
    G, Y0 = pow2(rng, -30, 20, n, d), pow2(rng, -30, 20, rows, d)
    idx = rng.integers(-1, rows - 1, n)                  # -1: skipped; row `rows - 1` is never named
    idx[rng.choice(n, 400, replace=False)] = 3           # a hub
    want, rev = Y0.copy(), Y0.copy()
    for b in range(n):
        if idx[b] >= 0:
            want[idx[b]] = want[idx[b]] + G[b]
    for b in reversed(range(n)):
        if idx[b] >= 0:
            rev[idx[b]] = rev[idx[b]] + G[b]
    assert not np.array_equal(bits(rev), bits(want))
    (gb, gv), (yb, yv) = wide(G), wide(Y0)
    ops.scatter_add_rows_ordered(gv, i32(idx), yv)
    torch.cuda.synchronize()
    got = yb.cpu().numpy()
    assert np.array_equal(bits(got[:, 4:4 + d]), bits(want))
    assert np.isnan(got[:, :4]).all() and np.isnan(got[:, 4 + d:]).all()
    assert np.array_equal(bits(got[rows - 1, 4:4 + d]), bits(Y0[rows - 1]))


def test_capacity_is_an_argument_error():
    from llmrec_b200 import ops
    z = torch.zeros(65537, dtype=torch.int32, device=cuda)
    with pytest.raises(RuntimeError, match="unsupported"):
        ops.bpr_slot_plan(z, z, z)
    with pytest.raises(RuntimeError, match="unsupported"):
        ops.scatter_add_rows_ordered(torch.zeros(131073, 4, device=cuda), torch.zeros(131073, dtype=torch.int32, device=cuda), torch.zeros(2, 4, device=cuda))


# ---------------------------------------------------------------------------------------------------------------------------------
# engines
# ---------------------------------------------------------------------------------------------------------------------------------
def _state(hp):
    o = hp.opt
    return [p.clone() for p in o.params] + [m.clone() for m in o.m] + [v.clone() for v in o.v]


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def _same_losses(a, b):
    """bit-equal loss sequences (a batch of one triplet keeps none: its loss is NaN, as in the reference)"""
    return np.array_equal(bits(a), bits(b))


def _tiny_run(tiny_root, extra, steps=10):
    """A Trainer on the tiny golden data set, `steps` batches of the host sampler cut to varying lengths B'."""
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir
    args = set_args(parse_args(["--data_path", tiny_root, "--dataset", "netflix", "--batch_size", "128", "--epoch", "1", "--debug", "--lr", "0.001"] + extra))
    try:
        M.set_seed(args.seed)
        gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size)
        batch_test.init(gen, args)
        tr = M.Trainer(data_config={}, data_generator=gen)
        M.set_seed(7)
        sizes, losses = set(), []
        for t in range(steps):
            users, pos, neg = tr.sample_batch()
            keep = len(users) - (7 * t) % 23              # every augmented edge of this data set passes the filter: vary B' here
            users, pos, neg = users[:keep], pos[:keep], neg[:keep]
            sizes.add(len(users))
            losses.append(tr.train_batch(users, pos, neg))
        torch.cuda.synchronize()
        return tr, _state(tr.hot), [float(x) for x in losses], sizes
    finally:
        set_args(parse_args([]))


TINY = [pytest.param(h, f, id=f"{'hoisted' if h else 'default'}-{f}") for h in (0, 1) for f in ("fp32", "bf16")]


@pytest.mark.parametrize("hoist,feat", TINY)
def test_tiny_trainers_are_bit_reproducible(tiny_root, hoist, feat, monkeypatch):
    base = ["--deterministic", "1", "--hoist_side", str(hoist), "--feat_dtype", feat]
    _, a, la, sizes = _tiny_run(tiny_root, base)
    _, b, lb, _ = _tiny_run(tiny_root, base)
    assert len(sizes) > 1, "the batches must vary in length"
    assert _same(a, b) and _same_losses(la, lb), "two graph-replayed runs differ"
    _, e, le, _ = _tiny_run(tiny_root, base + ["--cuda_graph", "0"])
    _, e2, le2, _ = _tiny_run(tiny_root, base + ["--cuda_graph", "0"])
    assert _same(e, e2) and _same_losses(le, le2), "two eager runs differ"
    if not hoist:       # the default engine's kernels see the same live rows either way; the hoisted one projects capacity-sized blocks under the graph
        assert _same(a, e) and _same_losses(la, le), "the eager run differs from the graph-replayed one"
    monkeypatch.setenv("LLMREC_BRANCHES", "0")
    _, c, lc, _ = _tiny_run(tiny_root, base)
    _, c2, lc2, _ = _tiny_run(tiny_root, base)
    assert _same(c, c2) and _same_losses(lc, lc2), "two single-chain runs differ"


def test_tiny_trainer_with_the_device_sampler_is_bit_reproducible(tiny_root):
    def run():
        tr, _, _, _ = _tiny_run(tiny_root, ["--deterministic", "1", "--device_sampler", "1"], steps=0)
        for _ in range(10):
            tr.train_next_batch()
        torch.cuda.synchronize()
        return _state(tr.hot)

    assert _same(run(), run())


def test_deterministic_trainer_meets_the_oracle_tolerances(tiny_root):
    """One step of the deterministic Trainer against the CPU oracle, at the tolerances of the default path's smoke run."""
    from oracle import llmrec_oracle as O
    from llmrec_b200 import main as M
    tr, _, _, _ = _tiny_run(tiny_root, ["--deterministic", "1", "--lr", "0.0001"], steps=0)
    data = O.load_dataset(os.path.join(tiny_root, "netflix_valid_item"))
    O.set_seed(2022)
    otr = O.OracleTrainer(data, O.OracleConfig(batch_size=128))
    M.set_seed(7)
    users, pos, neg = tr.sample_batch()
    loss = float(tr.train_batch(users, pos, neg))
    oloss, _ = otr.step(users, pos, neg)
    assert abs(loss - oloss) < 5e-5 * max(1.0, abs(oloss)), (loss, oloss)
    sd = tr.model_mm.state_dict()
    for k in O.PARAM_NAMES:
        np.testing.assert_allclose(sd[k].cpu().numpy(), otr.params[k].detach().numpy(), rtol=2e-4, atol=2e-6)


NETFLIX = (13187, 17366, 68933, 64, 2)
KEYS = ["k0", "k1", "k2", "k3", "k4"]
DIMS = dict(image=64, text=96, user=160, item=128)


def _engine(deterministic, hoisted=False, lr=1e-3):
    """The netflix-shaped graph of tests/test_live_items_gpu.py: every user has an edge, item popularity falls off as a power law."""
    from llmrec_b200.engine import HotPath, HotPathConfig
    from llmrec_b200.graph import BipartiteGraph
    from llmrec_b200.hoist import HoistedHotPath
    nu, ni, ne, d, L = NETFLIX
    rng = np.random.default_rng(0)
    rows = np.concatenate([np.arange(nu), rng.integers(0, nu, ne - nu)])
    w = 1.0 / (np.arange(ni) + 8.0) ** 0.8
    cols = rng.choice(ni, size=ne, p=w / w.sum())
    R = sp.csr_matrix((np.ones(rows.size, F), (rows, cols)), shape=(nu, ni))
    R.sum_duplicates(); R.data[:] = 1.0
    g = BipartiteGraph(R, cuda)
    gen = torch.Generator().manual_seed(0)
    p = {"user_id_embedding.weight": torch.randn(nu, d, generator=gen) * 0.1, "item_id_embedding.weight": torch.randn(ni, d, generator=gen) * 0.1}
    for k in ("image", "text", "user", "item"):
        p[k + "_trans.weight"] = torch.randn(d, DIMS[k], generator=gen) / DIMS[k] ** 0.5
        p[k + "_trans.bias"] = torch.randn(d, generator=gen) * 0.1
    feats = dict(image=torch.randn(ni, DIMS["image"], generator=gen).to(cuda), text=torch.randn(ni, DIMS["text"], generator=gen).to(cuda),
                 user=torch.randn(nu, DIMS["user"], generator=gen).to(cuda),
                 item={k: torch.randn(ni, DIMS["item"], generator=gen).to(cuda) for k in KEYS})
    cfg = HotPathConfig(embed_size=d, n_layers=L, batch_size=1024, deterministic=deterministic)
    ops_, params = (g.ui, g.iu, g.uiT, g.iuT), {k: v.to(cuda) for k, v in p.items()}
    hp = HoistedHotPath(ops_, params, feats, cfg, g.ones_propagated()) if hoisted else HotPath(ops_, params, feats, cfg)
    hp.set_optimizer(lr=lr)
    return hp


def _netflix_run(deterministic, hoisted=False, sizes=(1126, 1030, 1, 1100, 1128, 513, 1127, 2, 1090, 1128)):
    hp = _engine(deterministic, hoisted)
    rng = np.random.default_rng(4)
    w = 1.0 / (np.arange(hp.ni) + 8.0) ** 0.8               # popular items repeat within a batch, as positives and as negatives
    losses, grads = [], []
    for B in sizes:
        u = torch.from_numpy(rng.integers(0, hp.nu, B).astype(np.int32)).to(cuda)
        p, n = (torch.from_numpy(rng.choice(hp.ni, size=B, p=w / w.sum()).astype(np.int32)).to(cuda) for _ in range(2))
        losses.append(float(hp.train_step_graphed(u, p, n)))
        grads.append({k: v.clone() for k, v in hp.grads.items()})
    torch.cuda.synchronize()
    return hp, _state(hp), losses, grads


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_netflix_shaped_steps_are_bit_reproducible(hoisted):
    _, a, la, _ = _netflix_run(True, hoisted)
    _, b, lb, _ = _netflix_run(True, hoisted)
    assert _same(a, b) and _same_losses(la, lb)


def test_deterministic_steps_stay_within_the_spread_of_the_default_path():
    """After the same 6 steps: within the bound tests/test_live_items_gpu.py uses for two engines that differ by summation order."""
    lr, eps, sizes = 1e-3, 1e-8, (1126, 1030, 1, 1100, 1128, 513)
    ha, _, la, ga = _netflix_run(False, sizes=sizes)
    hb, _, lb, _ = _netflix_run(False, sizes=sizes)
    hd, _, ld, gd = _netflix_run(True, sizes=sizes)
    for k in ha.p:
        slack = torch.zeros_like(ha.p[k])
        for t, (x, y) in enumerate(zip(ga, gd)):
            dg = (y[k] - x[k]).abs()
            assert float(dg.max()) <= 1e-4 * float(x[k].abs().max()), (k, t, float(dg.max()), float(x[k].abs().max()))
            slack += dg
        spread = float((ha.p[k] - hb.p[k]).abs().max())
        bound = max(2 * spread, 1e-5) + 2 * lr / eps * slack
        assert bool(((hd.p[k] - ha.p[k]).abs() <= bound).all()), (k, spread, float((hd.p[k] - ha.p[k]).abs().max()))
    spread = max(abs(x - y) for x, y in zip(la, lb))
    assert max(abs(x - y) for x, y in zip(ld, la)) <= max(2 * spread, 1e-5 * max(1.0, abs(la[0]))), (la, lb, ld)


def test_uncovered_flags_raise(tiny_root):
    with pytest.raises(ValueError, match="tensor-core"):
        _tiny_run(tiny_root, ["--deterministic", "1", "--proj_mode", "fp32"], steps=0)
    with pytest.raises(ValueError, match="deterministic"):
        _tiny_run(tiny_root, ["--deterministic", "1", "--mask_rate", "0.1"], steps=0)
    with pytest.raises(ValueError, match="deterministic"):
        _tiny_run(tiny_root, ["--deterministic", "1", "--drop_rate", "0.1"], steps=0)
