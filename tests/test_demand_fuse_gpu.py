"""-m gpu: train_step's batch-row fusion (engine.HotPath._batch_rows / _fuse_fwd / _fuse_bwd with batch_rows=True) against the full-row
fusion it replaces.  The loss heads scatter with float atomics, so two whole steps agree only to rounding: the fusion is compared from a
shared snapshot of the loss gradients instead, bit for bit, at the netflix and movielens shapes; whole steps are compared old schedule
against new with the run-to-run spread of the old schedule as the yardstick."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu
cuda = "cuda"

SHAPES = {"netflix": (13187, 17366, 68933, 64, 2), "movielens": (12495, 10322, 57960, 128, 3)}
KEYS = ["k0", "k1", "k2", "k3", "k4"]
DIMS = dict(image=64, text=96, user=160, item=128)
BATCH = 1024


def _engine(name, seed=0, lr=1e-3):
    from llmrec_b200.engine import HotPath, HotPathConfig
    from llmrec_b200.graph import BipartiteGraph
    nu, ni, ne, d, L = SHAPES[name]
    rng = np.random.default_rng(0)
    rows = np.concatenate([np.arange(nu), rng.integers(0, nu, ne - nu)])
    w = 1.0 / (np.arange(ni) + 8.0) ** 0.8
    R = sp.csr_matrix((np.ones(ne, np.float32), (rows, rng.choice(ni, size=ne, p=w / w.sum()))), shape=(nu, ni))
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
    hp = HotPath((g.ui, g.iu, g.uiT, g.iuT), {k: v.to(cuda) for k, v in p.items()}, feats, HotPathConfig(embed_size=d, n_layers=L, batch_size=BATCH))
    hp.set_optimizer(lr=lr)
    assert hp.demand_fuse
    return hp


def _stage(hp, B, rng):
    """Write a batch of B' = B live triplets into the index buffer: users drawn from the first half of the user ids with repeats,
    the last ~10 % repeating earlier users with other items (augmented edges); the stale slots past B' hold in-range ids of rows
    that are NOT in the batch (the second half of each table).  -> (users, pos, neg) of the live part, int64 CPU."""
    nu, ni = hp.nu, hp.ni
    gi = hp.index_buffer(B)
    cap = gi.shape[1]
    n_aug = B // 11
    u = rng.integers(0, nu // 2, B)
    u[B - n_aug:] = u[rng.integers(0, max(1, B - n_aug), n_aug)]
    pi, ni_ = rng.integers(0, ni // 2, B), rng.integers(0, ni // 2, B)
    gi[0] = torch.from_numpy(rng.integers(nu // 2, nu, cap).astype(np.int32)).to(cuda)
    gi[1] = torch.from_numpy(rng.integers(ni // 2, ni, cap).astype(np.int32)).to(cuda)
    gi[2] = torch.from_numpy(rng.integers(ni // 2, ni, cap).astype(np.int32)).to(cuda)
    for r, v in enumerate((u, pi, ni_)):
        gi[r, :B] = torch.from_numpy(v.astype(np.int32)).to(cuda)
    gi[3, :2] = torch.tensor(hp.meta_row(B), dtype=torch.int32, device=cuda)
    return torch.from_numpy(u), torch.from_numpy(pi), torch.from_numpy(ni_)


def _grad_bufs(hp):
    return {"dUl": hp.dUl, "dIl": hp.dIl, "GFu": hp.GFu, "GFi": hp.GFi, "Gprof_u": hp.Gprof_u, "Gprof_i": hp.Gprof_i,
            "gU": hp.gU, "gI": hp.gI, **{"grad." + k: v for k, v in hp.grads.items()}}


def _loss_grads(hp):
    """Forward (full rows) + the first touch of the batch-row schedule + loss heads on the staged batch; -> snapshot."""
    gi = hp._gidx
    hp.forward()
    hp._grad_init(id_grads=True)
    hp.loss_and_output_grads(gi[0], gi[1], gi[2], gi[3], init_done=True)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in _grad_bufs(hp).items()}, hp.U.clone(), hp.I.clone()


def _restore(hp, snap):
    for k, v in _grad_bufs(hp).items():
        v.copy_(snap[k])


def _batch_fusion(hp):
    gi = hp._gidx
    hp._batch_rows(gi[0], gi[1], gi[2], gi[3])
    hp._fuse_fwd(batch_rows=True)
    hp._fuse_bwd(batch_rows=True)


@pytest.mark.parametrize("name", ["netflix", "movielens"])
def test_row_sets_are_the_unique_live_ids(name):
    hp = _engine(name)
    rng = np.random.default_rng(1)
    for B in (1, 7, 600, hp.batch_capacity()):
        u, p, n = _stage(hp, B, rng)
        gi = hp._gidx
        hp._batch_rows(gi[0], gi[1], gi[2], gi[3])
        assert hp.batch_u.count.is_cuda and hp.batch_i.count.is_cuda
        cu, ci = int(hp.batch_u.count), int(hp.batch_i.count)
        assert torch.equal(hp.batch_u.list[:cu].sort().values.cpu().long(), torch.unique(u))
        assert torch.equal(hp.batch_i.list[:ci].sort().values.cpu().long(), torch.unique(torch.cat([p, n])))


@pytest.mark.parametrize("name", ["netflix", "movielens"])
def test_batch_row_fusion_is_bit_identical_to_full_rows(name):
    """From one snapshot of the loss gradients: full-row fusion vs batch-row fusion (eager) vs the batch-row fusion replayed from a CUDA
    graph captured once and fed different B' -- every gradient buffer torch.equal, U / I torch.equal on the batch rows, and the rows
    outside the batch of U / I not written at all."""
    hp = _engine(name)
    rng = np.random.default_rng(2)
    _stage(hp, hp.batch_capacity(), rng)
    _loss_grads(hp)
    torch.cuda.synchronize()
    _batch_fusion(hp)                                  # warm-up: side streams and ctypes tables exist before the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _batch_fusion(hp)
    for B in (hp.batch_capacity(), 1, 5, 777):
        u, p, n = _stage(hp, B, rng)
        snap, U_full, I_full = _loss_grads(hp)
        hp._fuse_bwd()                                 # full rows
        torch.cuda.synchronize()
        full = {k: v.clone() for k, v in _grad_bufs(hp).items()}
        for run in ("eager", "graph"):
            _restore(hp, snap)
            hp.U.fill_(float("nan")); hp.I.fill_(float("nan"))
            if run == "eager":
                _batch_fusion(hp)
            else:
                graph.replay()
            torch.cuda.synchronize()
            for k, v in _grad_bufs(hp).items():
                assert torch.equal(v, full[k]), (name, B, run, k)
            ru, ri = torch.unique(u).to(cuda), torch.unique(torch.cat([p, n])).to(cuda)
            assert torch.equal(hp.U[ru], U_full[ru]) and torch.equal(hp.I[ri], I_full[ri]), (name, B, run)
            off_u = torch.ones(hp.nu, dtype=torch.bool, device=cuda); off_u[ru] = False
            off_i = torch.ones(hp.ni, dtype=torch.bool, device=cuda); off_i[ri] = False
            assert bool(hp.U[off_u].isnan().all()) and bool(hp.I[off_i].isnan().all()), (name, B, run)


def test_grad_init_first_touch_of_the_id_gradients():
    """_grad_init(id_grads=True) zeroes dUl / dIl and writes every other region exactly as _grad_init() does."""
    hp = _engine("netflix")
    rng = np.random.default_rng(3)
    _stage(hp, 300, rng)
    hp.forward()
    for t in _grad_bufs(hp).values():
        t.fill_(7.0)
    hp._grad_init()
    torch.cuda.synchronize()
    want = {k: v.clone() for k, v in _grad_bufs(hp).items()}
    loss = hp.loss.clone()
    hp._grad_init(id_grads=True)
    torch.cuda.synchronize()
    for k, v in _grad_bufs(hp).items():
        zeroed = k in ("dUl", "dIl", "grad.user_id_embedding.weight")          # dUl is the user table's gradient buffer
        assert torch.equal(v, torch.zeros_like(v) if zeroed else want[k]), k
    assert torch.equal(hp.loss, loss)


@pytest.mark.parametrize("name,branches", [("netflix", True), ("movielens", True), ("netflix", False)])
def test_whole_steps_match_the_full_row_schedule(name, branches):
    """Graphed whole steps on varying B' (branches=False: the single-chain schedule): parameters after 6 steps of the batch-row schedule
    differ from the full-row schedule's within twice the spread of two runs of the full-row schedule (the loss heads' float atomics),
    floor 1e-5 absolute -- a hundredth of what one step moves a parameter at lr 1e-3; the losses likewise."""
    def run(demand):
        hp = _engine(name)
        hp.demand_fuse, hp.branches = demand, branches
        rng = np.random.default_rng(4)
        losses = []
        for B in (1126, 1030, 1, 1100, 1128, 513):
            u, p, n = (torch.from_numpy(rng.integers(0, m, B).astype(np.int32)).to(cuda) for m in (hp.nu, hp.ni, hp.ni))
            losses.append(float(hp.train_step_graphed(u, p, n)))
        torch.cuda.synchronize()
        return losses, {k: v.clone() for k, v in hp.p.items()}

    la, pa = run(False)
    lb, pb = run(False)
    ln, pn = run(True)
    for k in pa:
        spread = float((pa[k] - pb[k]).abs().max())
        assert float((pn[k] - pa[k]).abs().max()) <= max(2 * spread, 1e-5), (name, k, spread)
    spread = max(abs(x - y) for x, y in zip(la, lb))
    assert max(abs(x - y) for x, y in zip(ln, la)) <= max(2 * spread, 1e-5 * max(1.0, abs(la[0]))), (la, lb, ln)
