"""-m gpu: `--device_sampler 2` (csrc/device_sampler_ref.cu) draws exactly the host sampler's batches and leaves `random` / `np.random`
exactly where the host sampler leaves them.  Every comparison is exact: against the reference's golden batches, against
host_native.BatchSampler batch after batch (netflix shape, several seeds, streams about to twist, every branch and edge), on the error
paths, and for whole Trainer runs and checkpoints across sampler modes."""
import os
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TINY_FLAGS = ["--batch_size", "128", "--epoch", "1", "--debug", "--seed", "2022", "--lr", "0.001"]


def _trainer(root, extra=()):
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir
    args = set_args(parse_args(["--data_path", root, "--dataset", "netflix"] + TINY_FLAGS + list(extra)))
    M.set_seed(args.seed)
    gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size, sampler=args.host_sampler)
    batch_test.init(gen, args)
    tr = M.Trainer(data_config={}, data_generator=gen)
    tr.logger.logging = lambda s: None
    return tr, M


def _sorted_rows(rowptr, col):
    rows = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
    return col[np.lexsort((col, rows))].astype(np.int32)


def _streams():
    return random.getstate(), np.random.get_state()


def _same_streams(a, b):
    return a[0] == b[0] and a[1][0] == b[1][0] and np.array_equal(a[1][1], b[1][1]) and a[1][2:] == b[1][2:]


def _compare(exist, rowptr, col, n_items, batch, aug=None, rate=0.0, n_batches=5, aug_limit=None):
    """n_batches batches from the current streams, host vs device; both end states must agree too."""
    from llmrec_b200.device_sampler import ReferenceDeviceSampler
    from llmrec_b200.host_native import BatchSampler
    aug_limit = n_items if aug_limit is None else aug_limit
    ap, an = aug if aug is not None else (None, None)
    start = _streams()
    host = BatchSampler(exist, rowptr, col, n_items, batch, ap, an, aug_limit=aug_limit)
    cap = 2 * batch + 8
    want = []
    for _ in range(n_batches):
        o = np.zeros((3, cap), dtype=np.int32)
        B = host.draw(o, rate)
        want.append(o[:, :B].copy())
    end = _streams()
    random.setstate(start[0]); np.random.set_state(start[1])
    ds = ReferenceDeviceSampler(exist, rowptr, col, _sorted_rows(rowptr, col), n_items, batch, ap, an, aug_limit, rate, "cuda")
    buf = torch.full((4, cap), -7, dtype=torch.int32, device="cuda")
    meta = torch.stack([torch.arange(cap + 1), torch.arange(cap + 1) // 2], 1).to(torch.int32).cuda().contiguous()
    for t, w in enumerate(want):
        ds.fill(buf, meta)
        B = int(buf[3, 0])
        assert B == w.shape[1] and int(buf[3, 1]) == B // 2, (t, B, w.shape[1])
        np.testing.assert_array_equal(buf[:3, :B].cpu().numpy(), w, err_msg=f"batch {t}")
    ds.sync_to_host()
    assert _same_streams(_streams(), end)
    return want


def _netflix_graph(seed=0):
    """13 187 users, 17 366 items, ~69 k edges, item popularity falling off as a power law; rows in the order they were drawn"""
    rng = np.random.default_rng(seed)
    nu, ni = 13187, 17366
    rows = []
    for _ in range(nu):
        r = np.unique((rng.pareto(1.0, int(rng.integers(1, 10))) * 30).astype(np.int64) % ni)
        rng.shuffle(r)
        rows.append(r)
    rowptr = np.zeros(nu + 1, dtype=np.int32)
    np.cumsum([len(r) for r in rows], out=rowptr[1:])
    col = np.concatenate(rows).astype(np.int32)
    aug_pos = rng.integers(0, ni + ni // 20, nu).astype(np.int32)                # some >= n_items: dropped
    aug_neg = rng.integers(0, ni, nu).astype(np.int32)
    return np.arange(nu, dtype=np.int32), rowptr, col, ni, (aug_pos, aug_neg)


def _set_pos(near):
    """move both streams' positions to `near` (a twist falls inside the next batch)"""
    v, st, g = random.getstate()
    random.setstate((v, st[:624] + (near,), g))
    name, key, _, hg, c = np.random.get_state()
    np.random.set_state((name, key, near, hg, c))


def test_golden_batches_of_the_reference(tiny_root, golden):
    tr, M = _trainer(tiny_root, ["--device_sampler", "2", "--cuda_graph", "0"])
    M.set_seed(2022)
    ds, hp = tr.device_sampler, tr.hot
    ds.upload_from_host()                                                          # draws the pending batch again, from the reseeded streams
    for b in range(3):
        ds.step_begin()
        ds.step_end()
        B = int(hp._gidx[3, 0])
        np.testing.assert_array_equal(hp._gidx[:3, :B].cpu().numpy(), golden[f"sampler/{b}"])


@pytest.mark.parametrize("seed,near", [(0, None), (1, None), (2022, None), (5, 620), (6, 623), (7, 624)])
def test_netflix_shape_matches_the_host_sampler(seed, near):
    exist, rowptr, col, ni, aug = _netflix_graph()
    random.seed(seed); np.random.seed(seed)
    if near is not None:
        _set_pos(near)
    _compare(exist, rowptr, col, ni, 1024, aug, 0.1, n_batches=200)


def _small_graph(nu=300, ni=50, seed=0, deg_hi=8):
    rng = np.random.default_rng(seed)
    rows = [rng.permutation(ni)[:int(rng.integers(1, deg_hi))] for _ in range(nu)]
    rowptr = np.zeros(nu + 1, dtype=np.int32)
    np.cumsum([len(r) for r in rows], out=rowptr[1:])
    return rowptr, np.concatenate(rows).astype(np.int32)


@pytest.mark.parametrize("n_exist,batch", [(2000, 1024), (300, 64), (100, 128), (7, 7), (5, 64)])
def test_user_branches(n_exist, batch):
    """pool branch (n_exist <= setsize), set branch, and batch > n_exist (independent draws)"""
    rowptr, col = _small_graph(nu=n_exist, ni=500)
    random.seed(n_exist); np.random.seed(batch)
    _compare(np.arange(n_exist, dtype=np.int32), rowptr, col, 500, batch, n_batches=20)


@pytest.mark.parametrize("batch,rate", [(1024, 0.1), (1024, 0.005), (64, 1.0), (256, 0.5), (40, 0.2)])
def test_augmentation_branches_and_filter(batch, rate):
    """aug pool and set branches; ids >= aug_limit are dropped; rate 1.0 with all ids valid fills B' to capacity"""
    nu, ni = 3000, 400
    rowptr, col = _small_graph(nu=nu, ni=ni, seed=3)
    rng = np.random.default_rng(1)
    ap = rng.integers(0, ni + 40, nu).astype(np.int32) if rate < 1 else rng.integers(0, ni, nu).astype(np.int32)
    an = rng.integers(0, ni, nu).astype(np.int32)
    random.seed(batch); np.random.seed(int(rate * 1000))
    want = _compare(np.arange(nu, dtype=np.int32), rowptr, col, ni, batch, (ap, an), rate, n_batches=10)
    if rate == 1.0:
        assert all(w.shape[1] == 2 * batch for w in want)


def test_degree_one_and_a_single_possible_negative():
    """degree 1: the positive consumes no word; degree n_items - 1: one item is left to be the negative"""
    ni = 40
    rng = np.random.default_rng(5)
    rows = [np.array([int(rng.integers(ni))]) if u % 3 else rng.permutation(ni)[:ni - 1] for u in range(90)]
    rowptr = np.zeros(91, dtype=np.int32)
    np.cumsum([len(r) for r in rows], out=rowptr[1:])
    col = np.concatenate(rows).astype(np.int32)
    random.seed(9); np.random.seed(9)
    want = _compare(np.arange(90, dtype=np.int32), rowptr, col, ni, 32, n_batches=30)
    for w in want:
        for u, n in zip(w[0], w[2]):
            assert n not in col[rowptr[u]:rowptr[u + 1]]


@pytest.mark.parametrize("case", ["no_train_items", "no_negative", "missing_aug"])
def test_errors_raise_the_host_samplers_exception(case):
    from llmrec_b200.device_sampler import ReferenceDeviceSampler
    from llmrec_b200.host_native import BatchSampler
    nu, ni = 50, 30
    rowptr, col = _small_graph(nu=nu, ni=ni, seed=2)
    ap = an = None
    rate = 0.0
    if case == "no_train_items":
        lens = np.diff(rowptr); lens[17] = 0
        col = np.concatenate([col[rowptr[u]:rowptr[u] + lens[u]] for u in range(nu)]).astype(np.int32)
        rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    if case == "no_negative":
        full = np.arange(ni, dtype=np.int32)
        rows = [full if u == 23 else col[rowptr[u]:rowptr[u + 1]] for u in range(nu)]
        col = np.concatenate(rows).astype(np.int32)
        rowptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    if case == "missing_aug":
        ap = np.full(nu, 1, dtype=np.int32); ap[11] = BatchSampler.MISSING
        an = np.full(nu, 2, dtype=np.int32)
        rate = 1.0
    random.seed(4); np.random.seed(4)
    start = _streams()
    host = BatchSampler(np.arange(nu), rowptr, col, ni, nu, ap, an)
    with pytest.raises((RuntimeError, KeyError)) as want:
        host.draw(np.zeros((3, 2 * nu + 8), dtype=np.int32), rate)
    random.setstate(start[0]); np.random.set_state(start[1])
    ds = ReferenceDeviceSampler(np.arange(nu), rowptr, col, _sorted_rows(rowptr, col), ni, nu, ap, an, ni, rate, "cuda")
    cap = 2 * nu + 8
    buf = torch.zeros((4, cap), dtype=torch.int32, device="cuda")
    meta = torch.stack([torch.arange(cap + 1), torch.arange(cap + 1)], 1).to(torch.int32).cuda().contiguous()
    for _ in range(3):                                                   # later calls draw nothing and do not fault
        ds.fill(buf, meta)
    torch.cuda.synchronize()
    assert int(buf[3, 0]) == nu and int(buf[:3, :nu].abs().sum()) == 0
    with pytest.raises(want.type) as got:
        ds.sync_to_host()
    assert str(got.value) == str(want.value)
    assert _same_streams(_streams(), start)                              # a failed sync leaves the host streams alone


def _run(root, mode, extra, steps=None):
    tr, M = _trainer(root, ["--device_sampler", str(mode), "--deterministic", "1"] + extra)
    seen = []
    step = tr.train_next_batch

    def rec():
        r = step()
        g = tr.hot._gidx
        seen.append(g[:3, :int(g[3, 0])].cpu().clone())
        return r
    tr.train_next_batch = rec
    if steps is None:
        tr.train()
    else:
        for _ in range(steps):
            tr.train_next_batch()
    torch.cuda.synchronize()
    return tr, seen


@pytest.mark.parametrize("graph,branches", [(1, True), (0, True), (1, False)])
def test_trainer_runs_are_bit_identical_to_host_sampled_ones(tiny_root, monkeypatch, graph, branches):
    if not branches:
        monkeypatch.setenv("LLMREC_BRANCHES", "0")
    a, ba = _run(tiny_root, 0, ["--cuda_graph", str(graph)])
    sa = _streams()
    b, bb = _run(tiny_root, 2, ["--cuda_graph", str(graph)])
    assert b.ref_sampler and len(ba) == len(bb) > 4
    for t, (x, y) in enumerate(zip(ba, bb)):
        assert torch.equal(x, y), f"batch {t}"
    assert _same_streams(_streams(), sa)
    ta, tb = a.hot.state_tensors(), b.hot.state_tensors()
    for k in ta:
        assert torch.equal(ta[k], tb[k]), k


@pytest.mark.parametrize("first,second,graph", [(0, 2, 1), (2, 0, 1), (2, 2, 0)])
def test_checkpoints_resume_across_sampler_modes(tiny_root, tmp_path, first, second, graph):
    n, k = 12, 5
    flags = ["--cuda_graph", str(graph)]
    full, bf = _run(tiny_root, first, flags, steps=n)
    if full.ref_sampler:
        full.device_sampler.sync_to_host()
    end = _streams()
    head, bh = _run(tiny_root, first, flags, steps=k)
    ck = os.path.join(str(tmp_path), "k.pt")
    head.save_checkpoint(ck)
    tail, bt = _run(tiny_root, second, flags + ["--resume", ck], steps=n - k)
    for t, (x, y) in enumerate(zip(bf, bh + bt)):
        assert torch.equal(x, y), f"batch {t}"
    if tail.ref_sampler:
        tail.device_sampler.sync_to_host()
    assert _same_streams(_streams(), end)
    tf, tt = full.hot.state_tensors(), tail.hot.state_tensors()
    for key in tf:
        assert torch.equal(tf[key], tt[key]), key


def test_device_sampler_1_is_unchanged(tiny_root):
    """mode 1 keeps its own {seed, step} stream and state layout"""
    tr, _ = _trainer(tiny_root, ["--device_sampler", "1", "--cuda_graph", "0"])
    assert not tr.ref_sampler and tuple(tr.device_sampler.state.shape) == (2,)


def test_checkpoint_taken_while_a_batch_is_pre_drawn_holds_the_streams_before_it(tiny_root, tmp_path):
    """batch k + 1 is already drawn when step k ends; the checkpoint holds the streams of a host-sampled run after k batches"""
    k = 5
    host, bh = _run(tiny_root, 0, ["--cuda_graph", "1"], steps=k)
    want = _streams()
    dev, bd = _run(tiny_root, 2, ["--cuda_graph", "1"], steps=k)
    ds = dev.device_sampler
    assert ds.next is not None and int(ds.next[3, 0]) >= 128                       # batch k + 1 is pre-drawn
    ck = os.path.join(str(tmp_path), "k.pt")
    dev.save_checkpoint(ck)
    assert _same_streams(_streams(), want)
    rng = torch.load(ck, weights_only=True)["rng"]
    assert tuple(rng["py_key"].tolist()) == want[0][1]
    assert np.array_equal(rng["np_key"].numpy().astype(np.uint32), want[1][1]) and rng["np_pos"] == want[1][2]
    host.train_next_batch(); dev.train_next_batch()                               # the pre-drawn batch is the one the host draws next
    torch.cuda.synchronize()
    assert torch.equal(host.hot._gidx[:, :int(host.hot._gidx[3, 0])].cpu()[:3], dev.hot._gidx[:, :int(dev.hot._gidx[3, 0])].cpu()[:3])
