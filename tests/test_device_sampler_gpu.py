"""-m gpu: `--device_sampler 1` (csrc/device_sampler.cu) draws exactly the batches of its host restatement (tests/device_sampler_model.py):
every launch's whole [4 x cap] buffer is compared with np.array_equal, and the step counter must advance by one per launch.  Covers the
netflix shape, 10 M exist users, every user and augmentation branch, invalid table entries, ties at both selection thresholds, users whose
rejection loop is exhausted, graph replay, and the Trainer's steps with and without a captured graph."""
import numpy as np
import pytest
import torch

import device_sampler_model as DM

pytestmark = pytest.mark.gpu

INT32_MIN = -(1 << 31)
# {seed, step} found by a one-off search over the restatement: a tie split by the users' threshold (10 M exist users, batch 1024) and
# one split by the augmented-edge threshold (batch 1024, n_aug 102); each test first checks on the restatement that the tie is there
USERS_TIE = (1, 1030)
AUG_TIE = (1, 5004810)


def _sampler(exist, rowptr, col, n_items, batch, aug=None, rate=0.0, aug_limit=None, seed=0):
    from llmrec_b200.device_sampler import DeviceSampler
    ap, an = aug if aug is not None else (None, None)
    return DeviceSampler(exist, rowptr, col, n_items, batch, ap, an, n_items if aug_limit is None else aug_limit, rate, "cuda", seed=seed)


def _model_args(ds, cap, meta):
    host = lambda t: None if t is None else t.cpu().numpy()
    return dict(exist=host(ds.exist), rowptr=host(ds.rowptr), col_sorted=host(ds.col), n_items=ds.n_items, batch=ds.batch, n_aug=ds.n_aug,
                aug_pos=host(ds.aug_pos) if ds.n_aug else None, aug_neg=host(ds.aug_neg) if ds.n_aug else None,
                n_aug_table=ds.aug_pos.numel() if ds.n_aug else 0, aug_limit=ds.aug_limit, meta_table=meta, cap=cap)


def _check(ds, steps, cap=None, start=None):
    """launch `steps` times from {seed, start}; each buffer must equal the restatement's; returns the buffers"""
    cap = ds.batch + ds.n_aug + 8 if cap is None else cap
    meta = DM.meta_table_for(cap)
    meta_d = torch.from_numpy(meta).cuda()
    kw = _model_args(ds, cap, meta)
    seed = int(ds.state[0])
    if start is not None:
        ds.state[1] = start
    step = int(ds.state[1])
    buf = torch.full((4, cap), -7, dtype=torch.int32, device="cuda")
    prev, out = buf.cpu().numpy(), []
    for t in range(steps):
        ds.fill(buf, meta_d)
        got = buf.cpu().numpy()
        want, nxt = DM.sample((seed, step + t), out=prev, **kw)
        assert int(ds.state[1]) == nxt == step + t + 1
        assert np.array_equal(got, want), f"seed {seed} step {step + t}: {np.argwhere(got != want)[:8].tolist()}"
        prev = got
        out.append(got)
    return out


def _netflix(seed=0, valid_tables=False):
    """13 187 users, 17 366 items, power-law item popularity, rows sorted; some augmentation ids >= n_items unless valid_tables"""
    rng = np.random.default_rng(seed)
    nu, ni = 13187, 17366
    rows = [np.unique((rng.pareto(1.0, int(rng.integers(1, 10))) * 30).astype(np.int64) % ni) for _ in range(nu)]
    rowptr, col = DM.csr(rows)
    ap = rng.integers(0, ni if valid_tables else ni + ni // 20, nu).astype(np.int32)
    an = rng.integers(0, ni, nu).astype(np.int32)
    return np.arange(nu, dtype=np.int32), rowptr, col, ni, (ap, an)


@pytest.mark.parametrize("seed", [0, 7, 2022])
def test_netflix_shape_matches_the_restatement(seed):
    exist, rowptr, col, ni, aug = _netflix()
    ds = _sampler(exist, rowptr, col, ni, 1024, aug, 0.1, seed=seed)
    bufs = _check(ds, 50)
    assert len({int(b[3, 0]) for b in bufs}) > 1                            # some augmented ids are dropped, varying B'


def _ten_million():
    rng = np.random.default_rng(3)
    n, ni = 10_000_000, 1000
    deg = rng.integers(1, 4, n)
    rowptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=rowptr[1:])
    rows = np.repeat(np.arange(n, dtype=np.int64), deg)
    col = np.sort(rows * ni + rng.integers(0, ni, len(rows))) % ni            # sorted within each row (repeats allowed)
    return np.arange(n, dtype=np.int32), rowptr.astype(np.int32), col.astype(np.int32), ni


def test_ten_million_users_and_a_tie_at_the_users_threshold():
    exist, rowptr, col, ni = _ten_million()
    seed, step = USERS_TIE
    n_tied, taken = DM.threshold_ties(DM.user_keys(DM.batch_base(seed, step), len(exist)), 1024)
    assert n_tied > taken >= 1                                              # the tie is split by the threshold
    ds = _sampler(exist, rowptr, col, ni, 1024, seed=seed)
    _check(ds, 2, start=step)
    ds.state[0] = 5
    _check(ds, 2, start=0)


def test_tie_at_the_augmented_threshold():
    """two batch positions share the n_aug-th smallest key: exactly n_aug positions are selected, the lower one of the pair"""
    exist, rowptr, col, ni, aug = _netflix(valid_tables=True)
    seed, step = AUG_TIE
    n_tied, taken = DM.threshold_ties(DM.aug_keys(DM.batch_base(seed, step), 1024), 102)
    assert n_tied > taken >= 1
    ds = _sampler(exist, rowptr, col, ni, 1024, aug, 0.1, seed=seed)
    (buf,) = _check(ds, 1, start=step)
    assert int(buf[3, 0]) == 1024 + 102


@pytest.mark.parametrize("n_exist,batch,rate,cap_extra", [
    (1, 1, 1.0, 0),          # one exist user
    (1, 16, 0.5, 3),         # one exist user, batch > n_exist
    (64, 64, 0.25, 0),       # batch == n_exist
    (5, 64, 0.1, 8),         # batch > n_exist: draws with replacement
    (300, 128, 0.0, 0),      # rate 0: no augmentation tables
    (300, 128, 1.0, 0),      # n_aug == batch, cap = batch + n_aug
    (300, 128, 1.5, 0),      # n_aug > batch: clamped to batch
    (2000, 1024, 0.1, 0),
])
def test_user_and_augmentation_branches(n_exist, batch, rate, cap_extra):
    rng = np.random.default_rng(n_exist + batch)
    nu, ni = n_exist + 20, 500
    rowptr, col = DM.csr([np.sort(rng.permutation(ni)[:int(rng.integers(1, 12))]) for _ in range(nu)])
    exist = np.sort(rng.permutation(nu)[:n_exist]).astype(np.int32)
    aug = None
    if rate > 0:
        aug = (rng.integers(0, ni, nu).astype(np.int32), rng.integers(0, ni, nu).astype(np.int32))
    ds = _sampler(exist, rowptr, col, ni, batch, aug, rate, seed=n_exist)
    assert ds.n_aug == (int(batch * rate) if aug is not None else 0)
    bufs = _check(ds, 20, cap=batch + ds.n_aug + cap_extra)
    if rate >= 1.0:
        assert all(int(b[3, 0]) == 2 * batch for b in bufs)                  # every position selected, every entry valid


def test_invalid_augmentation_entries_are_dropped():
    """INT32_MIN (uid missing from augmented_sample_dict), -1, aug_limit, and uids past the end of the tables: dropped, never raised"""
    rng = np.random.default_rng(8)
    nu, ni, batch = 400, 300, 256
    rowptr, col = DM.csr([np.sort(rng.permutation(ni)[:int(rng.integers(1, 12))]) for _ in range(nu)])
    n_tab = nu - 40                                                         # uids >= 360 are outside the tables
    ap = rng.integers(0, ni, n_tab).astype(np.int32)
    an = rng.integers(0, ni, n_tab).astype(np.int32)
    bad = rng.permutation(n_tab)[:n_tab // 2]
    for j, u in enumerate(bad):
        (ap if j % 2 else an)[u] = (INT32_MIN, -1, ni, INT32_MIN)[j % 4]
    ds = _sampler(np.arange(nu, dtype=np.int32), rowptr, col, ni, batch, (ap, an), 1.0, seed=4)
    bufs = _check(ds, 20, cap=2 * batch)
    kept = [int(b[3, 0]) - batch for b in bufs]
    assert 0 < min(kept) and max(kept) < batch


@pytest.mark.parametrize("seed", range(8))
def test_exhausted_rejection_never_returns_a_train_item(seed):
    """2^20 items: one user holds all but one (its negative must be the missing item), three hold all but 2, 3 and 4"""
    ni = 1 << 20
    rng = np.random.default_rng(100 + seed)
    missing = [np.sort(rng.permutation(ni)[:k]) for k in (1, 2, 3, 4)]
    rowptr, col = DM.csr([np.setdiff1d(np.arange(ni), m) for m in missing])
    ds = _sampler(np.arange(4, dtype=np.int32), rowptr, col, ni, 4, seed=seed)
    (buf,) = _check(ds, 1, cap=4)
    assert int(buf[2, 0]) == int(missing[0][0])
    for b in range(4):
        u = int(buf[0, b])
        assert int(buf[2, b]) in missing[u] and int(buf[1, b]) not in missing[u]


def test_graph_replay_equals_eager_launches_and_the_restatement():
    exist, rowptr, col, ni, aug = _netflix()
    k, cap = 6, 1024 + 102 + 8
    meta = torch.from_numpy(DM.meta_table_for(cap)).cuda()
    eager = _sampler(exist, rowptr, col, ni, 1024, aug, 0.1, seed=31)
    want = _check(eager, k, cap=cap)
    ds = _sampler(exist, rowptr, col, ni, 1024, aug, 0.1, seed=31)
    buf = torch.full((4, cap), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ds.fill(buf, meta)
    torch.cuda.synchronize()
    assert int(ds.state[1]) == 0 and int(buf[0, 0]) == -7                   # capturing launches nothing
    for t in range(k):
        g.replay()
        torch.cuda.synchronize()
        assert int(ds.state[1]) == t + 1
        assert np.array_equal(buf.cpu().numpy(), want[t]), t


def _trainer(root, extra):
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir
    args = set_args(parse_args(["--data_path", root, "--dataset", "netflix", "--batch_size", "128", "--epoch", "1", "--debug",
                                "--seed", "2022"] + list(extra)))
    M.set_seed(args.seed)
    gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size, sampler=args.host_sampler)
    batch_test.init(gen, args)
    tr = M.Trainer(data_config={}, data_generator=gen)
    tr.logger.logging = lambda s: None
    return tr, args


@pytest.mark.parametrize("graph", [0, 1])
def test_trainer_steps_read_the_restatements_batches(tiny_root, graph):
    """step n (0-based) trains on the batch of {args.seed, n}: the graph warm-up hands its batch back (state[1] -= 1)"""
    tr, args = _trainer(tiny_root, ["--device_sampler", "1", "--cuda_graph", str(graph)])
    ds, hp = tr.device_sampler, tr.hot
    meta = hp._meta_table.cpu().numpy()
    cap = int(hp._gidx.shape[1])
    kw = _model_args(ds, cap, meta)
    assert int(ds.state[0]) == args.seed and int(ds.state[1]) == 0
    for n in range(6):
        tr.train_next_batch()
        torch.cuda.synchronize()
        got = hp._gidx.cpu().numpy()
        want, _ = DM.sample((args.seed, n), **kw)
        Bp = int(want[3, 0])
        assert int(ds.state[1]) == n + 1
        assert np.array_equal(got[:3, :Bp], want[:3, :Bp]) and np.array_equal(got[3, :2], want[3, :2]), f"step {n}"


@pytest.mark.parametrize("case", ["no_train_items", "no_negative", "unsorted"])
def test_device_sampler_rejects_what_the_kernel_cannot_sample(case):
    from llmrec_b200.device_sampler import raise_sampler_error
    ni = 50
    rows = [np.arange(u % 7 + 1) * 3 for u in range(40)]
    if case == "no_train_items":
        rows[17] = np.zeros(0, dtype=np.int64)
    if case == "no_negative":
        rows[23] = np.arange(ni)
    if case == "unsorted":
        rows[9] = rows[9][::-1]
    rowptr, col = DM.csr(rows)
    if case == "unsorted":
        with pytest.raises(ValueError, match="row 9 is not sorted"):
            _sampler(np.arange(40, dtype=np.int32), rowptr, col, ni, 16)
        return
    with pytest.raises(RuntimeError) as want:
        raise_sampler_error(2 if case == "no_train_items" else 3)
    with pytest.raises(RuntimeError) as got:
        _sampler(np.arange(40, dtype=np.int32), rowptr, col, ni, 16)
    assert str(got.value) == str(want.value)
