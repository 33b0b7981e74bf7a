"""No GPU: the host restatement of the `--device_sampler 1` kernel (tests/device_sampler_model.py) against a brute-force statement of each
rule in Python integers, the distributions it draws (chi-square at fixed seeds, so deterministic), and the input checks of DeviceSampler."""
import numpy as np
import pytest
from scipy import stats

import device_sampler_model as DM

M64 = (1 << 64) - 1
INT32_MIN = -(1 << 31)


# ---- brute force, Python integers only -------------------------------------------------------------------------------------------------
def sm(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


class Rng:
    def __init__(self, base, ctr):
        self.base, self.ctr = base, ctr

    def next(self):
        self.ctr += 1
        return sm((self.base + 0xD1342543DE82EF95 * self.ctr) & M64) >> 32

    def below(self, n):
        return (self.next() * n) >> 32


def bf_sample(state, exist, rowptr, col, n_items, batch, n_aug, aug_pos, aug_neg, n_aug_table, aug_limit, meta_table, cap):
    """every rule by its plain statement: a full sort by (key, index), a set for membership, the complement listed in order"""
    seed, step = state
    base = sm(seed ^ sm(step))
    exist = [int(x) for x in exist]
    n = len(exist)
    buf = [[-7] * cap for _ in range(4)]
    if batch <= n:
        keys = [(sm(base ^ ((0xA5A5A5A5 + i * 0x9E3779B97F4A7C15) & M64)) >> 32, i) for i in range(n)]
        users = [exist[i] for i in sorted(i for _, i in sorted(keys)[:batch])]
    else:
        users = [exist[Rng(base ^ 0x1111, 4 * b).below(n)] for b in range(batch)]
    for b, u in enumerate(users):
        g = Rng(base ^ 0x2222, b << 20)
        row = [int(x) for x in col[rowptr[u]:rowptr[u + 1]]]
        members = set(row)
        p = row[g.below(len(row))] if row else 0
        c = None
        for _ in range(1 << 16):
            c = g.below(n_items)
            if c not in members:
                break
        else:
            c = [x for x in range(n_items) if x not in members][g.below(n_items - len(row))]
        buf[0][b], buf[1][b], buf[2][b] = u, p, c
    kept = []
    if n_aug > 0 and aug_pos is not None:
        k2 = [(sm(base ^ ((0x3333 + i * 0xD6E8FEB86659FD93) & M64)) >> 32, i) for i in range(batch)]
        for i in sorted(i for _, i in sorted(k2)[:min(n_aug, batch)]):
            u = users[i]
            if 0 <= u < n_aug_table and 0 <= aug_pos[u] < aug_limit and 0 <= aug_neg[u] < aug_limit:
                kept.append((u, int(aug_pos[u]), int(aug_neg[u])))
    kept = kept[:cap - batch]
    for j, (u, p, c) in enumerate(kept):
        buf[0][batch + j], buf[1][batch + j], buf[2][batch + j] = u, p, c
    buf[3][0], buf[3][1] = (int(x) for x in meta_table[batch + len(kept)])
    return np.array(buf, dtype=np.int32), step + 1


def _graph(nu, ni, seed, deg_lo=1, deg_hi=8):
    rng = np.random.default_rng(seed)
    return DM.csr([np.sort(rng.permutation(ni)[:int(rng.integers(deg_lo, deg_hi))]) for _ in range(nu)])


# ---- the restatement against the brute force --------------------------------------------------------------------------------------------
def test_splitmix_and_words_match_python_integers():
    rng = np.random.default_rng(0)
    x = rng.integers(0, 1 << 63, 2000, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, 2000, dtype=np.uint64)
    x[:3] = [0, M64, 1 << 63]
    assert [int(v) for v in DM.splitmix64(x)] == [sm(int(v)) for v in x]
    for b0, c0 in ((0, 0), (M64, 5), (0x2222 ^ 0xDEADBEEF12345678, 7 << 20)):
        g = Rng(b0, c0)
        want = [g.next() for _ in range(50)]
        assert [int(v) for v in DM.rng_words(b0, np.arange(c0 + 1, c0 + 51, dtype=np.uint64))] == want
    assert int(DM.below(0xFFFFFFFF, 7)) == 6 and int(DM.below(0, 7)) == 0


@pytest.mark.parametrize("n,k", [(50, 1), (50, 17), (50, 50), (1000, 999), (7, 3)])
def test_smallest_is_a_sort_by_key_then_index(n, k):
    rng = np.random.default_rng(n + k)
    for trial in range(20):
        keys = rng.integers(0, 6 if trial % 2 else 1 << 32, n).astype(np.uint64)      # heavy ties on odd trials
        want = sorted(i for _, i in sorted(zip(keys.tolist(), range(n)))[:k])
        assert DM.smallest(keys, k).tolist() == want


CASES = {   # name: (n_exist, n_users, n_items, batch, rate, table kind, cap extra)
    "subset": (40, 40, 30, 16, 0.25, "valid", 0),
    "batch_eq_n_exist": (12, 12, 30, 12, 0.5, "valid", 3),
    "with_replacement": (5, 5, 30, 23, 0.3, "valid", 0),
    "one_user": (1, 1, 9, 1, 1.0, "valid", 0),
    "no_tables": (40, 40, 30, 16, 0.0, None, 0),
    "n_aug_eq_batch": (40, 40, 30, 16, 1.0, "valid", 0),
    "n_aug_over_batch": (40, 40, 30, 16, 1.5, "valid", 0),
    "invalid_entries": (60, 60, 30, 32, 1.0, "invalid", 0),
    "exist_subset_of_users": (25, 80, 30, 16, 0.5, "invalid", 4),
}


def _case(name, seed=0):
    n_exist, nu, ni, batch, rate, tables, extra = CASES[name]
    rng = np.random.default_rng(seed)
    rowptr, col = _graph(nu, ni, seed, deg_hi=ni - 1)
    exist = np.sort(rng.permutation(nu)[:n_exist]).astype(np.int32)
    ap = an = None
    if tables:
        n_tab = nu if tables == "valid" else nu - 7                   # the last 7 uids are outside the tables
        ap = rng.integers(0, ni, n_tab).astype(np.int32)
        an = rng.integers(0, ni, n_tab).astype(np.int32)
        if tables == "invalid":
            bad = rng.permutation(n_tab)[:n_tab // 2]
            for j, u in enumerate(bad):
                t = ap if j % 2 else an
                t[u] = (INT32_MIN, -1, ni, ni + 5)[j % 4]
    n_aug = int(batch * rate) if ap is not None else 0
    cap = batch + n_aug + extra
    return dict(exist=exist, rowptr=rowptr, col_sorted=col, n_items=ni, batch=batch, n_aug=n_aug, aug_pos=ap, aug_neg=an,
                n_aug_table=0 if ap is None else len(ap), aug_limit=ni, meta_table=DM.meta_table_for(cap), cap=cap)


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_equals_the_brute_force(name):
    kw = _case(name)
    seen_kept = set()
    for seed, step in [(0, 0), (1, 0), (2022, 7), (M64, 3), (5, 1 << 40)] + [(9, s) for s in range(20)]:
        got, nxt = DM.sample((seed, step), **kw)
        want, _ = bf_sample((seed, step), kw["exist"], kw["rowptr"], kw["col_sorted"], kw["n_items"], kw["batch"], kw["n_aug"],
                            kw["aug_pos"], kw["aug_neg"], kw["n_aug_table"], kw["aug_limit"], kw["meta_table"], kw["cap"])
        assert nxt == step + 1
        np.testing.assert_array_equal(got, want, err_msg=f"{name} seed {seed} step {step}")
        seen_kept.add(int(got[3, 0]) - kw["batch"])
    if name == "invalid_entries":                                   # some selected positions are dropped, some kept
        assert max(seen_kept) < min(kw["n_aug"], kw["batch"]) and max(seen_kept) > 0


def test_missing_uids_are_dropped_not_raised():
    """mode 1 drops a uid missing from augmented_sample_dict (INT32_MIN) or outside the tables; upstream raises KeyError"""
    kw = _case("n_aug_eq_batch")
    kw["aug_pos"] = kw["aug_pos"].copy()
    kw["aug_pos"][kw["exist"][::2]] = INT32_MIN
    buf, _ = DM.sample((3, 0), **kw)
    B = kw["batch"]
    users = buf[0, :B]
    keep = [u for u in users if kw["aug_pos"][u] != INT32_MIN]
    assert 0 < len(keep) < B and buf[0, B:B + len(keep)].tolist() == keep and int(buf[3, 0]) == B + len(keep)


def test_exhausted_rejection_falls_back_to_the_rth_non_member():
    """rows holding all items but a few: after 2^16 rejected candidates the negative is the r-th non-member (never a train item)"""
    ni = 1 << 20
    missing = [[77], [5, 900000], [0, 1, ni - 1]]
    rowptr, col = DM.csr([np.setdiff1d(np.arange(ni), m) for m in missing])
    kw = dict(exist=np.arange(3, dtype=np.int32), rowptr=rowptr, col_sorted=col, n_items=ni, batch=3, n_aug=0, aug_pos=None,
              aug_neg=None, n_aug_table=0, aug_limit=ni, meta_table=DM.meta_table_for(3), cap=3)
    fell_back = 0
    for seed in range(4):
        got, _ = DM.sample((seed, 0), **kw)
        want, _ = bf_sample((seed, 0), *(kw[k] for k in ("exist", "rowptr", "col_sorted", "n_items", "batch", "n_aug", "aug_pos", "aug_neg",
                                                        "n_aug_table", "aug_limit", "meta_table", "cap")))
        np.testing.assert_array_equal(got, want)
        assert all(int(got[2, b]) in missing[b] for b in range(3))
        _, _, words = DM.draw_pos_neg(DM.batch_base(seed, 0), np.arange(3), rowptr, col, ni)
        fell_back += int((words == (1 << 16) + 2).sum())             # pos, 2^16 candidates, r
    assert fell_back >= 4                                            # ~0.94 for the one-hole row, ~0.88 / 0.83 for the others


def test_tie_detection_reports_split_ties():
    keys = np.array([5, 3, 3, 3, 9, 1], dtype=np.uint64)
    assert DM.threshold_ties(keys, 3) == (3, 2)                      # threshold 3: three equal keys, two of them selected
    assert DM.smallest(keys, 3).tolist() == [1, 2, 5]


# ---- distributions (chi-square, fixed seeds) --------------------------------------------------------------------------------------------
P_MIN = 1e-3


def _steps(kw, n, seed=11):
    return [DM.sample((seed, s), **kw)[0] for s in range(n)]


def test_user_inclusion_is_batch_over_n_exist():
    kw = _case("subset")
    counts = np.zeros(kw["exist"].max() + 1)
    for buf in _steps(kw, 3000):
        u = buf[0, :kw["batch"]]
        assert len(set(u.tolist())) == kw["batch"]
        counts[u] += 1
    c = counts[kw["exist"]]
    assert abs(c.mean() - 3000 * kw["batch"] / len(kw["exist"])) < 1e-9
    assert stats.chisquare(c).pvalue > P_MIN


def test_with_replacement_branch_is_uniform_over_exist():
    kw = _case("with_replacement")
    counts = np.zeros(kw["exist"].max() + 1)
    for buf in _steps(kw, 2000):
        np.add.at(counts, buf[0, :kw["batch"]], 1)
    assert stats.chisquare(counts[kw["exist"]]).pvalue > P_MIN


def test_pos_is_uniform_over_the_row_and_neg_over_its_complement():
    ni = 24
    rows = [np.array([3]), np.array([0, 7, 8, 20]), np.arange(0, ni, 2), np.setdiff1d(np.arange(ni), [4, 11, 12])]
    rowptr, col = DM.csr(rows)
    kw = dict(exist=np.arange(4, dtype=np.int32), rowptr=rowptr, col_sorted=col, n_items=ni, batch=4, n_aug=0, aug_pos=None, aug_neg=None,
              n_aug_table=0, aug_limit=ni, meta_table=DM.meta_table_for(4), cap=4)
    pc, nc = np.zeros((4, ni)), np.zeros((4, ni))
    for buf in _steps(kw, 4000):
        for b in range(4):
            u = buf[0, b]
            pc[u, buf[1, b]] += 1
            nc[u, buf[2, b]] += 1
    for u, row in enumerate(rows):
        comp = np.setdiff1d(np.arange(ni), row)
        assert pc[u].sum() == pc[u, row].sum() and nc[u, row].sum() == 0
        if len(row) > 1:
            assert stats.chisquare(pc[u, row]).pvalue > P_MIN, u
        assert stats.chisquare(nc[u, comp]).pvalue > P_MIN, u


def test_augmented_positions_are_a_uniform_subset():
    """batch 8, n_aug 2: all 28 position pairs equally likely"""
    rowptr, col = _graph(8, 30, 1)
    kw = dict(exist=np.arange(8, dtype=np.int32), rowptr=rowptr, col_sorted=col, n_items=30, batch=8, n_aug=2,
              aug_pos=np.arange(8, dtype=np.int32) + 100, aug_neg=np.arange(8, dtype=np.int32), n_aug_table=8, aug_limit=1 << 20,
              meta_table=DM.meta_table_for(10), cap=10)
    pairs = {}
    for buf in _steps(kw, 4200):
        assert int(buf[3, 0]) == 10
        pos_of = {int(u): i for i, u in enumerate(buf[0, :8])}
        sel = tuple(pos_of[int(u)] for u in buf[0, 8:10])
        assert sel[0] < sel[1]                                      # appended in position order
        pairs[sel] = pairs.get(sel, 0) + 1
    assert len(pairs) == 28
    assert stats.chisquare(list(pairs.values())).pvalue > P_MIN


# ---- DeviceSampler input checks (device="cpu": they run before anything touches a GPU) -------------------------------------------------
def _sampler(exist, rows, ni, **kw):
    from llmrec_b200.device_sampler import DeviceSampler
    rowptr, col = DM.csr(rows)
    return DeviceSampler(np.asarray(exist), rowptr, col, ni, 4, None, None, ni, 0.0, "cpu", **kw)


def test_device_sampler_accepts_valid_inputs_and_keeps_its_state_layout():
    ds = _sampler([0, 2], [[1, 3], [], [0, 0, 5]], 6, seed=9)           # user 1 is not an exist user; a repeated item is sorted too
    assert ds.state.tolist() == [9, 0] and ds.keys.numel() == 4 and ds.n_aug == 0


@pytest.mark.parametrize("case", ["no_train_items", "no_negative", "unsorted"])
def test_device_sampler_rejects_what_the_kernel_cannot_sample(case):
    from llmrec_b200.device_sampler import raise_sampler_error
    ni = 6
    rows = [[0, 2], [1, 4, 5], [3]]
    if case == "no_train_items":
        rows[1] = []
    if case == "no_negative":
        rows[2] = list(range(ni))
    if case == "unsorted":
        rows[1] = [1, 5, 4]
    if case == "unsorted":
        with pytest.raises(ValueError, match="row 1 is not sorted"):
            _sampler([0, 1, 2], rows, ni)
        return
    with pytest.raises(RuntimeError) as want:
        raise_sampler_error(2 if case == "no_train_items" else 3)
    with pytest.raises(RuntimeError) as got:
        _sampler([0, 1, 2], rows, ni)
    assert str(got.value) == str(want.value)
