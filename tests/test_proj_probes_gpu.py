"""-m gpu: the projection kernels on term-exact probe operands (tests/proj_probes.py), bit for bit.

On a probe every product the kernel forms is exact, its split of each operand is known in closed form, and every partial sum is
exact in fp32, so a correct kernel returns one fp32 value per output whatever its summation order: 3xTF32 on fp32 tables gives
sum (lo hi + hi lo + hi hi) + b (not the exact dot product), plain TF32 sum hi hi + b, bf16 / int8 tables the exact sum in mode 0 and
sum x w0 + b in mode 1, and the SIMT kernels the exact sum.  A dropped, duplicated or mispaired term fails `torch.equal`, where the
randn tests' tolerances let some through (tests/test_proj_probes_cpu.py).  Mode 0 on fp32 tables also proves the tensor cores ran:
the SIMT kernels would add the lo lo terms.

Cases: every width in modes 0, 1 and 2 on fp32, bf16 and int8 tables; n at stage, chunk and tile edges with k at and off the stage
width; X as a column slice of a wider table; strided Y / dY views with NaN around them (nothing outside a view is read or written);
row maps sorted with gaps and shuffled; an empty problem inside the group; a group large enough for the 256-wide tiles at d <= 128;
accumulate, and five problems sharing one dW / db; a shape only the SIMT kernels take (k = 130) in a group with tensor-core shapes.
Every call is made twice and must give the same bits."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import proj_probes as PP  # noqa: E402

pytestmark = pytest.mark.gpu

cuda = torch.device("cuda")
NAN = float("nan")
WIDTHS = [32, 64, 96, 128, 160, 192, 224, 256]
SMS = 132                     # H100 SXM
# n: one row, a stage (32 fp32 rows / 64 bf16 rows) and its neighbours, a 256-row chunk plus one, two chunk sizes; an empty problem
EDGE_N = {"f32": [1, 31, 32, 33, 63, 64, 65, 257, 1025, 2111, 0],
          "bf16": [1, 63, 64, 65, 127, 128, 129, 257, 1025, 2111, 0]}
# k: below one stage, one stage plus a ragged k8 / k16, a few stages, ragged, the netflix width (int8 tables: k % 16 == 0)
EDGE_K = {"f32": [4, 36, 100, 264, 1536], "bf16": [8, 40, 104, 264, 1536], "i8": [16, 48, 112, 272, 1536]}
BIG = {"f32": [(9000, 1536)] * 4 + [(8001, 100), (9001, 36), (7777, 4)],
       "bf16": [(9000, 1536)] * 4 + [(8001, 104), (9001, 40), (7777, 8)],
       "i8": [(9000, 1536)] * 4 + [(8001, 112), (9001, 48), (7777, 16)]}


def _kinds(path, mode):
    """(X kind, W / dY kind, nonzeros per X row / column) of proj_probes.KINDS for a table type and mode."""
    if mode == 2:
        return PP.KINDS["f32_simt" if path == "f32" else "bf16_simt"]
    return PP.KINDS["f32" if path == "f32" else "bf16"]


def _dev(p):
    return p.to(lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda))


def _table(path, X):
    """The table the kernels read for probe X: fp32 / bf16 as a column slice of a wider table (16 bytes into its row), int8 as
    feat_int8 rows that must dequantize to X exactly."""
    n, k = X.value.shape
    v = torch.from_numpy(X.value).to(cuda)
    if path == "i8":
        from llmrec_b200 import feat_int8 as F8
        T = F8.quantize(v)
        assert torch.equal(F8.dequantize(T, k), v)
        return T
    dt, lead = (torch.float32, 4) if path == "f32" else (torch.bfloat16, 8)
    wide = torch.zeros((max(n, 1), lead + k + 8), dtype=dt, device=cuda)[:n]     # an empty table is still an aligned slice
    wide[:, lead:lead + k] = v.to(dt)
    assert torch.equal(wide[:, lead:lead + k].float(), v)
    return wide[:, lead:lead + k]


def _view(vals, m, d):
    """[m x d] fp32 view into the middle of a NaN [m x 3d] buffer -> (view, buffer); vals (numpy) fills the view when given."""
    wide = torch.full((max(m, 1), 3 * d), NAN, device=cuda)[:m]
    if vals is not None:
        wide[:, d:2 * d] = torch.from_numpy(vals).to(cuda)
    return wide[:, d:2 * d], wide


def _assert_bits(got, want, what):
    g, w = got.contiguous().view(torch.int32), want.contiguous().view(torch.int32)
    if not torch.equal(g, w):
        bad = (g != w).nonzero()
        i = tuple(int(t) for t in bad[0])
        raise AssertionError(f"{what}: {bad.shape[0]} of {g.numel()} elements differ, first at {i}: got {float(got[i])!r}, want {float(want[i])!r}")


class Problem:
    """One projection problem on probes: X (table), W, b, dY (a strided view of m rows), an optional row map, the expected Y buffer
    and the product terms of dW."""

    def __init__(self, path, mode, n, k, d, seed, mapped=0, X=None, col_cap=None):
        xk, wk, cap = _kinds(path, mode)
        rng = np.random.default_rng(seed)
        self.n, self.k = n, k
        if X is None:
            Xp = PP.probe(xk, rng, (n, k), PP.pattern(n, k, cap, col_cap or cap, shift=seed))
            X = (_table(path, Xp), _dev(Xp))
        self.X, Xd = X
        Wp, bp = PP.probe(wk, rng, (d, k)), PP.probe(wk, rng, (d,))
        self.W, self.b = torch.from_numpy(Wp.value).to(cuda), torch.from_numpy(bp.value).to(cuda)
        self.m = 2 * n + 3 if mapped and n else n
        self.rows = None
        if mapped and n:                   # 1: sorted with gaps, 2: shuffled
            pick = rng.permutation(self.m)[:n]
            self.rows = torch.from_numpy(np.sort(pick) if mapped == 1 else pick).to(cuda, torch.int32).contiguous()
        dYp = PP.probe(wk, rng, (self.m, d))
        self.dY, _ = _view(dYp.value, self.m, d)
        Wd, dYd = _dev(Wp), _dev(dYp)
        Y = PP.expected(PP.term_pairs(Xd, Wd, mode), PP.fwd, [(torch.from_numpy(bp.full).to(cuda)[None, :], min(bp.units))])
        self.Y_want = torch.full((self.m, 3 * d), NAN, device=cuda)
        if self.rows is None:
            self.Y_want[:, d:2 * d] = Y
        else:
            self.Y_want[self.rows.long(), d:2 * d] = Y
        pair = dYd if self.rows is None else dYd.to(lambda a: a[self.rows.long()])
        self.dW_pairs = PP.term_pairs(Xd, pair, mode)
        self.dY64, self.dY_unit = dYd.full, min(dYp.units)

    def dW_want(self):
        return PP.expected(self.dW_pairs, PP.wgrad)


def _check_db(db, members, prior, what):
    """db = the members' colsum(dY) (+ prior: (tensor, unit)): bit for bit where every fp32 partial sum is exact (sum |dY| (+ |prior|)
    below 2^24 units), else against fp64 within the randn tests' bound."""
    total = sum(p.dY64.sum(0) for p in members)
    bound = sum(p.dY64.abs().sum(0) for p in members)
    unit = min(p.dY_unit for p in members)
    if prior is not None:
        total, bound, unit = total + prior[0].double(), bound + prior[0].double().abs(), min(unit, prior[1])
    if float(bound.max()) < 2.0 ** 24 * unit:
        _assert_bits(db, total.float(), what)
    else:
        n = max(1, sum(p.m for p in members))
        torch.testing.assert_close(db.double(), total, rtol=1e-4, atol=1e-4 * n ** 0.5, msg=lambda s: f"{what}: {s}")


def _run_group(probs, d, mode, what):
    """Forward then weight gradient of the group, each twice: bits against the expected values, NaN kept outside the views."""
    from llmrec_b200 import ops
    ys = [_view(None, p.m, d) for p in probs]
    fwd = [(p.X, p.W, p.b, y) + ((p.rows,) if p.rows is not None else ()) for p, (y, _) in zip(probs, ys)]
    for rep in range(2):
        ops.proj_fwd_group(fwd, d, mode)
        for i, (p, (_, wide)) in enumerate(zip(probs, ys)):
            _assert_bits(wide, p.Y_want, f"{what} fwd #{rep} problem {i} (n={p.n}, k={p.k}, map={p.rows is not None})")
    outs = [(torch.full((d, p.k), NAN, device=cuda), torch.full((d,), NAN, device=cuda)) for p in probs]
    wg = [(p.X, p.dY, dW, db, False) + ((p.rows,) if p.rows is not None else ()) for p, (dW, db) in zip(probs, outs)]
    for rep in range(2):
        ops.proj_wgrad_group(wg, d, mode)
        for i, (p, (dW, db)) in enumerate(zip(probs, outs)):
            w = f"{what} wgrad #{rep} problem {i} (n={p.n}, k={p.k}, map={p.rows is not None})"
            _assert_bits(dW, p.dW_want(), w)
            _check_db(db, [p], None, w + " db")


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("path", ["f32", "bf16", "i8"])
@pytest.mark.parametrize("d", WIDTHS)
def test_probes_at_stage_chunk_and_tile_edges(d, path, mode):
    """Eleven problems (two grouped launches, 128-wide tiles): n at stage and chunk edges and an empty problem, k at and off the
    stage width; every third problem row-mapped sorted with gaps, every third shuffled."""
    ns = EDGE_N["f32" if path == "f32" else "bf16"]
    ks = EDGE_K[path]
    probs = [Problem(path, mode, n, ks[i % len(ks)], d, seed=1000 * d + 10 * mode + i, mapped=i % 3) for i, n in enumerate(ns)]
    _run_group(probs, d, mode, f"{path} d={d} mode={mode}")


def _rows_per_chunk(n):   # wg_rows_per_chunk in proj_tc.cu
    return PP.rows_per_chunk(n)


def _uses_256_wide_tiles(dims):
    """The grouped launches pick 256-row / 256-feature tiles at d <= 128 when those still give every SM a unit (pick_mb)."""
    fwd = sum(-(-n // 256) for n, _ in dims)
    wg = sum(-(-k // 256) * -(-n // _rows_per_chunk(n)) for n, k in dims)
    return fwd >= SMS and wg >= SMS


@functools.lru_cache(maxsize=1)
def _big_tables(path):
    """(table, device probe) of each BIG problem, shared by the modes and widths."""
    xk, _, cap = PP.KINDS["f32" if path == "f32" else "bf16"]
    rng = np.random.default_rng(7)
    Xs = [PP.probe(xk, rng, (n, k), PP.pattern(n, k, cap, cap, shift=i)) for i, (n, k) in enumerate(BIG[path])]
    return [(_table(path, X), _dev(X)) for X in Xs]


@pytest.mark.parametrize("path", ["f32", "bf16", "i8"])
def test_probes_on_256_wide_tiles(path):
    """A group with enough units for the 256-row / 256-feature tiles (two m64 blocks per consumer) at d <= 128, modes 0 and 1,
    the first two problems row-mapped."""
    assert _uses_256_wide_tiles(BIG[path])
    Xs = _big_tables(path)
    for mode, d in ((0, 32), (0, 128), (1, 64)):
        probs = [Problem(path, mode, n, k, d, seed=d + i, mapped=i if i < 3 else 0, X=X) for i, ((n, k), X) in enumerate(zip(BIG[path], Xs))]
        _run_group(probs, d, mode, f"{path} d={d} mode={mode} 256-wide")


ACC = {"item_trans": ([(9000, 1536), (8000, 1536), (7001, 1536), (9000, 1536), (6000, 1536)], [False, True, True, True, True]),
       "single": ([(9000, 1536)], [True])}


@pytest.mark.parametrize("case", list(ACC))
@pytest.mark.parametrize("path", ["f32", "bf16", "i8"])
def test_probes_accumulate_and_shared_outputs(path, case, d=64):
    """Five problems sharing one dW / db (flags F, T, T, T, T: the first overwrites the prior), and one accumulating into a prior
    on the probes' grid.  The columns' nonzeros are split between the problems, so the shared sums stay exact."""
    from llmrec_b200 import ops
    dims, flags = ACC[case]
    _, wk, cap = PP.KINDS["f32" if path == "f32" else "bf16"]
    probs = [Problem(path, 0, n, k, d, seed=50 + i, col_cap=max(1, (cap - 3) // len(dims))) for i, (n, k) in enumerate(dims)]
    rng = np.random.default_rng(99)
    Pw, Pb = PP.probe(wk, rng, (d, dims[0][1])), PP.probe(wk, rng, (d,))
    prior_W, prior_b = torch.from_numpy(Pw.value).to(cuda), torch.from_numpy(Pb.value).to(cuda)
    dW, db = prior_W.clone(), prior_b.clone()
    for rep in range(2):
        dW.copy_(prior_W)
        db.copy_(prior_b)
        ops.proj_wgrad_group([(p.X, p.dY, dW, db, f) for p, f in zip(probs, flags)], d, 0)
        pairs = [t for p in probs for t in p.dW_pairs]
        want = PP.expected(pairs, PP.wgrad, [(torch.from_numpy(Pw.full).to(cuda), min(Pw.units))] if flags[0] else [])
        _assert_bits(dW, want, f"{path} d={d} {case} dW #{rep}")
        _check_db(db, probs, (prior_b, min(Pb.units)) if flags[0] else None, f"{path} d={d} {case} db #{rep}")


@pytest.mark.parametrize("path", ["f32", "bf16"])
@pytest.mark.parametrize("d", [32, 128, 256])
def test_probes_simt_fallback_group(d, path):
    """k = 130 has no tensor-core kernel, so its group of eight runs on the SIMT kernels, tensor-core shapes included: with coarse
    probes every problem gives the exact sums, and so mode 0 does not form the 3xTF32 terms there."""
    ks = [130, 36 if path == "f32" else 40, 1536, 264]
    probs = [Problem(path, 2, n, ks[i % 4], d, seed=300 + i, mapped=i % 3) for i, n in enumerate([1, 33, 65, 257, 130, 2111, 0, 64])]
    _run_group(probs, d, 0, f"{path} d={d} SIMT group")


def _sums_of_rows(rows, k, bf16):
    """Mode-1 forward with X = 1 and no bias: output j is the tensor cores' sum of W row j (k <= 16: one or two k8 steps, one k16)."""
    from llmrec_b200 import ops
    d = 32
    W = torch.zeros(d, k, dtype=torch.float64)
    for j, r in enumerate(rows):
        W[j, :len(r)] = torch.tensor(r, dtype=torch.float64)
    assert torch.equal(W.float().double(), W)
    W = W.float().to(cuda)
    X = torch.ones(64, k, device=cuda, dtype=torch.bfloat16 if bf16 else torch.float32)
    Y = torch.empty(64, d, device=cuda)
    ops.proj_fwd_group([(X, W, None, Y)], d, 1)
    assert bool((Y == Y[:1]).all())
    return [float(v) for v in Y[0, :len(rows)].cpu()]


@pytest.mark.parametrize("bf16", [False, True])
def test_tc_accumulation_rule(bf16):
    """How one wgmma adds its products to the fp32 accumulator, measured on TF32 (k8) and bf16 (k16) inputs through mode-1 calls
    with X = 1 (H100 80GB HBM3):
      - the step's products and the accumulator are added together: each is aligned to the largest exponent among them and cut
        toward zero 25 bits below it (2^-25 next to 1 survives, 2^-26 does not, wherever it sits in the step or in the accumulator);
      - the sum is rounded toward zero to fp32 (1 + 0.75 ulp -> 1, 1 + 1.75 ulp -> 1 + 1 ulp, the same in magnitude for negatives).
    Products are exact, so a step's result is exact whenever its terms sit on a grid of 2^(emax - 25): the probes' premise.

    The rule reproduces the error, not the bits, of the kernels on randn operands (fp32 emulation of the 3xTF32 / bf16 main loop with
    this rule per wgmma, against the H100): at the fingerprint shape (256 x 256, d = 64) and at 1000 rows of the netflix table
    (9000 x 1536, d = 64) the largest error against fp64 is the H100's to the digit (1.16e-5 and 4.89e-5 3xTF32; 5.1e-6 and 2.7e-5
    bf16), where an exact fp32 accumulation of the same terms stays at 2.1e-6 and 4.0e-6; but 4.3% of the 3xTF32 outputs and 1.1-1.5%
    of the bf16 ones differ from the H100 by one ulp (largest difference 2.4e-7), so the bits are not asserted.  The truncating
    accumulation, not a dropped term, is what puts the 3xTF32 engines above the fp32 bound."""
    k = 16 if bf16 else 8
    one_step = [[1, -1, 2.0 ** -25], [1, -1, 2.0 ** -26], [2.0 ** -25] + [0] * (k - 3) + [1, -1], [2.0 ** -26] + [0] * (k - 3) + [1, -1]]
    assert _sums_of_rows(one_step, k, bf16) == [2.0 ** -25, 0.0, 2.0 ** -25, 0.0]
    # the first step leaves 2^-j in the accumulator, the second adds 1 and -1
    acc = [[2.0 ** -25] + [0] * (k - 1) + [1, -1], [2.0 ** -26] + [0] * (k - 1) + [1, -1]]
    assert _sums_of_rows(acc, 2 * k, bf16) == [2.0 ** -25, 0.0]
    u = 2.0 ** -23
    rounding = [[1, 0.75 * u], [1, 1.75 * u], [-1, -0.75 * u], [-1, -1.75 * u], [1] + [-(2.0 ** -25)] * 7]
    assert _sums_of_rows(rounding, k, bf16) == [1.0, 1 + u, -1.0, -1 - u, 1 - 2.0 ** -22]
    rounding_acc = [[1] + [0] * (k - 1) + [0.75 * u], [-1] + [0] * (k - 1) + [-1.75 * u]]
    assert _sums_of_rows(rounding_acc, 2 * k, bf16) == [1.0, -1 - u]
