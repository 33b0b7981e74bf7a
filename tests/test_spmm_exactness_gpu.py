"""The propagation SpMM family (csrc/spmm.cu) and the row helpers of the hoisted and sharded paths (csrc/rows.cu) against exact fp64
references.  Every SpMM output element is held to its own error bound, derived from the sums it is made of, not to a blanket tolerance:

    plain:    |y^ - y| <= c u (deg_r + n_pieces_r + 3) |rs_r| sum_e |v_e cs_c x_cj| + u |z|            u = 2^-24, c = 2
    softmax:  the logit bound B_r = max_j of the above, carried through the softmax (a factor exp(2 B_r)), plus a few ulp for
              expf, the subtraction of the row max, the sum and the division

and to the identical-bits properties the kernels promise (ticket epilogue == second pass, reused tickets, concurrent operator copies,
TMA-staged kernel == register kernel, row list == tile kernel).  X padding columns, source rows the pattern never references and
masked-out source rows hold NaN; Y views sit between NaN columns, so a read outside X or a write outside Y fails the test.

GPU tests carry their own `gpu` mark: the bound's self-test (a dropped or doubled edge must fail it, an fp32 emulation of the
kernel's summation order must pass it) runs without a GPU."""
import copy
import functools
import itertools
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import scipy.sparse as sp
import torch

gpu = pytest.mark.gpu
cuda = "cuda"

U = 2.0 ** -24
C_BOUND = 2.0
TILES = (8, 16, 24, 120, 248)
WIDTHS = (4, 8, 16, 20, 32, 48, 64, 96, 128, 256, 512, 1536)
TEETH_MAX_DEG = 3 * 248       # one edge of a row stays above the worst-case bound (which grows like deg^2) up to this degree
RATIOS = {}                   # family -> largest error / bound seen (printed at the end of the module, e.g. with -s)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    if RATIOS:
        print("\nlargest error / bound per family: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(RATIOS.items())))


# ---------------------------------------------------------------------------------------------------------------------------------
# graphs and inputs (seeded; the TMA-staged comparison rebuilds them in child processes)
# ---------------------------------------------------------------------------------------------------------------------------------
class Graph:
    """CSR pattern with fp32 vals / rs / cs in [0.5, 1.5); the last `unref` source rows (and any never drawn) are never referenced."""

    def __init__(self, degs, n_cols, seed, unref=64):
        rng = np.random.default_rng(seed)
        self.deg = np.asarray(degs, np.int64)
        self.n_rows, self.n_cols = len(self.deg), int(n_cols)
        self.rowptr = np.concatenate([[0], np.cumsum(self.deg)]).astype(np.int64)
        self.col = rng.integers(0, self.n_cols - unref, int(self.rowptr[-1])).astype(np.int32)
        self.vals = rng.uniform(0.5, 1.5, self.col.size).astype(np.float32)
        self.rs = rng.uniform(0.5, 1.5, self.n_rows).astype(np.float32)
        self.cs = rng.uniform(0.5, 1.5, self.n_cols).astype(np.float32)
        self.referenced = np.zeros(self.n_cols, bool)
        self.referenced[self.col] = True
        self._dev = None

    def erow(self):
        return np.repeat(np.arange(self.n_rows), self.deg)

    def dev(self):
        if self._dev is None:
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
            self._dev = (t(self.rowptr.astype(np.int32)), t(self.col), t(self.vals), t(self.rs), t(self.cs))
        return self._dev

    def op(self, tile, max_rows=15, vals=True, rs=True, cs=True):
        from llmrec_b200.ops import CsrOperator, TilePlan
        rp, col, v, r, c = self.dev()
        plan = TilePlan(rp, self.n_rows, tile, max_rows)
        assert plan.tile_nnz == tile
        return CsrOperator(rp, col, self.n_rows, self.n_cols, vals=v if vals else None, rs=r if rs else None, cs=c if cs else None, plan=plan)


def boundary_degrees(tile, seed=0):
    """Rows at the planner's boundaries for one tile size: runs of more than 15 empty rows at the start, middle and end; degree
    tile - 1, tile, tile + 1 and exact multiples; a 15-row group ending exactly at tile non-zeros (its 15th row-end byte is the
    largest); 16 one-entry rows; degrees 7, 8, 9, 31, 32, 33 and 248 + those; random short rows."""
    rng = np.random.default_rng(seed + tile)
    q = tile // 15
    degs = [0] * 17
    degs += [tile, tile + 1, 2 * tile, 3 * tile, tile - 1, 1, 0, tile, 2 * tile + 1]
    degs += [0] * 20
    degs += [q] * 14 + [tile - 14 * q]
    degs += [1] * 16
    degs += rng.integers(0, min(tile, 40) + 1, 200).tolist()
    degs += [7, 8, 9, 31, 32, 33] + [248 + r for r in (7, 8, 9, 31, 32, 33)]
    degs += [q] * 14 + [tile - 14 * q, 0, 0]
    degs += [0] * 18
    return np.array(degs, np.int64)


@functools.lru_cache(maxsize=None)
def boundary_graph(tile):
    return Graph(boundary_degrees(tile), 3000, seed=tile)


@functools.lru_cache(maxsize=None)
def powerlaw_graph():
    """1500 rows of power-law degree, two hub rows of more than 10^4 entries."""
    rng = np.random.default_rng(7)
    degs = np.minimum(rng.zipf(1.6, 1500), 2000)
    degs[[3, 900]] = (12001, 25003)
    degs[100:130] = 0
    return Graph(degs, 6000, seed=8)


@functools.lru_cache(maxsize=None)
def rowlist_graph():
    """40 000 rows: mostly short, some of a few hundred entries, five hubs of thousands."""
    rng = np.random.default_rng(9)
    degs = rng.integers(0, 20, 40000)
    degs[rng.choice(40000, 200, replace=False)] = rng.integers(100, 300, 200)
    degs[[0, 1, 2, 17, 39999]] = (6000, 3000, 4500, 249, 5000)
    return Graph(degs, 20000, seed=10)


@functools.lru_cache(maxsize=None)
def bulk_graph():
    """For the TMA-staged kernel at tile 248: complete-row tiles of 1 to 31 groups of 8, degrees 7, 8, 9, 31, 32, 33 mod 248, a hub row
    split into 301 pieces, runs of empty rows."""
    rng = np.random.default_rng(11)
    degs = [0] * 20 + rng.integers(0, 41, 3000).tolist()
    degs += [248 * k + r for k in (0, 1, 2, 3) for r in (7, 8, 9, 31, 32, 33)]
    degs += [0] * 17 + [248 * 300 + 5] + rng.integers(1, 249, 600).tolist() + [0] * 16
    for k in range(1, 32):                  # a tile of exactly k groups (the last one partial unless k % 3 == 0), cut off by a long row
        degs += [8 * k - k % 3, 249]
    return Graph(degs, 40000, seed=12)


def x_values(rng, n, d):
    """magnitudes in [0.5, 2), random signs: every term of a sum is far from zero, so one dropped edge is never invisible"""
    return (rng.uniform(0.5, 2.0, (n, d)) * rng.choice([-1.0, 1.0], (n, d))).astype(np.float32)


def mask_words(keep):
    """uint32 bitmask over rows (RowSet layout: (n + 31) // 32 + 1 words) as an int32 CUDA tensor"""
    words = np.zeros((keep.size + 31) // 32 + 1, np.uint32)
    idx = np.nonzero(keep)[0]
    np.bitwise_or.at(words, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
    return torch.from_numpy(words.view(np.int32)).to(cuda)


# ---------------------------------------------------------------------------------------------------------------------------------
# fp64 reference and bound
# ---------------------------------------------------------------------------------------------------------------------------------
def reference(g, Xs, Zs, softmax, tile, vals=True, rs=True, cs=True, keep_src=None, extra=0):
    """[(y, bound)] per segment for Y_s = epi(diag(rs) P(vals) diag(cs) X_s) + Z_s in fp64 (module docstring).  keep_src: masked-out
    source rows contribute nothing; extra: partial sums added on top of the pieces (8 for the one-CTA-per-row kernel)."""
    erow = g.erow()
    w = (g.vals.astype(np.float64) if vals else np.ones(g.col.size)) * (g.cs[g.col].astype(np.float64) if cs else 1.0)
    sel = np.ones(g.col.size, bool) if keep_src is None else keep_src[g.col]
    A = sp.csr_matrix((w[sel], (erow[sel], g.col[sel])), shape=(g.n_rows, g.n_cols))
    Aa = abs(A)
    r = g.rs.astype(np.float64) if rs else np.ones(g.n_rows)
    npc = np.where(g.deg > tile, -(-g.deg // tile), 0)
    K = (g.deg + npc + 3 + extra).astype(np.float64)[:, None]
    out = []
    for X, Z, sm in zip(Xs, Zs, softmax):
        a = r[:, None] * (A @ X)
        B = C_BOUND * U * K * (np.abs(r)[:, None] * (Aa @ np.abs(X)))
        z = np.zeros_like(a) if Z is None else Z
        if sm:
            m = a.max(1, keepdims=True)
            e = np.exp(a - m)
            s = e / e.sum(1, keepdims=True)
            arg = 2.0 * B.max(1, keepdims=True) + C_BOUND * U * (np.abs(a - m) + a.shape[1] + 8)
            rel = np.minimum(s * np.expm1(np.minimum(arg, 700.0)), 2.0)       # a softmax output lies in [0, 1] (hub rows reach the cap)
            out.append((s + z, rel + U * (s + np.abs(z)) + 2.0 ** -126))
        else:
            out.append((a + z, B + U * np.abs(z)))
    return out


def ratio_of(got, y, bound):
    err = np.abs(got - y)
    return np.divide(err, bound, out=np.where(err == 0, 0.0, np.inf), where=bound > 0)


def check(got, y, bound, family, what="", rows=None):
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    if rows is not None:
        got, y, bound = got[rows], y[rows], bound[rows]
    assert np.isfinite(got).all(), f"{what}: {int((~np.isfinite(got)).sum())} non-finite outputs (unwritten, or a NaN source row was read)"
    ratio = ratio_of(got, y, bound)
    RATIOS[family] = max(RATIOS.get(family, 0.0), float(ratio.max(initial=0.0)))
    if ratio.size and ratio.max() > 1.0:
        k = np.unravel_index(np.argmax(ratio), ratio.shape)
        raise AssertionError(f"{what}: {int((ratio > 1).sum())} elements beyond the fp64 bound; worst at {k}: got {got[k]!r}, "
                             f"want {y[k]!r}, error {abs(got[k] - y[k]):.3g} > bound {bound[k]:.3g}")


# ---------------------------------------------------------------------------------------------------------------------------------
# launching column views of wide NaN-padded buffers
# ---------------------------------------------------------------------------------------------------------------------------------
def layout(nseg, d, off, gap):
    return off + nseg * (d + gap), [off + s * (d + gap) for s in range(nseg)]


def make_inputs(g, d, nseg, z, seed, xoff=4, off=4, zoff=None, gap=4, keep_src=None):
    """numpy X / Z blocks and the device buffers holding them as column views; NaN everywhere outside the views, on unreferenced
    and on masked-out source rows.  z: None, 'sep' (its own buffer) or 'alias' (Z is Y, Y prefilled with Z)."""
    rng = np.random.default_rng(seed)
    zoff = off if zoff is None else zoff
    WX, cx = layout(nseg, d, xoff, gap)
    WY, cy = layout(nseg, d, off, gap)
    WZ, cz = layout(nseg, d, zoff, gap)
    Xw = np.full((g.n_cols, WX), np.nan, np.float32)
    Yw = np.full((g.n_rows, WY), np.nan, np.float32)
    Zw = np.full((g.n_rows, WZ), np.nan, np.float32)
    dead = ~g.referenced if keep_src is None else ~(g.referenced & keep_src)
    Xs, Zs = [], []
    for s in range(nseg):
        x = x_values(rng, g.n_cols, d)
        x[dead] = np.nan
        Xw[:, cx[s]:cx[s] + d] = x
        Xs.append(x.astype(np.float64))
        if z:
            zz = x_values(rng, g.n_rows, d)
            (Yw if z == "alias" else Zw)[:, (cy if z == "alias" else cz)[s]:(cy if z == "alias" else cz)[s] + d] = zz
            Zs.append(zz.astype(np.float64))
        else:
            Zs.append(None)
    dev = lambda a: torch.from_numpy(a).to(cuda)
    return dict(Xs=Xs, Zs=Zs, X=dev(Xw), Y=dev(Yw), Z=dev(Zw) if z == "sep" else None, cx=cx, cy=cy, cz=cz, d=d, nseg=nseg, z=z)


def seg_list(io, softmax):
    d, X, Y = io["d"], io["X"], io["Y"]
    segs = []
    for s in range(io["nseg"]):
        Zv = None
        if io["z"] == "alias":
            Zv = Y[:, io["cy"][s]:io["cy"][s] + d]
        elif io["z"] == "sep":
            Zv = io["Z"][:, io["cz"][s]:io["cz"][s] + d]
        segs.append((X[:, io["cx"][s]:io["cx"][s] + d], Y[:, io["cy"][s]:io["cy"][s] + d], Zv, bool(softmax[s])))
    return segs


def run_segments(op, g, d, nseg, *, tile, softmax=None, z=None, seed=0, vals=True, rs=True, cs=True, keep_src=None, src_mask=None,
                 family="register", check_result=True, **lay):
    """one op.apply over nseg column views; checks that nothing beside the Y views changed and every view element is within its
    fp64 bound; returns the Y views on the host (for identical-bits comparisons)"""
    softmax = softmax or [False] * nseg
    io = make_inputs(g, d, nseg, z, seed, keep_src=keep_src, **lay)
    op.apply(seg_list(io, softmax), src_mask=src_mask)
    Yh = io["Y"].cpu()
    outs = [Yh[:, c:c + d] for c in io["cy"]]
    if check_result:
        pad = np.ones(Yh.shape[1], bool)
        for c in io["cy"]:
            pad[c:c + d] = False
        assert bool(torch.isnan(Yh[:, torch.from_numpy(pad)]).all()), "a column beside the Y views was written"
        refs = reference(g, io["Xs"], io["Zs"], softmax, tile, vals, rs, cs, keep_src)
        for s, ((y, b), got) in enumerate(zip(refs, outs)):
            check(got, y, b, family + (" +Z" if z else ""), f"d={d} nseg={nseg} segment {s} softmax={softmax[s]} z={z}")
    return outs


def no_tickets(op):
    """the same operator with its long rows reduced by the spmm_finish_kernel second pass"""
    o = copy.copy(op)
    o.plan = copy.copy(op.plan)
    o.plan.tickets, o.plan.scratch = None, None
    return o


def pow2_softmax_ok(d):
    return d % 4 == 0 and (d // 4) & (d // 4 - 1) == 0 and d <= 128


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU: the bound has teeth, and a correct fp32 summation passes it
# ---------------------------------------------------------------------------------------------------------------------------------
def perturbed(g, kind):
    """g with, in every row of 1 .. TEETH_MAX_DEG entries, its first or last edge dropped, or its middle edge counted twice"""
    h = copy.copy(g)
    rows = np.nonzero((g.deg >= 1) & (g.deg <= TEETH_MAX_DEG))[0]
    pick = {"drop_first": g.rowptr[rows], "drop_last": g.rowptr[rows + 1] - 1, "double_middle": g.rowptr[rows] + g.deg[rows] // 2}[kind]
    erow = g.erow()
    if kind == "double_middle":
        order = np.argsort(np.concatenate([erow, erow[pick]]), kind="stable")
        col, vals, erow2 = (np.concatenate([a, a[pick]])[order] for a in (g.col, g.vals, erow))
    else:
        keep = np.ones(g.col.size, bool)
        keep[pick] = False
        col, vals, erow2 = g.col[keep], g.vals[keep], erow[keep]
    h.col, h.vals = col, vals
    h.deg = np.bincount(erow2, minlength=g.n_rows).astype(np.int64)
    h.rowptr = np.concatenate([[0], np.cumsum(h.deg)])
    return h, rows


def emulate_fp32(g, X, tile, softmax):
    """fp32 with the kernel's order (sequential per piece of <= tile entries, pieces added in order, then rs) but a separate rounding
    for every product and sum (the kernel uses fma): a correct kernel that the bound must accept"""
    X32 = X.astype(np.float32)
    w = g.vals * g.cs[g.col]
    erow = g.erow()
    loc = np.arange(g.col.size) - g.rowptr[erow]
    split = g.deg[erow] > tile
    piece, pos = np.where(split, loc // tile, 0), np.where(split, loc % tile, loc)
    acc = np.zeros((g.n_rows, int(piece.max(initial=0)) + 1, X.shape[1]), np.float32)
    for k in range(int(pos.max(initial=-1)) + 1):
        s = pos == k
        acc[erow[s], piece[s]] = acc[erow[s], piece[s]] + w[s, None] * X32[g.col[s]]
    tot = np.zeros((g.n_rows, X.shape[1]), np.float32)
    for p in range(acc.shape[1]):
        tot = tot + acc[:, p]
    a = tot * g.rs[:, None]
    if softmax:
        e = np.exp(a - a.max(1, keepdims=True))
        a = e * (np.float32(1) / e.sum(1, keepdims=True))
    return a.astype(np.float64)


@pytest.mark.parametrize("tile", TILES)
def test_bound_rejects_a_dropped_or_doubled_edge_and_accepts_fp32(tile):
    g = boundary_graph(tile)
    variants = {k: perturbed(g, k) for k in ("drop_first", "drop_last", "double_middle")}
    for i, d in enumerate(WIDTHS):
        rng = np.random.default_rng(d)
        X = x_values(rng, g.n_cols, d).astype(np.float64)
        for sm in ((False, True) if pow2_softmax_ok(d) else (False,)):
            (y, bound), = reference(g, [X], [None], [sm], tile)
            assert (ratio_of(emulate_fp32(g, X, tile, sm), y, bound) <= 1.0).all(), (d, sm)
            for kind, (h, rows) in variants.items():
                (y2, _), = reference(h, [X], [None], [sm], tile)
                worst = ratio_of(y2, y, bound).max(1)[rows]
                # a softmax forgets a shift shared by all columns: an edge whose x row is nearly constant across a narrow segment
                # can hide behind the bound (1 row in ~1300 at d = 8); plain outputs must show every edge
                missed = rows[worst <= 1.0]
                assert missed.size <= (0.01 * rows.size if sm else 0), (kind, d, sm, missed[:5], g.deg[missed[:5]])


# ---------------------------------------------------------------------------------------------------------------------------------
# sweeps against fp64
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", ("boundary", "powerlaw"))
@pytest.mark.parametrize("max_rows", (1, 7, 15))
@pytest.mark.parametrize("tile", TILES)
def test_tile_plans_match_fp64(tile, max_rows, kind):
    g = boundary_graph(tile) if kind == "boundary" else powerlaw_graph()
    op = g.op(tile, max_rows)
    d = (4, 8, 16, 20, 32, 64, 128)[(TILES.index(tile) + max_rows) % 7]
    sm = [pow2_softmax_ok(d), False]
    run_segments(op, g, d, 2, tile=tile, softmax=sm, z="sep", seed=tile + max_rows)
    run_segments(op, g, d, 1, tile=tile, seed=tile * max_rows + 1)                     # the same operator again: tickets were reset


WIDTH_CASES = [(4, 1), (4, 33), (8, 5), (16, 2), (20, 7), (32, 16), (48, 17), (64, 33), (96, 7), (128, 16), (128, 17), (256, 5),
               (256, 16), (512, 1), (512, 5), (768, 1), (1536, 1), (1536, 2)]


@gpu
@pytest.mark.parametrize("d,nseg", WIDTH_CASES)
def test_widths_and_segment_counts_match_fp64(d, nseg):
    """lane groups of 8, 16 and 32, 1 to 48 column windows, launches chunked at 16 segments (scratch and tickets reused), both sides of
    the ticket threshold (nseg * d = 2048)"""
    g = powerlaw_graph()
    tile = 248 if WIDTH_CASES.index((d, nseg)) % 2 == 0 else 16
    op = g.op(tile)
    sm = [pow2_softmax_ok(d) and s % 2 == 0 for s in range(nseg)]
    run_segments(op, g, d, nseg, tile=tile, softmax=sm, z="sep", seed=d * nseg)


@gpu
@pytest.mark.parametrize("z", (None, "sep", "alias"))
@pytest.mark.parametrize("vals,rs,cs", list(itertools.product((False, True), repeat=3)))
def test_scaling_and_epilogue_variants(vals, rs, cs, z):
    g = powerlaw_graph()
    op = g.op(120, vals=vals, rs=rs, cs=cs)
    for i, sm in enumerate(([False] * 3, [True, False, True], [True] * 3)):
        run_segments(op, g, 32, 3, tile=120, softmax=sm, z=z, seed=i, vals=vals, rs=rs, cs=cs)


SCALAR_CASES = [("unaligned X", 32, 2, False), ("unaligned Z", 64, 3, False), ("odd d", 7, 2, True), ("odd d", 33, 17, False),
                ("softmax f4 not a power of two", 48, 2, True), ("softmax f4 not a power of two", 96, 1, True), ("softmax above 128", 256, 2, True)]


@gpu
@pytest.mark.parametrize("why,d,nseg,sm", SCALAR_CASES)
def test_scalar_fallback_matches_fp64_and_refuses_a_source_mask(why, d, nseg, sm):
    g = powerlaw_graph()
    op = g.op(248)
    lay = dict(xoff=1) if why == "unaligned X" else dict(zoff=1) if why == "unaligned Z" else {}
    softmax = [sm and s % 2 == 0 for s in range(nseg)]
    run_segments(op, g, d, nseg, tile=248, softmax=softmax, z="sep", seed=d, family="scalar", **lay)
    io = make_inputs(g, d, nseg, "sep", 0, **lay)
    with pytest.raises(RuntimeError, match="source-row mask"):
        op.apply(seg_list(io, softmax), src_mask=mask_words(np.ones(g.n_cols, bool)))
    assert bool(torch.isnan(io["Y"]).all())                                     # refused before any launch


@gpu
@pytest.mark.parametrize("vals", (False, True))
def test_source_mask_with_long_row_pieces(vals):
    g = powerlaw_graph()
    op = g.op(248, vals=vals, cs=False)
    assert op.plan.n_split > 0 and op.plan.tickets is not None
    keep = np.random.default_rng(5).random(g.n_cols) < 0.6
    m = mask_words(keep)
    run_segments(op, g, 64, 2, tile=248, softmax=[True, False], z="sep", vals=vals, cs=False, keep_src=keep, src_mask=m, seed=1)
    run_segments(op, g, 128, 17, tile=248, vals=vals, cs=False, keep_src=keep, src_mask=m, seed=2)      # chunked: 16 + 1 segments


# ---------------------------------------------------------------------------------------------------------------------------------
# identical bits
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("d,nseg", [(16, 1), (128, 1), (64, 8), (128, 16)])
def test_ticket_epilogue_equals_the_second_pass(d, nseg):
    """pieces of a long row added by the last piece to finish (tickets) == spmm_finish_kernel: one and several column windows"""
    g = powerlaw_graph()
    op = g.op(248)
    assert op.plan.tickets is not None and op.plan.n_split > 0
    for sm in (False, True):
        softmax = [sm and s % 2 == 0 for s in range(nseg)]
        a = run_segments(op, g, d, nseg, tile=248, softmax=softmax, z="sep", seed=d + nseg)
        b = run_segments(no_tickets(op), g, d, nseg, tile=248, softmax=softmax, z="sep", seed=d + nseg)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), (d, nseg, sm)


@gpu
def test_wide_launch_above_the_ticket_threshold_equals_each_segment_alone():
    """16 x 256 columns (second pass) and 16 x 128 + 1 (tickets, chunked) give each segment the bits it has when launched alone"""
    g = powerlaw_graph()
    op = g.op(248)
    for d, nseg in ((256, 16), (128, 17)):
        io = make_inputs(g, d, nseg, "sep", seed=d)
        segs = seg_list(io, [False] * nseg)
        op.apply(segs)
        wide = [y.clone() for _, y, _, _ in segs]
        io["Y"].fill_(float("nan"))
        for s in range(nseg):
            op.apply([segs[s]])
            assert torch.equal(segs[s][1], wide[s]), (d, nseg, s)


@gpu
def test_reused_tickets_match_a_fresh_operator():
    """one operator alternates launches of 1 and 16 column windows, lane groups of 8 and 32, with and without softmax; the tickets
    each launch leaves behind must not change the next one"""
    g = powerlaw_graph()
    op = g.op(248)
    for i, (d, nseg, sm) in enumerate([(128, 1, False), (128, 16, False), (128, 1, True), (4, 1, False), (128, 16, True),
                                       (16, 1, True), (128, 1, False), (64, 8, True)]):
        a = run_segments(op, g, d, nseg, tile=248, softmax=[sm] * nseg, seed=i, check_result=False)
        b = run_segments(g.op(248), g, d, nseg, tile=248, softmax=[sm] * nseg, seed=i, check_result=False)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), (i, d, nseg, sm)
        assert not any(bool(torch.isnan(x).any()) for x in a)


@gpu
def test_branch_copies_on_two_streams_match_sequential_launches():
    """op and op.branch() share a plan but own scratch and tickets: overlapping launches give the sequential bits"""
    g = powerlaw_graph()
    op = g.op(248)
    br = op.branch()
    ios = [make_inputs(g, 128, 4, "sep", seed=s) for s in (1, 2)]
    segs = [seg_list(io, [True, False, False, True]) for io in ios]
    op.apply(segs[0]); br.apply(segs[1])
    want = [io["Y"].clone() for io in ios]
    for io in ios:
        io["Y"].fill_(float("nan"))
    cur = torch.cuda.current_stream()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(cur); s2.wait_stream(cur)
    for _ in range(4):
        with torch.cuda.stream(s1):
            op.apply(segs[0])
        with torch.cuda.stream(s2):
            br.apply(segs[1])
    cur.wait_stream(s1); cur.wait_stream(s2)
    torch.cuda.synchronize()
    for io, w in zip(ios, want):
        assert torch.equal(io["Y"].nan_to_num(7.0), w.nan_to_num(7.0))


BULK_VARIANTS = [dict(vals=True, rs=True, cs=False, sm=False, z=None), dict(vals=False, rs=True, cs=False, sm=True, z=None),
                 dict(vals=True, rs=True, cs=True, sm=False, z="sep"), dict(vals=False, rs=True, cs=False, sm=True, z="alias")]


def bulk_runs():
    """(tile, variant, Y view) for every leg of the TMA-staged comparison; X is contiguous (the staged kernel copies 512-byte rows)"""
    g = bulk_graph()
    out = []
    for tile in (248, 16):
        for i, v in enumerate(BULK_VARIANTS):
            op = g.op(tile, vals=v["vals"], rs=v["rs"], cs=v["cs"])
            y, = run_segments(op, g, 128, 1, tile=tile, softmax=[v["sm"]], z=v["z"], seed=i, vals=v["vals"], rs=v["rs"], cs=v["cs"],
                              check_result=False, xoff=0, off=0, zoff=0, gap=0)
            out.append(y.numpy().copy())
    return out


_BULK_CHILD = r"""
import sys, numpy as np
sys.path[:0] = [%r, %r]
import test_spmm_exactness_gpu as T
np.save(sys.argv[1], np.stack(T.bulk_runs()))
"""


@gpu
def test_tma_staged_kernel_equals_the_register_kernel_at_every_ring_position():
    """LLMREC_SPMM_BULK (read once per process) forces spmm_bulk_kernel on or off, so each leg runs in its own process.  At tile 248
    the tiles hold 1 to 31 groups of 8 rows: the 3-stage mbarrier ring wraps up to ten times per tile and every column/weight
    prefetch slot is used."""
    g = bulk_graph()
    t = g.op(248).plan.tiles.cpu().numpy()
    assert set(range(1, 32)) <= set((-(-(t[:, 3] - t[:, 2]) // 8)).tolist())
    here = os.path.dirname(os.path.abspath(__file__))
    legs = []
    with tempfile.TemporaryDirectory() as tmp:
        for flag in ("0", "1"):
            path = os.path.join(tmp, f"bulk{flag}.npy")
            r = subprocess.run([sys.executable, "-c", _BULK_CHILD % (os.path.dirname(here), here), path], env=dict(os.environ, LLMREC_SPMM_BULK=flag),
                               capture_output=True, text=True, timeout=300)
            assert r.returncode == 0, r.stderr[-3000:]
            legs.append(np.load(path))
    reg, bulk = legs
    for k, (tile, v) in enumerate(itertools.product((248, 16), BULK_VARIANTS)):
        io = make_inputs(g, 128, 1, v["z"], k % len(BULK_VARIANTS), xoff=0, off=0, zoff=0, gap=0)
        (y, b), = reference(g, io["Xs"], io["Zs"], [v["sm"]], tile, v["vals"], v["rs"], v["cs"])
        check(reg[k], y, b, "register" + (" +Z" if v["z"] else ""), f"register kernel, tile {tile} {v}")
        check(bulk[k], y, b, "bulk" + (" +Z" if v["z"] else ""), f"staged kernel, tile {tile} {v}")
        assert np.array_equal(reg[k], bulk[k]), (tile, v, int((reg[k] != bulk[k]).sum()))


# ---------------------------------------------------------------------------------------------------------------------------------
# row lists
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("cta", (False, True))
@pytest.mark.parametrize("d", (32, 64, 128))
def test_row_lists_match_fp64_and_the_tile_kernel(d, cta):
    """10^5 list entries (several passes of either persistent grid) with duplicates and -1; the device-side count below, at and above
    max_rows.  Rows of <= tile_nnz entries take the tile kernel's terms in its order: identical bits (for the one-CTA-per-row kernel
    only rows of <= 32 entries, which warp 0 sums alone; longer rows are added as 8 warp partials)."""
    g = rowlist_graph()
    op = g.op(248)
    rng = np.random.default_rng(d + cta)
    lst = np.concatenate([rng.permutation(g.n_rows), rng.integers(0, g.n_rows, 40000), np.full(20000, -1)]).astype(np.int32)
    rng.shuffle(lst)
    rows_dev = torch.from_numpy(lst).to(cuda)
    same_order = g.deg <= (32 if cta else 248)
    for i, (sm, z) in enumerate(((False, None), (True, "sep"))):
        full = make_inputs(g, d, 1, z, seed=i)
        op.apply(seg_list(full, [sm]))
        want = full["Y"][:, full["cy"][0]:full["cy"][0] + d].cpu()
        (y, b), = reference(g, full["Xs"], full["Zs"], [sm], 248, extra=8 if cta else 0)
        for count, max_rows in ((lst.size, lst.size), (60000, lst.size), (lst.size, 70000)):
            io = make_inputs(g, d, 1, z, seed=i)
            X, Y, Z, _ = seg_list(io, [sm])[0]
            cnt = torch.tensor([count], dtype=torch.int32, device=cuda)
            op.apply_rows((X, Y, Z, sm), rows_dev, cnt, max_rows=max_rows, cta_per_row=cta)
            Yh = io["Y"].cpu()
            got = Yh[:, io["cy"][0]:io["cy"][0] + d].clone()
            listed = np.zeros(g.n_rows, bool)
            head = lst[:min(count, max_rows)]
            listed[head[head >= 0]] = True
            assert bool(torch.isnan(got[torch.from_numpy(~listed)]).all()), "an unlisted row was written"
            Yh[:, io["cy"][0]:io["cy"][0] + d] = float("nan")
            assert bool(torch.isnan(Yh).all()), "a column beside the Y view was written"
            check(got, y, b, "rows" + (" +Z" if z else ""), f"d={d} cta={cta} softmax={sm} count={count} max_rows={max_rows}", rows=listed)
            sel = torch.from_numpy(listed & same_order)
            assert torch.equal(got[sel], want[sel]), (d, cta, sm, count, int((got[sel] != want[sel]).sum()))


# ---------------------------------------------------------------------------------------------------------------------------------
# stand-alone softmax kernels
# ---------------------------------------------------------------------------------------------------------------------------------
def softmax_ref(a, argerr=0.0):
    """fp64 softmax of rows of `a` and a bound for an fp32 kernel: argerr = extra absolute error of each exponent's argument"""
    m = a.max(1, keepdims=True)
    e = np.exp(a - m)
    s = e / e.sum(1, keepdims=True)
    return s, s * np.expm1(C_BOUND * U * (np.abs(a - m) + a.shape[1] + 8) + argerr) + U * s + 2.0 ** -126


def strided(n, d, off=3, fill=None):
    """an n x d view at column `off` of an n x (d + 7) buffer; NaN (or `fill`) outside the view"""
    buf = torch.full((n, d + 7), float("nan"), device=cuda)
    v = buf[:, off:off + d]
    if fill is not None:
        v.copy_(torch.from_numpy(fill))
    return buf, v


@gpu
@pytest.mark.parametrize("d", (1, 20, 32, 33, 64, 128, 256))
def test_standalone_softmax_forward_and_backward(d):
    from llmrec_b200 import ops
    rng = np.random.default_rng(d)
    n = 1000
    x = (rng.standard_normal((n, d)) * 4).astype(np.float32)
    xb, X = strided(n, d, fill=x)
    yb, Y = strided(n, d)
    ops.row_softmax(X, out=Y)
    s, bound = softmax_ref(x.astype(np.float64))
    check(Y, s, bound, "softmax", f"row_softmax d={d}")
    assert bool(torch.isnan(yb[:, :3]).all() and torch.isnan(yb[:, 3 + d:]).all())
    S = Y.double().cpu().numpy()
    gr = x_values(rng, n, d)
    gb, G = strided(n, d, off=1, fill=gr)
    t = (gr.astype(np.float64) * S).sum(1, keepdims=True)
    want = S * (gr - t)
    tb = C_BOUND * U * (d / 32 + 6) * np.abs(gr * S).sum(1, keepdims=True)
    bound = C_BOUND * (np.abs(S) * (tb + U * (np.abs(gr) + np.abs(t))) + U * np.abs(want))
    ob, O = strided(n, d, off=4)
    ops.row_softmax_bwd(Y, G, out=O)
    check(O, want, bound, "softmax", f"row_softmax_bwd d={d}")
    assert bool(torch.isnan(ob[:, :4]).all() and torch.isnan(ob[:, 4 + d:]).all())
    lst = np.concatenate([[5, 5, -1, 17, -1], rng.permutation(n)[:600]]).astype(np.int32)
    rb, R = strided(n, d, off=4)
    ops.row_softmax_bwd_rows(Y, G, R, torch.from_numpy(lst).to(cuda), torch.tensor([590], dtype=torch.int32, device=cuda))
    listed = np.zeros(n, bool)
    listed[lst[:590][lst[:590] >= 0]] = True
    check(R, want, bound, "softmax", f"row_softmax_bwd_rows d={d}", rows=listed)
    assert bool(torch.isnan(R[torch.from_numpy(~listed).to(cuda)]).all())
    assert torch.equal(R[torch.from_numpy(listed).to(cuda)], O[torch.from_numpy(listed).to(cuda)])


# ---------------------------------------------------------------------------------------------------------------------------------
# csrc/rows.cu: the propagation epilogue and batch gathers of the hoisted and sharded paths
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
def test_gather_rows_float4_and_scalar_branches():
    from llmrec_b200 import ops
    rng = np.random.default_rng(1)
    table = torch.from_numpy(x_values(rng, 500, 72)).to(cuda)
    idx = torch.tensor([3, -1, 0, 499, 3, -1, 250] * 20, dtype=torch.int32, device=cuda)
    for c0, d in ((4, 64), (1, 20), (5, 1)):                          # float4 rows; unaligned; one column (dist.py's scale gather)
        X = table[:, c0:c0 + d]
        buf = torch.full((idx.numel(), d + 12), float("nan"), device=cuda)
        out = buf[:, 8:8 + d]
        ops.gather_rows(X, idx, out)
        want = torch.where((idx >= 0)[:, None], X[idx.clamp(min=0).long()], torch.zeros_like(out))
        assert torch.equal(out, want), d
        assert bool(torch.isnan(buf[:, :8]).all() and torch.isnan(buf[:, 8 + d:]).all())
    assert bool((table[0] != 0).all())                                # a -1 that read row 0 would show


@gpu
def test_scatter_add_rows_duplicates_and_negative_ids():
    from llmrec_b200 import ops
    rng = np.random.default_rng(2)
    n, d, m = 300, 64, 2000
    y0 = x_values(rng, n, d)
    gr = x_values(rng, m, d)
    idx = rng.integers(-1, 40, m).astype(np.int32)                    # ~50 hits per row, and -1
    buf = torch.full((n, d + 8), float("nan"), device=cuda)
    Y = buf[:, 4:4 + d]
    Y.copy_(torch.from_numpy(y0))
    gb = torch.from_numpy(np.concatenate([gr, gr], 1)).to(cuda)
    ops.scatter_add_rows(gb[:, d:], torch.from_numpy(idx).to(cuda), Y)
    want = torch.from_numpy(y0).double().index_add(0, torch.from_numpy(idx[idx >= 0]).long(), torch.from_numpy(gr[idx >= 0]).double())
    cnt = np.bincount(idx[idx >= 0], minlength=n)[:, None]
    absum = np.abs(y0).astype(np.float64)
    np.add.at(absum, idx[idx >= 0], np.abs(gr[idx >= 0]))
    check(Y, want.numpy(), C_BOUND * U * (cnt + 1) * absum, "row helpers", "scatter_add_rows")
    assert bool(torch.isnan(buf[:, :4]).all() and torch.isnan(buf[:, 4 + d:]).all())


@gpu
@pytest.mark.parametrize("d", (1, 20, 64, 128, 256))
def test_row_scale_softmax_in_place_and_out_of_place(d):
    from llmrec_b200 import ops
    rng = np.random.default_rng(d)
    n = 700
    x = (rng.standard_normal((n, d)) * 3).astype(np.float32)
    sc = rng.uniform(0.5, 1.5, n).astype(np.float32)
    for scale in (None, torch.from_numpy(sc).to(cuda)):
        for smx in (False, True):
            _, X = strided(n, d, fill=x)
            yb, Y = strided(n, d, off=4)
            ops.row_scale_softmax(X, scale, Y, smx)
            a = x.astype(np.float64) * (sc[:, None] if scale is not None else 1.0)
            if smx:
                s, bound = softmax_ref(a, C_BOUND * U * (np.abs(a) + np.abs(a).max(1, keepdims=True)))
            else:
                s, bound = a, U * np.abs(a)
            check(Y, s, bound, "softmax", f"row_scale_softmax d={d} scale={scale is not None} softmax={smx}")
            assert bool(torch.isnan(yb[:, :4]).all() and torch.isnan(yb[:, 4 + d:]).all())
            ib, I = strided(n, d, off=4, fill=x)
            ops.row_scale_softmax(I, scale, I, smx)                       # in place, as dist.py calls it
            assert torch.equal(I, Y), (d, scale is not None, smx)


@gpu
def test_rowset_marks_and_compacts_against_a_python_set():
    from llmrec_b200 import ops
    rng = np.random.default_rng(3)
    n = 1000                                                           # not a multiple of 32
    degs = rng.integers(0, 6, 100)
    degs[42] = 15000                                                   # hub row
    rowptr = np.concatenate([[0], np.cumsum(degs)]).astype(np.int32)
    col = rng.integers(0, n - 40, int(rowptr[-1])).astype(np.int32)
    t = lambda a: torch.from_numpy(np.asarray(a, np.int32)).to(cuda)
    rs = ops.RowSet(n, cuda)

    def compacted():
        c = int(rs.count[0])
        lst = rs.list[:c].cpu().tolist()
        assert len(lst) == len(set(lst))
        words = rs.mask.cpu().numpy().view(np.uint32)
        bits = {32 * w + b for w in range(words.size) for b in range(32) if words[w] >> b & 1}
        assert bits == set(lst)
        return set(lst)

    for rows, ids in (([3, -1, 42, 7, 3], [5, -1, 999, 0, 31, 32]), ([-1, 8], [998, -1, 63, 64]), ([], [-1])):
        rs.clear()
        if rows:
            rs.add_neighbors(t(rowptr), t(col), t(rows))
        rs.add_ids(t(ids))
        rs.compact()
        want = {int(c) for r in rows if r >= 0 for c in col[rowptr[r]:rowptr[r + 1]]} | {i for i in ids if i >= 0}
        assert compacted() == want, (rows, ids)
