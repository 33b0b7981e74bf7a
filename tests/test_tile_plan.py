"""Host-side SpMM tile planner (llmrec_spmm_plan_tiles): every row is covered exactly once, nnz bounds hold."""
import numpy as np
import pytest

from llmrec_b200 import _native as N


def _plan(rowptr, tile_nnz, max_rows=15):
    lib = N.lib()
    rp = np.ascontiguousarray(rowptr, dtype=np.int32)
    n = len(rp) - 1
    counts = np.zeros(3, np.int32)
    assert lib.llmrec_spmm_plan_tiles(rp.ctypes.data, n, tile_nnz, max_rows, None, None, None, counts.ctypes.data) == 0
    tiles = np.zeros((max(counts[0], 1), 8), np.int32); srow = np.zeros(max(counts[1], 1), np.int32); sfirst = np.zeros(counts[1] + 1, np.int32)
    assert lib.llmrec_spmm_plan_tiles(rp.ctypes.data, n, tile_nnz, max_rows, tiles.ctypes.data, srow.ctypes.data, sfirst.ctypes.data, counts.ctypes.data) == 0
    return tiles[:counts[0]], srow[:counts[1]], sfirst, counts


def test_plan_covers_rows_once():
    rng = np.random.default_rng(0)
    for trial in range(20):
        n = int(rng.integers(1, 400))
        deg = rng.integers(0, 6, n)
        heavy = rng.integers(0, n, 3)
        deg[heavy] += rng.integers(50, 700, 3)
        if trial % 5 == 0:
            deg[:] = 0
        rp = np.concatenate([[0], np.cumsum(deg)])
        T = int(rng.choice([8, 32, 64, 248]))
        tiles, srow, sfirst, counts = _plan(rp, T)
        seen = np.zeros(n, int)
        covered = np.zeros(int(rp[-1]), int)
        for i, (r0, nr, e0, e1) in enumerate(tiles[:, :4]):
            deltas = tiles[i, 4:].view(np.uint8)
            if nr:
                assert (e0 + deltas[:nr].astype(np.int64) == rp[r0 + 1:r0 + nr + 1]).all()
            assert e1 - e0 <= T or (nr == 1 and False)
            if nr == 0:
                assert i < counts[2] and rp[r0 + 1] - rp[r0] > T and rp[r0] <= e0 < e1 <= rp[r0 + 1]
            else:
                assert i >= counts[2] and 1 <= nr <= 15 and e0 == rp[r0] and e1 == rp[r0 + nr]
                seen[r0:r0 + nr] += 1
            covered[e0:e1] += 1
        assert (covered == 1).all()
        long_rows = np.nonzero(deg > T)[0]
        assert (seen[deg <= T] == 1).all() and (seen[long_rows] == 0).all()
        assert srow.tolist() == long_rows.tolist()
        for j, r in enumerate(srow):
            pcs = tiles[sfirst[j]:sfirst[j + 1], :4]
            assert (pcs[:, 0] == r).all() and pcs[0, 2] == rp[r] and pcs[-1, 3] == rp[r + 1]


@pytest.mark.parametrize("max_rows", (1, 7, 15))
@pytest.mark.parametrize("tile", (8, 248))
def test_plan_at_the_boundaries(tile, max_rows):
    """The boundary graphs of the kernel exactness tests: a row of exactly tile_nnz entries stays whole, one of tile_nnz + 1 is cut
    into exactly 2 pieces (k * tile_nnz into k); groups hold at most max_rows rows, and their row-end bytes are the row ends."""
    from test_spmm_exactness_gpu import boundary_degrees
    deg = boundary_degrees(tile)
    rp = np.concatenate([[0], np.cumsum(deg)])
    tiles, srow, sfirst, counts = _plan(rp, tile, max_rows)
    whole = {}
    for i, (r0, nr, e0, e1) in enumerate(tiles[:, :4]):
        deltas = tiles[i, 4:].view(np.uint8)
        if nr:
            assert nr <= max_rows and e1 - e0 <= tile and e0 == rp[r0] and e1 == rp[r0 + nr]
            assert (e0 + deltas[:nr].astype(np.int64) == rp[r0 + 1:r0 + nr + 1]).all() and (deltas[nr:] == 0).all()
            for r in range(r0, r0 + nr):
                whole[r] = whole.get(r, 0) + 1
        else:
            j = int(np.searchsorted(srow, r0))
            assert srow[j] == r0 and tuple(deltas.view(np.int32)[:3]) == (j, sfirst[j], sfirst[j + 1] - sfirst[j])
    pieces = dict(zip(srow.tolist(), np.diff(sfirst).tolist()))
    assert set(whole) | set(pieces) == set(range(len(deg))) and not set(whole) & set(pieces)
    assert all(v == 1 for v in whole.values())
    for r, dg in enumerate(deg):
        if dg <= tile:
            assert r in whole, (r, dg)
        else:
            assert pieces[r] == -(-dg // tile), (r, dg)
            if dg == tile + 1:
                assert pieces[r] == 2
    assert {tile, tile + 1, 2 * tile, 3 * tile} <= set(deg.tolist())
