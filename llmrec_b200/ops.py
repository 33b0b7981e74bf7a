"""Thin tensor-level wrappers over the C ABI (include/llmrec_b200.h).

PyTorch supplies device memory and the current CUDA stream only; every op below is one or more
launches of the hand-written sm_90a kernels.  2-D operands must be row-major views
(stride(1) == 1); column slices of wider buffers are fine (the leading dimension is passed).
"""
from __future__ import annotations

import copy
import ctypes as C
import os

import numpy as np
import torch

from . import _native as N
from . import feat_int8


STATS = {"launches": 0}     # kernels of libllmrec_b200 launched through this module (bench.py reports it)


def _count(n=1):
    STATS["launches"] += n


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _mat(t: torch.Tensor, name="operand"):
    if t.dim() != 2 or t.dtype != torch.float32 or not t.is_cuda or (t.shape[1] > 1 and t.stride(1) != 1):
        raise ValueError(f"{name}: need a CUDA fp32 row-major 2-D tensor, got {tuple(t.shape)} {t.dtype} {t.device} strides {t.stride()}")
    return t


def _ld(t):
    return int(t.stride(0)) if t.shape[0] > 1 else int(max(t.stride(0), t.shape[1]))


def _i32(t, name="index"):
    if t.dtype != torch.int32 or not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{name}: need a contiguous CUDA int32 tensor")
    return t


DEFAULT_TILE_NNZ = int(os.environ.get("LLMREC_SPMM_TILE", "0"))      # 0 = size tiles from the graph


def auto_tile_nnz(nnz):
    """16 non-zeros per tile on small graphs (parallelism and short dependent-load chains; 8 would cut
    ordinary rows into pieces), growing to 248 on large ones (amortised
    index reads, few long-row pieces)."""
    t = nnz // 65536
    return int(min(248, max(16, (t // 8) * 8)))


class TilePlan:
    """nnz-bounded work decomposition of a CSR pattern (llmrec_spmm_plan_tiles); shared by the operators
    that use the same pattern (forward of one direction, backward of the other)."""

    def __init__(self, rowptr_dev, n_rows, tile_nnz=0, max_rows=15):
        rp = np.ascontiguousarray(rowptr_dev.cpu().numpy().astype(np.int32))
        tile_nnz = int(tile_nnz) or DEFAULT_TILE_NNZ or auto_tile_nnz(int(rp[-1]))
        lib = N.lib()
        counts = np.zeros(3, dtype=np.int32)
        N.check(lib.llmrec_spmm_plan_tiles(rp.ctypes.data, n_rows, tile_nnz, max_rows, None, None, None, counts.ctypes.data), "spmm_plan")
        tiles = np.zeros((max(int(counts[0]), 1), 8), dtype=np.int32)
        srow = np.zeros(max(int(counts[1]), 1), dtype=np.int32)
        sfirst = np.zeros(int(counts[1]) + 1, dtype=np.int32)
        N.check(lib.llmrec_spmm_plan_tiles(rp.ctypes.data, n_rows, tile_nnz, max_rows, tiles.ctypes.data, srow.ctypes.data,
                                           sfirst.ctypes.data, counts.ctypes.data), "spmm_plan")
        dev = rowptr_dev.device
        self.tiles, self.split_row, self.split_first = (torch.from_numpy(a).to(dev) for a in (tiles, srow, sfirst))
        self.n_tiles, self.n_split, self.n_split_tiles = (int(c) for c in counts)
        self.tile_nnz, self.scratch = tile_nnz, None
        # per (long row, column window) tickets: the last piece to finish reduces the row inside the same launch (self-resetting)
        self.tickets = torch.zeros(max(self.n_split, 1) * 64, dtype=torch.int32, device=dev) if self.n_split else None


class CsrOperator:
    """One sparse operator  Y = diag(rs) . P(vals) . diag(cs) . X  over a CSR pattern P."""

    def __init__(self, rowptr, col, n_rows, n_cols, vals=None, rs=None, cs=None, tile_nnz=0, plan=None):
        self.rowptr, self.col = _i32(rowptr, "rowptr"), _i32(col, "col")
        self.vals, self.rs, self.cs = vals, rs, cs
        self.n_rows, self.n_cols = int(n_rows), int(n_cols)
        self.nnz = int(col.numel())
        self.plan = plan if plan is not None else TilePlan(self.rowptr, self.n_rows, tile_nnz)

    def branch(self):
        """The same operator with its own long-row scratch and tickets, for launches that may overlap launches of `self` (or of an
        operator sharing its plan) on another stream."""
        o, k = copy.copy(self), copy.copy(self.plan)
        k.scratch = None
        k.tickets = torch.zeros_like(self.plan.tickets) if self.plan.tickets is not None else None
        o.plan = k
        return o

    def _tiling_struct(self, width):
        k = self.plan
        need = k.n_split_tiles * width
        if need and (k.scratch is None or k.scratch.numel() < need):
            if k.scratch is not None:
                _retired.append(k.scratch)
            k.scratch = torch.empty(need, dtype=torch.float32, device=self.rowptr.device)
        return N.SpmmTiling(_p(k.tiles), _p(k.split_row), _p(k.split_first), _p(k.scratch), k.n_tiles, k.n_split, k.n_split_tiles, 0, _p(k.tickets), None)

    def apply_rows(self, seg, rows, count, max_rows=None, src_mask=None, cta_per_row=False):
        """Row-list form (llmrec_spmm_rows_f32): only rows[0 .. count[0]) are computed and written.  seg = (X, Y, Z|None, softmax);
        rows: int32 CUDA list, count: int32[1] CUDA (device-side length), src_mask: optional uint32/int32 bitmask over source rows."""
        X, Y, Z, sm = seg
        _mat(X, "spmm X"); _mat(Y, "spmm Y")
        d = int(X.shape[1])
        if X.shape[0] != self.n_cols or Y.shape[0] != self.n_rows or Y.shape[1] != d:
            raise ValueError("spmm_rows: shape mismatch")
        sg = N.SpmmSeg(_p(X), _p(Y), _p(Z) if Z is not None else None, _ld(X), _ld(Y), _ld(Z) if Z is not None else 0, N.SPMM_SOFTMAX if sm else 0, 0)
        mx = int(rows.numel()) if max_rows is None else int(max_rows)
        N.check(N.lib().llmrec_spmm_rows_f32(_p(self.rowptr), _p(self.col), _p(self.vals), _p(self.rs), _p(self.cs), d, C.byref(sg),
                                              _p(_i32(rows)), _p(count), mx, _p(src_mask), 1 if cta_per_row else 0, _stream()), "spmm_rows")
        _count()

    def apply(self, segs, src_mask=None):
        """segs: list of (X, Y, Z_or_None, softmax: bool); all share d = X.shape[1].  src_mask: optional bitmask over the SOURCE rows
        (rows of X): a clear bit promises an all-zero row, whose fetch is skipped."""
        if not segs:
            return
        d = int(segs[0][0].shape[1])
        arr = (N.SpmmSeg * len(segs))()
        for i, (X, Y, Z, sm) in enumerate(segs):
            _mat(X, "spmm X"); _mat(Y, "spmm Y")
            if X.shape[0] != self.n_cols or Y.shape[0] != self.n_rows or X.shape[1] != d or Y.shape[1] != d:
                raise ValueError(f"spmm: shape mismatch X{tuple(X.shape)} Y{tuple(Y.shape)} for operator {self.n_rows}x{self.n_cols}")
            arr[i] = N.SpmmSeg(_p(X), _p(Y), _p(Z) if Z is not None else None, _ld(X), _ld(Y), _ld(Z) if Z is not None else 0,
                               N.SPMM_SOFTMAX if sm else 0, 0)
        til = self._tiling_struct(d * min(len(segs), N.MAX_SEG))
        til.src_mask = src_mask.data_ptr() if src_mask is not None else None
        N.check(N.lib().llmrec_spmm_csr_f32(_p(self.rowptr), _p(self.col), _p(self.vals), _p(self.rs), _p(self.cs),
                                             self.n_rows, self.n_cols, d, arr, len(segs), C.byref(til), _stream()), "spmm")
        _count(-(-len(segs) // N.MAX_SEG))


def row_softmax(X, out=None):
    out = torch.empty_like(X) if out is None else out
    N.check(N.lib().llmrec_row_softmax_f32(_p(_mat(X)), _ld(X), _p(_mat(out)), _ld(out), X.shape[0], X.shape[1], _stream()), "row_softmax")
    _count()
    return out


def row_softmax_bwd(S, dS, out=None):
    out = torch.empty((S.shape[0], S.shape[1]), dtype=torch.float32, device=S.device) if out is None else out
    N.check(N.lib().llmrec_row_softmax_bwd_f32(_p(_mat(S)), _ld(S), _p(_mat(dS)), _ld(dS), _p(_mat(out)), _ld(out),
                                                S.shape[0], S.shape[1], _stream()), "row_softmax_bwd")
    _count()
    return out


def row_softmax_bwd_rows(S, dS, out, rows, count, max_rows=None):
    mx = int(rows.numel()) if max_rows is None else int(max_rows)
    N.check(N.lib().llmrec_row_softmax_bwd_rows_f32(_p(_mat(S)), _ld(S), _p(_mat(dS)), _ld(dS), _p(_mat(out)), _ld(out), _p(_i32(rows)), _p(count), mx,
                                                     S.shape[1], _stream()), "row_softmax_bwd_rows")
    _count()
    return out


class RowSet:
    """A set of row ids living on the device: uint32 bitmask + compacted id list + its length, rebuilt every step without a host sync."""

    def __init__(self, n, device):
        self.n = int(n)
        self.mask = torch.zeros((self.n + 31) // 32 + 1, dtype=torch.int32, device=device)
        self.list = torch.zeros(max(self.n, 1), dtype=torch.int32, device=device)
        self.count = torch.zeros(1, dtype=torch.int32, device=device)

    def clear(self):
        N.check(N.lib().llmrec_fill_f32(_p(self.mask), self.mask.numel(), 0.0, _stream()), "fill")
        N.check(N.lib().llmrec_fill_f32(_p(self.count), 1, 0.0, _stream()), "fill")
        _count(2)

    def add_neighbors(self, rowptr, col, rows):
        """every column id of the CSR rows named in `rows` (int32 CUDA list; entries < 0 skipped)"""
        N.check(N.lib().llmrec_mark_neighbors(_p(_i32(rowptr)), _p(_i32(col)), _p(_i32(rows)), rows.numel(), _p(self.mask), _stream()), "mark_neighbors")
        _count()

    def add_ids(self, ids, n=None):
        """n: optional int32 CUDA tensor whose first entry is the live length (ids[0 .. min(n[0], len(ids))) are marked; no host sync)"""
        if n is None:
            N.check(N.lib().llmrec_mark_ids(_p(_i32(ids)), ids.numel(), _p(self.mask), _stream()), "mark_ids")
        else:
            N.check(N.lib().llmrec_mark_ids_rows(_p(_i32(ids)), _p(_i32(n, "live length")), ids.numel(), _p(self.mask), _stream()), "mark_ids_rows")
        _count()

    def compact(self):
        N.check(N.lib().llmrec_compact_mask(_p(self.mask), self.n, _p(self.list), _p(self.count), _stream()), "compact_mask")
        _count()


def zero_rows(Y, idx):
    N.check(N.lib().llmrec_zero_rows_f32(_p(_mat(Y)), _ld(Y), _p(_i32(idx)), idx.numel(), Y.shape[1], _stream()), "zero_rows")
    _count()


def assign_rows(G, idx, Y):
    N.check(N.lib().llmrec_assign_rows_f32(_p(_mat(G)), _ld(G), _p(_i32(idx)), idx.numel(), G.shape[1], _p(_mat(Y)), _ld(Y), _stream()), "assign_rows")
    _count()


PROJ_MODE = {"3xtf32": 0, "tf32": 1, "fp32": 2}


_scratch = {}


_retired = []     # outgrown scratch buffers stay allocated: a captured CUDA graph may still hold their addresses


def _get_scratch(key, n, device, zero=False):
    t = _scratch.get(key)
    if t is None or t.numel() < n:
        if t is not None:
            _retired.append(t)
        t = _scratch[key] = (torch.zeros if zero else torch.empty)(max(int(n), 1), dtype=torch.float32, device=device)
    return t


FEAT_DTYPES = (torch.float32, torch.bfloat16, torch.int8)     # element types of the side-feature table X the projections accept


def _feat(X, name="X"):
    """X of a projection: a CUDA fp32 or bf16 row-major 2-D tensor (column slices fine), or an int8 table (feat_int8)."""
    if X.dim() != 2 or X.dtype not in FEAT_DTYPES or not X.is_cuda or (X.shape[1] > 1 and X.stride(1) != 1):
        raise ValueError(f"{name}: need a CUDA fp32, bf16 or int8 row-major 2-D tensor, got {tuple(X.shape)} {X.dtype} {X.device} strides {X.stride()}")
    return X


def _feat_k(X, k, what):
    """Logical width of X for a problem whose weights are k wide: X's width, or for an int8 table the k its row pitch must hold."""
    if X.dtype == torch.int8:
        if X.shape[1] != feat_int8.pitch(k):
            raise ValueError(f"{what}: an int8 table of width k = {k} has rows of {feat_int8.pitch(k)} bytes, got {X.shape[1]}")
        return k
    return int(X.shape[1])


_PROBLEMS = {torch.float32: (N.ProjFwdProblem, N.ProjWgradProblem, "f32"), torch.bfloat16: (N.ProjFwdProblemBf16, N.ProjWgradProblemBf16, "bf16"),
             torch.int8: (N.ProjFwdProblemI8, N.ProjWgradProblemI8, "i8")}


def _group_dtype(Xs, what):
    """The one X dtype of a grouped call: a bf16 / int8 group runs the _bf16 / _i8 entry points, and one call never mixes them."""
    dt = {X.dtype for X in Xs}
    if len(dt) != 1:
        raise ValueError(f"{what}: every problem of one call must share the X dtype, got {sorted(str(t) for t in dt)}")
    return dt.pop()


def _f32(t, name):
    if t is not None and t.dtype != torch.float32:
        raise ValueError(f"{name}: must be fp32 (only the feature table X may be bf16 or int8), got {t.dtype}")
    return t


def _row_map(rows, n, what):
    """Optional row map of a projection problem: None, or a contiguous CUDA int32 list of the problem's n X rows."""
    if rows is not None and (_i32(rows, what + " rows").dim() != 1 or rows.numel() != n):
        raise ValueError(f"{what}: a row map needs one entry per X row ({n}), got {tuple(rows.shape)}")
    return rows


def _problem_array(prob_type, n, mapped):
    """ctypes array of n problems; with row maps, followed in the same block by their n llmrec_proj_row_map records (the layout the
    grouped entry points read when a problem flags LLMREC_PROJ_ROW_MAP).  -> (problems, records | None, block)"""
    if not mapped:
        arr = (prob_type * n)()
        return arr, None, arr

    class Block(C.Structure):
        _fields_ = [("probs", prob_type * n), ("maps", N.ProjRowMap * n)]
    blk = Block()
    return blk.probs, blk.maps, blk


def proj_fwd_group(problems, d, mode=0):
    """problems: list of (X[n x k], W[d x k], bias[d]|None, out[m x d] [, rows]).  One grouped launch (wgmma) --
    the 8 nn.Linear calls of Models.py:145-150.  Problems sharing W share the split buffer.  X is fp32, bf16 or an int8 table
    (feat_int8; k is then W's width) -- all problems alike; W, bias and out are fp32.  rows (optional, int32 CUDA [n]): X row r is
    written to out[rows[r]], the other rows of out are left untouched (without it m == n and row r goes to out[r]); a written row
    gets the bits of the full-table call."""
    dt = _group_dtype([_feat(pr[0]) for pr in problems], "proj_fwd")
    bf16 = dt != torch.float32             # bf16 and int8 run the bf16 kernels: W as bf16 terms
    prob_t, _, suffix = _PROBLEMS[dt]
    arr, recs, _blk = _problem_array(prob_t, len(problems), any(len(pr) > 4 and pr[4] is not None for pr in problems))
    for i, (X, W, b, out, *rows) in enumerate(problems):
        _mat(out); _f32(W, "proj_fwd W"); _f32(b, "proj_fwd bias")
        n, k = int(X.shape[0]), _feat_k(X, int(W.shape[1]) if W.dim() == 2 else -1, "proj_fwd")
        rows = _row_map(rows[0] if rows else None, n, "proj_fwd")
        if not W.is_contiguous() or tuple(W.shape) != (d, k) or out.shape[1] != d or (rows is None and out.shape[0] != n):
            raise ValueError("proj_fwd: bad shapes")
        # the bf16 kernels read W as bf16 terms in modes 0 and 1: 3dk (or dk) bf16 in the 2dk floats of the fp32 hi/lo split
        ws = _get_scratch(("wsplit", W.data_ptr()), 2 * d * k, X.device) if mode == 0 or (bf16 and mode == 1) else None
        arr[i] = prob_t(_p(X), _p(W), _p(b), _p(out), _p(ws), _ld(X), _ld(out), n, k, 0 if rows is None else N.PROJ_ROW_MAP)
        if rows is not None:
            recs[i] = N.ProjRowMap(_p(rows), int(out.shape[0]))
    lib = N.lib()
    if bf16:
        N.check(getattr(lib, "llmrec_proj_fwd_group_" + suffix)(arr, len(problems), d, mode, _stream()), "proj_fwd_group_" + suffix)
    else:
        N.check(lib.llmrec_proj_fwd_group_f32(arr, len(problems), d, mode, _stream()), "proj_fwd_group")
    _count((2 if mode == 0 or (bf16 and mode == 1) else 1) * -(-len(problems) // 8))


def proj_fwd(X, W, b, out, mode=0):
    """out[n x d] = X[n x k] W[d x k]^T + b  (nn.Linear; Models.py:145-150)."""
    proj_fwd_group([(X, W, b, out)], W.shape[0], mode)
    return out


def proj_wgrad_group(problems, d, mode=0):
    """problems: list of (X[n x k], dY[m x d], dW[d x k], db[d]|None, accumulate [, rows]).  dW (+)= dY^T X ; db (+)= colsum(dY).
    X is fp32, bf16 or an int8 table (feat_int8; k is then dW's width) -- all problems alike; dY, dW and db are fp32.  rows (optional,
    int32 CUDA [n]): X row r pairs with dY[rows[r]] (without it m == n); db still sums all m rows of dY, so it gets the bits of the
    full-table call, and dW differs from it by rounding."""
    dt = _group_dtype([_feat(pr[0]) for pr in problems], "proj_wgrad")
    _, prob_t, suffix = _PROBLEMS[dt]
    arr, recs, _blk = _problem_array(prob_t, len(problems), any(len(pr) > 5 and pr[5] is not None for pr in problems))
    for i, (X, dY, dW, db, acc, *rows) in enumerate(problems):
        _mat(dY); _f32(dW, "proj_wgrad dW"); _f32(db, "proj_wgrad db")
        n, k = int(X.shape[0]), _feat_k(X, int(dW.shape[1]) if dW.dim() == 2 else -1, "proj_wgrad")
        rows = _row_map(rows[0] if rows else None, n, "proj_wgrad")
        if not dW.is_contiguous() or tuple(dW.shape) != (d, k) or dY.shape[1] != d or (rows is None and dY.shape[0] != n):
            raise ValueError("proj_wgrad: bad shapes")
        flags = (N.WGRAD_ACCUMULATE if acc else 0) | (0 if rows is None else N.PROJ_ROW_MAP)
        arr[i] = prob_t(_p(X), _p(dY), _p(dW), _p(db), _ld(X), _ld(dY), n, k, flags)
        if rows is not None:
            recs[i] = N.ProjRowMap(_p(rows), int(dY.shape[0]))
    lib = N.lib()
    name = "llmrec_proj_wgrad_group" + ("" if dt == torch.float32 else "_" + suffix)
    need = int(getattr(lib, name + "_scratch")(arr, len(problems), d, mode))
    scratch = _get_scratch(("wgrad", problems[0][0].device.index), need, problems[0][0].device, zero=True) if need else None     # holds a ticket word
    if dt != torch.float32:
        N.check(getattr(lib, name)(arr, len(problems), d, mode, _p(scratch), need, _stream()), "proj_wgrad_group_" + suffix)
    else:
        N.check(lib.llmrec_proj_wgrad_group_f32(arr, len(problems), d, mode, _p(scratch), need, _stream()), "proj_wgrad_group")
    _count(4 if need else len(problems))


def proj_wgrad(X, dY, dW, db, accumulate=False, mode=0):
    """dW[d x k] (+)= dY^T X ; db[d] (+)= colsum(dY)."""
    proj_wgrad_group([(X, dY, dW, db, accumulate)], dY.shape[1], mode)


def _ptr_table(tensors):
    arr = (C.c_void_p * max(1, len(tensors)))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr() if t is not None else None
    return arr


def _ld_table(tensors):
    arr = (C.c_int64 * max(1, len(tensors)))()
    for i, t in enumerate(tensors):
        arr[i] = _ld(t) if t is not None else 0
    return arr


def _row_list(rows, count, max_rows, what):
    """(rows, count, max_rows) of a row-list launch with a device-side length: rows[0 .. min(count[0], max_rows)) are processed."""
    if rows is None:
        raise ValueError(f"{what}: a device-side count needs a row list")
    mx = int(rows.numel()) if max_rows is None else min(int(max_rows), int(rows.numel()))
    return _i32(rows), _i32(count, "count"), mx


def fuse_fwd(layers, sides, coefs, out, rows=None, compact=False, count=None, max_rows=None):
    """out = mean(layers) + sum_t coefs[t] * normalize(sides[t])   (Models.py:185-197).
    rows: only these rows; compact=True: layers are read at rows[b], sides and out are [len(rows) x d] blocks indexed by b.
    count: int32[1] CUDA tensor, the live length of `rows` (only rows[0 .. min(count[0], max_rows)) are fused; no host sync)."""
    for t in list(layers) + list(sides) + [out]:
        _mat(t)
    cf = (C.c_float * max(1, len(coefs)))(*[float(c) for c in coefs])
    if count is not None:
        if compact:
            raise ValueError("fuse_fwd: the device-count form is not compact")
        rows, count, mx = _row_list(rows, count, max_rows, "fuse_fwd")
        N.check(N.lib().llmrec_fuse_fwd_rows_f32(_ptr_table(layers), _ld_table(layers), len(layers), _ptr_table(sides), _ld_table(sides), cf,
                                                  len(sides), _p(out), _ld(out), _p(rows), _p(count), mx, out.shape[1], _stream()), "fuse_fwd_rows")
        _count()
        return out
    n = out.shape[0] if rows is None else rows.numel()
    if compact:
        if rows is None:
            raise ValueError("fuse_fwd: compact form needs a row list")
        n = -n
    N.check(N.lib().llmrec_fuse_fwd_f32(_ptr_table(layers), _ld_table(layers), len(layers), _ptr_table(sides), _ld_table(sides), cf,
                                         len(sides), _p(out), _ld(out), _p(rows), n, out.shape[1], _stream()), "fuse_fwd")
    _count()
    return out


def fuse_bwd(g, n_layers, d_layer, sides, coefs, d_sides, accumulate, rows=None, count=None, max_rows=None):
    """count: as for fuse_fwd; a row listed twice would be processed twice (accumulate=True adds twice): pass a set (RowSet.list).
    Negative entries of `rows` are skipped, as in the forward."""
    _mat(g)
    cf = (C.c_float * max(1, len(coefs)))(*[float(c) for c in coefs])
    dl = (_p(d_layer), _ld(d_layer) if d_layer is not None else 0)
    if count is not None:
        rows, count, mx = _row_list(rows, count, max_rows, "fuse_bwd")
        N.check(N.lib().llmrec_fuse_bwd_rows_f32(_p(g), _ld(g), n_layers, *dl, _ptr_table(sides), _ld_table(sides), cf, _ptr_table(d_sides),
                                                  _ld_table(d_sides), len(sides), 1 if accumulate else 0, _p(rows), _p(count), mx, g.shape[1],
                                                  _stream()), "fuse_bwd_rows")
        _count()
        return
    n = g.shape[0] if rows is None else rows.numel()
    N.check(N.lib().llmrec_fuse_bwd_f32(_p(g), _ld(g), n_layers, *dl,
                                         _ptr_table(sides), _ld_table(sides), cf, _ptr_table(d_sides), _ld_table(d_sides), len(sides),
                                         1 if accumulate else 0, _p(rows), n, g.shape[1], _stream()), "fuse_bwd")
    _count()


def bpr_work(n_heads, B, device):
    return torch.zeros(int(N.lib().llmrec_bpr_work_elems(n_heads, B)), dtype=torch.float32, device=device)


def bpr_slot_plan(users, pos, neg, meta=None, plan=None):
    """Slot plan of the ordered row gradients (llmrec_bpr_slot_plan): the batch's user slots and pos | neg item slots sorted by (row, slot).
    It reads the index arrays (and meta[0]) only.  plan: int32 CUDA buffer of llmrec_bpr_slot_plan_elems(B) entries to fill (made when None).
    Capacities past 65 536 triplets raise."""
    B = int(users.numel())
    need = int(N.lib().llmrec_bpr_slot_plan_elems(B))
    if plan is None:
        plan = torch.zeros(need, dtype=torch.int32, device=users.device)
    if _i32(plan, "plan").numel() < need:
        raise ValueError("bpr_slot_plan: plan buffer too small for this capacity")
    N.check(N.lib().llmrec_bpr_slot_plan(_p(_i32(users)), _p(_i32(pos)), _p(_i32(neg)), B, _p(meta), _p(plan), _stream()), "bpr_slot_plan")
    _count(2)
    return plan


def bpr_heads(heads, users, pos, neg, n_keep, regs0_over_bs, out, loss, work, meta=None, ordered=None):
    """heads: list of (XU, XI, GU|None, GI|None, w_mf, w_emb).  See include/llmrec_b200.h.
    meta: optional int32 CUDA tensor {live B', n_keep}; users/pos/neg/work are then sized for the capacity B.
    ordered: a `bpr_slot_plan` of the same index arrays: the row gradients are then accumulated in the fixed order of
    llmrec_bpr_heads_ordered_f32 (bit-reproducible) instead of with float atomics; loss and `out` are the same either way."""
    arr = (N.BprHead * len(heads))()
    d = int(heads[0][0].shape[1])
    for i, (XU, XI, GU, GI, wmf, wemb) in enumerate(heads):
        _mat(XU); _mat(XI)
        arr[i] = N.BprHead(_p(XU), _p(XI), _p(GU), _p(GI), _ld(XU), _ld(XI), _ld(GU) if GU is not None else 0,
                           _ld(GI) if GI is not None else 0, float(wmf), float(wemb))
    B = int(users.numel())
    if work.numel() < N.lib().llmrec_bpr_work_elems(len(heads), B):
        raise ValueError("bpr_heads: work buffer too small for this capacity")
    args = (arr, len(heads), _p(_i32(users)), _p(_i32(pos)), _p(_i32(neg)), B, int(n_keep), _p(meta), float(regs0_over_bs), d, _p(out), _p(loss), _p(work))
    if ordered is not None:
        if _i32(ordered, "plan").numel() < N.lib().llmrec_bpr_slot_plan_elems(B):
            raise ValueError("bpr_heads: the slot plan was built for a smaller capacity")
        N.check(N.lib().llmrec_bpr_heads_ordered_f32(*args, _p(ordered), _stream()), "bpr_heads_ordered")
    else:
        N.check(N.lib().llmrec_bpr_heads_f32(*args, _stream()), "bpr_heads")
    _count(2)


_ginit = {}


def grad_init(regions, loss):
    """regions: list of (G, X|None, c): G = c*X (or 0) written once; loss = sum 0.5*c*|X|^2 (overwritten).  One launch."""
    arr = (N.GradRegion * len(regions))()
    for i, (G, X, c) in enumerate(regions):
        _mat(G)
        if X is not None and tuple(_mat(X).shape) != tuple(G.shape):
            raise ValueError("grad_init: X and G shapes differ")
        arr[i] = N.GradRegion(_p(G), _p(X), _ld(G), _ld(X) if X is not None else 0, G.shape[0], G.shape[1], float(c))
    key = loss.device.index
    sc = _ginit.get(key)
    if sc is None:
        sc = _ginit[key] = torch.zeros(int(N.lib().llmrec_grad_init_scratch()), dtype=torch.float32, device=loss.device)
    N.check(N.lib().llmrec_grad_init_f32(arr, len(regions), _p(loss), _p(sc), _stream()), "grad_init")
    _count()


_partial = {}


def sqnorm_grad(X, G, c, accumulate, loss):
    """loss += c*0.5*sum(X^2); G = (G if accumulate else 0) + c*X   (feat_reg, main.py:151-156)."""
    _mat(X)
    part = _partial.get(X.device.index)
    if part is None:
        part = _partial[X.device.index] = torch.empty(1024, dtype=torch.float32, device=X.device)
    N.check(N.lib().llmrec_sqnorm_grad_f32(_p(X), _ld(X), _p(G), _ld(G) if G is not None else 0, X.shape[0], X.shape[1], float(c),
                                            1 if accumulate else 0, _p(loss), _p(part), _stream()), "sqnorm_grad")
    _count(2)


class AdamW:
    """Dense fused AdamW over a fixed list of parameter tensors (torch.optim.AdamW defaults)."""

    def __init__(self, params, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01):
        self.params = [p for p in params]
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        dev = self.params[0].device
        self.m = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params]
        self.v = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in self.params]
        self.state = torch.zeros(4, dtype=torch.float64, device=dev)
        self._n = (C.c_int64 * len(self.params))(*[p.numel() for p in self.params])

    def advance(self):
        """bump the device-side step counter / bias corrections once per optimizer step (before any step_tensor)"""
        N.check(N.lib().llmrec_adamw_advance(_p(self.state), self.lr, self.betas[0], self.betas[1], _stream()), "adamw_advance")
        _count()

    def step_tensor(self, i, grad, row_mask=None):
        """update parameter i alone (after advance()): lets independent tables be updated at different points of a step, e.g. the
        user table while an item-side exchange is in flight"""
        lib, p = N.lib(), self.params[i]
        if row_mask is not None:
            N.check(lib.llmrec_adamw_step_rows_f32(_p(p), _p(grad), _p(self.m[i]), _p(self.v[i]), p.shape[0], p.shape[1], _p(row_mask), _p(self.state),
                                                    self.lr, self.betas[0], self.betas[1], self.eps, self.wd, _stream()), "adamw_step_rows")
        else:
            n = (C.c_int64 * 1)(p.numel())
            N.check(lib.llmrec_adamw_step_f32(_ptr_table([p.data]), _ptr_table([grad]), _ptr_table([self.m[i]]), _ptr_table([self.v[i]]), n, 1, _p(self.state),
                                               self.lr, self.betas[0], self.betas[1], self.eps, self.wd, _stream()), "adamw_step")
        _count()

    def step(self, grads, row_masks=None):
        """row_masks: optional list (one entry per parameter) of RowSet-style bitmasks or None: a masked [n x w] parameter reads its
        gradient only on the flagged rows and takes the g = 0 update elsewhere (row-sparse gradients of a dense AdamW)."""
        lib = N.lib()
        N.check(lib.llmrec_adamw_advance(_p(self.state), self.lr, self.betas[0], self.betas[1], _stream()), "adamw_advance")
        dense = [i for i in range(len(self.params)) if not (row_masks and row_masks[i] is not None)]
        for i in range(len(self.params)):
            if i in dense:
                continue
            p = self.params[i]
            N.check(lib.llmrec_adamw_step_rows_f32(_p(p), _p(grads[i]), _p(self.m[i]), _p(self.v[i]), p.shape[0], p.shape[1], _p(row_masks[i]), _p(self.state),
                                                    self.lr, self.betas[0], self.betas[1], self.eps, self.wd, _stream()), "adamw_step_rows")
            _count()
        if dense:
            ps, gs, ms, vs = ([x[i] for i in dense] for x in ([p.data for p in self.params], grads, self.m, self.v))
            n = (C.c_int64 * len(dense))(*[self.params[i].numel() for i in dense])
            N.check(lib.llmrec_adamw_step_f32(_ptr_table(ps), _ptr_table(gs), _ptr_table(ms), _ptr_table(vs), n, len(dense), _p(self.state),
                                               self.lr, self.betas[0], self.betas[1], self.eps, self.wd, _stream()), "adamw_step")
        _count(1 + -(-len(dense) // 16))


SCORE_MODE = {"3xtf32": 0, "fp32": 2}
_score_scratch = {}


def _score_topk_scratch(need, device):
    """The per-device scratch of score_topk / score_topk_among, grown to `need` fp32 elements (None while nothing was needed)."""
    key = device.index
    scratch = _score_scratch.get(key)
    if need and (scratch is None or scratch.numel() < need):
        if scratch is not None:
            _retired.append(scratch)
        scratch = _score_scratch[key] = torch.empty(need, dtype=torch.float32, device=device)
    return scratch


def score_topk(U, I, users, mask_rowptr, mask_col, K, mode=0, want_vals=False):
    """Top-K item ids per user among items not in the user's mask row; ties -> lowest id."""
    _mat(U); _mat(I)
    nb, ni, d = int(users.numel()), int(I.shape[0]), int(I.shape[1])
    idx = torch.empty((nb, K), dtype=torch.int32, device=U.device)
    val = torch.empty((nb, K), dtype=torch.float32, device=U.device) if want_vals else None
    scratch = _score_topk_scratch(int(N.lib().llmrec_score_topk_scratch(nb, ni, d, K, mode)), U.device)
    N.check(N.lib().llmrec_score_topk_f32(_p(U), _ld(U), _p(I), _ld(I), _p(_i32(users)), nb, ni, d, _p(mask_rowptr), _p(mask_col), K,
                                           _p(idx), _p(val), mode, _p(scratch), scratch.numel() if scratch is not None else 0,
                                           _stream()), "score_topk")
    _count(3)
    return (idx, val) if want_vals else idx


def score_topk_among(U, I, users, among, mask_rowptr, mask_col, K, mode=0, want_vals=False):
    """score_topk over the catalog rows `among` of I (int32 device ids, strictly ascending): mask rows and returned ids are global
    item ids, a masked id outside `among` is ignored, ties -> lowest id, K <= among.numel()."""
    _mat(U); _mat(I)
    nb, na, d = int(users.numel()), int(among.numel()), int(I.shape[1])
    idx = torch.empty((nb, K), dtype=torch.int32, device=U.device)
    val = torch.empty((nb, K), dtype=torch.float32, device=U.device) if want_vals else None
    scratch = _score_topk_scratch(int(N.lib().llmrec_score_topk_among_scratch(nb, na, d, K, mode)), U.device)
    N.check(N.lib().llmrec_score_topk_among_f32(_p(U), _ld(U), _p(I), _ld(I), _p(_i32(users)), nb, _p(_i32(among, "among")), na, d,
                                                 _p(mask_rowptr), _p(mask_col), K, _p(idx), _p(val), mode, _p(scratch),
                                                 scratch.numel() if scratch is not None else 0, _stream()), "score_topk_among")
    _count(3)
    return (idx, val) if want_vals else idx


GROUP_AGG = {"mean": 0, "min": 1, "max": 2}     # LLMREC_AGG_MEAN / _MIN / _MAX
GROUP_MAX_MEMBERS = 64     # one wgmma M tile: a group never straddles a tile of llmrec_score_topk_group_f32


def score_topk_group(U, I, member_rowptr, members, among, mask_rowptr, mask_col, K, agg="mean", mode=0, want_vals=False):
    """Top-K per group of users (llmrec_score_topk_group_f32): group g's members are rows members[member_rowptr[g] ..
    member_rowptr[g+1]) of U (1..64, ascending, distinct; member_rowptr is read on the host), its score of an item the mean (fp32 sum
    in member order, then one division), min or max of the members' exact chains (a NaN member makes it NaN).  among: None (the
    catalog is I) or int32 device ids, strictly ascending; mask rows are indexed by group and hold global ids.  Ties -> lowest id;
    NaN / -inf group scores never returned; padded with -1 / -inf."""
    _mat(U); _mat(I)
    if agg not in GROUP_AGG:
        raise ValueError(f"agg = {agg!r}: one of {tuple(GROUP_AGG)}")
    rp = member_rowptr.detach().to("cpu", torch.int32).contiguous()
    ng, d = int(rp.numel()) - 1, int(I.shape[1])
    ni = int(I.shape[0]) if among is None else int(among.numel())
    idx = torch.empty((ng, K), dtype=torch.int32, device=U.device)
    val = torch.empty((ng, K), dtype=torch.float32, device=U.device) if want_vals else None
    scratch = _score_topk_scratch(int(N.lib().llmrec_score_topk_group_scratch(_p(rp), ng, ni, d, K, mode)), U.device)
    N.check(N.lib().llmrec_score_topk_group_f32(_p(U), _ld(U), _p(I), _ld(I), _p(rp), _p(_i32(members, "members")), ng,
                                                 _p(None if among is None else _i32(among, "among")), ni, d, _p(mask_rowptr), _p(mask_col),
                                                 K, GROUP_AGG[agg], _p(idx), _p(val), mode, _p(scratch),
                                                 scratch.numel() if scratch is not None else 0, _stream()), "score_topk_group")
    _count(3)
    return (idx, val) if want_vals else idx


RERANK_MAX_K = 1024        # LLMREC_RERANK_MAX_K: the selection width of llmrec_rerank_f32


def score_pairs(U, I, qrow, item):
    """fp32[n]: <U[qrow[p]], I[item[p]]> as one sequential fp32 FMA chain (the bits score_topk returns for the same pair)."""
    _mat(U); _mat(I)
    n = int(qrow.numel())
    if int(item.numel()) != n:
        raise ValueError(f"score_pairs: {n} query rows but {int(item.numel())} items")
    out = torch.empty(n, dtype=torch.float32, device=U.device)
    N.check(N.lib().llmrec_score_pairs_f32(_p(U), _ld(U), _p(I), _ld(I), _p(_i32(qrow)), _p(_i32(item)), n, int(I.shape[1]), _p(out),
                                            _stream()), "score_pairs")
    _count()
    return out


def rerank(U, I, qrow, cand_rowptr, cand_col, mask_rowptr, mask_col, K):
    """(ids int32 [m x K], scores fp32 [m x K]): per query row r, the K best of its candidate row (CSR) scored against U[qrow[r]] by
    (score desc, id asc); ids outside [0, I.shape[0]) and ids of mask row qrow[r] dropped, repeats kept once, padded with -1 / -inf."""
    _mat(U); _mat(I)
    m = int(qrow.numel())
    idx = torch.empty((m, K), dtype=torch.int32, device=U.device)
    val = torch.empty((m, K), dtype=torch.float32, device=U.device)
    N.check(N.lib().llmrec_rerank_f32(_p(U), _ld(U), _p(I), _ld(I), _p(_i32(qrow)), m, _p(_i32(cand_rowptr)), _p(_i32(cand_col)),
                                       _p(mask_rowptr), _p(mask_col), int(I.shape[0]), int(I.shape[1]), int(K), _p(idx), _p(val),
                                       _stream()), "rerank")
    _count()
    return idx, val


EXPLAIN_MAX_TOP = 64       # LLMREC_EXPLAIN_MAX_TOP: the selection width of llmrec_explain_f32


def explain(own_src, last_src, side_usr, side_src, coefs, id_src, I, qrow, su, hist_rowptr, hist_col, targets, n_layers, top=0):
    """Exact split of <U[qrow[b]], I[targets[b, p]]> over query b's history (llmrec_explain_f32): own_src / last_src = Ul[0] / Ul[L] and
    side_usr = the fused side rows of the user side, indexed by qrow; side_src = their item-side sources and id_src = Il[0 .. L-2], indexed
    by history id; su fp32 [m] the queries' row scales; hist_rowptr / hist_col an int32 CSR of ascending history ids; targets int32
    [m x P] (-1 = padding).  -> (contrib fp32 [P * nnz x (1 + n_side)], own fp32 [m x P], last fp32 [m x P], top_ids int32 [m x P x top]
    or None, top_vals fp32 or None)."""
    for t in [own_src, last_src, I] + list(side_usr) + list(side_src) + list(id_src):
        _mat(t)
    m, P = int(targets.shape[0]), int(targets.shape[1])
    if len(side_usr) != len(side_src) or len(coefs) != len(side_usr) or int(su.numel()) != m or int(qrow.numel()) != m:
        raise ValueError("explain: one user-side row, one source and one coefficient per side term; one qrow and su per query")
    nnz, dev = int(hist_col.numel()), I.device
    C_ = 1 + len(side_usr)
    contrib = torch.empty((P * nnz, C_), dtype=torch.float32, device=dev)
    own = torch.empty((m, P), dtype=torch.float32, device=dev)
    last = torch.empty((m, P), dtype=torch.float32, device=dev)
    top = int(top or 0)
    tids = torch.empty((m, P, top), dtype=torch.int32, device=dev) if top else None
    tvals = torch.empty((m, P, top), dtype=torch.float32, device=dev) if top else None
    if su.dtype != torch.float32 or not su.is_cuda or not su.is_contiguous():
        raise ValueError("explain: su needs a contiguous CUDA fp32 vector")
    cf = (C.c_float * max(1, len(coefs)))(*[float(c) for c in coefs])
    N.check(N.lib().llmrec_explain_f32(_p(own_src), _ld(own_src), _p(last_src), _ld(last_src), _ptr_table(side_usr), _ld_table(side_usr),
                                        _ptr_table(side_src), _ld_table(side_src), cf, len(side_usr), _ptr_table(id_src), _ld_table(id_src),
                                        len(id_src), _p(I), _ld(I), int(I.shape[0]), int(I.shape[1]), int(n_layers), _p(_i32(qrow)), _p(su), m,
                                        _p(_i32(hist_rowptr)), _p(_i32(hist_col)), _p(_i32(targets.reshape(-1), "targets")), P, _p(contrib),
                                        _p(own), _p(last), top, _p(tids), _p(tvals), _stream()), "explain")
    _count(2 if top else 1)
    return contrib, own, last, tids, tvals


def diversify(X, pool_ids, pool_scores, K, lam):
    """Greedy maximal-marginal-relevance selection (llmrec_diversify_f32): per query row b, K entries of the pool (pool_ids [m x P], any
    integer dtype, ids outside [0, X.shape[0]) are padding; pool_scores fp32 [m x P]) in pick order, by lam * score - (1 - lam) * the
    largest cosine to an earlier pick, cosines the fmaf chain over the normalised rows X.  -> (ids int64 [m x K], scores fp32 [m x K],
    sims fp32 [m x K]: each pick's largest cosine when picked, -inf for the first), padded with -1 / -inf / -inf."""
    _mat(X)
    m, P = int(pool_ids.shape[0]), int(pool_ids.shape[1])
    if tuple(pool_scores.shape) != (m, P) or pool_scores.dtype != torch.float32 or not pool_scores.is_cuda:
        raise ValueError(f"diversify: pool_scores needs a CUDA fp32 [{m} x {P}] tensor like pool_ids, got {tuple(pool_scores.shape)} "
                         f"{pool_scores.dtype}")
    n = int(X.shape[0])
    ids = pool_ids.to(X.device)
    ids = torch.where((ids < 0) | (ids >= n), torch.full_like(ids, -1), ids).to(torch.int32).contiguous()
    sc = pool_scores.contiguous()
    out_i = torch.empty((m, K), dtype=torch.int32, device=X.device)
    out_v = torch.empty((m, K), dtype=torch.float32, device=X.device)
    out_s = torch.empty((m, K), dtype=torch.float32, device=X.device)
    N.check(N.lib().llmrec_diversify_f32(_p(X), _ld(X), _p(ids), _p(sc), P, m, P, n, int(X.shape[1]), int(K), C.c_float(float(lam)),
                                          _p(out_i), _p(out_v), _p(out_s), _stream()), "diversify")
    _count()
    return out_i.long(), out_v, out_s


def topk_hits(idx, users, truth_rowptr, truth_col):
    hits = torch.empty(idx.shape, dtype=torch.uint8, device=idx.device)
    N.check(N.lib().llmrec_topk_hits(_p(_i32(idx)), idx.shape[0], idx.shape[1], _p(_i32(users)), _p(_i32(truth_rowptr)), _p(_i32(truth_col)),
                                      _p(hits), _stream()), "topk_hits")
    _count()
    return hits


def user_auc(U, I, users, mask_rowptr, mask_col, truth_rowptr, truth_col):
    """fp32[n] per-user ROC-AUC over the candidates (test_flag='full', batch_test.py:38-68)."""
    _mat(U); _mat(I)
    out = torch.empty(users.numel(), dtype=torch.float32, device=U.device)
    N.check(N.lib().llmrec_user_auc_f32(_p(U), _ld(U), _p(I), _ld(I), _p(_i32(users)), users.numel(), I.shape[0], I.shape[1], _p(mask_rowptr), _p(mask_col),
                                         _p(_i32(truth_rowptr)), _p(_i32(truth_col)), _p(out), _stream()), "user_auc")
    _count()
    return out


def row_scale_softmax(X, scale, out, softmax):
    N.check(N.lib().llmrec_row_scale_softmax_f32(_p(_mat(X)), _ld(X), _p(scale), _p(_mat(out)), _ld(out), X.shape[0], X.shape[1],
                                                  1 if softmax else 0, _stream()), "row_scale_softmax")
    _count()
    return out


def row_normalize(X, out=None):
    """out = X / max(||X||_2, 1e-12) row by row (F.normalize(X, dim=1)); out may be X."""
    out = torch.empty((X.shape[0], X.shape[1]), dtype=torch.float32, device=X.device) if out is None else out
    if tuple(out.shape) != tuple(X.shape):
        raise ValueError(f"row_normalize: out {tuple(out.shape)} differs from X {tuple(X.shape)}")
    N.check(N.lib().llmrec_row_normalize_f32(_p(_mat(X)), _ld(X), _p(_mat(out)), _ld(out), X.shape[0], X.shape[1], _stream()), "row_normalize")
    _count()
    return out


def gather_rows(X, idx, out):
    N.check(N.lib().llmrec_gather_rows_f32(_p(_mat(X)), _ld(X), _p(_i32(idx)), idx.numel(), X.shape[1], _p(_mat(out)), _ld(out), _stream()), "gather_rows")
    _count()
    return out


def scatter_add_rows(G, idx, Y):
    N.check(N.lib().llmrec_scatter_add_rows_f32(_p(_mat(G)), _ld(G), _p(_i32(idx)), idx.numel(), G.shape[1], _p(_mat(Y)), _ld(Y), _stream()), "scatter_add_rows")
    _count()


def scatter_add_rows_ordered(G, idx, Y, scratch=None):
    """Y[idx[b]] += G[b] one fp32 add at a time in ascending b (idx[b] < 0 skipped): the bit-reproducible form of scatter_add_rows.
    scratch: int32 CUDA buffer of 2 * len(idx) entries; pass a persistent one under CUDA-graph capture, and one per concurrent call."""
    n = int(idx.numel())
    need = int(N.lib().llmrec_scatter_add_rows_ordered_scratch(n))
    if scratch is None:
        scratch = torch.empty(max(need, 1), dtype=torch.int32, device=idx.device)
    N.check(N.lib().llmrec_scatter_add_rows_ordered_f32(_p(_mat(G)), _ld(G), _p(_i32(idx)), n, G.shape[1], _p(_mat(Y)), _ld(Y),
                                                         _p(_i32(scratch, "scratch")), scratch.numel(), _stream()), "scatter_add_rows_ordered")
    _count(2)


def _scale_col(t):
    """1-D fp32 CUDA view (a column of a row-major table) -> (pointer, element stride)."""
    if t is None:
        return C.c_void_p(0), 0
    if t.dim() != 1 or t.dtype != torch.float32 or not t.is_cuda:
        raise ValueError("scale: need a 1-D fp32 CUDA tensor (a column view is fine)")
    return C.c_void_p(t.data_ptr()), int(t.stride(0)) if t.numel() > 1 else 1


def rank1_add(blocks):
    """blocks: list of (Y[n x w], scale[n] (1-D view), bias[w]):  Y += scale (x) bias.  One launch."""
    arr = (N.Rank1Block * len(blocks))()
    for i, (Y, sc, b) in enumerate(blocks):
        _mat(Y)
        ptr, lds = _scale_col(sc)
        arr[i] = N.Rank1Block(_p(Y), ptr, _p(b), _ld(Y), lds, Y.shape[0], Y.shape[1], 0)
    N.check(N.lib().llmrec_rank1_add_f32(arr, len(blocks), _stream()), "rank1_add")
    _count()


def scaled_colsum(terms, out, accumulate=False):
    """out[c] (+)= sum over terms (G[n x w], scale[n] | None) of sum_r scale[r] * G[r, c].  One launch, deterministic."""
    w = int(out.numel())
    arr = (N.ColsumTerm * len(terms))()
    for i, (G, sc) in enumerate(terms):
        _mat(G)
        if G.shape[1] != w:
            raise ValueError("scaled_colsum: width mismatch")
        ptr, lds = _scale_col(sc)
        arr[i] = N.ColsumTerm(_p(G), ptr, _ld(G), lds, G.shape[0])
    key = ("colsum", out.device.index, w)
    sc_ = _scratch.get(key)
    if sc_ is None:
        sc_ = _scratch[key] = torch.zeros(int(N.lib().llmrec_scaled_colsum_scratch(w)), dtype=torch.float32, device=out.device)
    N.check(N.lib().llmrec_scaled_colsum_f32(arr, len(terms), w, _p(out), 1 if accumulate else 0, _p(sc_), _stream()), "scaled_colsum")
    _count()


def feat_reg_gram(W, b, G, h, n2, c, dW, db, loss):
    """feat_reg over all rows through the Gram matrix G[k x k] of a propagated table (include/llmrec_b200.h).
    The kernels read W, G and dW as dense row-major blocks and b, h, db as unit-stride vectors."""
    if W.dim() != 2:
        raise ValueError(f"feat_reg_gram: W must be 2-D, got {tuple(W.shape)}")
    d, k = W.shape
    for name, t, shape in (("W", W, (d, k)), ("G", G, (k, k)), ("dW", dW, (d, k)), ("b", b, (d,)), ("db", db, (d,)), ("h", h, (k,)),
                           ("loss", loss, None)):
        if t is None and name in ("b", "db", "h", "loss"):
            continue
        if t is None or t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or (shape is not None and tuple(t.shape) != shape) \
                or (shape is None and t.numel() < 1):
            got = "None" if t is None else f"{tuple(t.shape)} {t.dtype} {t.device} strides {t.stride()}"
            raise ValueError(f"feat_reg_gram: {name} must be a contiguous CUDA fp32 tensor of shape {shape or '[>= 1]'}, got {got}")
    key = ("gram", W.device.index, d, k)
    sc_ = _scratch.get(key)
    if sc_ is None:
        sc_ = _scratch[key] = torch.zeros(int(N.lib().llmrec_feat_reg_gram_scratch(d, k)), dtype=torch.float32, device=W.device)
    N.check(N.lib().llmrec_feat_reg_gram_f32(_p(W), _p(b), _p(G), _p(h), float(n2), d, k, float(c), _p(dW), _p(db), _p(loss), _p(sc_), _stream()), "feat_reg_gram")
    _count(2)


def fill(t, v):
    N.check(N.lib().llmrec_fill_f32(_p(t), t.numel(), float(v), _stream()), "fill")
