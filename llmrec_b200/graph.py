"""Device-resident bipartite interaction graph for the propagation kernels.

The reference builds two fp32 COO tensors, ui = diag((deg_u+1e-8)^-1/2) R and
iu = diag((deg_i+1e-8)^-1/2) R^T (main.py:84-91,114-134), and torch re-coalesces / converts them to
CSR inside every torch.sparse.mm call.  Here the binary pattern R is stored ONCE as int32 CSR plus
the CSR of its transpose and two fp32 scale vectors; the four operators the path needs are views:

    ui   = diag(su) R          rows=users   pattern CSR(R)    row scale su
    iu   = diag(si) R^T        rows=items   pattern CSR(R^T)  row scale si
    ui^T = R^T diag(su)        rows=items   pattern CSR(R^T)  col scale su     (backward of ui)
    iu^T = R diag(si)          rows=users   pattern CSR(R)    col scale si     (backward of iu)

HBM layout: rowptr int32[n+1], col int32[nnz], scales fp32[n]; forward operators carry no value array, the two
transpose operators carry w[e] = scale[col[e]] (fp32[nnz]).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import torch

from .ops import CsrOperator


def inv_sqrt_degree(mat: sp.spmatrix) -> np.ndarray:
    """(rowsum + 1e-8)^-1/2 in float64 with inf -> 0, as csr_norm does (main.py:114-118)."""
    deg = np.asarray(mat.sum(1)).reshape(-1).astype(np.float64)
    s = np.power(deg + 1e-8, -0.5)
    s[np.isinf(s)] = 0.0
    return s


def history_matrix(rowptr, col, n_items: int, what: str = "histories", unit: str = "item id") -> sp.csr_matrix:
    """m interaction histories given at call time (int CSR over item ids: rowptr[m+1], col[nnz]; arrays, lists or tensors on any
    device) -> the binary [m x n_items] CSR with sorted rows, a repeated id within a row collapsed as BipartiteGraph does for R.
    An id outside [0, n_items) raises ValueError.  The same holds for the user lists of new items (columns = user ids); `what` and
    `unit` name the input in the error messages."""
    as_np = lambda a: (a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)).astype(np.int64).reshape(-1)
    rp, c = as_np(rowptr), as_np(col)
    if rp.size < 1 or rp[0] != 0 or np.any(np.diff(rp) < 0) or rp[-1] != c.size:
        raise ValueError(f"{what}: rowptr must start at 0, never decrease and end at len(col) = {c.size}")
    if c.size and (c.min() < 0 or c.max() >= n_items):
        bad = int(c[(c < 0) | (c >= n_items)][0])
        raise ValueError(f"{what}: {unit} {bad} is outside [0, {n_items})")
    m = rp.size - 1
    R = sp.csr_matrix((np.ones(c.size, dtype=np.float32), c, rp), shape=(m, n_items))
    R.sum_duplicates()
    R.sort_indices()
    R.data[:] = 1.0
    if R.nnz >= 2 ** 31:
        raise ValueError(f"{what} too large for int32 CSR")
    return R


def histories_csr(histories, n_items: int, what: str = "histories", unit: str = "item id") -> sp.csr_matrix:
    """`history_matrix` of either form a caller may hold: a (rowptr, col) pair (a tuple of two arrays / tensors), or a sequence of
    item-id lists, one per history."""
    if isinstance(histories, tuple) and len(histories) == 2 and all(hasattr(a, "shape") for a in histories):
        return history_matrix(histories[0], histories[1], n_items, what, unit)
    rows = [np.asarray(list(h), dtype=np.int64).reshape(-1) for h in histories]
    rp = np.zeros(len(rows) + 1, dtype=np.int64)
    rp[1:] = np.cumsum([r.size for r in rows])
    return history_matrix(rp, np.concatenate(rows) if rows else np.zeros(0, np.int64), n_items, what, unit)


class BipartiteGraph:
    def __init__(self, train_mat: sp.spmatrix, device, tile_nnz: int = 0):
        R = sp.csr_matrix(train_mat)
        R.sum_duplicates()
        R.sort_indices()
        Rt = sp.csr_matrix(R.T)
        Rt.sort_indices()
        self.n_users, self.n_items = R.shape
        self.nnz = int(R.nnz)
        if self.nnz >= 2 ** 31:
            raise ValueError("graph too large for int32 CSR")
        if not np.all(R.data == 1):
            raise ValueError("BipartiteGraph expects a binary interaction matrix (use operators_from_coo for weighted graphs)")
        dev = torch.device(device)
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a.astype(dt))).to(dev)
        self.rowptr_u, self.col_u = t(R.indptr, np.int32), t(R.indices, np.int32)
        self.rowptr_i, self.col_i = t(Rt.indptr, np.int32), t(Rt.indices, np.int32)
        self.su = t(inv_sqrt_degree(R), np.float32)
        self.si = t(inv_sqrt_degree(Rt), np.float32)
        nu, ni = self.n_users, self.n_items
        self.ui = CsrOperator(self.rowptr_u, self.col_u, nu, ni, rs=self.su, tile_nnz=tile_nnz)
        self.iu = CsrOperator(self.rowptr_i, self.col_i, ni, nu, rs=self.si, tile_nnz=tile_nnz)
        # transposes: the column scale is gathered ONCE into a per-nnz weight array (coalesced with col in the kernel,
        # no dependent cs[col] load); same pattern -> same tile plan as the forward operator of the other direction
        self.w_uiT = self.su[self.col_i.long()].contiguous()
        self.w_iuT = self.si[self.col_u.long()].contiguous()
        self.uiT = CsrOperator(self.rowptr_i, self.col_i, ni, nu, vals=self.w_uiT, plan=self.iu.plan)
        self.iuT = CsrOperator(self.rowptr_u, self.col_u, nu, ni, vals=self.w_iuT, plan=self.ui.plan)
        self.device = dev

    def ones_propagated(self):
        """cu = ui.1, ci = iu.ui.1, ri = iu.1, ru = ui.iu.1 -- the propagated ones-vectors that multiply the Linear biases when the
        side-feature propagation is hoisted (hoist.py); computed with the propagation kernel itself on [n x 4] blocks."""
        new = lambda n: torch.empty(n, 4, dtype=torch.float32, device=self.device)
        one_i, one_u = torch.ones(self.n_items, 4, device=self.device), torch.ones(self.n_users, 4, device=self.device)
        cu, ci, ri, ru = new(self.n_users), new(self.n_items), new(self.n_items), new(self.n_users)
        self.ui.apply([(one_i, cu, None, False)])
        self.iu.apply([(cu, ci, None, False)])
        self.iu.apply([(one_u, ri, None, False)])
        self.ui.apply([(ri, ru, None, False)])
        return dict(cu=cu[:, 0].contiguous(), ci=ci[:, 0].contiguous(), ri=ri[:, 0].contiguous(), ru=ru[:, 0].contiguous())

    # the reference-facing COO tensors (what Trainer.ui_graph / iu_graph hold; main.py:128-134)
    def coo_tensors(self):
        def coo(rowptr, col, scale, shape):
            rp = rowptr.to(torch.int64)
            rows = torch.repeat_interleave(torch.arange(shape[0], device=self.device), rp[1:] - rp[:-1])
            idx = torch.stack([rows, col.to(torch.int64)])
            t = torch.sparse_coo_tensor(idx, scale[rows], shape)
            return t
        ui = coo(self.rowptr_u, self.col_u, self.su, (self.n_users, self.n_items))
        iu = coo(self.rowptr_i, self.col_i, self.si, (self.n_items, self.n_users))
        ui._llmrec_ops = (self.ui, self.uiT)
        iu._llmrec_ops = (self.iu, self.iuT)
        return ui, iu


def operators_from_coo(A: torch.Tensor):
    """(forward, backward) CsrOperators for an arbitrary fp32 sparse COO matrix (valued CSR path)."""
    cached = getattr(A, "_llmrec_ops", None)
    if cached is not None:
        return cached

    def csr(M):
        M = M.coalesce()
        idx, val = M.indices(), M.values().to(torch.float32).contiguous()
        n_rows, n_cols = M.shape
        counts = torch.bincount(idx[0], minlength=n_rows)
        rowptr = torch.zeros(n_rows + 1, dtype=torch.int64, device=val.device)
        rowptr[1:] = torch.cumsum(counts, 0)
        return CsrOperator(rowptr.to(torch.int32), idx[1].to(torch.int32).contiguous(), n_rows, n_cols, vals=val)

    ops = (csr(A), csr(A.t()))
    try:
        A._llmrec_ops = ops
    except Exception:
        pass
    return ops
