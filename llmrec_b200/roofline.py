"""Roofline denominators and the algorithmic byte counts of SURVEY.md 8(d) (fp32, int32 indices), shared by bench.py's legs."""
from __future__ import annotations

import json
import os

from .sides import SideLayout

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def peaks():
    """-> (HBM GB/s, dense bf16 TFLOP/s, source): MEASURED_PEAKS.json when present, else the H100 SXM data-sheet figures."""
    p = os.path.join(REPO, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        j = json.load(open(p))
        return float(j["hbm_gbs"]), float(j.get("bf16_tflops", 989.0)), "measured"
    return 3350.0, 989.0, "H100 SXM data sheet"


def spmm_bytes(nnz, M, N, d, segs=1):
    """Y[M x d] = diag(s) R X[N x d] for `segs` operands sharing the pattern: every operand touched once."""
    return 4 * nnz + 4 * (M + 1) + 4 * M + segs * (4 * d * N + 4 * d * M)


def proj_bytes(n, k, d, x_bytes=4):
    """Y[n x d] = X[n x k] W^T (or its weight gradient): X read once at x_bytes per element (4 fp32, 2 bf16, 1 int8 -- plus the
    int8 table's fp32 row scale, 4 per row), fp32 W and Y."""
    return x_bytes * n * k + (4 * n if x_bytes == 1 else 0) + 4 * k * d + 4 * n * d


def step_bytes(hp, nnz):
    """Algorithmic bytes per kernel family for one training step of engine.HotPath `hp`."""
    nu, ni, d, S, L = hp.nu, hp.ni, hp.d, hp.S, hp.L
    out = {}
    if hp.has_feats:
        f, p = hp.feats, hp.p
        nl = getattr(hp, "n_live", ni)         # the item-side problems read the live items' rows only (engine.HotPath._build_live_items)
        w = SideLayout(hp.keys, d).weights                   # the S item-side blocks, then the user profile
        k = lambda name: int(p[name + ".weight"].shape[1])      # logical widths from the weights (an int8 row also holds its scale)
        gemms = [(nl, k(name)) for name in w[:-1]] + [(nu, k(w[-1]))]
        xb = f["image"].element_size()
        out["proj_fwd"] = out["proj_wgrad"] = sum(proj_bytes(n, k, d, xb) for n, k in gemms)
    sp = lambda M, N, segs: spmm_bytes(nnz, M, N, d, segs)
    out["spmm_fwd"] = sp(nu, ni, S + 1) + sp(ni, nu, S + 2) + sp(nu, ni, 2) + (sp(ni, nu, 1) if L >= 2 else 0)
    out["spmm_bwd"] = sp(ni, nu, 1) + sp(nu, ni, S + 2) + sp(ni, nu, S + 1) + (sp(nu, ni, 1) + sp(ni, nu, 1) if L >= 2 else 0)
    out["adamw"] = 28 * sum(p.numel() for p in hp.opt.params)
    T = (3 + len(hp.keys)) if hp.has_feats else 0
    # rows fused per step: every user and item, or with train_step's batch-row fusion the batch's distinct users and items (the row
    # counts of the last row sets built -- a host read, so call this outside any timed region) plus one int32 id per row
    n_fused, ids = nu + ni, 0
    if getattr(hp, "demand_fuse", False):
        n_fused = int(hp.batch_u.count.item()) + int(hp.batch_i.count.item())
        ids = 4 * n_fused
    fuse = 4 * d * n_fused * ((L + 1) + T + 1) + ids
    out["fuse_fwd"] = fuse
    out["fuse_bwd"] = fuse + 4 * d * n_fused * T
    return out
