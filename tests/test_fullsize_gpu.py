"""-m gpu: size-independent properties of the DEFAULT kernels at the full sizes of BASELINE.json's netflix / movielens
configurations (linearity, adjoint identity, idempotence, sortedness, exclusion) -- parity at shapes where every persistent
kernel runs many tiles per CTA, which the tiny golden dataset cannot exercise."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
cuda = "cuda"


FULL = {"netflix": (13187, 17366, 68933, 64), "movielens": (12495, 10322, 57960, 128)}


def _full_graph(name):
    import scipy.sparse as sp
    from llmrec_b200.graph import BipartiteGraph
    nu, ni, ne, d = FULL[name]
    rng = np.random.default_rng(0)
    rows = np.concatenate([np.arange(nu), rng.integers(0, nu, ne - nu)])
    w = 1.0 / (np.arange(ni) + 8.0) ** 0.8
    cols = rng.choice(ni, size=ne, p=w / w.sum())
    R = sp.csr_matrix((np.ones(ne, np.float32), (rows, cols)), shape=(nu, ni))
    R.sum_duplicates(); R.data[:] = 1.0
    return BipartiteGraph(R, cuda), R, d


@pytest.mark.parametrize("name", ["netflix", "movielens"])
def test_fullsize_propagation_is_linear_and_matches_fp64(name):
    g, R, d = _full_graph(name)
    gen = torch.Generator().manual_seed(1)
    nu, ni = R.shape
    X, Z = torch.randn(ni, d, generator=gen).to(cuda), torch.randn(ni, d, generator=gen).to(cuda)
    out = [torch.empty(nu, d, device=cuda) for _ in range(3)]
    g.ui.apply([(X, out[0], None, False)])
    g.ui.apply([(Z, out[1], None, False)])
    g.ui.apply([(2.0 * X - 0.5 * Z, out[2], None, False)])
    torch.testing.assert_close(out[2], 2.0 * out[0] - 0.5 * out[1], rtol=1e-5, atol=1e-5)           # linearity
    again = torch.empty_like(out[0])
    g.ui.apply([(X, again, None, False)])
    assert torch.equal(again, out[0])                                                                # run-to-run identical (no atomics)
    deg = np.asarray(R.sum(1)).reshape(-1)
    ref = torch.from_numpy(np.power(deg + 1e-8, -0.5))[:, None] * torch.from_numpy((R @ X.cpu().double().numpy()))
    torch.testing.assert_close(out[0].cpu().double(), ref, rtol=1e-5, atol=1e-6)
    # adjoint identity <ui X, Y> == <X, ui^T Y> ties the forward operator to the backward one
    Y = torch.randn(nu, d, generator=gen).to(cuda)
    back = torch.empty(ni, d, device=cuda)
    g.uiT.apply([(Y, back, None, False)])
    a, b = (out[0].double() * Y.double()).sum(), (X.double() * back.double()).sum()
    assert abs(float(a - b)) <= 1e-5 * max(1.0, abs(float(a)))


@pytest.mark.parametrize("name", ["netflix", "movielens"])
def test_fullsize_projection_matches_fp64_and_is_linear(name):
    from llmrec_b200 import ops
    nu, ni, _, d = FULL[name]
    gen = torch.Generator().manual_seed(2)
    X = torch.randn(ni, 1536, generator=gen).to(cuda)
    W = (torch.randn(d, 1536, generator=gen) / 1536 ** 0.5).to(cuda)
    b = torch.randn(d, generator=gen).to(cuda)
    Y = torch.empty(ni, d, device=cuda)
    ops.proj_fwd_group([(X, W, b, Y)], d, 0)
    ref = X.double() @ W.double().t() + b.double()
    torch.testing.assert_close(Y.double(), ref, rtol=1e-4, atol=1e-4)
    Y2 = torch.empty_like(Y)
    ops.proj_fwd_group([(X, 2.0 * W, None, Y2)], d, 0)                      # exact in binary: scaling W by 2 scales every product by 2
    assert torch.equal(Y2, 2.0 * (Y - b))  or torch.allclose(Y2, 2.0 * (Y - b), rtol=1e-6, atol=1e-6)
    dY = torch.randn(ni, d, generator=gen).to(cuda)
    dW, db = torch.empty(d, 1536, device=cuda), torch.empty(d, device=cuda)
    ops.proj_wgrad_group([(X, dY, dW, db, False)], d, 0)
    torch.testing.assert_close(dW.double(), dY.double().t() @ X.double(), rtol=1e-4, atol=1e-4 * ni ** 0.5)
    torch.testing.assert_close(db.double(), dY.double().sum(0), rtol=1e-4, atol=1e-3)


def test_fullsize_scoring_topk_properties():
    """13 187 users x 17 366 items, K = 50: lists are sorted by exact score (ties by id), contain no train item, are
    identical between the tensor-core and the exact SIMT path and between two runs, and nothing outside beats the K-th entry."""
    from llmrec_b200 import ops
    nu, ni, ne, d = FULL["netflix"]
    g, R, _ = _full_graph("netflix")
    gen = torch.Generator().manual_seed(3)
    U, I = torch.randn(nu, d, generator=gen).to(cuda), torch.randn(ni, d, generator=gen).to(cuda)
    users = torch.arange(nu, dtype=torch.int32, device=cuda)
    idx, val = ops.score_topk(U, I, users, g.rowptr_u, g.col_u, 50, mode=0, want_vals=True)
    idx2 = ops.score_topk(U, I, users, g.rowptr_u, g.col_u, 50, mode=0)
    assert torch.equal(idx, idx2)                                                                    # idempotent
    exact, exact_val = ops.score_topk(U, I, users, g.rowptr_u, g.col_u, 50, mode=2, want_vals=True)
    assert torch.equal(idx, exact)                                                                   # rescoring makes the lists exact
    assert torch.equal(val.view(torch.int32), exact_val.view(torch.int32))                           # same fp32 FMA order: same bits
    S = U @ I.t()                                                                                    # fp32 scores, dense (0.9 GB)
    rows = torch.repeat_interleave(torch.arange(nu, device=cuda), (g.rowptr_u[1:] - g.rowptr_u[:-1]).long())
    S[rows, g.col_u.long()] = float("-inf")                                                          # train items are not candidates
    picked = torch.gather(S, 1, idx.long())
    assert bool(torch.isfinite(picked).all())                                                        # no train item was ranked
    assert bool((picked[:, :-1] >= picked[:, 1:] - 1e-5).all())                                      # descending
    S.scatter_(1, idx.long(), float("-inf"))
    assert bool((S.max(dim=1).values <= picked[:, -1] + 1e-5).all())                                 # nothing outside beats the K-th




def test_tma_staged_spmm_is_bit_identical_to_the_register_kernel():
    """LLMREC_SPMM_BULK=1 routes d = 128 single-operand products through spmm_bulk_kernel (neighbour rows staged in shared memory by
    cp.async.bulk + mbarriers): same tile plan, same summation order -> bit-identical output; softmax epilogue, addend, long rows."""
    import subprocess
    import sys
    code = r"""
import os, sys, numpy as np, torch
sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests"))
from test_fullsize_gpu import _full_graph
res = {}
g, R, d = _full_graph("movielens")
nu, ni = R.shape
gen = torch.Generator().manual_seed(4)
X, Z = torch.randn(ni, d, generator=gen).cuda(), torch.randn(nu, d, generator=gen).cuda()
Xu = torch.randn(nu, d, generator=gen).cuda()
out = []
for sm, z in ((False, None), (True, None), (False, Z)):
    Y = torch.empty(nu, d, device="cuda"); g.ui.apply([(X, Y, z, sm)]); out.append(Y.cpu())
Yi = torch.empty(ni, d, device="cuda"); g.iu.apply([(Xu, Yi, None, False)]); out.append(Yi.cpu())       # item rows: long rows -> pieces + finish pass
torch.save(out, sys.argv[1])
""" % ((os.path.dirname(os.path.dirname(os.path.abspath(__file__))),) * 2)
    import tempfile
    outs = []
    for flag in ("0", "1"):
        with tempfile.NamedTemporaryFile(suffix=".pt") as f:
            r = subprocess.run([sys.executable, "-c", code, f.name], env=dict(os.environ, LLMREC_SPMM_BULK=flag), capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, r.stderr[-2000:]
            outs.append(torch.load(f.name))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_grouped_projections_many_tiles_per_cta_match_fp64():
    """The grouped launches at the bench's own shape: 8 problems (k = 1536 x6, 768, 512), ~1056 row tiles / ~700 wgrad items, i.e. many
    CTAs per SM with ring wrap-around and problem changes across the grid -- against fp64."""
    from llmrec_b200 import ops
    nu, ni, _, d = FULL["netflix"]
    gen = torch.Generator().manual_seed(11)
    dims = [(ni, 1536)] * 5 + [(nu, 1536), (ni, 768), (ni, 512)]
    Xs = [torch.randn(n, k, generator=gen).to(cuda) for n, k in dims]
    Ws = [(torch.randn(d, k, generator=gen) / k ** 0.5).to(cuda) for _, k in dims]
    bs = [torch.randn(d, generator=gen).to(cuda) for _ in dims]
    Ys = [torch.empty(n, d, device=cuda) for n, _ in dims]
    for rep in range(2):                                        # second launch: barriers / rings start from a used state
        ops.proj_fwd_group([(X, W, b, Y) for X, W, b, Y in zip(Xs, Ws, bs, Ys)], d, 0)
    for X, W, b, Y in zip(Xs, Ws, bs, Ys):
        torch.testing.assert_close(Y.double(), X.double() @ W.double().t() + b.double(), rtol=1e-4, atol=1e-4)
    dYs = [torch.randn(n, d, generator=gen).to(cuda) for n, _ in dims]
    dWs = [torch.empty(d, k, device=cuda) for _, k in dims]
    dbs = [torch.empty(d, device=cuda) for _ in dims]
    for rep in range(2):
        ops.proj_wgrad_group([(X, dY, dW, db, False) for X, dY, dW, db in zip(Xs, dYs, dWs, dbs)], d, 0)
    for X, dY, dW, db in zip(Xs, dYs, dWs, dbs):
        torch.testing.assert_close(dW.double(), dY.double().t() @ X.double(), rtol=1e-4, atol=1e-4 * X.shape[0] ** 0.5)
        torch.testing.assert_close(db.double(), dY.double().sum(0), rtol=1e-4, atol=1e-3)
