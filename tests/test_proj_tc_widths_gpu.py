"""-m gpu: the tensor-core projections at every tile shape they pick -- widths d = 32 / 96 / 256, k not a multiple of 32, plain
TF32 (mode 1), and grouped launches large enough for the 256-wide tiles (d <= 128) -- against fp64."""
import pytest
import torch

pytestmark = pytest.mark.gpu

cuda = torch.device("cuda")
# mode 0 (3xTF32): fp32-class; mode 1 (plain TF32 operands, ~2^-11 per product): relative to |Y| ~ 1 and |dW| ~ sqrt(n)
TOL = {0: 1e-4, 1: 5e-3}


def _check(Xs, d, mode, seed):
    from llmrec_b200 import ops
    g = torch.Generator().manual_seed(seed)
    Ws = [(torch.randn(d, X.shape[1], generator=g) / X.shape[1] ** 0.5).to(cuda) for X in Xs]
    bs = [torch.randn(d, generator=g).to(cuda) for _ in Xs]
    wides = [torch.empty(X.shape[0], 3 * d, device=cuda) for X in Xs]
    Ys = [w[:, d:2 * d] for w in wides]                                              # strided output views
    ops.proj_fwd_group(list(zip(Xs, Ws, bs, Ys)), d, mode)
    tol = TOL[mode]
    for X, W, b, Y in zip(Xs, Ws, bs, Ys):
        torch.testing.assert_close(Y.double(), X.double() @ W.double().t() + b.double(), rtol=tol, atol=tol)
    dYs = [torch.randn(X.shape[0], 3 * d, generator=g).to(cuda)[:, d:2 * d] for X in Xs]   # strided dY views (like the GPi blocks)
    dWs = [torch.empty(d, X.shape[1], device=cuda) for X in Xs]
    dbs = [torch.empty(d, device=cuda) for _ in Xs]
    for _ in range(2):                                                               # second call: rings and tickets start used
        ops.proj_wgrad_group(list(zip(Xs, dYs, dWs, dbs, [False] * len(Xs))), d, mode)
    for X, dY, dW, db in zip(Xs, dYs, dWs, dbs):
        n = X.shape[0]
        torch.testing.assert_close(dW.double(), dY.double().t() @ X.double(), rtol=tol, atol=tol * n ** 0.5)
        torch.testing.assert_close(db.double(), dY.double().sum(0), rtol=1e-4, atol=1e-4 * n ** 0.5)


@pytest.mark.parametrize("n,k,d,mode", [(1000, 512, 32, 0), (700, 256, 256, 0), (777, 100, 96, 0), (513, 100, 64, 0),
                                        (1000, 512, 64, 1), (300, 1536, 128, 1), (450, 68, 160, 1), (257, 36, 224, 0)])
def test_single_projection_widths_and_edges(n, k, d, mode):
    g = torch.Generator().manual_seed(n + k + d)
    _check([torch.randn(n, k, generator=g).to(cuda)], d, mode, seed=d)


@pytest.mark.parametrize("d,mode", [(128, 0), (128, 1), (96, 0), (32, 0)])
def test_grouped_projections_on_256_wide_tiles(d, mode):
    """Enough row tiles / wgrad items that the launches use 256-row / 256-feature tiles, with mixed k (one not a multiple of 32)."""
    g = torch.Generator().manual_seed(d + mode)
    dims = [(9000, 1536)] * 5 + [(8000, 100), (9001, 768)]
    _check([torch.randn(n, k, generator=g).to(cuda) for n, k in dims], d, mode, seed=3 * d + mode)
