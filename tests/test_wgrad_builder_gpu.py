"""-m gpu: with fp32 tables in mode 0 the weight-gradient kernel builds its B operand (dY^T, hi and lo) from dY inside the kernel.

Each stage's B tile is gathered from the caller's strided dY through the optional row map, split and written in the swizzled layout
wgmma reads; rows past n must be zeros.  bf16 tables and mode 1 take dY^T from `dyt_split` by TMA and run the same cases.  These cases sit on the builder's edges -- n around one stage (32 rows, 64 for bf16 tables),
row chunks ending mid-stage, an empty problem beside non-empty ones, dY as a column block of a wider matrix, row maps with gaps and
out of order, every width in both tile forms, fp32 and bf16 tables, modes 0 and 1 -- against fp64, and a repeated call must give
the same bits.  An identity row map must give the bits of no map."""
import pytest
import torch

pytestmark = pytest.mark.gpu

cuda = torch.device("cuda")
NAN = float("nan")
WIDTHS = [32, 64, 96, 128, 160, 192, 224, 256]
# mode 0: fp32-class (3xTF32, or exact bf16 products); mode 1: plain TF32 operands, or dY truncated to bf16 with a bf16 table
TOL = {(False, 0): 1e-4, (False, 1): 5e-3, (True, 0): 1e-4, (True, 1): 2e-2}
# n: one row, one stage and its neighbours (32 fp32 rows / 64 bf16 rows per stage), a row chunk of 256 plus one row, an empty problem
EDGES = [(1, 40), (31, 264), (32, 8), (33, 1536), (63, 40), (64, 264), (65, 8), (1025, 264), (0, 40), (2111, 72)]
BIG = [(9000, 1536)] * 5                       # 150 items at 256 features: the 256-wide tile form at d <= 128


def _gen(seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def _table(g, n, k, bf16, lead=8, pad=8):
    """X[n x k] as a column slice of a wider table, 16 bytes into its row (ld a multiple of 8 elements for bf16)."""
    T = torch.randn((n, lead + k + pad), generator=g, device=cuda)
    return (T.to(torch.bfloat16) if bf16 else T)[:, lead:lead + k]


def _case(dims, d, mode, bf16, seed, mapped):
    """(problems, references): dY is a column block of a [m x 3d] matrix; with `mapped`, X row r pairs with dY[rows[r]], rows a
    sorted subset with gaps (even problems) or a shuffled one (odd problems) of m = 2n + 3 rows."""
    g = _gen(seed)
    probs, refs = [], []
    for i, (n, k) in enumerate(dims):
        X = _table(g, n, k, bf16)
        mapped_i = mapped and n > 0                # an empty problem takes no map
        m = 2 * n + 3 if mapped_i else n
        dY = torch.randn((m, 3 * d), generator=g, device=cuda)[:, d:2 * d]
        dW, db = torch.full((d, k), NAN, device=cuda), torch.full((d,), NAN, device=cuda)
        pr = (X, dY, dW, db, False)
        if mapped_i:
            pick = torch.randperm(m, generator=g, device=cuda)[:n]
            rows = (torch.sort(pick).values if i % 2 == 0 else pick).to(torch.int32).contiguous()
            pr += (rows,)
            dYr = dY[rows.long()]
        else:
            dYr = dY
        probs.append(pr)
        refs.append((dYr.double().t() @ X.double(), dY.double().sum(0)))
    return probs, refs


def _run_and_check(probs, refs, d, mode, bf16):
    from llmrec_b200 import ops
    ops.proj_wgrad_group(probs, d, mode)
    first = [(p[2].clone(), p[3].clone()) for p in probs]
    tol = TOL[(bf16, mode)]
    for p, (rW, rb) in zip(probs, refs):
        n = p[0].shape[0]
        torch.testing.assert_close(p[2].double(), rW, rtol=tol, atol=tol * max(n, 1) ** 0.5, msg=lambda s: f"dW n={n} k={p[0].shape[1]}: {s}")
        torch.testing.assert_close(p[3].double(), rb, rtol=1e-4, atol=1e-4 * max(n, 1) ** 0.5, msg=lambda s: f"db n={n}: {s}")
    ops.proj_wgrad_group(probs, d, mode)
    for p, (W0, b0) in zip(probs, first):
        assert torch.equal(p[2].view(torch.int32), W0.view(torch.int32)), "dW changed on a second call"
        assert torch.equal(p[3].view(torch.int32), b0.view(torch.int32)), "db changed on a second call"


@pytest.mark.parametrize("mapped", [False, True])
@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("d", WIDTHS)
def test_builder_edges(d, mode, bf16, mapped):
    """Stage and chunk edges, an empty problem and strided dY (ten problems: two grouped launches, 128-wide tiles)."""
    probs, refs = _case(EDGES, d, mode, bf16, seed=d * 10 + mode, mapped=mapped)
    _run_and_check(probs, refs, d, mode, bf16)


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("d", [32, 64, 96, 128])
def test_builder_wide_tiles(d, mode, bf16):
    """Enough items for the 256-feature tiles (two m64 blocks per consumer), row-mapped as the live-item tables are."""
    probs, refs = _case(BIG, d, mode, bf16, seed=1000 + d, mapped=True)
    _run_and_check(probs, refs, d, mode, bf16)


@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("d", [64, 128])
def test_identity_map_is_no_map(d, bf16):
    from llmrec_b200 import ops
    dims = [(33, 264), (2111, 1536), (1, 8)]
    probs, _ = _case(dims, d, 0, bf16, seed=7, mapped=False)
    ops.proj_wgrad_group(probs, d, 0)
    plain = [p[2].clone() for p in probs]
    ident = [(X, dY, torch.full_like(dW, NAN), torch.full_like(db, NAN), False, torch.arange(X.shape[0], dtype=torch.int32, device=cuda))
             for X, dY, dW, db, _ in probs]
    ops.proj_wgrad_group(ident, d, 0)
    for a, p in zip(plain, ident):
        assert torch.equal(a.view(torch.int32), p[2].view(torch.int32))
