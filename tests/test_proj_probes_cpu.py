"""The term-exact probes (tests/proj_probes.py) against a CPU emulator of the tensor-core projection main loop: fp32 arithmetic in k8
(bf16: k16) wgmma steps over 32- (64-) deep stages, the operand split of tf32_hi and bf16_split3.

The emulator gives the expected bits on every probe case, and each kernel defect of proj_probes.MUTATIONS changes them.  The
tolerance check of tests/test_tc_exactness_gpu.py and tests/test_feat_bf16_gpu.py (randn operands against fp64, rtol = atol = 1e-4,
atol scaled by sqrt(n) for dW), run on the same emulator with the same shapes, misses one of those defects: the bf16 X*w2 term
missing on the last k16 step moves results by less than a tenth of the tolerance.  The dropped and mispaired 3xTF32 terms it does
catch -- by 2x to 14x the tolerance: the truncating split leaves lo up to 2^-10 |x|, so a lo*hi or hi*lo term is ~4e-4 relative, not
fp32-rounding sized."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import proj_probes as PP  # noqa: E402

D = 64
PROBE_DIMS = {"f32": [(1, 4), (33, 36), (65, 100), (257, 264), (300, 1536), (2111, 40)],
              "bf16": [(1, 8), (65, 40), (129, 104), (257, 264), (300, 1536), (2111, 40)]}


def _case(path, mode, n, k, seed):
    """(X probe, W probe, bias probe, dY probe): X sparse (proj_probes.pattern), W / dY dense."""
    xk, wk, cap = PP.KINDS[path]
    rng = np.random.default_rng(seed)
    X = PP.probe(xk, rng, (n, k), PP.pattern(n, k, cap, cap, shift=seed))
    return X, PP.probe(wk, rng, (D, k)), PP.probe(wk, rng, (D,)), PP.probe(wk, rng, (n, D))


def _expect(path, mode, n, k, seed):
    X, W, b, dY = _case(path, mode, n, k, seed)
    Y = PP.expected(PP.term_pairs(X, W, mode), PP.fwd, [(b.full[None, :], min(b.units))])
    dW = PP.expected(PP.term_pairs(X, dY, mode), PP.wgrad)
    return X, W, b, dY, Y, dW


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("path", ["f32", "bf16"])
def test_emulator_gives_the_probe_bits(path, mode):
    """Every probe case, forward and weight gradient: the emulated kernel equals the expected values bit for bit."""
    bf16 = path == "bf16"
    for i, (n, k) in enumerate(PROBE_DIMS[path]):
        X, W, b, dY, Y, dW = _expect(path, mode, n, k, seed=i)
        assert np.array_equal(PP.emulate_fwd(X.value, W.value, b.value, mode, bf16), Y), (path, mode, n, k)
        assert np.array_equal(PP.emulate_wgrad(X.value, dY.value, mode, bf16), dW), (path, mode, n, k)


def test_probe_value_does_not_depend_on_summation_order():
    """One probe output (bias included) summed term by term in fp32 in 200 random orders: always the same value."""
    rng = np.random.default_rng(0)
    X, W, b, _, Y, _ = _expect("f32", 0, 1, 1536, seed=3)
    terms = np.concatenate([(a[0] * w[0]) for a, _, w, _ in PP.term_pairs(X, W, 0)] + [b.full[:1]])
    assert np.count_nonzero(terms) > 3 * 40
    for _ in range(200):
        acc = np.float32(0)
        for t in rng.permutation(terms):
            acc = np.float32(acc + np.float32(t))
        assert acc == Y[0, 0]


MUTATION_DIMS = [(257, 1536), (2111, 128)]      # k a multiple of 64: the last k16 step of a stage holds real columns


@pytest.mark.parametrize("name", list(PP.MUTATIONS))
def test_every_mutation_changes_the_probe_bits(name):
    """Each defect of proj_probes.MUTATIONS gives wrong bits on the probes, in each direction it applies to."""
    path, dirs, rule = PP.MUTATIONS[name]
    bf16 = path == "bf16"
    for i, (n, k) in enumerate(MUTATION_DIMS):
        X, W, b, dY, Y, dW = _expect(path, 0, n, k, seed=10 + i)
        if "fwd" in dirs:
            assert not np.array_equal(PP.emulate_fwd(X.value, W.value, b.value, 0, bf16, rule), Y), (name, n, k)
        if "wgrad" in dirs:
            assert not np.array_equal(PP.emulate_wgrad(X.value, dY.value, 0, bf16, rule), dW), (name, n, k)


# the shapes of the tolerance tests (tests/test_tc_exactness_gpu.py, tests/test_feat_bf16_gpu.py): small n and k at stage edges, and
# the netflix table (9000 x 1536)
RANDN_DIMS = {"f32": [(n, k) for n in (1, 63, 65, 257) for k in (4, 36, 100, 1536)] + [(9000, 1536)],
              "bf16": [(n, k) for n in (1, 63, 65, 257) for k in (8, 40, 104, 1536)] + [(9000, 1536)]}
MISSED_BY_RANDN = {"bf16_w2_last_k16"}


def _randn_check_fails(name):
    """Does today's randn tolerance check reject the mutated emulator on any of its shapes?"""
    path, dirs, rule = PP.MUTATIONS[name]
    bf16 = path == "bf16"
    rng = np.random.default_rng(1)
    for n, k in RANDN_DIMS[path]:
        X = rng.standard_normal((n, k)).astype(np.float32)
        X = PP.bf16_trunc(X) if bf16 else X
        W = (rng.standard_normal((D, k)) / k ** 0.5).astype(np.float32)
        b = rng.standard_normal(D).astype(np.float32)
        dY = rng.standard_normal((n, D)).astype(np.float32)
        X64 = X.astype(np.float64)
        if "fwd" in dirs:
            Y = PP.emulate_fwd(X, W, b, 0, bf16, rule)
            if not np.allclose(Y, X64 @ W.T.astype(np.float64) + b, rtol=1e-4, atol=1e-4):
                return True
        if "wgrad" in dirs:
            dW = PP.emulate_wgrad(X, dY, 0, bf16, rule)
            if not np.allclose(dW, dY.T.astype(np.float64) @ X64, rtol=1e-4, atol=1e-4 * n ** 0.5):
                return True
    return False


def test_randn_tolerance_check_misses_what_the_probes_catch():
    """The unmutated emulator passes the randn check; of the mutations, exactly MISSED_BY_RANDN pass it too."""
    missed = {name for name in PP.MUTATIONS if not _randn_check_fails(name)}
    assert missed == MISSED_BY_RANDN
    none = {"none": ("f32", ("fwd", "wgrad"), None), "none_bf16": ("bf16", ("fwd", "wgrad"), None)}
    saved = dict(PP.MUTATIONS)
    try:
        PP.MUTATIONS.update(none)
        assert not _randn_check_fails("none") and not _randn_check_fails("none_bf16")
    finally:
        PP.MUTATIONS.clear()
        PP.MUTATIONS.update(saved)


def test_precondition_rejects_sums_past_2_to_24_units():
    """A dot product of 800 tf32 probe pairs (about 800 x 6.25 x 2^12 > 2^24 units of 2^-12) is refused; 256 pairs (the forward's
    row cap) are accepted."""
    rng = np.random.default_rng(2)
    for nnz, ok in ((256, True), (800, False)):
        X, W = PP.probe("tf32", rng, (1, nnz)), PP.probe("tf32", rng, (1, nnz))
        if ok:
            PP.expected(PP.term_pairs(X, W, 0), PP.fwd)
        else:
            with pytest.raises(ValueError, match="probe precondition"):
                PP.expected(PP.term_pairs(X, W, 0), PP.fwd)
    with pytest.raises(ValueError, match="probe precondition"):      # a bf16 column of 60 nonzeros at unit 2^-17
        X = PP.probe("int", rng, (60, 1))
        PP.expected(PP.term_pairs(X, PP.probe("bf16", rng, (60, 4)), 0), PP.wgrad)


def test_probe_splits_are_the_closed_form():
    """The kernels' split rules give the closed-form parts for every sign and digit (probe() asserts it), and the int probes survive
    the int8 table format unchanged."""
    rng = np.random.default_rng(4)
    for kind in ("tf32", "bf16", "int", "coarse"):
        PP.probe(kind, rng, (64, 64))
    import torch
    from llmrec_b200 import feat_int8 as F8
    X = PP.probe("int", rng, (100, 48), PP.pattern(100, 48, 12, 12))
    T = F8.quantize(torch.from_numpy(X.value))
    assert torch.equal(F8.dequantize(T, 48), torch.from_numpy(X.value))
