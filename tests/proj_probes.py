"""Term-exact probe operands for the projection kernels (proj_tc.cu, proj_simt.cu), their expected values, and a CPU emulator of
the tensor-core main loop.

A probe is an operand pair whose every product term is exact, whose split inside the kernel is known in closed form, and whose
every partial sum is exact in fp32.  Then a correct kernel returns ONE fp32 value per output, in any accumulation order and under
any rounding or alignment rule that keeps 24 bits, and a term that is dropped, duplicated or paired with the wrong operand changes it.

Values (s = +-1, a in {2, 3}, c, c1, c2 in {1, 2, 3}):
  tf32    s (a + c 2^-12)                tf32_hi = s a, lo = s c 2^-12, both TF32-exact.  The fp32 tables in modes 0 and 1.
  bf16    s (a + c1 2^-8 + c2 2^-17)     bf16_split3 = (s a, s c1 2^-8, s c2 2^-17).  W / dY beside a bf16 or int8 table.
  int     s c                            bf16-exact (and int8-exact: dequantize(quantize(X)) == X).  bf16 / int8 tables.
  coarse  s (a + c 2^-6)                 x w exact in fp32: the SIMT kernels (mode 2, shapes the tensor cores refuse).
The expected value of an output is the exact (fp64) sum of the terms the kernel forms, from the closed-form split:
  fp32 mode 0   sum (lo hi + hi lo + hi hi) + b      -- not the exact dot product: lo lo is not formed
  fp32 mode 1   sum hi hi + b
  bf16 mode 0   sum x (w0 + w1 + w2) + b = the exact sum;   mode 1: sum x w0 + b
  SIMT          sum x w + b
`expected` refuses (ValueError) any case where some output's sum of |terms| (bias and prior included) reaches 2^24 units, the unit
being a power of two that divides every term."""
import numpy as np

STAGE = {"f32": 32, "bf16": 64}       # k (forward) / rows (weight gradient) per pipeline stage
STEP = {"f32": 8, "bf16": 16}         # k per wgmma: k8 (tf32), k16 (bf16)


# ---- the kernels' operand rules, restated (tc_common.cuh) ------------------------------------------------------------------------
def tf32_hi(x):
    """Top 19 bits of fp32 x (sign, exponent, 10 mantissa bits): truncation, as tf32_hi in the kernels."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def bf16_trunc(x):
    x = np.ascontiguousarray(x, dtype=np.float32)
    return (x.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def bf16_split3(v):
    """v -> (w0, w1, w2), bf16-exact, w0 + w1 + w2 = v: bf16_split3 in the kernels."""
    v = np.asarray(v, dtype=np.float32)
    h = bf16_trunc(v)
    r = (v - h).astype(np.float32)
    m = bf16_trunc(r)
    return h, m, bf16_trunc((r - m).astype(np.float32))


# ---- probe values with their closed-form split -----------------------------------------------------------------------------------
class Probe:
    """An operand: `value` (fp32, as the caller passes it), `parts` (its split terms in fp64, by construction: (hi, lo) for tf32,
    (w0, w1, w2) for bf16, (value,) for int and coarse), `full` (the value in fp64) and `units` (a power of two dividing every entry of
    each part).  `to(f)` maps parts and full (to a torch device, say): `expected` then runs there."""

    def __init__(self, kind, value, parts, full, units):
        self.kind, self.value, self.parts, self.full, self.units = kind, value, parts, full, units

    def to(self, f):
        return Probe(self.kind, self.value, tuple(f(p) for p in self.parts), f(self.full), self.units)


def _digits(rng, shape):
    return rng.choice([-1.0, 1.0], shape), rng.integers(2, 4, shape).astype(np.float64), rng.integers(1, 4, shape).astype(np.float64)


def probe(kind, rng, shape, mask=None):
    """Probe values of `kind` ("tf32", "bf16", "int", "coarse"); zero where mask is False.  Checks that the kernels' split of every
    value is the closed form."""
    s, a, c = _digits(rng, shape)
    if mask is not None:
        s = np.where(mask, s, 0.0)
    if kind == "tf32":
        parts = (s * a, s * c * 2.0 ** -12)
    elif kind == "bf16":
        parts = (s * a, s * c * 2.0 ** -8, s * rng.integers(1, 4, shape) * 2.0 ** -17)
    elif kind == "int":
        parts = (s * c,)
    elif kind == "coarse":
        parts = (s * (a + c * 2.0 ** -6),)
    else:
        raise ValueError(kind)
    full = sum(parts)
    value = full.astype(np.float32)
    assert np.array_equal(value.astype(np.float64), full), "probe value is not fp32-exact"
    if kind == "tf32":
        hi = tf32_hi(value)
        assert np.array_equal(hi, parts[0]) and np.array_equal(value - hi, parts[1]) and np.array_equal(tf32_hi(value - hi), parts[1])
    elif kind == "bf16":
        assert all(np.array_equal(w, e) for w, e in zip(bf16_split3(value), parts))
    elif kind == "int":
        assert np.array_equal(bf16_trunc(value), value)
    return Probe(kind, value, parts, full, tuple(_unit(p) for p in parts))


def pattern(n, k, row_cap, col_cap, shift=0):
    """Sparsity of X [n x k]: X[r, c] != 0 iff (r + c + shift) % q == 0, q the smallest period that keeps at most row_cap nonzeros in
    a row and col_cap in a column.  When q <= k every row has a nonzero and every column does when q <= n: every k position of every
    stage, every row of every tile (both consumer warpgroups, every m64 block), and in the weight gradient every dY row meets an x."""
    q = max(1, -(-k // row_cap), -(-n // col_cap))
    r, c = np.arange(n)[:, None], np.arange(k)[None, :]
    return (r + c + shift) % q == 0


# per table probe kind: (X kind, W / dY kind in modes 0 and 1, nonzeros per X row / column); mode 2 (SIMT) takes "coarse" W / dY
KINDS = {"f32": ("tf32", "tf32", 256), "bf16": ("int", "bf16", 12), "i8": ("int", "bf16", 12), "f32_simt": ("coarse", "coarse", 256),
         "bf16_simt": ("int", "coarse", 256)}


# ---- expected values ---------------------------------------------------------------------------------------------------------------
def _unit(x):
    """Largest power of two dividing every nonzero entry of x (fp64); inf for an all-zero x."""
    v = np.abs(np.asarray(x, np.float64))
    v = v[v != 0]
    if v.size == 0:
        return np.inf
    m, e = np.frexp(v)
    mi = (m * 2.0 ** 53).astype(np.int64)
    low = (mi & -mi).astype(np.float64)
    return float(np.min(np.ldexp(low, e - 53)))


def term_pairs(x, w, mode):
    """[(x part, its unit, w part, its unit)] for every product the kernel forms.  x: the table's probe (tf32, int or coarse); w: the
    fp32 operand's (W in the forward, dY in the weight gradient)."""
    if mode == 2 or w.kind == "coarse":
        return [(x.full, min(x.units), w.full, min(w.units))]
    if w.kind == "tf32":
        (xh, xl), (wh, wl) = x.parts, w.parts
        (uxh, uxl), (uwh, uwl) = x.units, w.units
        return [(xl, uxl, wh, uwh), (xh, uxh, wl, uwl), (xh, uxh, wh, uwh)] if mode == 0 else [(xh, uxh, wh, uwh)]
    if w.kind == "bf16":
        (xv,), (w0, w1, w2), (ux,) = x.parts, w.parts, x.units
        pairs = [(xv, ux, w2, w.units[2]), (xv, ux, w1, w.units[1]), (xv, ux, w0, w.units[0])]
        return pairs if mode == 0 else pairs[2:]
    raise ValueError(w.kind)


def _f32(t):
    return t.astype(np.float32) if isinstance(t, np.ndarray) else t.float()


def _f64(t):
    return t.astype(np.float64) if isinstance(t, np.ndarray) else t.double()


def expected(pairs, contract, extras=()):
    """fp32 result of sum over pairs of contract(x part, w part) plus the extras ((array, unit): bias, prior dW), exact in fp64 (numpy
    arrays or torch tensors).  Raises ValueError unless every output's sum of |terms| stays below 2^24 units, so that every fp32
    partial sum of the terms, in any order, is exact."""
    total = sum(contract(a, b) for a, _, b, _ in pairs)
    bound = sum(contract(abs(a), abs(b)) for a, _, b, _ in pairs)
    unit = min(ua * ub for _, ua, _, ub in pairs)
    for e, ue in extras:
        total, bound, unit = total + e, bound + abs(e), min(unit, ue)
    if unit == np.inf:
        unit = 1.0
    worst = float(bound.max()) if min(bound.shape, default=1) > 0 else 0.0
    if worst >= 2.0 ** 24 * unit:
        raise ValueError(f"probe precondition: sum |terms| = 2^{np.log2(worst / unit):.2f} units of 2^{np.log2(unit):.0f}, not below 2^24")
    out = _f32(total)
    assert bool((_f64(out) == total).all()), "an exact fp32 sum is not exact"
    return out


def fwd(a, b):            # Y [n x d] = X [n x k] W [d x k]^T
    return a @ b.T


def wgrad(a, b):          # dW [d x k] = dY [n x d]^T X [n x k]
    return b.T @ a


def colsum_exact(dy, n_rows):
    """db = colsum(dY) [d] when n_rows max|dY| stays below 2^24 units of dY (exact in any order), else None."""
    v = dy.full
    if v.shape[0] == 0:
        return _f32(v.sum(0))
    if n_rows * float(abs(v).max()) >= 2.0 ** 24 * min(dy.units):
        return None
    return _f32(v.sum(0))


# ---- CPU emulator of the tensor-core main loop ---------------------------------------------------------------------------------------
def _split_terms(A, B, mode, bf16):
    """Operands as the wgmmas read them, in issue order: [(name, A part, B part)].  A = the table side (X, or X^T), B = the fp32 side
    (W, or dY^T); the tensor cores read a TF32 operand's top 19 bits."""
    if bf16:
        if mode == 1:
            return [("x*w0", A, bf16_trunc(B))]
        w0, w1, w2 = bf16_split3(B)
        return [("x*w2", A, w2), ("x*w1", A, w1), ("x*w0", A, w0)]
    ah, bh = tf32_hi(A), tf32_hi(B)
    if mode == 1:
        return [("hi*hi", ah, bh)]
    al, bl = tf32_hi(A - ah), tf32_hi(B - bh)
    return [("lo*hi", al, bh), ("hi*lo", ah, bl), ("hi*hi", ah, bh)]


def emulate_unit(A, B, mode, bf16, mutation=None):
    """out [M x N] = A [M x K] B [N x K]^T as one work unit of the kernel: K in stages of 32 (bf16: 64), each stage in k8 (k16)
    steps, one wgmma per term per step whose exact product sum is rounded to fp32 and added to the fp32 accumulator.
    mutation(term, stage, kk, last_stage) -> None, "drop", or "shift" (the term pairs A column j with B column j + 1)."""
    A, B = np.asarray(A, np.float32), np.asarray(B, np.float32)
    path = "bf16" if bf16 else "f32"
    st, step = STAGE[path], STEP[path]
    K = A.shape[1]
    kp = -(-K // st) * st
    A = np.pad(A, ((0, 0), (0, kp - K)))
    B = np.pad(B, ((0, 0), (0, kp - K + 1)))          # one zero column past the end for "shift"
    terms = _split_terms(A, B, mode, bf16)
    acc = np.zeros((A.shape[0], B.shape[0]), np.float32)
    n_st = kp // st
    for s in range(n_st):
        for kk in range(st // step):
            j = s * st + kk * step
            for name, a, b in terms:
                m = mutation(name, s, kk, n_st - 1) if mutation else None
                if m == "drop":
                    continue
                o = 1 if m == "shift" else 0
                acc = (acc + (a[:, j:j + step].astype(np.float64) @ b[:, j + o:j + o + step].astype(np.float64).T).astype(np.float32)).astype(np.float32)
    return acc


def emulate_fwd(X, W, bias, mode, bf16=False, mutation=None):
    Y = emulate_unit(X, W, mode, bf16, mutation)
    return Y if bias is None else (Y + np.asarray(bias, np.float32)[None, :]).astype(np.float32)


def rows_per_chunk(n):   # wg_rows_per_chunk in proj_tc.cu
    r = 2048
    while r > 256 and n // r < 4:
        r //= 2
    return r


def emulate_wgrad(X, dY, mode, bf16=False, mutation=None, prior=None):
    """dW [d x k]: one unit per row chunk (A = X^T, B = dY^T over the chunk's rows), the chunk partials summed in fp32 as the reduce
    kernel does (four interleaved slices, combined pairwise), then the prior under accumulate."""
    X, dY = np.asarray(X, np.float32), np.asarray(dY, np.float32)
    n = X.shape[0]
    rpc = rows_per_chunk(n)
    sl = [np.zeros((dY.shape[1], X.shape[1]), np.float32) for _ in range(4)]
    for i, r0 in enumerate(range(0, n, rpc)):
        part = emulate_unit(X[r0:r0 + rpc].T, dY[r0:r0 + rpc].T, mode, bf16, mutation)   # [k x d]
        sl[i % 4] = (sl[i % 4] + part.T).astype(np.float32)
    dW = ((sl[0] + sl[1]).astype(np.float32) + (sl[2] + sl[3]).astype(np.float32)).astype(np.float32)
    return dW if prior is None else (dW + np.asarray(prior, np.float32)).astype(np.float32)


# The kernel defects the probes must catch (tests/test_proj_probes_cpu.py), as emulator mutations: (table path, directions, rule).
MUTATIONS = {
    # the lo*hi wgmma skipped at k8 step kk = 3 of every stage
    "drop_lohi_kk3": ("f32", ("fwd", "wgrad"), lambda t, s, kk, last: "drop" if t == "lo*hi" and kk == 3 else None),
    # the hi*lo wgmma skipped on the unit's last stage
    "drop_hilo_last_stage": ("f32", ("fwd", "wgrad"), lambda t, s, kk, last: "drop" if t == "hi*lo" and s == last else None),
    # lo*hi of one k8 step (stage 0, kk = 1) pairs x_k with w_{k+1}
    "pair_shift_lohi": ("f32", ("fwd", "wgrad"), lambda t, s, kk, last: "shift" if t == "lo*hi" and s == 0 and kk == 1 else None),
    # the bf16 X*w2 wgmma missing on the unit's last k16 step
    "bf16_w2_last_k16": ("bf16", ("fwd", "wgrad"), lambda t, s, kk, last: "drop" if t == "x*w2" and s == last and kk == 3 else None),
    # the weight-gradient builder's lo tile zero past row 16 of a stage: hi*lo loses stage rows 16..31 (k8 steps 2 and 3)
    "builder_lo_rows16": ("f32", ("wgrad",), lambda t, s, kk, last: "drop" if t == "hi*lo" and kk >= 2 else None),
}
