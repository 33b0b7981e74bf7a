"""Elementwise fp64 bounds shared by the exactness tests: the check that records each family's largest error / bound ratio, and
one AdamW step in fp64 with its bound (tests/test_step_tail_exactness_gpu.py derives it; tests/test_step_sequence_fp64_gpu.py holds
whole runs of training steps to it).  TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np
import torch

U = 2.0 ** -24
RATIOS = {}                       # family -> largest error / bound ratio seen by `check`


def ratio_of(got, y, bound):
    err = np.abs(np.asarray(got, np.float64) - y)
    return np.divide(err, bound, out=np.where(err == 0, 0.0, np.inf), where=bound > 0)


def passes(got, y, bound):
    """every element within its bound (a NaN fails)"""
    return bool(np.all(ratio_of(got, y, bound) <= 1.0))


def check(got, y, bound, family, what=""):
    got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    y, bound = np.broadcast_to(y, got.shape), np.broadcast_to(bound, got.shape)
    assert np.isfinite(got).all(), f"{what}: {int((~np.isfinite(got)).sum())} non-finite outputs (unwritten, or a NaN row was read)"
    ratio = ratio_of(got, y, bound)
    RATIOS[family] = max(RATIOS.get(family, 0.0), float(ratio.max(initial=0.0)))
    if ratio.size and ratio.max() > 1.0:
        k = np.unravel_index(np.argmax(ratio), ratio.shape)
        raise AssertionError(f"{what}: {int((ratio > 1).sum())} elements beyond the fp64 bound; worst at {k}: got {got[k]!r}, "
                             f"want {y[k]!r}, error {abs(got[k] - y[k]):.3g} > bound {bound[k]:.3g}")


def adamw_ref(p, g, m, v, t, lr, b1, b2, eps, wd):
    """one AdamW step in fp64 from fp32 state -> [(p', bound), (m', bound), (v', bound)]"""
    f = lambda z: float(np.float32(z))
    b1f, b2f, epsf = f(b1), f(b2), f(eps)
    decay = 1.0 - f(lr) * f(wd)
    step, bc2s = lr / (1.0 - b1 ** t), math.sqrt(1.0 - b2 ** t)
    p, g, m, v = (a.astype(np.float64) for a in (p, g, m, v))
    p1 = p * decay
    m1 = m + (1 - b1f) * (g - m)
    v1 = v * b2f + (1 - b2f) * g * g
    den = np.sqrt(v1) / bc2s + epsf
    upd = step * m1 / den
    p2 = p1 - upd
    bm = 8 * U * (np.abs(m) + (1 - b1f) * (np.abs(g) + np.abs(m)))
    bv = 8 * U * (v * b2f + (1 - b2f) * g * g)
    bp = 2 * U * (2 * np.abs(p1) + np.abs(p2)) + step / den * bm + 24 * U * np.abs(upd)
    return [(p2, bp), (m1, bm), (v1, bv)]



def state_ok(st, t, lr, b1, b2):
    """the device's step size lr / (1 - b1^t) and sqrt(1 - b2^t) against Python's, to a few double ulp of pow, amplified by the
    cancellation in 1 - b^t"""
    e = 2.0 ** -52
    ok1 = abs(st[1] - lr / (1 - b1 ** t)) <= st[1] * 4 * e * (b1 ** t / (1 - b1 ** t) + 2)
    ok2 = abs(st[2] - math.sqrt(1 - b2 ** t)) <= st[2] * 4 * e * (b2 ** t / (1 - b2 ** t) + 2)
    return ok1 and ok2
