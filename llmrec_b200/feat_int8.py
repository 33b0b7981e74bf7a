"""The int8 side-feature table format (--feat_dtype int8; include/llmrec_b200.h, the _i8 projection entry points).

A table of n rows and logical width k is ONE contiguous int8 tensor [n x P], P = pitch(k) = roundup(k, 16) + 16.  Row r holds
    bytes [0, k)                    the int8 values q (|q| <= 127),
    bytes [k, roundup(k, 16))       zero,
    bytes [roundup(k, 16), +4)      the row's fp32 scale 2^e,
    the rest of the row             zero.
The scale lives inside the row, so everything that moves rows (the live-item compaction X[live], row maps, TMA boxes) keeps working
on one tensor; P is a multiple of 16, a legal TMA row stride.

Every stored value q * 2^e is exactly a bf16 number (at most 7 significant bits, a normal fp32 for e in [-126, 120]), so an int8
table is a lossless 2x compression of one bf16 table X~ = dequantize(table): the projection kernels compute exactly what the bf16
kernels compute on X~.  This module is the only code that knows the layout.
"""
from __future__ import annotations

import numpy as np
import torch

E_MIN, E_MAX = -126, 120          # scale exponents: every non-zero q * 2^e stays a normal fp32 (and an exact bf16)
Q_MAX = 127


def scale_offset(k: int) -> int:
    """Byte offset of a row's scale: roundup(k, 16)."""
    return (int(k) + 15) // 16 * 16


def pitch(k: int) -> int:
    """Row pitch in bytes of a table of logical width k."""
    return scale_offset(k) + 16


def k_capacity(p: int) -> int:
    """The largest logical width a row pitch p holds (k itself is fixed by the weights that read the table: any k in
    (k_capacity - 16, k_capacity] has this pitch)."""
    if p < 16 or p % 16:
        raise ValueError(f"not an int8 table row pitch: {p}")
    return p - 16


def _exponents(m: np.ndarray) -> np.ndarray:
    """Smallest integer e with m <= 127 * 2^e, per row (m = max |x| > 0, fp64 holding fp32 values): exact, through frexp."""
    _, E = np.frexp(m)                                   # m = f 2^E, f in [0.5, 1): 127 * 2^(E-8) < m < 2^E
    e = E.astype(np.int64) - 7
    return np.where(m <= np.ldexp(float(Q_MAX), e), e, e + 1)


def quantize(x) -> torch.Tensor:
    """fp32 / bf16 [n x k] (tensor or array) -> int8 table [n x pitch(k)] on x's device (CPU for arrays).
    Per row: e = the smallest integer with max|x| <= 127 * 2^e, clamped below at -126; q = round_half_even(x * 2^-e) (the
    multiplication is exact); a row whose q are all zero (an all-zero row, or a clamped one that rounds to zero) gets scale 1.
    Raises ValueError on non-finite input or on a row that would need e > 120.  Draws no random numbers.
    quantize(dequantize(T)) == T byte for byte."""
    t = torch.as_tensor(x)
    dev = t.device
    a = t.detach().to("cpu", torch.float32).numpy().astype(np.float64)
    if a.ndim != 2:
        raise ValueError(f"quantize: need a 2-D table, got shape {tuple(a.shape)}")
    n, k = a.shape
    if not np.isfinite(a).all():
        raise ValueError("quantize: the table holds non-finite values")
    m = np.abs(a).max(axis=1) if k else np.zeros(n)
    nz = m > 0
    e = np.zeros(n, dtype=np.int64)
    e[nz] = _exponents(m[nz])
    if (e > E_MAX).any():
        raise ValueError(f"quantize: row {int(np.argmax(e > E_MAX))} needs a scale above 2^{E_MAX} (max |x| too large)")
    e = np.maximum(e, E_MIN)
    q = np.rint(np.ldexp(a, -e[:, None]))                 # exact scaling; rint rounds half to even
    e[~(q != 0).any(axis=1)] = 0                          # a row that is all zero in q (a clamped tiny row too): scale 1, as its dequantization
    out = np.zeros((n, pitch(k)), dtype=np.int8)
    out[:, :k] = q.astype(np.int8)
    s = scale_offset(k)
    out[:, s:s + 4] = np.ldexp(np.ones(n, dtype=np.float32), e.astype(np.int32)).astype(np.float32).view(np.int8).reshape(n, 4)
    return torch.empty(out.shape, dtype=torch.int8, device=dev).copy_(torch.from_numpy(out))   # row-major strides even when empty


def scales(T: torch.Tensor, k: int) -> torch.Tensor:
    """fp32 [n] row scales of an int8 table of logical width k."""
    s = scale_offset(k)
    raw = torch.empty((T.shape[0], 4), dtype=torch.int8, device=T.device).copy_(T[:, s:s + 4])   # row-major even when empty
    return raw.view(torch.float32).reshape(-1)


def dequantize(T: torch.Tensor, k: int, dtype=torch.float32) -> torch.Tensor:
    """int8 table of logical width k -> [n x k] table of q * 2^e in fp32 or bf16 (exact in both)."""
    if T.dtype != torch.int8 or T.dim() != 2 or T.shape[1] != pitch(k):
        raise ValueError(f"dequantize: need an int8 [n x {pitch(k)}] table for k = {k}, got {tuple(T.shape)} {T.dtype}")
    x = T[:, :k].float() * scales(T, k)[:, None]
    return x.to(dtype)


def nbytes(T: torch.Tensor) -> int:
    """Bytes of an int8 table, scales and padding included."""
    return T.numel() * T.element_size()
