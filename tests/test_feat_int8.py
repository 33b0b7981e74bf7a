"""CPU checks of --feat_dtype int8: the flag, the row-scaled int8 table format of feat_int8 (exponent choice, rounding, clamps,
layout, exactness in bf16, idempotence), MM_Model's int8 buffers and the roofline byte counts."""
import numpy as np
import pytest
import torch

from llmrec_b200 import feat_int8 as F8


def _args(*extra):
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility.parser import parse_args
    return set_args(parse_args(["--debug"] + list(extra)))


def test_flag_choices():
    from llmrec_b200.utility.parser import parse_args
    assert parse_args([]).feat_dtype == "fp32"
    assert parse_args(["--feat_dtype", "int8"]).feat_dtype == "int8"
    assert parse_args(["--feat_dtype", "bf16"]).feat_dtype == "bf16"
    with pytest.raises(SystemExit):
        parse_args(["--feat_dtype", "fp16"])


def _rows(seed=0, n=64, k=40):
    rng = np.random.default_rng(seed)
    mag = 2.0 ** rng.integers(-20, 20, size=(n, 1))
    return (rng.standard_normal((n, k)) * mag).astype(np.float32)


def _exp(T, k):
    return torch.log2(F8.scales(T, k)).round().long()


def test_layout_and_padding():
    for k in (1, 15, 16, 17, 40, 512, 1536):
        x = _rows(k, n=9, k=k)
        T = F8.quantize(x)
        assert T.dtype == torch.int8 and T.is_contiguous() and tuple(T.shape) == (9, F8.pitch(k))
        assert F8.pitch(k) % 16 == 0 and F8.pitch(k) == (k + 15) // 16 * 16 + 16 and F8.k_capacity(F8.pitch(k)) >= k
        s = F8.scale_offset(k)
        assert (T[:, k:s] == 0).all() and (T[:, s + 4:] == 0).all()
        assert F8.nbytes(T) == 9 * F8.pitch(k)


def test_smallest_exponent_and_error_bound():
    x = _rows(1, n=256, k=96)
    T = F8.quantize(x)
    k = x.shape[1]
    q = T[:, :k].long()
    e = _exp(T, k)
    qmax = q.abs().max(1).values
    assert ((qmax >= 64) & (qmax <= 127)).all()                     # smallest e (no row is clamped here): max|x| > 127 * 2^(e-1)
    m = torch.from_numpy(np.abs(x).max(1)).double()
    assert (m <= 127.0 * torch.pow(2.0, e.double())).all() and (m > 127.0 * torch.pow(2.0, e.double() - 1)).all()
    xt = F8.dequantize(T, k).double()
    err = (torch.from_numpy(x).double() - xt).abs()
    assert (err <= torch.pow(2.0, e.double() - 1)[:, None]).all()


def test_round_half_even_on_exact_ties():
    # scale 2^0 (max 100 -> e = 0): 0.5 -> 0, 1.5 -> 2, 2.5 -> 2, -0.5 -> 0, -1.5 -> -2, -3.5 -> -4
    x = np.array([[100.0, 0.5, 1.5, 2.5, -0.5, -1.5, -3.5, 3.5]], dtype=np.float32)
    T = F8.quantize(x)
    assert float(F8.scales(T, 8)[0]) == 1.0
    assert T[0, :8].tolist() == [100, 0, 2, 2, 0, -2, -4, 4]


def test_zero_rows_and_clamps():
    tiny = np.full((1, 16), 3.0 * 2.0 ** -124, dtype=np.float32)   # would want e = -130: clamped to -126, q = 12
    vanish = np.full((1, 16), 1e-40, dtype=np.float32)             # subnormal: rounds to q = 0 at 2^-126 -> an all-zero row
    big = np.full((1, 16), 2.0 ** 126, dtype=np.float32)            # 2^126 <= 127 * 2^120
    x = np.concatenate([np.zeros((1, 16), np.float32), tiny, vanish, big])
    T = F8.quantize(x)
    sc = F8.scales(T, 16)
    assert float(sc[0]) == 1.0 and (T[0, :16] == 0).all()
    assert float(sc[1]) == 2.0 ** -126 and (T[1, :16] == 12).all()
    assert float(sc[2]) == 1.0 and (T[2, :16] == 0).all()
    assert float(sc[3]) == 2.0 ** 120 and (T[3, :16] == 64).all()
    assert torch.equal(F8.quantize(F8.dequantize(T, 16)), T)
    with pytest.raises(ValueError):
        F8.quantize(np.full((1, 4), 2.0 ** 127 * 1.5, dtype=np.float32))   # needs e > 120
    for bad in (np.nan, np.inf, -np.inf):
        y = np.ones((2, 4), np.float32)
        y[1, 2] = bad
        with pytest.raises(ValueError):
            F8.quantize(y)


def test_dequantized_values_are_exact_bf16_and_quantize_is_idempotent():
    x = np.concatenate([_rows(2, n=200, k=48), np.zeros((1, 48), np.float32), np.full((1, 48), 3e-39, np.float32)])
    T = F8.quantize(x)
    xf = F8.dequantize(T, 48)
    xb = F8.dequantize(T, 48, torch.bfloat16)
    assert torch.equal(xb.float(), xf) and torch.equal(xf.bfloat16().float(), xf)
    assert torch.equal(F8.quantize(xf), T) and torch.equal(F8.quantize(xb), T)
    assert torch.equal(F8.quantize(xf.numpy()), T)


def _inputs(seed=0):
    rng = np.random.default_rng(seed)
    nu, ni = 37, 53
    f = lambda n, k: (rng.standard_normal((n, k)) * 3.0).astype(np.float32)
    return nu, ni, f(ni, 32), f(ni, 64), f(nu, 96), {"title": f(ni, 40), "genre": f(ni, 40), "year": f(ni, 40)}


def _model(feat_dtype):
    from llmrec_b200.Models import MM_Model
    _args("--feat_dtype", feat_dtype, "--embed_size", "32")
    nu, ni, img, txt, usr, att = _inputs()
    torch.manual_seed(2022)
    m = MM_Model(nu, ni, 32, [32, 32], [0.1, 0.1], img, txt, usr, att)
    return m, (img, txt, usr, att)


def _feature_buffers(m):
    return [m.image_feats, m.text_feats, m.user_feats] + [m.item_feats[k] for k in m._item_keys]


def test_int8_buffers_are_the_quantized_inputs():
    m, (img, txt, usr, att) = _model("int8")
    raw = [img, txt, usr] + [att[k] for k in m._item_keys]
    for buf, x in zip(_feature_buffers(m), raw):
        assert buf.dtype == torch.int8 and buf.is_contiguous() and buf.shape[1] == F8.pitch(x.shape[1])
        assert torch.equal(buf, F8.quantize(x))


def test_int8_parameters_are_bit_identical_to_fp32_construction():
    a, _ = _model("fp32")
    b, _ = _model("int8")
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert pa.keys() == pb.keys()
    for k in pa:
        assert pa[k].dtype == torch.float32 and torch.equal(pa[k], pb[k]), k


def test_int8_feature_bytes():
    a, (img, txt, usr, att) = _model("fp32")
    b, _ = _model("int8")
    nbytes = lambda m: sum(t.numel() * t.element_size() for t in _feature_buffers(m))
    want = sum(x.shape[0] * F8.pitch(x.shape[1]) for x in [img, txt, usr] + list(att.values()))
    assert nbytes(b) == want
    assert nbytes(b) < nbytes(a) / 2


def test_roofline_int8_bytes():
    from types import SimpleNamespace

    from llmrec_b200.roofline import proj_bytes, step_bytes
    n, k, d = 17366, 1536, 64
    assert proj_bytes(n, k, d, 1) == n * k + 4 * n + 4 * k * d + 4 * n * d
    assert proj_bytes(n, k, d, 2) == 2 * n * k + 4 * k * d + 4 * n * d
    # step_bytes takes k from the weights, not from the int8 row pitch
    m, (img, txt, usr, att) = _model("int8")
    p = {name: prm.data for name, prm in m.named_parameters()}
    feats = dict(image=m.image_feats, text=m.text_feats, user=m.user_feats, item=m.item_feats)
    hp = SimpleNamespace(nu=37, ni=53, d=32, S=2 + len(att), L=2, has_feats=True, feats=feats, p=p, keys=list(att),
                         opt=SimpleNamespace(params=list(p.values())), demand_fuse=False)
    got = step_bytes(hp, nnz=100)
    want = sum(proj_bytes(53, x.shape[1], 32, 1) for x in [img, txt] + list(att.values())) + proj_bytes(37, usr.shape[1], 32, 1)
    assert got["proj_fwd"] == got["proj_wgrad"] == want
