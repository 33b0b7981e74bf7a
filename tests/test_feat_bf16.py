"""CPU checks of --feat_dtype: the flag, the bf16 feature buffers of MM_Model (rounding, parameter parity, bytes) and the
projection byte counts of roofline."""
import numpy as np
import pytest
import torch


def _args(*extra):
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility.parser import parse_args
    return set_args(parse_args(["--debug"] + list(extra)))


def test_flag_default_and_choices():
    from llmrec_b200.utility.parser import parse_args
    assert parse_args([]).feat_dtype == "fp32"
    assert parse_args(["--feat_dtype", "bf16"]).feat_dtype == "bf16"
    with pytest.raises(SystemExit):
        parse_args(["--feat_dtype", "fp16"])


def _inputs(seed=0):
    rng = np.random.default_rng(seed)
    nu, ni = 37, 53
    f = lambda n, k: (rng.standard_normal((n, k)) * 3.0).astype(np.float32)
    return nu, ni, f(ni, 32), f(ni, 64), f(nu, 96), {"title": f(ni, 96), "genre": f(ni, 96), "year": f(ni, 96)}


def _model(feat_dtype):
    from llmrec_b200.Models import MM_Model
    _args("--feat_dtype", feat_dtype, "--embed_size", "32")
    nu, ni, img, txt, usr, att = _inputs()
    torch.manual_seed(2022)
    m = MM_Model(nu, ni, 32, [32, 32], [0.1, 0.1], img, txt, usr, att)
    return m, (img, txt, usr, att)


def _feature_buffers(m):
    return [m.image_feats, m.text_feats, m.user_feats] + [m.item_feats[k] for k in m._item_keys]


def test_bf16_buffers_are_rne_rounding_of_the_inputs():
    m, (img, txt, usr, att) = _model("bf16")
    raw = [img, txt, usr] + [att[k] for k in m._item_keys]
    for buf, x in zip(_feature_buffers(m), raw):
        assert buf.dtype == torch.bfloat16 and buf.is_contiguous()
        assert torch.equal(buf, torch.from_numpy(x).to(torch.bfloat16))
        # round-to-nearest-even by hand on the bits: add 0x7fff + lsb, drop the low half
        b = torch.from_numpy(x).view(torch.int32).to(torch.int64) & 0xffffffff
        rne = ((b + 0x7fff + ((b >> 16) & 1)) >> 16) << 16
        want = torch.from_numpy(rne.to(torch.int64).numpy().astype(np.uint32).view(np.float32))
        assert torch.equal(buf.float(), want)


def test_bf16_parameters_are_bit_identical_to_fp32_construction():
    a, _ = _model("fp32")
    b, _ = _model("bf16")
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert pa.keys() == pb.keys()
    for k in pa:
        assert pa[k].dtype == torch.float32 and torch.equal(pa[k], pb[k]), k
    for buf in _feature_buffers(a):
        assert buf.dtype == torch.float32


def test_bf16_feature_bytes_are_exactly_half():
    a, _ = _model("fp32")
    b, _ = _model("bf16")
    nbytes = lambda m: sum(t.numel() * t.element_size() for t in _feature_buffers(m))
    assert nbytes(a) == 2 * nbytes(b) > 0


def test_roofline_proj_bytes_by_element_size():
    from llmrec_b200.roofline import proj_bytes
    n, k, d = 17366, 1536, 64
    assert proj_bytes(n, k, d) == proj_bytes(n, k, d, 4) == 4 * n * k + 4 * k * d + 4 * n * d
    assert proj_bytes(n, k, d, 2) == 2 * n * k + 4 * k * d + 4 * n * d
