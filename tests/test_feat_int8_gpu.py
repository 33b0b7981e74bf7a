"""-m gpu: int8 side-feature tables (--feat_dtype int8).

An int8 table (llmrec_b200/feat_int8.py) encodes the bf16 table X~ = dequantize(table) exactly, and the _i8 projection entry points
must give the BITS of the _bf16 entry points on X~: the tensor-core kernels expand q * 2^e to bf16 in shared memory, in the layout the
bf16 TMA load writes, before the unchanged bf16 consumers; the SIMT kernels widen q * 2^e on load.  Then the whole engine: on a dataset
whose features already hold X~, --feat_dtype int8 trains like --feat_dtype bf16 (and the hoisted engine like fp32)."""
import os
import pickle
import shutil

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

cuda = torch.device("cuda")
NAN = float("nan")
WIDTHS = [32, 64, 96, 128, 160, 192, 224, 256]
TINY_FLAGS = ["--batch_size", "128", "--epoch", "1", "--debug", "--seed", "2022"]


def _gen(seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def _tables(g, n, k, spread=True):
    """-> (int8 table [n x pitch(k)], the bf16 table X~ it encodes [n x k]) on the device.  Rows of very different magnitudes, a
    zero row when n > 2."""
    from llmrec_b200 import feat_int8 as F8
    x = torch.randn(n, k, generator=g, device=cuda)
    if spread:
        x = x * torch.pow(2.0, torch.randint(-12, 12, (n, 1), generator=g, device=cuda).float())
    if n > 2:
        x[n // 2] = 0
    T = F8.quantize(x)
    return T, F8.dequantize(T, k, torch.bfloat16)


def _equal(a, b):
    return a.shape == b.shape and torch.equal(a, b)


def _fwd_pair(Ts, Xbs, Ws, bs, d, mode, rows=None, m=None):
    from llmrec_b200 import ops
    outs = []
    for Xs in (Ts, Xbs):
        Ys = [torch.full((m[i] if m else X.shape[0], 3 * d), NAN, device=cuda)[:, d:2 * d] for i, X in enumerate(Xs)]
        probs = [(X, W, b, Y) + ((rows[i],) if rows else ()) for i, (X, W, b, Y) in enumerate(zip(Xs, Ws, bs, Ys))]
        ops.proj_fwd_group(probs, d, mode)
        outs.append(Ys)
    return outs


def _wgrad_pair(Ts, Xbs, dYs, d, mode, acc=None, prior=None, rows=None):
    from llmrec_b200 import ops
    outs = []
    for Xs in (Ts, Xbs):
        dWs = [prior[i][0].clone() if prior else torch.full((d, Xbs[i].shape[1]), NAN, device=cuda) for i in range(len(Xs))]
        dbs = [(prior[i][1].clone() if prior else torch.full((d,), NAN, device=cuda)) for i in range(len(Xs))]
        probs = [(X, dY, dW, db, acc[i] if acc else False) + ((rows[i],) if rows else ())
                 for i, (X, dY, dW, db) in enumerate(zip(Xs, dYs, dWs, dbs))]
        ops.proj_wgrad_group(probs, d, mode)
        outs.append((dWs, dbs))
    return outs


def _check_case(dims, d, mode, seed):
    g = _gen(seed)
    pairs = [_tables(g, n, k) for n, k in dims]
    Ts, Xbs = [p[0] for p in pairs], [p[1] for p in pairs]
    Ws = [torch.randn(d, k, generator=g, device=cuda) / k ** 0.5 for _, k in dims]
    bs = [torch.randn(d, generator=g, device=cuda) for _ in dims]
    Yi, Yb = _fwd_pair(Ts, Xbs, Ws, bs, d, mode)
    for (n, k), a, b in zip(dims, Yi, Yb):
        assert _equal(a, b), f"fwd d={d} mode={mode} n={n} k={k}: max diff {float((a - b).abs().max()) if a.numel() else 0}"
    dYs = [torch.randn(n, 2 * d, generator=g, device=cuda)[:, :d] for n, _ in dims]
    (dWi, dbi), (dWb, dbb) = _wgrad_pair(Ts, Xbs, dYs, d, mode)
    for (n, k), a, b, c, e in zip(dims, dWi, dWb, dbi, dbb):
        assert _equal(a, b), f"wgrad d={d} mode={mode} n={n} k={k}: max diff {float((a - b).abs().max())}"
        assert _equal(c, e), f"db d={d} mode={mode} n={n} k={k}"


# n: 1, tile - 1 / tile / tile + 1 for the 128- and 256-row tiles, not multiples of either; k: one and several 64-wide stages, ragged
SMALL = [(1, 16), (127, 48), (128, 64), (129, 80), (255, 112), (256, 1536), (257, 208), (1000, 512)]
BIG = [(9000, 1536)] * 4 + [(8001, 112), (9001, 48), (7777, 16)]                 # >= 132 units at 256 wide: 256-row / feature tiles


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("d", WIDTHS)
def test_int8_projection_bit_identical_to_bf16_on_dequantized_table(d, mode):
    """Forward Y, weight gradient dW and bias gradient db of int8 tables equal the bf16 entry points on X~, bit for bit, at every
    width and mode, on 128-wide tiles (small n) and on a group large enough for 256-wide tiles at d <= 128."""
    _check_case(SMALL, d, mode, seed=10 * d + mode)
    if mode != 2:
        _check_case(BIG, d, mode, seed=10 * d + mode + 1)


def test_int8_empty_problem_and_row_maps_and_accumulate():
    from llmrec_b200 import feat_int8 as F8
    d, g = 64, _gen(5)
    dims = [(300, 128), (0, 128), (1000, 64)]
    pairs = [_tables(g, n, k) for n, k in dims]
    Ts, Xbs = [p[0] for p in pairs], [p[1] for p in pairs]
    assert Ts[1].shape == (0, F8.pitch(128))
    Ws = [torch.randn(d, k, generator=g, device=cuda) for _, k in dims]
    bs = [torch.randn(d, generator=g, device=cuda) for _ in dims]
    # row maps: X row r -> Y row rows[r] of a taller output
    m = [700, 5, 1500]
    rows = [torch.randperm(mm, generator=torch.Generator().manual_seed(i))[:n].to(cuda, torch.int32) for i, ((n, _), mm) in enumerate(zip(dims, m))]
    Yi, Yb = _fwd_pair(Ts, Xbs, Ws, bs, d, 0, rows=rows, m=m)
    for a, b in zip(Yi, Yb):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))
    dYs = [torch.randn(mm, d, generator=g, device=cuda) for mm in m]
    prior = [(torch.randn(d, k, generator=g, device=cuda), torch.randn(d, generator=g, device=cuda)) for _, k in dims]
    for acc in ([False] * 3, [True] * 3):
        (dWi, dbi), (dWb, dbb) = _wgrad_pair(Ts, Xbs, dYs, d, 0, acc=acc, prior=prior, rows=rows)
        for a, b, c, e in zip(dWi, dWb, dbi, dbb):
            assert torch.equal(a, b) and torch.equal(c, e)


NETFLIX = [("image", 17366, 512), ("text", 17366, 768)] + [(f"att{j}", 17366, 1536) for j in range(5)] + [("user", 13187, 1536)]


def test_int8_grouped_netflix_shaped_launch():
    """The 8 projections of a netflix-shaped step in one grouped call at d = 64 in modes 0 and 1: five attribute tables sharing
    item_trans (W, dW and db; accumulate F,T,T,T,T), bit-identical to the bf16 call on X~."""
    d, g = 64, _gen(7)
    pairs = {name: _tables(g, n, k, spread=False) for name, n, k in NETFLIX}
    W = {"image": torch.randn(d, 512, generator=g, device=cuda) / 512 ** 0.5, "text": torch.randn(d, 768, generator=g, device=cuda) / 768 ** 0.5,
         "item": torch.randn(d, 1536, generator=g, device=cuda) / 1536 ** 0.5, "user": torch.randn(d, 1536, generator=g, device=cuda) / 1536 ** 0.5}
    wk = lambda name: "item" if name.startswith("att") else name
    b = {key: torch.randn(d, generator=g, device=cuda) for key in W}
    dY = {name: torch.randn(n, d, generator=g, device=cuda) for name, n, _ in NETFLIX}
    from llmrec_b200 import ops
    for mode in (0, 1):
        res = []
        for which in (0, 1):
            X = {name: pairs[name][which] for name in pairs}
            Y = {name: torch.empty(n, d, device=cuda) for name, n, _ in NETFLIX}
            ops.proj_fwd_group([(X[name], W[wk(name)], b[wk(name)], Y[name]) for name, _, _ in NETFLIX], d, mode)
            out = {key: (torch.empty(d, W[key].shape[1], device=cuda), torch.empty(d, device=cuda)) for key in W}
            atts = [name for name, _, _ in NETFLIX if name.startswith("att")]
            probs = [(X[name], dY[name], *out["item"], j > 0) for j, name in enumerate(atts)]
            probs += [(X["user"], dY["user"], *out["user"], False), (X["text"], dY["text"], *out["text"], False),
                      (X["image"], dY["image"], *out["image"], False)]
            ops.proj_wgrad_group(probs, d, mode)
            res.append((Y, out))
        for name in res[0][0]:
            assert torch.equal(res[0][0][name], res[1][0][name]), (mode, name)
        for key in W:
            assert torch.equal(res[0][1][key][0], res[1][1][key][0]) and torch.equal(res[0][1][key][1], res[1][1][key][1]), (mode, key)


FALLBACKS = [("k % 16 != 0", 64, 40, 0), ("k % 16 != 0, mode 1", 128, 24, 1), ("d = 48", 48, 64, 0)]


@pytest.mark.parametrize("case", [c[0] for c in FALLBACKS])
def test_int8_simt_fallbacks_equal_bf16_simt(case):
    """Shapes the int8 tensor-core path does not take run the SIMT kernels, which widen q * 2^e on load: bit-identical to the bf16
    SIMT kernel (mode 2) on X~ -- the weight gradient at n <= 1024 (one row chunk; above, the chunks' atomics may round differently)."""
    _, d, k, mode = next(c for c in FALLBACKS if c[0] == case)
    g = _gen(d + k + mode)
    for n in (1, 700, 1024):
        T, Xb = _tables(g, n, k)
        from llmrec_b200 import ops
        W, b = torch.randn(d, k, generator=g, device=cuda), torch.randn(d, generator=g, device=cuda)
        Y, Yb = torch.empty(n, d, device=cuda), torch.empty(n, d, device=cuda)
        ops.proj_fwd_group([(T, W, b, Y)], d, mode)
        ops.proj_fwd_group([(Xb, W, b, Yb)], d, 2)
        assert torch.equal(Y, Yb), (case, n)
        dY = torch.randn(n, d, generator=g, device=cuda)
        dW, db, dWb, dbb = torch.empty(d, k, device=cuda), torch.empty(d, device=cuda), torch.empty(d, k, device=cuda), torch.empty(d, device=cuda)
        ops.proj_wgrad_group([(T, dY, dW, db, False)], d, mode)
        ops.proj_wgrad_group([(Xb, dY, dWb, dbb, False)], d, 2)
        assert torch.equal(dW, dWb) and torch.equal(db, dbb), (case, n)


def test_int8_dtype_and_pitch_rejections():
    from llmrec_b200 import ops
    d, g = 64, _gen(3)
    T, Xb = _tables(g, 100, 64)
    W, b, Y = torch.randn(d, 64, device=cuda), torch.randn(d, device=cuda), torch.empty(100, d, device=cuda)
    dY, dW = torch.randn(100, d, device=cuda), torch.empty(d, 64, device=cuda)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(T, W, b, Y), (Xb, W, b, Y)], d, 0)               # mixed group
    with pytest.raises(ValueError):
        ops.proj_wgrad_group([(T, dY, dW, None, False), (Xb.float(), dY, dW, None, True)], d, 0)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(T, W.bfloat16(), b, Y)], d, 0)                   # W, Y, dY must be fp32
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(T, W, b, Y.bfloat16())], d, 0)
    with pytest.raises(ValueError):
        ops.proj_wgrad_group([(T, dY.bfloat16(), dW, None, False)], d, 0)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(T[:, :64], W, b, Y)], d, 0)                      # a row without its scale: pitch != pitch(k)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(T, torch.randn(d, 32, device=cuda), b, Y)], d, 0)  # k = 32 has another pitch
    with pytest.raises(ValueError):
        ops.proj_wgrad_group([(T, dY, torch.empty(d, 80, device=cuda), None, False)], d, 0)


# ------------------------------------------------------------------------------------------------------------------------------
# the engine
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dequantized_root(tiny_root, tmp_path_factory):
    """A copy of the tiny dataset whose feature tables hold X~ = dequantize(quantize(x)) (stored as fp32): --feat_dtype int8 quantizes
    them back to the same bytes, --feat_dtype bf16 rounds them to themselves, and fp32 reads them as they are."""
    from llmrec_b200 import feat_int8 as F8
    root = str(tmp_path_factory.mktemp("tiny_i8")) + "/"
    src = os.path.join(tiny_root, "netflix_valid_item")
    dst = os.path.join(root, "netflix_valid_item")
    shutil.copytree(src, dst)

    def rnd(a):
        a = np.ascontiguousarray(a, dtype=np.float32)
        return F8.dequantize(F8.quantize(a), a.shape[1]).numpy()

    for name in ("image_feat.npy", "text_feat.npy"):
        np.save(os.path.join(dst, name), rnd(np.load(os.path.join(src, name))))
    path = os.path.join(dst, "augmented_user_init_embedding")
    with open(path, "rb") as f:
        usr = pickle.load(f)
    with open(path, "wb") as f:
        pickle.dump(rnd(np.array([usr[i] for i in range(len(usr))]) if not isinstance(usr, np.ndarray) else usr), f)
    path = os.path.join(dst, "augmented_atttribute_embedding_dict")
    with open(path, "rb") as f:
        att = pickle.load(f)
    with open(path, "wb") as f:
        pickle.dump({k: rnd(np.array([v[i] for i in range(len(v))]) if not isinstance(v, np.ndarray) else v) for k, v in att.items()}, f)
    return root


def _trainer(root, extra=()):
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir
    args = set_args(parse_args(["--data_path", root, "--dataset", "netflix"] + TINY_FLAGS + list(extra)))
    M.set_seed(args.seed)
    gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size, sampler=args.host_sampler)
    batch_test.init(gen, args)
    return M.Trainer(data_config={}, data_generator=gen), gen, M


def _feature_buffers(m):
    return [m.image_feats, m.text_feats, m.user_feats] + [m.item_feats[k] for k in m._item_keys]


def _assert_same_run(a, b, gen, steps):
    """The tolerances of the bf16 engine comparison (the loss heads' float atomics)."""
    from llmrec_b200.utility import batch_test
    for i in range(steps):
        u, p, n = a.sample_batch()
        torch.cuda.manual_seed(1000 + i)
        la = float(a.train_batch(u, p, n))
        torch.cuda.manual_seed(1000 + i)
        lb = float(b.train_batch(u, p, n))
        assert abs(la - lb) <= 2e-5 * max(1.0, abs(la)), (i, la, lb)
    sa, sb = a.model_mm.state_dict(), b.model_mm.state_dict()
    for k in sa:
        if not k.startswith("batch_norm"):
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-4, atol=1e-6, msg=k)
    Ua, Ia = (t.clone() for t in a.hot.forward())
    Ub, Ib = b.hot.forward()
    torch.testing.assert_close(Ub, Ua, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(Ib, Ia, rtol=1e-4, atol=1e-6)
    users = list(gen.test_set.keys())
    batch_test.init(gen, a.args)
    ra = a.test(users, False)
    batch_test.init(gen, b.args)
    rb = b.test(users, False)
    for key in ("recall", "ndcg"):
        assert abs(float(ra[key][1]) - float(rb[key][1])) <= 1e-4, (key, ra[key], rb[key])


@pytest.mark.parametrize("engine", ["default_eager", "default_graph", "hoisted_graph"])
def test_int8_engine_on_dequantized_tables(dequantized_root, engine):
    """--feat_dtype int8 against bf16 (default engine, eager and graphed) and against fp32 (hoisted engine, whose one-time products
    widen the int8 tables to the same fp32 values) on the X~ dataset, same init and batches, 6 steps."""
    from llmrec_b200 import feat_int8 as F8
    flags = {"default_eager": ["--cuda_graph", "0"], "default_graph": ["--cuda_graph", "1"],
             "hoisted_graph": ["--cuda_graph", "1", "--hoist_side", "1"]}[engine]
    ref_dtype = "fp32" if engine == "hoisted_graph" else "bf16"
    a, gen, M = _trainer(dequantized_root, flags + ["--feat_dtype", ref_dtype])
    b, _, _ = _trainer(dequantized_root, flags + ["--feat_dtype", "int8"])
    for ta, tb in zip(_feature_buffers(a.model_mm), _feature_buffers(b.model_mm)):
        assert tb.dtype == torch.int8 and torch.equal(ta.float(), F8.dequantize(tb, ta.shape[1]))
    if engine == "hoisted_graph":
        assert b.hoisted and torch.equal(a.hot.TU, b.hot.TU) and torch.equal(a.hot.TI, b.hot.TI)
    M.set_seed(5)
    _assert_same_run(a, b, gen, 6)


def test_int8_step_uses_the_i8_entry_points(dequantized_root, monkeypatch):
    from llmrec_b200 import _native as N
    b, gen, M = _trainer(dequantized_root, ["--cuda_graph", "0", "--feat_dtype", "int8"])
    lib = N.lib()
    calls = {}
    for name in ("llmrec_proj_fwd_group_f32", "llmrec_proj_wgrad_group_f32", "llmrec_proj_fwd_group_bf16", "llmrec_proj_wgrad_group_bf16",
                 "llmrec_proj_fwd_group_i8", "llmrec_proj_wgrad_group_i8"):
        fn = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *args, _fn=fn, _n=name: (calls.__setitem__(_n, calls.get(_n, 0) + 1), _fn(*args))[1])
    M.set_seed(8)
    u, p, n = b.sample_batch()
    b.train_batch(u, p, n)
    torch.cuda.synchronize()
    assert calls.get("llmrec_proj_fwd_group_i8") and calls.get("llmrec_proj_wgrad_group_i8"), calls
    assert set(calls) == {"llmrec_proj_fwd_group_i8", "llmrec_proj_wgrad_group_i8"}, calls


@pytest.mark.parametrize("flags", [["--mask", "1"], ["--mask_rate", "0.1"]])
def test_int8_with_mask_branch_raises(dequantized_root, flags):
    with pytest.raises(ValueError, match="feat_dtype int8"):
        _trainer(dequantized_root, ["--feat_dtype", "int8"] + flags)
