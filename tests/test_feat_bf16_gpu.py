"""-m gpu: bf16 side-feature tables (--feat_dtype bf16).

The bf16 projection kernels must compute what the fp32 kernels compute on the upcast table: the 3-way bf16 split of W / dY
loses no product term, so mode 0 is held to fp64 of the upcast table at fp32-class accuracy; mode 1 rounds W / dY to bf16 on
the tensor cores; shapes the tensor-core path does not take run the SIMT kernel, bit-identical to the fp32 SIMT kernel on the
upcast table.  Then the whole engine: a bf16 run on a dataset whose features are already bf16 values equals the fp32 run on it."""
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
TOL = {0: 1e-4, 1: 3e-2}      # mode 0: fp32-class; mode 1: W / dY truncated to bf16 (2^-8 relative per product on average)
SMS = 132                     # H100 SXM
TINY_FLAGS = ["--batch_size", "128", "--epoch", "1", "--debug", "--seed", "2022"]


def _gen(seed):
    return torch.Generator(device=cuda).manual_seed(seed)


def _ld(t):
    from llmrec_b200 import ops
    return ops._ld(t)


def _table(g, n, k, lead=8, pad=8, positive=False):
    """bf16 X[n x k] as a column slice of a wider bf16 table: ld = lead + k + pad (a multiple of 8 for k % 8 == 0), the slice
    starting 16 bytes into its row."""
    shape = (n, lead + k + pad)
    T = 1.0 + torch.rand(shape, generator=g, device=cuda) if positive else torch.randn(shape, generator=g, device=cuda)
    return T.to(torch.bfloat16)[:, lead:lead + k]


def _assert_tc(d, X, out):
    """The operands satisfy the bf16 tensor-core preconditions, so no case tests the SIMT fallback instead."""
    assert d % 32 == 0 and 32 <= d <= 256 and X.dtype == torch.bfloat16
    assert X.shape[1] % 8 == 0 and _ld(X) % 8 == 0 and X.data_ptr() % 16 == 0
    assert _ld(out) % 4 == 0 and out.data_ptr() % 16 == 0


def _rows_per_chunk(n):   # wg_rows_per_chunk in proj_tc.cu
    r = 2048
    while r > 256 and n // r < 4:
        r //= 2
    return r


def _uses_256_wide_tiles(dims):
    fwd = sum(-(-n // 256) for n, _ in dims)
    wg = sum(-(-k // 256) * -(-n // _rows_per_chunk(n)) for n, k in dims)
    return fwd >= SMS and wg >= SMS


# ------------------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------------------
SMALL = [(n, k) for n in (1, 63, 65, 257) for k in (8, 40, 104, 1536)]          # 16 problems, k % 64 != 0 included
BIG = [(9000, 1536)] * 4 + [(8001, 104), (9001, 40), (7777, 8)]                 # >= 132 units at 256 wide


def _projection_case(dims, d, mode, seed):
    """Forward and weight gradient against fp64 of the upcast table, strided outputs framed by NaN, then a second call that
    reuses the split buffers, rings and colsum ticket and must give the same bits."""
    from llmrec_b200 import ops
    g = _gen(seed)
    Xs = [_table(g, n, k) for n, k in dims]
    Ws = [torch.randn(d, k, generator=g, device=cuda) / k ** 0.5 for _, k in dims]
    bs = [torch.randn(d, generator=g, device=cuda) for _ in dims]
    wides = [torch.full((n, 3 * d), NAN, device=cuda) for n, _ in dims]
    Ys = [w[:, d:2 * d] for w in wides]
    for X, Y in zip(Xs, Ys):
        _assert_tc(d, X, Y)
    ops.proj_fwd_group(list(zip(Xs, Ws, bs, Ys)), d, mode)
    tol = TOL[mode]
    for (n, k), X, W, b, Y, wide in zip(dims, Xs, Ws, bs, Ys, wides):
        torch.testing.assert_close(Y.double(), X.double() @ W.double().t() + b.double(), rtol=tol, atol=tol, msg=lambda m: f"fwd n={n} k={k}: {m}")
        assert bool(wide[:, :d].isnan().all() and wide[:, 2 * d:].isnan().all()), f"fwd n={n} k={k} wrote outside its view"
    first = [Y.clone() for Y in Ys]
    ops.proj_fwd_group(list(zip(Xs, Ws, bs, Ys)), d, mode)
    assert all(torch.equal(a, Y) for a, Y in zip(first, Ys)), "second forward call differs"

    dYs = [torch.randn(n, 3 * d, generator=g, device=cuda)[:, d:2 * d] for n, _ in dims]
    runs = []
    for _ in range(2):
        dWs = [torch.full((d, k), NAN, device=cuda) for _, k in dims]
        dbs = [torch.full((d,), NAN, device=cuda) for _ in dims]
        for X, dY in zip(Xs, dYs):
            _assert_tc(d, X, dY)
        ops.proj_wgrad_group(list(zip(Xs, dYs, dWs, dbs, [False] * len(dims))), d, mode)
        runs.append((dWs, dbs))
    for (n, k), X, dY, dW, db, dW2, db2 in zip(dims, Xs, dYs, *runs[0], *runs[1]):
        torch.testing.assert_close(dW.double(), dY.double().t() @ X.double(), rtol=tol, atol=tol * n ** 0.5, msg=lambda m: f"wgrad n={n} k={k}: {m}")
        torch.testing.assert_close(db.double(), dY.double().sum(0), rtol=1e-4, atol=1e-4 * n ** 0.5, msg=lambda m: f"db n={n} k={k}: {m}")
        assert torch.equal(dW, dW2) and torch.equal(db, db2), f"second wgrad call differs n={n} k={k}"


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("d", WIDTHS)
def test_bf16_projection_every_width_mode_and_tile(d, mode):
    """128-wide tiles on small problems (n = 1 .. 257, k = 8 .. 1536 with ragged last 64-wide k-blocks), then a group large enough
    for 256-wide tiles at d <= 128, forward and weight gradient against fp64 of the upcast table."""
    _projection_case(SMALL[:8], d, mode, seed=10 * d + mode)
    _projection_case(SMALL[8:], d, mode, seed=10 * d + mode + 1)
    assert _uses_256_wide_tiles(BIG)
    _projection_case(BIG, d, mode, seed=10 * d + mode + 2)


def _max_rel(got, ref):
    return float(((got.double() - ref) / ref).abs().max())


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("d", WIDTHS)
def test_bf16_precision_fingerprint(d, mode, capsys):
    """All operands in [1, 2), so nothing cancels.  Mode 0 drops no product term (X is exact, W / dY = t0 + t1 + t2 exactly):
    within 5e-5 of fp64, and not the SIMT bits.  Mode 1 truncates W / dY to bf16 (8 significand bits, ~2.6e-3 relative on
    average for values in [1, 2)): its error must lie in (1e-3, 1e-2), which proves W / dY were rounded to bf16 on the tensor cores."""
    from llmrec_b200 import ops
    g = _gen(d + mode)
    n, k = 256, 256
    X = _table(g, n, k, positive=True)
    W = 1.0 + torch.rand(d, k, generator=g, device=cuda)
    dY = (1.0 + torch.rand(n, 3 * d, generator=g, device=cuda))[:, d:2 * d]
    Y = torch.empty(n, d, device=cuda)
    _assert_tc(d, X, Y)
    _assert_tc(d, X, dY)
    ops.proj_fwd_group([(X, W, None, Y)], d, mode)
    dW, db = torch.empty(d, k, device=cuda), torch.empty(d, device=cuda)
    ops.proj_wgrad_group([(X, dY, dW, db, False)], d, mode)
    fwd = _max_rel(Y, X.double() @ W.double().t())
    wg = _max_rel(dW, dY.double().t() @ X.double())
    with capsys.disabled():
        print(f"\nbf16 fingerprint d={d} mode={mode}: fwd max rel {fwd:.3e}, wgrad max rel {wg:.3e}")
    assert _max_rel(db, dY.double().sum(0)) < 5e-5
    if mode == 0:
        assert fwd < 5e-5 and wg < 5e-5, (fwd, wg)
        Y2, dW2 = torch.empty_like(Y), torch.empty_like(dW)
        ops.proj_fwd_group([(X, W, None, Y2)], d, 2)
        ops.proj_wgrad_group([(X, dY, dW2, None, False)], d, 2)
        assert not torch.equal(Y, Y2) and not torch.equal(dW, dW2)
    else:
        assert 1e-3 < fwd < 1e-2 and 1e-3 < wg < 1e-2, (fwd, wg)


NETFLIX = [("image", 17366, 512), ("text", 17366, 768)] + [(f"att{j}", 17366, 1536) for j in range(5)] + [("user", 13187, 1536)]


def test_bf16_grouped_netflix_shaped_launch():
    """The 8 projections of a netflix-shaped step in one grouped call at d = 64, mode 0: five attribute tables sharing item_trans
    (W, dW and db; accumulate F,T,T,T,T).  Against fp64; two weight-gradient runs from the same prior are bitwise equal; an empty
    problem in the group gives the same bits as the group without it."""
    from llmrec_b200 import ops
    d, g = 64, _gen(7)
    X = {name: _table(g, n, k) for name, n, k in NETFLIX}
    W = {"image": torch.randn(d, 512, generator=g, device=cuda) / 512 ** 0.5, "text": torch.randn(d, 768, generator=g, device=cuda) / 768 ** 0.5,
         "item": torch.randn(d, 1536, generator=g, device=cuda) / 1536 ** 0.5, "user": torch.randn(d, 1536, generator=g, device=cuda) / 1536 ** 0.5}
    wk = lambda name: "item" if name.startswith("att") else name
    b = {key: torch.randn(d, generator=g, device=cuda) for key in W}
    Y = {name: torch.full((n, d), NAN, device=cuda) for name, n, _ in NETFLIX}
    probs = [(X[name], W[wk(name)], b[wk(name)], Y[name]) for name, _, _ in NETFLIX]
    ops.proj_fwd_group(probs, d, 0)
    for name, _, _ in NETFLIX:
        torch.testing.assert_close(Y[name].double(), X[name].double() @ W[wk(name)].double().t() + b[wk(name)].double(), rtol=1e-4, atol=1e-4)
    E = _table(g, 300, 1536)[:0]
    Ye = torch.empty(0, d, device=cuda)
    Y2 = {name: torch.empty_like(Y[name]) for name in Y}
    ops.proj_fwd_group([(X[name], W[wk(name)], b[wk(name)], Y2[name]) for name, _, _ in NETFLIX[:4]] + [(E, W["item"], b["item"], Ye)]
                       + [(X[name], W[wk(name)], b[wk(name)], Y2[name]) for name, _, _ in NETFLIX[4:7]], d, 0)
    ops.proj_fwd_group([(X["user"], W["user"], b["user"], Y2["user"])], d, 0)
    for name in Y:
        assert torch.equal(Y[name], Y2[name]), name

    dY = {name: torch.randn(n, d, generator=g, device=cuda) for name, n, _ in NETFLIX}
    prior = {key: (torch.randn(d, W[key].shape[1], generator=g, device=cuda), torch.randn(d, generator=g, device=cuda)) for key in W}

    def wgrad(with_empty):
        out = {key: (p[0].clone(), p[1].clone()) for key, p in prior.items()}
        atts = [name for name, _, _ in NETFLIX if name.startswith("att")]
        probs = [(X[name], dY[name], *out["item"], j > 0) for j, name in enumerate(atts)]
        if with_empty:
            probs.insert(2, (E, torch.empty(0, d, device=cuda), *out["item"], True))
        probs += [(X["user"], dY["user"], *out["user"], False), (X["text"], dY["text"], *out["text"], False),
                  (X["image"], dY["image"], *out["image"], False)]
        ops.proj_wgrad_group(probs, d, 0)
        return out

    r1, r2, r3 = wgrad(False), wgrad(False), wgrad(True)
    for key in W:
        assert torch.equal(r1[key][0], r2[key][0]) and torch.equal(r1[key][1], r2[key][1]), f"{key}: weight gradient not reproducible"
        assert torch.equal(r1[key][0], r3[key][0]) and torch.equal(r1[key][1], r3[key][1]), f"{key}: an empty problem changed the bits"
    members = {"item": [f"att{j}" for j in range(5)], "user": ["user"], "text": ["text"], "image": ["image"]}
    for key, names in members.items():
        refW = sum(dY[nm].double().t() @ X[nm].double() for nm in names)
        refb = sum(dY[nm].double().sum(0) for nm in names)
        n = sum(X[nm].shape[0] for nm in names)
        torch.testing.assert_close(r1[key][0].double(), refW, rtol=1e-4, atol=1e-4 * n ** 0.5)
        torch.testing.assert_close(r1[key][1].double(), refb, rtol=1e-4, atol=1e-4 * n ** 0.5)


FALLBACKS = [("k % 8 != 0", 64, 36, 0), ("d = 48", 48, 104, 0), ("mode 2", 64, 104, 2)]


@pytest.mark.parametrize("case", [c[0] for c in FALLBACKS])
def test_bf16_fallbacks_equal_fp32_simt_on_upcast_table(case):
    """Shapes the bf16 tensor-core path does not take (k % 8 != 0, d not a multiple of 32) and mode 2 run the SIMT kernel with X
    widened on load: bit-identical to the fp32 SIMT kernel on the upcast table.  The weight gradient is too at n <= 1024 (one row
    chunk); above that the SIMT kernel's atomics across chunks may round differently, so n = 3000 is held to fp64 instead."""
    from llmrec_b200 import ops
    _, d, k, mode = next(c for c in FALLBACKS if c[0] == case)
    g = _gen(d + k + mode)
    for n in (1, 700, 1024, 3000):
        X = _table(g, n, k, lead=4, pad=4)
        Xf = X.float()
        W = torch.randn(d, k, generator=g, device=cuda) / k ** 0.5
        b = torch.randn(d, generator=g, device=cuda)
        Y, Yf = torch.empty(n, d, device=cuda), torch.empty(n, d, device=cuda)
        ops.proj_fwd_group([(X, W, b, Y)], d, mode)
        ops.proj_fwd_group([(Xf, W, b, Yf)], d, 2)
        assert torch.equal(Y, Yf), (case, n)
        dY = torch.randn(n, 2 * d, generator=g, device=cuda)[:, :d]
        dW, db, dWf, dbf = torch.empty(d, k, device=cuda), torch.empty(d, device=cuda), torch.empty(d, k, device=cuda), torch.empty(d, device=cuda)
        ops.proj_wgrad_group([(X, dY, dW, db, False)], d, mode)
        ops.proj_wgrad_group([(Xf, dY, dWf, dbf, False)], d, 2)
        if n <= 1024:
            assert torch.equal(dW, dWf) and torch.equal(db, dbf), (case, n)
        else:
            torch.testing.assert_close(dW.double(), dY.double().t() @ Xf.double(), rtol=1e-4, atol=1e-4 * n ** 0.5)
            torch.testing.assert_close(db.double(), dY.double().sum(0), rtol=1e-4, atol=1e-4 * n ** 0.5)


def test_bf16_mixed_or_wrong_dtypes_are_rejected():
    from llmrec_b200 import ops
    d, g = 64, _gen(3)
    X, Xf = _table(g, 100, 64), torch.randn(100, 64, device=cuda)
    W, b, Y = torch.randn(d, 64, device=cuda), torch.randn(d, device=cuda), torch.empty(100, d, device=cuda)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(X, W, b, Y), (Xf, W, b, Y)], d, 0)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(X, W.bfloat16(), b, Y)], d, 0)
    with pytest.raises(ValueError):
        ops.proj_fwd_group([(X, W, b, Y.bfloat16())], d, 0)
    dY, dW = torch.randn(100, d, device=cuda), torch.empty(d, 64, device=cuda)
    with pytest.raises(ValueError):
        ops.proj_wgrad_group([(X, dY.bfloat16(), dW, None, False)], d, 0)
    with pytest.raises(ValueError):
        ops.proj_wgrad_group([(Xf, dY, dW, None, False), (X, dY, dW, None, True)], d, 0)


# ------------------------------------------------------------------------------------------------------------------------------
# the engine
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def rounded_root(tiny_root, tmp_path_factory):
    """A copy of the tiny dataset whose feature tables hold bf16 values (RNE-rounded, stored as fp32): --feat_dtype bf16 on it
    keeps exactly the values the fp32 run reads."""
    root = str(tmp_path_factory.mktemp("tiny_bf16")) + "/"
    src = os.path.join(tiny_root, "netflix_valid_item")
    dst = os.path.join(root, "netflix_valid_item")
    shutil.copytree(src, dst)
    rnd = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(torch.bfloat16).float().numpy()
    for name in ("image_feat.npy", "text_feat.npy"):
        np.save(os.path.join(dst, name), rnd(np.load(os.path.join(src, name))))
    path = os.path.join(dst, "augmented_user_init_embedding")
    with open(path, "rb") as f:
        usr = pickle.load(f)
    with open(path, "wb") as f:
        pickle.dump(rnd(usr), f)
    path = os.path.join(dst, "augmented_atttribute_embedding_dict")
    with open(path, "rb") as f:
        att = pickle.load(f)
    with open(path, "wb") as f:
        pickle.dump({k: rnd(v) for k, v in att.items()}, f)
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


def _step(tr, u, p, n, i):
    torch.cuda.manual_seed(1000 + i)          # both trainers draw from the one CUDA generator (dropout masks)
    return float(tr.train_batch(u, p, n))


def _assert_same_run(a, b, gen, steps):
    from llmrec_b200.utility import batch_test
    for i in range(steps):
        u, p, n = a.sample_batch()
        la, lb = _step(a, u, p, n, i), _step(b, u, p, n, i)
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
def test_bf16_engine_matches_fp32_on_rounded_tables(rounded_root, engine):
    """--feat_dtype bf16 against fp32 on the pre-rounded dataset, same init and the same batches (their lengths vary with the
    augmented edges) for 6 steps: losses, parameters, the eval forward and test() metrics agree to fp32 reassociation level.
    The hoisted engine's propagated tables TU / TI are bit-identical: the one-time SpMMs read the same values."""
    flags = {"default_eager": ["--cuda_graph", "0"], "default_graph": ["--cuda_graph", "1"],
             "hoisted_graph": ["--cuda_graph", "1", "--hoist_side", "1"]}[engine]
    a, gen, M = _trainer(rounded_root, flags)
    b, _, _ = _trainer(rounded_root, flags + ["--feat_dtype", "bf16"])
    assert all(t.dtype == torch.bfloat16 for t in _feature_buffers(b.model_mm))
    for ta, tb in zip(_feature_buffers(a.model_mm), _feature_buffers(b.model_mm)):
        assert torch.equal(ta, tb.float())
    if engine == "hoisted_graph":
        assert b.hoisted and torch.equal(a.hot.TU, b.hot.TU) and torch.equal(a.hot.TI, b.hot.TI)
    M.set_seed(5)
    _assert_same_run(a, b, gen, 6)


def test_bf16_dropout_step_matches_fp32(rounded_root):
    """--drop_rate 0.2 (the eager masked-branch step, dropout on the projections only) takes bf16 tables as well."""
    a, gen, M = _trainer(rounded_root, ["--drop_rate", "0.2"])
    b, _, _ = _trainer(rounded_root, ["--drop_rate", "0.2", "--feat_dtype", "bf16"])
    assert a.masked_mode and b.masked_mode
    M.set_seed(6)
    _assert_same_run(a, b, gen, 1)


def test_bf16_plumbing(rounded_root, monkeypatch):
    """On the device the tables are bf16 at half the bytes; a bf16 step launches as many library kernels as an fp32 step (no
    per-step conversion) and reaches the projections through the _bf16 entry points only; the default run stays on _f32."""
    from llmrec_b200 import _native as N
    from llmrec_b200 import ops
    a, gen, M = _trainer(rounded_root, ["--cuda_graph", "0"])
    b, _, _ = _trainer(rounded_root, ["--cuda_graph", "0", "--feat_dtype", "bf16"])
    fa, fb = _feature_buffers(a.model_mm), _feature_buffers(b.model_mm)
    assert all(t.is_cuda and t.dtype == torch.float32 for t in fa) and all(t.is_cuda and t.dtype == torch.bfloat16 for t in fb)
    assert sum(t.numel() * t.element_size() for t in fa) == 2 * sum(t.numel() * t.element_size() for t in fb)
    lib = N.lib()
    calls = {}
    for name in ("llmrec_proj_fwd_group_f32", "llmrec_proj_wgrad_group_f32", "llmrec_proj_fwd_group_bf16", "llmrec_proj_wgrad_group_bf16"):
        fn = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *args, _fn=fn, _n=name: (calls.__setitem__(_n, calls.get(_n, 0) + 1), _fn(*args))[1])
    M.set_seed(8)
    u, p, n = a.sample_batch()
    launches = []
    for tr in (a, b):
        calls.clear()
        l0 = ops.STATS["launches"]
        tr.train_batch(u, p, n)
        torch.cuda.synchronize()
        launches.append(ops.STATS["launches"] - l0)
        seen = dict(calls)
        if tr is a:
            assert seen.get("llmrec_proj_fwd_group_f32") and seen.get("llmrec_proj_wgrad_group_f32"), seen
            assert not seen.get("llmrec_proj_fwd_group_bf16") and not seen.get("llmrec_proj_wgrad_group_bf16"), seen
        else:
            assert seen.get("llmrec_proj_fwd_group_bf16") and seen.get("llmrec_proj_wgrad_group_bf16"), seen
            assert not seen.get("llmrec_proj_fwd_group_f32") and not seen.get("llmrec_proj_wgrad_group_f32"), seen
    assert launches[0] == launches[1] > 0, launches


@pytest.mark.parametrize("flags", [["--mask", "1"], ["--mask_rate", "0.1"]])
def test_bf16_with_mask_branch_raises(rounded_root, flags):
    with pytest.raises(ValueError, match="feat_dtype bf16"):
        _trainer(rounded_root, ["--feat_dtype", "bf16"] + flags)
