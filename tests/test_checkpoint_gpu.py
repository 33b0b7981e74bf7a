"""-m gpu: checkpoints on the real kernels (Trainer.save_checkpoint / load_checkpoint, --save_dir / --resume / --eval_only).

The experiment: run A takes N steps; run B takes k steps and saves, a FRESH Trainer resumes (a load before its first graph replay),
goes on to step k2 and saves again, takes two steps more, loads the second checkpoint into its live, already replayed graph, and
finishes.  With --deterministic 1 the parameters, AdamW moments, the fp64 step block and the device sampler state of A and B are
bit-identical, on the default and the hoisted engine, graph or eager, fp32 / bf16 / int8 tables, host or device sampler; the batches
of every step are identical with or without the flag.  Each configuration is executed once."""
import contextlib
import os
import re
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
cuda = torch.device("cuda")


@contextlib.contextmanager
def _flags(tiny_root, extra):
    """the process-wide args of a tiny run -> a function that builds Trainers under them (seeded like main(): seed, build, then --resume)"""
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir
    base = ["--data_path", tiny_root, "--dataset", "netflix", "--batch_size", "128", "--debug", "--lr", "0.001"] + extra

    def build(more=()):
        args = set_args(parse_args(base + list(more)))
        M.set_seed(args.seed)
        gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size, sampler=args.host_sampler)
        batch_test.init(gen, args)
        return M.Trainer(data_config={}, data_generator=gen)

    try:
        yield build
    finally:
        set_args(parse_args([]))


def _steps(tr, n, batches):
    for _ in range(n):
        tr.train_next_batch()
        g = tr.hot._gidx.cpu()                                  # the step's batch: rows users / pos / neg, row 3 = {B', n_keep}
        B = int(g[3, 0])
        batches.append((g[:3, :B].clone(), g[3, :2].clone()))


def _state(tr):
    torch.cuda.synchronize()
    s = {k: t.clone() for k, t in tr.hot.state_tensors().items()}
    if tr.device_sampler is not None:
        s["device_sampler"] = tr.device_sampler.state.clone()
    return s


def _ab(tiny_root, tmp_path, extra, N=10, k=3, k2=6):
    """-> (state, batches) of the uninterrupted run A and of the twice-restored run B"""
    ck1, ck2 = str(tmp_path / "k.pt"), str(tmp_path / "k2.pt")
    with _flags(tiny_root, extra) as build:
        a, ba = build(), []
        _steps(a, N, ba)
        sa = _state(a)
        b1, bb = build(), []
        _steps(b1, k, bb)
        b1.save_checkpoint(ck1)
        del b1
        b2 = build(["--resume", ck1])                           # loaded before the first replay: survives the warm-up step's undo
        ptrs = [t.data_ptr() for t in b2.hot.state_tensors().values()]
        _steps(b2, k2 - k, bb)
        b2.save_checkpoint(ck2)
        _steps(b2, 2, [])                                       # two steps that are thrown away
        b2.load_checkpoint(ck2)                                 # into the live graph, followed by more replays
        _steps(b2, N - k2, bb)
        assert [t.data_ptr() for t in b2.hot.state_tensors().values()] == ptrs, "a state tensor was rebound"
        return sa, ba, _state(b2), bb


def _same_batches(ba, bb):
    assert len(ba) == len(bb)
    for t, ((x, mx), (y, my)) in enumerate(zip(ba, bb)):
        assert torch.equal(mx, my) and torch.equal(x, y), f"the batch of step {t + 1} differs"


CONFIGS = [pytest.param(["--hoist_side", str(h), "--feat_dtype", f], id=f"{'hoisted' if h else 'default'}-{f}-graph") for h in (0, 1) for f in ("fp32", "bf16", "int8")]
CONFIGS += [pytest.param(["--hoist_side", str(h), "--cuda_graph", "0"], id=f"{'hoisted' if h else 'default'}-fp32-eager") for h in (0, 1)]
CONFIGS += [pytest.param(["--device_sampler", "1", "--cuda_graph", str(g)], id=f"default-fp32-device_sampler-{'graph' if g else 'eager'}") for g in (1, 0)]
CONFIGS += [pytest.param(["--host_sampler", "python"], id="default-fp32-python_sampler-graph")]


@pytest.mark.parametrize("extra", CONFIGS)
def test_restored_deterministic_run_is_bit_identical(tiny_root, tmp_path, extra):
    sa, ba, sb, bb = _ab(tiny_root, tmp_path, ["--deterministic", "1"] + extra)
    _same_batches(ba, bb)
    assert sa.keys() == sb.keys() and float(sa["state"][0]) == 10.0
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_restored_default_run_draws_the_same_batches_and_stays_within_the_run_to_run_spread(tiny_root, tmp_path):
    """Without --deterministic: the batches are integer work and still identical; the parameters of A and B differ by no more than
    8 x what two uninterrupted runs differ by (the float atomics' spread), with a floor of 1e-5 where that spread is ~0 -- a state
    that was not restored shows up at 1e-3 (lr x steps)."""
    sa, ba, sb, bb = _ab(tiny_root, tmp_path, [])
    _same_batches(ba, bb)
    with _flags(tiny_root, []) as build:
        a2, ba2 = build(), []
        _steps(a2, 10, ba2)
        sa2 = _state(a2)
    _same_batches(ba, ba2)
    assert torch.equal(sa["state"], sb["state"])
    for key in sa:
        if key.startswith("model/"):
            spread = float((sa[key] - sa2[key]).abs().max())
            diff = float((sa[key] - sb[key]).abs().max())
            assert diff <= max(8 * spread, 1e-5), (key, diff, spread)


@pytest.mark.parametrize("hoisted", [False, True], ids=["default", "hoisted"])
def test_netflix_shaped_restore_is_bit_identical(hoisted, tmp_path):
    """10 graph-replayed steps at the netflix shape against 5 steps, a save, a fresh engine, a load and 5 more"""
    sys.path.insert(0, HERE)
    import test_deterministic_gpu as D
    from llmrec_b200 import checkpoint
    sizes = (1126, 1030, 1, 1100, 1128, 513, 1127, 2, 1090, 1128)
    rng = np.random.default_rng(4)
    nu, ni = D.NETFLIX[:2]
    w = 1.0 / (np.arange(ni) + 8.0) ** 0.8
    i32 = lambda a: torch.from_numpy(a.astype(np.int32)).to(cuda)
    batches = [(i32(rng.integers(0, nu, B)), i32(rng.choice(ni, size=B, p=w / w.sum())), i32(rng.choice(ni, size=B, p=w / w.sum()))) for B in sizes]

    def run(hp, some):
        for u, p, n in some:
            hp.train_step_graphed(u, p, n)
        torch.cuda.synchronize()
        return hp

    a = run(D._engine(True, hoisted), batches)
    b1 = run(D._engine(True, hoisted), batches[:5])
    path = str(tmp_path / "n.pt")
    fp = dict(must=dict(n_users=nu, n_items=ni), recorded={})
    host = checkpoint.to_host(checkpoint.engine_tensors(b1))
    model, optim = checkpoint.engine_sections(host, b1.opt)
    loop = dict(epoch=0, batch=5, epoch_stats=torch.zeros(4), best_recall=0.0, stopping_step=0, test_ret=None, n_interactions=0)
    checkpoint.write(path, model, optim, checkpoint.rng_state(cuda), loop, fp)
    del b1
    b2 = D._engine(True, hoisted)
    _, saved, _ = checkpoint.read(path, fp, b2.state_tensors())
    b2.load_state(saved)
    run(b2, batches[5:])
    sa, sb = a.state_tensors(), b2.state_tensors()
    assert float(sa["state"][0]) == 10.0
    for key in sa:
        assert torch.equal(sa[key], sb[key]), key


def test_save_dir_adds_no_launch_and_no_synchronize_to_a_step(tiny_root, tmp_path, monkeypatch):
    from llmrec_b200 import ops
    counts = {}
    for name, extra in (("plain", []), ("saving", ["--save_dir", str(tmp_path / "ck")])):
        with _flags(tiny_root, ["--cuda_graph", "0"] + extra) as build:
            tr = build()
            tr.train_next_batch()                               # sizes the lazily allocated buffers
            n0 = ops.STATS["launches"]
            tr.train_next_batch()
            counts[name] = ops.STATS["launches"] - n0
            torch.cuda.synchronize()
    assert counts["plain"] == counts["saving"] > 0, counts
    with _flags(tiny_root, ["--save_dir", str(tmp_path / "ck")]) as build:
        tr = build()
        tr.train_next_batch()                                   # captures the graph
        torch.cuda.synchronize()
        syncs, real = [0], torch.cuda.synchronize
        monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: (syncs.__setitem__(0, syncs[0] + 1), real(*a, **k))[1])
        for _ in range(3):
            tr.train_next_batch()
        assert syncs[0] == 0
        tr.save_checkpoint(str(tmp_path / "ck" / "x.pt"))
        assert syncs[0] == 1, "saving synchronises once, for the device-to-host copies"
    assert sorted(os.listdir(tmp_path / "ck")) == ["x.pt"]      # steps alone wrote nothing


def _lines(logs):
    return [re.sub(r"\[[0-9.]+s( \+ [0-9.]+s)?\]", "[]", s) for s in logs if s.startswith(("Epoch ", "Test_Recall", "#####"))]


def test_killed_and_resumed_training_logs_the_uninterrupted_epochs_and_best_pt_evaluates_exactly(tiny_root, tmp_path, monkeypatch):
    """Trainer.train() end to end: 3 epochs against 2 epochs, a new Trainer with --resume last.pt and the third; then --eval_only 1
    on best.pt against the metrics of the epoch that wrote it (the same forward, scoring and top-K on the same bits)."""
    from llmrec_b200 import main as M
    logs = []
    monkeypatch.setattr(M.Logger, "logging", lambda self, s: logs.append(str(s)))
    da, db = str(tmp_path / "a"), str(tmp_path / "b")
    flags = ["--deterministic", "1", "--verbose", "1"]
    with _flags(tiny_root, flags) as build:
        a = build(["--epoch", "3", "--save_dir", da])
        best_a, _ = a.train()
        la, sa, ret_a = _lines(logs), _state(a), a._loop["test_ret"]
        del logs[:]
        build(["--epoch", "2", "--save_dir", db]).train()
        l1 = _lines(logs)
        del logs[:]
        b = build(["--epoch", "3", "--resume", os.path.join(db, "last.pt")])
        best_b, _ = b.train()
        assert l1 + _lines(logs) == la and len([s for s in la if s.startswith("Epoch ")]) == 3
        assert best_a == best_b
        sb = _state(b)
        for key in sa:
            assert torch.equal(sa[key], sb[key]), key
        del logs[:]
        e = build(["--resume", os.path.join(da, "best.pt"), "--eval_only", "1"])
        before = _state(e)
        ret = e.evaluate()
        after = _state(e)
        assert all(torch.equal(before[k], after[k]) for k in before), "--eval_only took a training step"
        for key in ("recall", "precision", "hit_ratio", "ndcg"):
            assert np.array_equal(ret[key], ret_a[key]), key
        assert ret["recall"][1] == best_a
        line = [s for s in logs if s.startswith("recall=[")]
        assert len(line) == 1 and any(line[0] in s for s in la)
