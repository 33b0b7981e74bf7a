"""Checkpoints without a GPU (llmrec_b200/checkpoint.py, Trainer.save_checkpoint / load_checkpoint, --save_dir / --resume / --eval_only).

Format level, on hand-made tensors: padded views are saved without their padding and loaded back in place; the file loads with
weights_only=True and its `model` section goes into MM_Model.load_state_dict; a failed save keeps the previous file; every malformed
file raises before a tensor of the target changes.

Trainer level, on the kernel stand-ins of tests/ops_emulator.py in spawned workers (as tests/test_trainer_emulated.py): a run that is
interrupted in the middle of its second epoch, saved and resumed by a NEW process draws the batches, logs the epoch lines and ends with
the parameters and moments of the uninterrupted run, exactly (the stand-ins are deterministic); best.pt evaluates to the metrics of the
epoch that wrote it; a run without --save_dir creates no file."""
import os
import pickle
import re
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from llmrec_b200 import checkpoint
from llmrec_b200.engine import PARAM_ORDER, HotPath

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


# ---------------------------------------------------------------------------------------------------------------------------------
# format level
# ---------------------------------------------------------------------------------------------------------------------------------
class _Engine(HotPath):
    """HotPath's state_tensors / load_state over a hand-made optimizer"""

    def __init__(self, opt, names):
        self.opt, self._opt_names = opt, names


def _wide(a, off=3, gap=5):
    n, d = a.shape
    buf = torch.full((n, off + d + gap), float("nan"))
    buf[:, off:off + d] = a
    return buf, buf[:, off:off + d]


def _engine(seed, shapes=None):
    g = torch.Generator().manual_seed(seed)
    shapes = shapes or {"user_id_embedding.weight": (7, 4), "item_id_embedding.weight": (9, 4), "image_trans.bias": (4,)}
    bufs, params = {}, []
    for k, s in shapes.items():
        t = torch.randn(*s, generator=g)
        if len(s) == 2:
            bufs[k], t = _wide(t)                          # a view with a leading dimension larger than its width
        params.append(t)
    opt = SimpleNamespace(params=params, m=[torch.randn(*s, generator=g) for s in shapes.values()],
                          v=[torch.rand(*s, generator=g) for s in shapes.values()],
                          state=torch.tensor([5.0, 0.25, 0.5, 0.0], dtype=torch.float64), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, wd=0.01)
    return _Engine(opt, list(shapes)), bufs


def _fingerprint(eng, **over):
    must = dict(n_users=7, n_items=9, params={k[6:]: tuple(t.shape) for k, t in eng.state_tensors().items() if k.startswith("model/")})
    must.update(over)
    return dict(must=must, recorded=dict(lr=1e-3, seed=1))


def _loop():
    return dict(epoch=1, batch=3, epoch_stats=torch.arange(4, dtype=torch.float32), best_recall=0.5, stopping_step=2, test_ret=None, n_interactions=11)


def _save(eng, path, fingerprint=None, loop=None):
    host = checkpoint.to_host(checkpoint.engine_tensors(eng))
    model, optim = checkpoint.engine_sections(host, eng.opt)
    checkpoint.write(path, model, optim, checkpoint.rng_state(torch.device("cpu")), loop or _loop(), fingerprint or _fingerprint(eng))


def _copy(eng, bufs):
    return [t.clone() for t in list(eng.state_tensors().values()) + list(bufs.values())]


def _unchanged(eng, bufs, before):
    return all(torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)) for a, b in zip(_copy(eng, bufs), before))


def test_round_trip_saves_views_without_padding_and_loads_them_in_place(tmp_path):
    src, _ = _engine(1)
    path = str(tmp_path / "a.pt")
    _save(src, path)
    raw = torch.load(path, weights_only=True)              # a plain dict of tensors and scalars: no project class is unpickled
    assert raw["format"] == 1 and set(raw["model"]) == set(src._opt_names) == set(raw["optim"]["m"]) == set(raw["optim"]["v"])
    for k, t in raw["model"].items():
        assert t.is_contiguous() and t.dtype == torch.float32 and t.untyped_storage().nbytes() == 4 * t.numel(), k
    assert raw["optim"]["state"].dtype == torch.float64 and raw["optim"]["state"].tolist() == [5.0, 0.25, 0.5, 0.0]
    assert (raw["optim"]["lr"], raw["optim"]["betas"], raw["optim"]["eps"], raw["optim"]["weight_decay"]) == (1e-3, (0.9, 0.999), 1e-8, 0.01)
    dst, bufs = _engine(2)
    ptrs = [t.data_ptr() for t in dst.state_tensors().values()]
    ck, saved, diffs = checkpoint.read(path, _fingerprint(dst), dst.state_tensors())
    assert diffs == [] and ck["loop"]["batch"] == 3
    dst.load_state(saved)
    assert [t.data_ptr() for t in dst.state_tensors().values()] == ptrs, "a tensor was rebound"
    for (k, a), b in zip(dst.state_tensors().items(), src.state_tensors().values()):
        assert torch.equal(a, b), k
    for k, buf in bufs.items():
        assert torch.isnan(buf[:, :3]).all() and torch.isnan(buf[:, -5:]).all(), k


def test_rng_streams_round_trip(tmp_path):
    import random
    random.seed(3); np.random.seed(4); torch.manual_seed(5)
    random.gauss(0, 1); np.random.standard_normal()        # both generators hold a cached gaussian
    eng, _ = _engine(1)
    path = str(tmp_path / "a.pt")
    _save(eng, path)
    want = (random.random(), random.gauss(0, 1), np.random.randint(0, 1 << 30), np.random.standard_normal(), torch.rand(3).tolist())
    ck, _, _ = checkpoint.read(path, _fingerprint(eng), eng.state_tensors())
    checkpoint.set_rng_state(ck["rng"], torch.device("cpu"))
    assert (random.random(), random.gauss(0, 1), np.random.randint(0, 1 << 30), np.random.standard_normal(), torch.rand(3).tolist()) == want


def test_model_section_goes_into_the_reference_module(tmp_path, golden):
    from llmrec_b200.Models import MM_Model
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility.parser import parse_args
    from oracle import llmrec_oracle as O
    names = sorted(k[len("epoch1/"):] for k in golden.files if k.startswith("epoch1/") and k.endswith((".weight", ".bias")))
    assert names == sorted(PARAM_ORDER) == sorted(O.PARAM_NAMES)
    shapes = {k: tuple(golden["epoch1/" + k].shape) for k in PARAM_ORDER}
    src, _ = _engine(3, shapes)
    path = str(tmp_path / "a.pt")
    _save(src, path)
    model = torch.load(path)["model"]
    assert sorted(model) == names
    set_args(parse_args(["--embed_size", str(shapes["image_trans.bias"][0])]))
    try:
        z = lambda n, k: np.zeros((n, k), np.float32)
        nu, ni = shapes["user_id_embedding.weight"][0], shapes["item_id_embedding.weight"][0]
        mm = MM_Model(nu, ni, shapes["image_trans.bias"][0], [64, 64], [0.1, 0.1], z(ni, shapes["image_trans.weight"][1]), z(ni, shapes["text_trans.weight"][1]),
                      z(nu, shapes["user_trans.weight"][1]), {"title": z(ni, shapes["item_trans.weight"][1])})
    finally:
        set_args(parse_args([]))
    res = mm.load_state_dict(model, strict=False)
    assert res.unexpected_keys == [] and all(k.startswith("batch_norm") for k in res.missing_keys)
    for k, t in src.state_tensors().items():
        if k.startswith("model/"):
            assert torch.equal(mm.state_dict()[k[6:]], t)


def test_a_failed_save_keeps_the_previous_checkpoint(tmp_path, monkeypatch):
    eng, _ = _engine(1)
    path = str(tmp_path / "last.pt")
    _save(eng, path)
    before = open(path, "rb").read()

    def half(obj, f):
        f.write(b"x" * 100)
        raise OSError("disk full")

    monkeypatch.setattr(torch, "save", half)
    eng.opt.state[0] = 6.0
    with pytest.raises(OSError, match="disk full"):
        _save(eng, path)
    assert open(path, "rb").read() == before and os.listdir(tmp_path) == ["last.pt"]


def test_malformed_files_raise_and_touch_nothing(tmp_path):
    src, _ = _engine(1)
    good = str(tmp_path / "good.pt")
    _save(src, good)
    blob = open(good, "rb").read()
    bad = str(tmp_path / "bad.pt")

    def edited(fn):
        ck = torch.load(good, weights_only=True)
        fn(ck)
        torch.save(ck, bad)
        return bad

    def truncated():
        open(bad, "wb").write(blob[:len(blob) // 2])
        return bad

    other, _ = _engine(1, {"user_id_embedding.weight": (7, 4), "item_id_embedding.weight": (8, 4), "image_trans.bias": (4,)})
    cases = [
        (truncated, "not a readable checkpoint"),
        (lambda: edited(lambda ck: ck.update(format=2)), "format 2"),
        (lambda: edited(lambda ck: ck["optim"]["m"].pop("image_trans.bias")), "'m/image_trans.bias' is missing"),
        (lambda: edited(lambda ck: ck.pop("rng")), "'rng' is missing"),
        (lambda: edited(lambda ck: ck["loop"].pop("stopping_step")), "loop/stopping_step"),
        (lambda: edited(lambda ck: ck["model"].update({"item_id_embedding.weight": torch.zeros(8, 4)})), "item_id_embedding.weight' is \\(8, 4\\)"),
        (lambda: edited(lambda ck: ck["optim"].update(state=torch.zeros(4))), "'state' is \\(4,\\) torch.float32"),
        (lambda: edited(lambda ck: ck["fingerprint"]["must"].update(n_items=10)), "n_items is 10 in the checkpoint and 9 in this run"),
    ]
    for make, msg in cases:
        dst, bufs = _engine(2)
        before = _copy(dst, bufs)
        with pytest.raises(ValueError, match=msg):
            checkpoint.read(make(), _fingerprint(dst), dst.state_tensors())
        assert _unchanged(dst, bufs, before), msg
    # a checkpoint of another model: the set of parameter shapes is part of what must match
    _save(other, bad, fingerprint=_fingerprint(other))
    dst, bufs = _engine(2)
    with pytest.raises(ValueError, match="params is"):
        checkpoint.read(bad, _fingerprint(dst), dst.state_tensors())
    # recorded fields that differ are reported, not raised
    fp = _fingerprint(dst)
    fp["recorded"]["lr"] = 5e-4
    assert checkpoint.read(good, fp, dst.state_tensors())[2] == ["lr: 0.001 -> 0.0005"]
    with pytest.raises(ValueError, match="per rank"):
        checkpoint.engine_tensors(object())


def test_flags_that_cannot_be_combined_raise(monkeypatch):
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility.parser import parse_args
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    base = ["--debug"]
    try:
        for extra, msg in ((["--eval_only", "1"], "--resume"), (["--resume", "x.pt", "--mask", "1"], "--mask"),
                           (["--resume", "x.pt", "--drop_rate", "0.1"], "--drop_rate"), (["--save_dir", "d", "--mask_rate", "0.1"], "--mask_rate")):
            set_args(parse_args(base + extra))
            with pytest.raises(ValueError, match=msg):
                M.Trainer(data_config={})
    finally:
        set_args(parse_args([]))


def test_help_texts_describe_the_supported_branches():
    from llmrec_b200.utility.parser import build_parser
    text = build_parser().format_help()
    assert "not supported here" not in text and "only 0 is supported" not in text
    for flag in ("--save_dir", "--save_every", "--resume", "--eval_only"):
        assert flag in text


# ---------------------------------------------------------------------------------------------------------------------------------
# the whole Trainer on the kernel stand-ins
# ---------------------------------------------------------------------------------------------------------------------------------
class _Slot:
    def __init__(self, cap):
        self.host = torch.zeros((4, cap), dtype=torch.int32)
        self.np = self.host.numpy()
        self.event = SimpleNamespace(synchronize=lambda: None, record=lambda: None)


class _Stop(Exception):
    pass


def _worker(rank, root, extra, stop_after, ck_path, out_path, cwd):
    """One Trainer run in a fresh process.  stop_after: save to ck_path after that many steps and die (None: run to the end)."""
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    os.chdir(cwd)
    import ops_emulator
    ops_emulator.install()
    from llmrec_b200 import Models, main as M, ops
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir

    class AdamW(ops_emulator.AdamW):
        """the stand-in with its step count where ops.AdamW keeps it: in a fp64[4] `state` block"""

        def __init__(self, *a, **k):
            self.state = torch.zeros(4, dtype=torch.float64)
            super().__init__(*a, **k)

        t = property(lambda self: int(self.state[0]), lambda self, v: self.state.__setitem__(0, float(v)))

    ops.AdamW = AdamW
    Models._on_device = lambda t: True
    M._StagingSlot = _Slot
    torch.cuda.is_available = lambda: True
    torch.cuda.synchronize = lambda *a, **k: None
    torch.cuda.manual_seed_all = lambda s: None
    args = set_args(parse_args(["--data_path", root, "--dataset", "netflix", "--batch_size", "128", "--epoch", "2", "--debug", "--seed", "2022",
                                "--cuda_graph", "0", "--proj_mode", "fp32", "--lr", "0.001"] + extra))
    M.set_seed(args.seed)                                       # as main(): seed, build (the model's and the Decoder's draws), then --resume
    gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size, sampler=args.host_sampler)
    batch_test.init(gen, args)
    logs, batches, steps = [], [], [0]
    orig_logging = M.Logger.logging
    M.Logger.logging = lambda self, s: logs.append(str(s))
    tr = M.Trainer(data_config={}, data_generator=gen, device="cpu")
    assert (tr._batch_sampler is not None) == (args.host_sampler == "native")
    push, step = tr._push, tr.train_next_batch

    def recording_push(slot, B):
        batches.append(slot.np[:3, :B].copy())
        return push(slot, B)

    def counted_step():
        if steps[0] == stop_after:                              # a step boundary of train()'s loop
            tr.save_checkpoint(ck_path)
            raise _Stop
        steps[0] += 1
        return step()

    tr._push, tr.train_next_batch = recording_push, counted_step
    res = None
    try:
        res = tr.evaluate() if args.eval_only else tr.train()
    except _Stop:
        pass
    M.Logger.logging = orig_logging
    state = {k: t.clone() for k, t in tr.hot.state_tensors().items()}
    ret = tr._loop["test_ret"] if not args.eval_only else res
    pickle.dump(dict(logs=logs, batches=batches, state=state, result=None if args.eval_only else res and res[0],
                     ret=None if ret is None else {k: np.asarray(v).tolist() for k, v in ret.items()}, files=sorted(os.listdir(cwd))), open(out_path, "wb"))


def _run(tmp, name, root, extra, stop_after=None, ck_path=None):
    cwd = os.path.join(tmp, name + "_cwd")
    os.makedirs(cwd)
    out_path = os.path.join(tmp, name + ".pkl")
    mp.spawn(_worker, args=(root, extra, stop_after, ck_path, out_path, cwd), nprocs=1, join=True)
    return pickle.load(open(out_path, "rb"))


def _epoch_lines(logs):
    """the per-epoch log lines without their wall-clock times"""
    return [re.sub(r"\[[0-9.]+s( \+ [0-9.]+s)?\]", "[]", s) for s in logs if s.startswith("Epoch ") or s.startswith("Test_Recall") or s.startswith("#####")]


@pytest.mark.parametrize("sampler", ["native", "python"])
def test_interrupted_and_resumed_run_equals_the_uninterrupted_one(tiny_root, tmp_path, sampler):
    tmp = str(tmp_path)
    flags = ["--host_sampler", sampler]
    save_dir = os.path.join(tmp, "ckpt")
    a = _run(tmp, "a", tiny_root, flags + ["--save_dir", save_dir])
    n_batch = len(a["batches"]) // 2
    assert len(a["batches"]) == 2 * n_batch and n_batch > 3
    ck = os.path.join(tmp, "mid.pt")
    b1 = _run(tmp, "b1", tiny_root, flags, stop_after=n_batch + 3, ck_path=ck)
    assert len(b1["batches"]) == n_batch + 3 and b1["files"] == []            # no --save_dir: the run itself wrote nothing
    loop = torch.load(ck, weights_only=True)["loop"]
    assert (loop["epoch"], loop["batch"]) == (1, 3)
    b2 = _run(tmp, "b2", tiny_root, flags + ["--resume", ck])
    assert len(b2["batches"]) == n_batch - 3
    for t, (x, y) in enumerate(zip(a["batches"], b1["batches"] + b2["batches"])):
        assert np.array_equal(x, y), f"batch {t} differs"
    la, lb = _epoch_lines(a["logs"]), _epoch_lines(b1["logs"]) + _epoch_lines(b2["logs"])
    assert len(la) >= 2 and la == lb
    assert a["result"] == b2["result"] and a["ret"] == b2["ret"]
    assert a["state"].keys() == b2["state"].keys() and float(a["state"]["state"][0]) == 2 * n_batch
    for k in a["state"]:
        assert torch.equal(a["state"][k], b2["state"][k]), k
    # --save_dir changed nothing of the run and wrote last.pt / best.pt, nothing else
    assert sorted(os.listdir(save_dir)) == ["best.pt", "last.pt"]
    last = torch.load(os.path.join(save_dir, "last.pt"), weights_only=True)
    assert (last["loop"]["epoch"], last["loop"]["batch"]) == (2, 0)
    for k in PARAM_ORDER:
        assert torch.equal(last["model"][k], a["state"]["model/" + k])
    if sampler == "native":
        # best.pt holds the parameters that scored best_recall: evaluating it gives that epoch's metrics, exactly
        best = os.path.join(save_dir, "best.pt")
        e = _run(tmp, "e", tiny_root, flags + ["--resume", best, "--eval_only", "1"])
        assert e["batches"] == [] and e["ret"] == a["ret"] and a["ret"]["recall"][1] == a["result"]
        line = [s for s in e["logs"] if s.startswith("recall=[")]
        assert len(line) == 1 and any(line[0] in s for s in a["logs"] if s.startswith("Epoch "))
