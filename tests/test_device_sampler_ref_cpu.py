"""`--device_sampler 2` on the CPU kernel stand-ins (tests/ops_emulator.py, tests/ops_emulator_sampler.py): the Trainer plumbing of the
device sampler on the reference's streams -- batches equal to the host sampler's, `random` / `np.random` handed back after train() while the
next batch is pre-drawn, checkpoints that resume across sampler modes, and the host-side error path."""
import os
import pickle
import random
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)


class _Stop(Exception):
    pass


class _Slot:
    def __init__(self, cap):
        self.host = torch.zeros((4, cap), dtype=torch.int32)
        self.np = self.host.numpy()

        class _Ev:
            def record(self):
                pass

            def synchronize(self):
                pass
        self.event = _Ev()


def _worker(rank, root, extra, stop_after, ck_path, out_path):
    sys.path.insert(0, HERE); sys.path.insert(0, REPO)
    torch.set_num_threads(2)
    import ops_emulator
    import ops_emulator_sampler
    ops_emulator.install()
    ops_emulator_sampler.install()
    from llmrec_b200 import Models, main as M, ops
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir

    class AdamW(ops_emulator.AdamW):
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
    M.set_seed(args.seed)
    gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size, sampler=args.host_sampler)
    batch_test.init(gen, args)
    M.Logger.logging = lambda self, s: None
    tr = M.Trainer(data_config={}, data_generator=gen, device="cpu")
    assert tr.ref_sampler == (args.device_sampler == 2)
    batches, steps = [], [0]
    step = tr.train_next_batch

    def counted_step():
        if steps[0] == stop_after:
            tr.save_checkpoint(ck_path)
            raise _Stop
        steps[0] += 1
        r = step()
        g = tr.hot._gidx
        batches.append(g[:3, :int(g[3, 0])].numpy().copy())
        return r

    tr.train_next_batch = counted_step
    try:
        tr.train()
    except _Stop:
        pass
    pickle.dump(dict(batches=batches, state={k: t.clone() for k, t in tr.hot.state_tensors().items()},
                     py=random.getstate(), np=np.random.get_state()), open(out_path, "wb"))


def _run(tmp, name, root, extra, stop_after=None, ck_path=None):
    out = os.path.join(tmp, name + ".pkl")
    mp.spawn(_worker, args=(root, extra, stop_after, ck_path, out), nprocs=1, join=True)
    return pickle.load(open(out, "rb"))


def _same_np_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def test_trainer_draws_the_host_samplers_batches_and_hands_the_streams_back(tiny_root, tmp_path):
    a = _run(str(tmp_path), "host", tiny_root, ["--device_sampler", "0"])
    b = _run(str(tmp_path), "dev", tiny_root, ["--device_sampler", "2"])
    assert len(a["batches"]) == len(b["batches"]) > 4
    for t, (x, y) in enumerate(zip(a["batches"], b["batches"])):
        assert np.array_equal(x, y), f"batch {t} differs"
    assert any(x.shape[1] > 128 for x in a["batches"])                    # augmented edges were drawn
    for k in a["state"]:
        assert torch.equal(a["state"][k], b["state"][k]), k
    assert a["py"] == b["py"] and _same_np_state(a["np"], b["np"])


@pytest.mark.parametrize("first,second", [("0", "2"), ("2", "0")])
def test_checkpoint_resumes_across_sampler_modes(tiny_root, tmp_path, first, second):
    tmp = str(tmp_path)
    full = _run(tmp, "full", tiny_root, ["--device_sampler", first])
    n = len(full["batches"])
    ck = os.path.join(tmp, "mid.pt")
    k = n // 2 + 1                                                       # inside the second epoch
    b1 = _run(tmp, "b1", tiny_root, ["--device_sampler", first], stop_after=k, ck_path=ck)
    b2 = _run(tmp, "b2", tiny_root, ["--device_sampler", second, "--resume", ck])
    assert len(b1["batches"]) == k and len(b2["batches"]) == n - k
    for t, (x, y) in enumerate(zip(full["batches"], b1["batches"] + b2["batches"])):
        assert np.array_equal(x, y), f"batch {t} differs"
    for key in full["state"]:
        assert torch.equal(full["state"][key], b2["state"][key]), key
    assert full["py"] == b2["py"] and _same_np_state(full["np"], b2["np"])


def _sampler(rowptr, col, n_items, batch, exist=None, aug=None, rate=0.0):
    from llmrec_b200.device_sampler import ReferenceDeviceSampler
    n_users = len(rowptr) - 1
    exist = np.arange(n_users) if exist is None else exist
    ap, an = aug if aug is not None else (None, None)
    return ReferenceDeviceSampler(exist, rowptr, col, col, n_items, batch, ap, an, n_items, rate, "cpu")


@pytest.fixture
def stand_in():
    sys.path.insert(0, HERE)
    import ops_emulator_sampler
    from llmrec_b200.device_sampler import ReferenceDeviceSampler
    saved = ReferenceDeviceSampler._launch
    ops_emulator_sampler.install()
    yield
    ReferenceDeviceSampler._launch = saved


@pytest.mark.parametrize("case", ["no_train_items", "no_negative", "missing_aug"])
def test_errors_raise_the_host_samplers_exception_and_stick(stand_in, case):
    from llmrec_b200.host_native import BatchSampler
    random.seed(3); np.random.seed(3)
    rowptr, col, n_items = np.array([0, 2, 4, 6]), np.array([0, 1, 1, 2, 0, 2]), 4
    aug = None
    if case == "no_train_items":
        rowptr = np.array([0, 2, 2, 4])
        col = col[:4]
    if case == "no_negative":
        rowptr, col, n_items = np.array([0, 2, 4, 6]), np.array([0, 1, 0, 1, 0, 1]), 2
    if case == "missing_aug":
        aug = (np.array([1, BatchSampler.MISSING, 1], dtype=np.int32), np.array([2, 2, 2], dtype=np.int32))
    ds = _sampler(rowptr, col, n_items, 3, aug=aug, rate=1.0 if aug else 0.0)
    host = BatchSampler(np.arange(3), rowptr, col, n_items, 3, *(aug or (None, None)))
    before = (random.getstate(), np.random.get_state())
    with pytest.raises((RuntimeError, KeyError)) as want:
        host.draw(np.zeros((3, 16), dtype=np.int32), 1.0 if aug else 0.0)
    random.setstate(before[0]); np.random.set_state(before[1])
    buf, meta = torch.full((4, 6), 7, dtype=torch.int32), torch.tensor([[b, b] for b in range(7)], dtype=torch.int32)
    ds.fill(buf, meta)
    with pytest.raises(want.type) as got:
        ds.sync_to_host()
    assert str(got.value) == str(want.value)
    assert (buf[:3, :3] == 0).all() and buf[3, 0] == 3                   # the placeholder batch
    ds.fill(buf, meta)                                                    # the error sticks: nothing is drawn
    with pytest.raises(want.type):
        ds.check()
    ds.upload_from_host()
    ds.check()
