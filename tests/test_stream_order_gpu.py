"""-m gpu: the step schedules keep every cross-stream dependency (tests/stream_order.py records every launch and sync and checks
happens-before), and the check sees the edges a schedule change could drop.

Scenarios: each engine runs two consecutive eager steps (B' = 1126, then B' = 8) with branches on, so the second step is also checked
against the first step's side lanes; the graph path records its warm-up step, the snapshot / undo and the capture; the Trainer runs the
device samplers (with the sampler's own pre-draw stream), the host staging ring past its four slots and the eager mask branch, then the
serving calls.  Mutations: each drops one edge of a real engine with monkeypatch, and the check must name the pair and the buffer."""
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import step_fp64_cases as SC  # noqa: E402
import stream_order as SO  # noqa: E402

pytestmark = pytest.mark.gpu

TINY_FLAGS = ["--batch_size", "128", "--epoch", "1", "--debug", "--seed", "2022"]


@pytest.fixture
def recorder(monkeypatch):
    from llmrec_b200 import main as M
    rec = SO.Recorder().install(monkeypatch, trainer_module=M)
    yield rec
    rec.uninstall()


def _ops_buffers():
    from llmrec_b200 import ops
    return dict(scratch=ops._scratch, ginit=ops._ginit, score_scratch=ops._score_scratch, retired=ops._retired)


def _name_streams(rec, hp, sampler=None):
    for lane, st in hp._side.items():
        rec.name_stream(st, f"lane {lane}")
    if sampler is not None and getattr(sampler, "_side", None) is not None:
        rec.name_stream(sampler._side, "sampler")


def _races(rec, **roots):
    """(race descriptions, full report)"""
    races = rec.races()
    names = SO.buffer_names(**roots, ops=_ops_buffers())
    return [rec.describe(r, names) for r in races], rec.report(races, names)


def _assert_clean(rec, **roots):
    descr, report = _races(rec, **roots)
    assert not descr, "cross-stream races:\n" + report
    assert len({a.stream for a in rec.clocks.accesses}) >= 2, "no side stream was recorded"


def _expect(rec, *parts, **roots):
    """a race whose description names every one of `parts` (launch names, buffer)"""
    descr, report = _races(rec, **roots)
    hits = [d for d in descr if all(p in d for p in parts)]
    assert hits, f"no race names {parts}; found:\n{report or '(none)'}"


def _dev(batch):
    return [torch.from_numpy(x).cuda() for x in batch]


def _two_steps(rec, hp, name):
    batches = [_dev(SC._batch(name, w)) for w in ("B1126", "small")]
    torch.cuda.synchronize()
    rec.on = True
    for u, p, n in batches:
        hp.train_step(u, p, n)
    rec.on = False
    torch.cuda.synchronize()
    _name_streams(rec, hp)


# ---- the real schedules ----------------------------------------------------------------------------------------------------------

ENGINES = {
    "netflix": dict(name="netflix"), "movielens": dict(name="movielens"), "odd": dict(name="odd"),
    "netflix-det": dict(name="netflix", det=True), "netflix-bf16": dict(name="netflix", dtype="bf16"),
    "netflix-int8": dict(name="netflix", dtype="int8"), "odd-mode2": dict(name="odd", mode=2),
    "hoisted-netflix": dict(name="netflix", hoisted=True), "hoisted-netflix-det": dict(name="netflix", hoisted=True, det=True),
}


@pytest.mark.parametrize("case", list(ENGINES))
def test_engine_steps_have_no_unordered_conflict(recorder, case):
    kw = dict(ENGINES[case])
    name = kw.pop("name")
    hp = SC._engine(name, **kw)
    assert hp.branches
    _two_steps(recorder, hp, name)
    lanes = {hp._side[k].cuda_stream for k in (0, 1)}
    assert lanes <= {a.stream for a in recorder.clocks.accesses if a.name.startswith("llmrec_")}     # both lanes launched kernels
    _assert_clean(recorder, hp=hp)


def test_graph_capture_has_no_unordered_conflict_and_replays_match_eager(recorder):
    batches = [_dev(SC._batch("netflix", w)) for w in ("B1126", "small", "B1126")]
    ref = SC._engine("netflix")
    want = []
    for u, p, n in batches:
        ref.train_step(u, p, n)
        want.append(ref.loss.item())
    del ref
    hp = SC._engine("netflix")
    torch.cuda.synchronize()
    recorder.on = True                                                 # warm-up step, snapshot / undo and capture
    hp.train_step_graphed(*batches[0])
    recorder.on = False
    got = [hp.loss.item()]
    for u, p, n in batches[1:]:                                        # replays, not recorded
        hp.train_step_graphed(u, p, n)
        got.append(hp.loss.item())
    assert hp._graph is not None and recorder.clocks.graph_end
    side = {a.stream for a in recorder.clocks.accesses} - {recorder.main} - {st.cuda_stream for st in hp._side.values()}
    assert side, "the capture's launches were not recorded"            # (they run on the capture stream)
    _name_streams(recorder, hp)
    _assert_clean(recorder, hp=hp)
    np.testing.assert_allclose(got, want, rtol=1e-5)


def _trainer(root, extra):
    from llmrec_b200 import main as M
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility import batch_test
    from llmrec_b200.utility.load_data import Data
    from llmrec_b200.utility.parser import parse_args, resolve_dataset_dir
    args = set_args(parse_args(["--data_path", root, "--dataset", "netflix"] + TINY_FLAGS + list(extra)))
    M.set_seed(args.seed)
    gen = Data(path=resolve_dataset_dir(args.data_path, args.dataset), batch_size=args.batch_size, sampler=args.host_sampler)
    batch_test.init(gen, args)
    return M.Trainer(data_config={}, data_generator=gen)


@pytest.fixture
def restore_args():
    yield
    from llmrec_b200.runtime import set_args
    from llmrec_b200.utility.parser import parse_args
    set_args(parse_args([]))


def _train(rec, tr, steps):
    torch.cuda.synchronize()
    rec.on = True
    for _ in range(steps):
        tr.train_next_batch()
    return tr


def _serve(tr):
    tr.recommend(users=[0, 1, 2], K=5)
    tr.rerank([[1, 2, 3], [4, 5, 6]], users=[0, 1], K=2)
    tr.explain([[1, 2]], users=[0])
    tr.similar_items([0, 1], K=3)
    tr.recommend_groups([[0, 1], [2]], K=3)


TRAINERS = {
    "graph-device-sampler-1": (["--cuda_graph", "1", "--device_sampler", "1"], 2, True),
    "graph-device-sampler-2": (["--cuda_graph", "1", "--device_sampler", "2"], 2, True),
    "host-sampler-ring": (["--cuda_graph", "0"], 6, True),
    "mask-branch": (["--cuda_graph", "0", "--mask", "1", "--mask_rate", "0.1", "--drop_rate", "0.2"], 2, False),
}


@pytest.mark.parametrize("case", list(TRAINERS))
def test_trainer_steps_and_serving_have_no_unordered_conflict(recorder, restore_args, tiny_root, case):
    extra, steps, serve = TRAINERS[case]
    tr = _train(recorder, _trainer(tiny_root, extra), steps)
    if serve:                                                          # against whatever the last step left in flight
        _serve(tr)
    recorder.on = False
    torch.cuda.synchronize()
    if case == "host-sampler-ring":
        assert sum(a.name == "host write" for a in recorder.clocks.accesses) == steps > len(tr._slots)
    sampler = getattr(tr.device_sampler, "_side", None)
    if sampler is not None:                                            # the pre-draw ran on the sampler's own stream
        assert sampler.cuda_stream in {a.stream for a in recorder.clocks.accesses}
    _name_streams(recorder, tr.hot, tr.device_sampler)
    _assert_clean(recorder, hp=tr.hot, tr=tr)


# ---- mutations: each drops one edge, and the check names the pair and the buffer ---------------------------------------------------


class _NeverRecorded(torch.cuda.Event):
    def record(self, stream=None):
        pass


def test_mutation_dropped_id_layers_wait(recorder, monkeypatch):
    hp = SC._engine("netflix")
    monkeypatch.setattr(hp, "_ev_ids", _NeverRecorded(), raising=False)   # the wait becomes a no-op
    _two_steps(recorder, hp, "netflix")
    _expect(recorder, "llmrec_spmm_csr_f32 [lane 0] writes", "llmrec_fuse_fwd_rows_f32 [main] reads", "hp.Il[", hp=hp)


def test_mutation_join_drops_the_row_set_lane(recorder, monkeypatch):
    hp = SC._engine("netflix")
    join = hp._join
    monkeypatch.setattr(hp, "_join", lambda lanes=None: None if lanes is not None and list(lanes) == [1] else join(lanes))
    _two_steps(recorder, hp, "netflix")
    _expect(recorder, "llmrec_compact_mask [lane 1] writes", "llmrec_fuse_fwd_rows_f32", "hp.batch_", hp=hp)


def test_mutation_id_layers_share_the_primary_operators(recorder, monkeypatch):
    hp = SC._engine("odd")
    assert hp.ui.plan.n_split_tiles > 0 and hp.iu.plan.n_split_tiles > 0
    primary = (hp.ui, hp.iu, hp.uiT, hp.iuT)
    monkeypatch.setattr(hp, "_opset", lambda k: primary)
    _two_steps(recorder, hp, "odd")
    _expect(recorder, "llmrec_spmm_csr_f32 [lane 0] writes tiling_host[0].s", "llmrec_spmm_csr_f32 [main] writes tiling_host[0].s",
            ".plan.", hp=hp)


def test_mutation_fork_without_wait_stream(recorder, monkeypatch):
    hp = SC._engine("netflix")

    def fork(thunk, lane=0):                                           # HotPath._fork without st.wait_stream(current)
        st = hp._side.get(lane)
        if st is None:
            st = hp._side[lane] = torch.cuda.Stream(device=hp.E_u.device)
        with torch.cuda.stream(st):
            thunk()
        hp._forked.add(lane)

    monkeypatch.setattr(hp, "_fork", fork)
    _two_steps(recorder, hp, "netflix")
    _expect(recorder, "llmrec_spmm_csr_f32 [main] writes segs_host[", "llmrec_grad_init_f32 [lane 0] reads regions_host[", "hp.Fu", hp=hp)


def test_mutation_sampler_fork_recorded_before_the_copy(recorder, restore_args, tiny_root, monkeypatch):
    from llmrec_b200.device_sampler import ReferenceDeviceSampler

    def step_begin(self):                                              # _ev_fork recorded BEFORE index_buffer.copy_(self.next)
        self.host_is_current = False
        main = torch.cuda.current_stream(self.device)
        self._ev_fork.record(main)
        self.index_buffer.copy_(self.next)
        self._side.wait_event(self._ev_fork)
        with torch.cuda.stream(self._side):
            self._predraw()
            self._ev_done.record(self._side)

    monkeypatch.setattr(ReferenceDeviceSampler, "step_begin", step_begin)
    tr = _train(recorder, _trainer(tiny_root, ["--cuda_graph", "0", "--device_sampler", "2"]), 2)
    recorder.on = False
    torch.cuda.synchronize()
    _name_streams(recorder, tr.hot, tr.device_sampler)
    _expect(recorder, "aten::copy_ [main] reads", "llmrec_device_sample_batch_ref [sampler] writes", "device_sampler.next", hp=tr.hot, tr=tr)


def test_mutation_staging_slot_wait_skipped(recorder, restore_args, tiny_root, monkeypatch):
    from llmrec_b200 import main as M

    class Slot(M._StagingSlot):                                        # _next_slot's slot.event.synchronize() does nothing
        def __init__(self, cap):
            super().__init__(cap)
            self.event = types.SimpleNamespace(record=self.event.record, synchronize=lambda: None)

    monkeypatch.setattr(M, "_StagingSlot", Slot)
    tr = _train(recorder, _trainer(tiny_root, ["--cuda_graph", "0"]), 6)
    recorder.on = False
    torch.cuda.synchronize()
    _expect(recorder, "aten::copy_ [main] reads", "host write [host] writes", "tr._slots[", hp=tr.hot, tr=tr)
