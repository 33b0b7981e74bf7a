"""-m "not gpu": the pieces of the stream-ordering check (tests/stream_order.py) that need no GPU -- the header's roles against the ctypes
binding, the ABI decoding on fake device memory, and the happens-before checker on hand-written traces."""
import ctypes as C
import inspect
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import stream_order as SO  # noqa: E402
from llmrec_b200 import _native as N  # noqa: E402

HDR = SO.parse_header()

STRUCTS = {"llmrec_spmm_seg": N.SpmmSeg, "llmrec_spmm_tiling": N.SpmmTiling, "llmrec_proj_fwd_problem": N.ProjFwdProblem,
           "llmrec_proj_wgrad_problem": N.ProjWgradProblem, "llmrec_proj_fwd_problem_bf16": N.ProjFwdProblemBf16,
           "llmrec_proj_wgrad_problem_bf16": N.ProjWgradProblemBf16, "llmrec_proj_fwd_problem_i8": N.ProjFwdProblemI8,
           "llmrec_proj_wgrad_problem_i8": N.ProjWgradProblemI8, "llmrec_proj_row_map": N.ProjRowMap, "llmrec_bpr_head": N.BprHead,
           "llmrec_grad_region": N.GradRegion, "llmrec_rank1_block": N.Rank1Block, "llmrec_colsum_term": N.ColsumTerm}


def _is_pointer_type(t):
    return t in (C.c_void_p, C.c_char_p) or (isinstance(t, type) and issubclass(t, C._Pointer))


# ---- the header against the binding ----------------------------------------------------------------------------------------------


def test_header_parse_covers_the_binding_with_roles():
    assert set(HDR.functions) == set(N.SIGNATURES)
    for fn, params in HDR.functions.items():
        argtypes = N.SIGNATURES[fn][1]
        assert len(params) == len(argtypes), fn
        for p, t in zip(params, argtypes):
            assert (p.stars > 0 or p.ctype == "llmrec_stream_t") == _is_pointer_type(t), (fn, p.name, p.ctype, t)
        if HDR.stream_param(fn) is None:
            continue
        assert params[-1].ctype == "llmrec_stream_t", fn                 # the stream is the last argument
        r = SO.roles(HDR, fn)
        ptrs = [p.name for p in params if p.stars]
        assert sorted(r) == sorted(ptrs), fn                             # every pointer parameter has a role
        for name, (kind, what) in r.items():
            assert kind in ("dev", "table", "structs", "host")
            if kind == "structs":
                assert what in HDR.structs and SO.field_roles(HDR, what), (fn, name)
    # spot checks of the const-correct roles
    assert SO.roles(HDR, "llmrec_adamw_step_f32")["p_host"] == ("table", SO.WRITE)
    assert SO.roles(HDR, "llmrec_adamw_step_f32")["g_host"] == ("table", SO.READ)
    assert SO.roles(HDR, "llmrec_fuse_fwd_f32")["layers_host"] == ("table", SO.READ)
    assert SO.roles(HDR, "llmrec_fuse_fwd_f32")["out"] == ("dev", SO.WRITE)
    assert SO.roles(HDR, "llmrec_explain_f32")["coef"] == ("host", None)
    assert SO.roles(HDR, "llmrec_spmm_csr_f32")["segs_host"] == ("structs", "llmrec_spmm_seg")
    assert SO.field_roles(HDR, "llmrec_spmm_tiling") == {"tiles": "r", "split_row": "r", "split_first": "r", "scratch": "w",
                                                        "split_tickets": "w", "src_mask": "r"}


def test_ctypes_structures_follow_the_header_typedefs():
    assert set(STRUCTS) == set(HDR.structs)
    for name, cls in STRUCTS.items():
        fields = HDR.structs[name]
        assert [f for f, _ in cls._fields_] == [f.name for f in fields], name
        roles = SO.field_roles(HDR, name)
        for (fname, t), f in zip(cls._fields_, fields):
            assert _is_pointer_type(t) == (f.stars > 0), (name, fname)
            if f.stars:
                assert roles[fname] in (SO.READ, SO.WRITE)
    for base, flag in SO.ROW_MAP_FLAG.items():                       # the flags word that announces a row map is an integer field
        for sfx in ("", "_bf16", "_i8"):
            assert [f.ctype for f in HDR.structs[base + sfx] if f.name == flag] == ["int32_t"]
    assert SO.ROW_MAP_BIT == N.PROJ_ROW_MAP


def test_length_map_names_real_parameters():
    for (fn, name), n in SO.LENGTHS.items():
        params = {p.name: p for p in HDR.functions[fn]}
        assert name in params and params[name].stars > 0, (fn, name)
        assert HDR.stream_param(fn) is not None, fn
        if isinstance(n, str):
            arg = n.partition("+")[0]
            assert arg in params and params[arg].stars == 0 and params[arg].ctype.startswith("int"), (fn, n)
    for fn in HDR.functions:
        if HDR.stream_param(fn) is None:
            continue
        for p in SO.host_array_params(HDR, fn):
            assert (fn, p.name) in SO.LENGTHS, f"{fn}: no length for host array {p.name}"


def test_wait_stream_goes_through_record_and_wait():
    """Only Event.record / Event.wait are wrapped: Stream.wait_event and wait_stream must reach them, once each."""
    src = lambda f: inspect.getsource(f).split('"""')[-1]
    assert "event.wait(self)" in src(torch.cuda.Stream.wait_event)
    assert "self.wait_event(stream.record_event())" in src(torch.cuda.Stream.wait_stream)
    assert "event.record(self)" in src(torch.cuda.Stream.record_event)


# ---- ABI decoding on fake device memory ------------------------------------------------------------------------------------------


class _FakeBlocks:
    def __init__(self, blocks):
        self.blocks = sorted(blocks)

    def find(self, p):
        for s, n in self.blocks:
            if s <= p < s + n:
                return s, n
        return None


def _fake_recorder(blocks):
    rec = SO.Recorder()
    rec._blocks = _FakeBlocks(blocks)
    rec.on = True
    return rec


def test_abi_calls_are_decoded_element_by_element():
    A, B, RP, COL, TI, SC, TK = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000, 0x70000
    rec = _fake_recorder([(A, 0x8000), (B, 0x8000), (RP, 0x1000), (COL, 0x1000), (TI, 0x1000), (SC, 0x1000), (TK, 0x1000)])
    segs = (N.SpmmSeg * 2)()
    segs[0] = N.SpmmSeg(A, B, None, 256, 256, 0, 0, 0)                # column block 0 (64 wide) of a 256-wide buffer
    segs[1] = N.SpmmSeg(A + 4 * 64, B + 4 * 64, B + 4 * 64, 256, 256, 256, 0, 0)
    til = N.SpmmTiling(TI, None, None, SC, 3, 0, 0, 0, TK, None)
    rec._abi("llmrec_spmm_csr_f32", (C.c_void_p(RP), C.c_void_p(COL), C.c_void_p(0), C.c_void_p(0), C.c_void_p(0), 10, 12, 64, segs, 2,
                                      C.byref(til), C.c_void_p(0x99)))
    a = rec.clocks.accesses[-1]
    assert a.stream == 0x99 and a.name == "llmrec_spmm_csr_f32"
    assert sorted(e.label for e in a.reads) == ["col", "rowptr", "segs_host[0].X", "segs_host[1].X", "segs_host[1].Z", "tiling_host[0].tiles"]
    assert sorted(e.label for e in a.writes) == ["segs_host[0].Y", "segs_host[1].Y", "tiling_host[0].scratch", "tiling_host[0].split_tickets"]
    y0 = [e for e in a.writes if e.label == "segs_host[0].Y"][0]
    y1 = [e for e in a.writes if e.label == "segs_host[1].Y"][0]
    assert y0.blocks == [(B, 10, 256, 1024)] and not y0.overlaps(y1)  # narrowed: disjoint column blocks of one allocation
    x0 = [e for e in a.reads if e.label == "segs_host[0].X"][0]
    assert x0.blocks == [(A, 12, 256, 1024)]

    # a grouped projection with row maps: the records after the problems are decoded too
    from llmrec_b200 import ops
    arr, recs, blk = ops._problem_array(N.ProjWgradProblem, 2, True)
    arr[0] = N.ProjWgradProblem(A, B, SC, TK, 64, 64, 5, 64, N.WGRAD_ACCUMULATE | N.PROJ_ROW_MAP)
    arr[1] = N.ProjWgradProblem(A, B, SC, None, 64, 64, 5, 64, 0)
    recs[0] = N.ProjRowMap(RP, 7)
    recs[1] = N.ProjRowMap(COL, 7)                                    # unflagged problem: its record is ignored
    rec._abi("llmrec_proj_wgrad_group_f32", (arr, 2, 64, 0, C.c_void_p(TI), 100, C.c_void_p(0x98)))
    a = rec.clocks.accesses[-1]
    assert sorted(e.label for e in a.reads) == ["probs_host[0].X", "probs_host[0].dY", "probs_host[1].X", "probs_host[1].dY", "row_maps[0].rows"]
    assert sorted(e.label for e in a.writes) == ["probs_host[0].dW", "probs_host[0].db", "probs_host[1].dW", "scratch"]

    # a pointer table: one access per element, with the table's role
    p_tab, g_tab = (C.c_void_p * 2)(A, B), (C.c_void_p * 2)(SC, TK)
    rec._abi("llmrec_adamw_step_f32", (p_tab, g_tab, p_tab, p_tab, (C.c_int64 * 2)(4, 4), 2, C.c_void_p(TI), 1e-3, 0.9, 0.999, 1e-8, 0.0,
                                        C.c_void_p(0x97)))
    a = rec.clocks.accesses[-1]
    assert sorted(e.label for e in a.reads) == ["g_host[0]", "g_host[1]", "state"]
    assert len(a.writes) == 6

    with pytest.raises(AssertionError, match="outside every block"):
        rec._abi("llmrec_fill_f32", (C.c_void_p(0x123), 4, 0.0, C.c_void_p(0x99)))
    with pytest.raises(AssertionError, match="is device memory"):   # a host-side planner handed device memory
        rec._abi("llmrec_spmm_plan_tiles", (C.c_void_p(RP), 10, 16, 15, None, None, None, C.c_void_p(0)))
    counts = np.zeros(3, dtype=np.int32)
    rec._abi("llmrec_spmm_plan_tiles", (counts.ctypes.data, 10, 16, 15, None, None, None, counts.ctypes.data))


# ---- the happens-before checker on hand-written traces ----------------------------------------------------------------------------


def _ext(key, start=0, n=64):
    return SO.Extent(("dev", key), [(key + start, 1, n, n)], f"buf{key:#x}")


class _Ev:
    pass


MAIN, SIDE, THIRD = 1, 2, 3


def test_fork_and_join():
    ck, X = SO.Clocks(), _ext(0x1000)
    ck.access(MAIN, "write X", [], [X])
    fork = _Ev()
    ck.record(fork, MAIN)
    ck.wait(fork, SIDE)
    ck.access(SIDE, "read X", [X], [])
    assert ck.races() == []                                            # forked after the write
    ck.access(MAIN, "write X again", [], [X])
    r = ck.races()
    assert len(r) == 1 and (r[0].a.name, r[0].b.name) == ("read X", "write X again")
    ck2, X = SO.Clocks(), _ext(0x1000)
    ck2.access(SIDE, "read X", [X], [])
    join = _Ev()
    ck2.record(join, SIDE)
    ck2.wait(join, MAIN)
    ck2.access(MAIN, "write X", [], [X])
    assert ck2.races() == []                                           # joined before the write


def test_wait_binds_to_the_latest_record_before_it():
    ck, X, ev = SO.Clocks(), _ext(0x1000), _Ev()
    ck.record(ev, MAIN)                                                # step 1's record
    ck.access(MAIN, "write X", [], [X])
    ck.record(ev, MAIN)                                                # re-recorded after the write
    ck.wait(ev, SIDE)
    ck.access(SIDE, "read X", [X], [])
    assert ck.races() == []
    ck2, X, ev = SO.Clocks(), _ext(0x1000), _Ev()
    ck2.record(ev, MAIN)
    ck2.wait(ev, SIDE)                                                 # binds to the first record
    ck2.access(MAIN, "write X", [], [X])
    ck2.record(ev, MAIN)                                               # a later record does not reach back
    ck2.access(SIDE, "read X", [X], [])
    assert len(ck2.races()) == 1


def test_wait_on_a_never_recorded_event_adds_no_edge():
    ck, X = SO.Clocks(), _ext(0x1000)
    ck.access(MAIN, "write X", [], [X])
    ck.wait(_Ev(), SIDE)
    ck.access(SIDE, "read X", [X], [])
    assert len(ck.races()) == 1


def test_wait_stream_is_record_plus_wait():
    ck, X = SO.Clocks(), _ext(0x1000)
    ck.access(MAIN, "write X", [], [X])
    ev = _Ev()                                                         # Stream.wait_stream: record_event() on MAIN, wait_event on SIDE
    ck.record(ev, MAIN)
    ck.wait(ev, SIDE)
    ck.access(SIDE, "write X", [], [X])
    ck.access(THIRD, "read X", [X], [])                                # a third stream is ordered after neither
    r = ck.races()
    assert {(x.a.name, x.b.name) for x in r} == {("write X", "read X")} and len(r) == 2


def test_synchronize_is_a_barrier():
    for sync in ("device", "stream", "event"):
        ck, X = SO.Clocks(), _ext(0x1000)
        ck.access(MAIN, "write X", [], [X])
        ev = _Ev()
        ck.record(ev, MAIN)
        {"device": ck.device_sync, "stream": lambda: ck.stream_sync(MAIN), "event": lambda: ck.event_sync(ev)}[sync]()
        ck.access(SIDE, "read X", [X], [])                             # launched after the host waited
        assert ck.races() == [], sync
    ck, X = SO.Clocks(), _ext(0x1000)
    ck.access(MAIN, "write X", [], [X])
    ck.stream_sync(THIRD)                                              # another stream's sync orders nothing
    ck.access(SIDE, "read X", [X], [])
    assert len(ck.races()) == 1


def test_host_writes():
    ck, slot = SO.Clocks(), SO.Extent(("host", 0x5000), [(0x5000, 1, 64, 64)], "slot.host")
    ck.access(SO.HOST, "host write", [], [slot])
    ck.access(MAIN, "aten::copy_", [slot], [_ext(0x1000)])             # the H2D copy is enqueued after the host wrote the slot
    assert ck.races() == []
    ev = _Ev()
    ck.record(ev, MAIN)
    ck.event_sync(ev)                                                  # the slot's event
    ck.access(SO.HOST, "host write", [], [slot])
    assert ck.races() == []
    ck.access(MAIN, "aten::copy_", [slot], [_ext(0x1000)])
    ck.access(SO.HOST, "host write", [], [slot])                       # rewritten without waiting for the copy
    r = ck.races()
    assert len(r) == 1 and r[0].b.name == "host write" and r[0].b.stream == SO.HOST


def test_strided_extents_overlap_exactly():
    t = torch.zeros(10, 8)
    e = lambda v: SO.tensor_extent(v)
    assert not e(t[:, 0:4]).overlaps(e(t[:, 4:8]))
    assert e(t[:, 2:6]).overlaps(e(t[:, 4:8]))
    assert not e(t[0:5]).overlaps(e(t[5:10]))
    assert e(t[4:6, 7:8]).overlaps(e(t[5]))
    assert not e(t[:, 3]).overlaps(e(t[:, 4]))                        # two columns
    assert e(t.t()[3]).overlaps(e(t[:, 3]))                           # the same column through a transpose
    assert not e(t[::2]).overlaps(e(t[1::2]))                         # even and odd rows
    assert not e(t[:, 0:4]).overlaps(e(torch.zeros(10, 8)[:, 0:4]))   # another allocation
    # against brute force: row blocks of random geometry inside one allocation
    rng = np.random.default_rng(0)
    for _ in range(3000):
        blk = []
        for _ in range(2):
            n, w = int(rng.integers(1, 6)), int(rng.integers(1, 9))
            ld = int(rng.integers(w, 12)) if n > 1 else w
            blk.append((int(rng.integers(0, 40)), n, w, ld))
        cover = [set(s + i * ld + j for i in range(n) for j in range(w)) for s, n, w, ld in blk]
        assert SO._blocks_overlap(*blk) == bool(cover[0] & cover[1]), blk
