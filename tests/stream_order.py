"""Ordering check of the launches of a training step across CUDA streams.  TEST INFRASTRUCTURE ONLY: the product never imports it.

A step is a DAG of streams (HotPath._fork / _join, the hoisted engine's forks, the device sampler's pre-draw stream, the host staging
ring).  A missing edge is a race that an idle GPU usually hides: the two launches run one after the other anyway and every value test
passes.  This module finds such races from the recorded order alone, without running anything twice:

Recorder
  ABI calls   `_native._lib` is replaced by a proxy (`N.lib()` returns `_lib` when it is set).  Every `llmrec_*` call is recorded with its
              stream -- its own `llmrec_stream_t` argument, not torch's current stream -- and the device memory it reads and writes.  The
              roles come from include/llmrec_b200.h, which is const-correct: `const T*` is a read, `T*` a write (taken as read-and-write).
              Host pointer tables (`float* const* p_host`, `const float* const* layers_host`, ...) and host struct arrays (`segs_host`,
              the projection problems and the row-map records that follow them, BPR heads, gradient regions, rank-1 blocks, colsum terms)
              are decoded element by element, each field with the role its const-ness gives it in the header typedef.  LENGTHS names the
              argument that holds each array's length.  A function without a stream argument (planners, `*_scratch` queries, host
              samplers) must not be handed device memory; the proxy asserts that.
              One ABI call is one unit on its stream.  The library's only internal branch, the bias column sums of the grouped
              weight-gradient calls, runs on a library-owned stream forked from the call's stream and is joined back into it before the
              call returns (proj_tc.cu, llmrec_proj_wgrad_group_*), so no launch of the call outlives it on another stream.
  torch ops   a TorchDispatchMode records every aten op that touches a CUDA tensor, on torch.cuda.current_stream(): writes from the
              schema (alias_info.is_write) and from the outputs, reads from the other tensor arguments (pinned host tensors included, so
              an H2D copy out of a staging slot reads that slot).  Pure view and metadata ops are skipped.
  syncs       Event.record / wait / synchronize, Stream.synchronize and torch.cuda.synchronize are wrapped.  Stream.wait_event calls
              Event.wait and Stream.wait_stream calls record_event (Event.record) + wait_event (torch/cuda/streams.py), so wrapping the
              Event methods sees every edge exactly once.  One vector clock per stream and one for the host; a launch joins the host's
              clock (it is enqueued after everything the host has waited for); waiting on an event that was never recorded adds no edge,
              as in CUDA.  A captured CUDA graph's launches are recorded while the capture runs; a replay orders the replaying stream
              after the end of the capture.
  host ring   Trainer._next_slot hands out a pinned staging slot for the host to fill: that is recorded as a host write of `slot.host`.

Extents
  An ABI pointer maps to the caching-allocator block that contains it (torch.cuda.memory_snapshot(): segment address plus block sizes);
  a device pointer outside every allocated block is an error, so nothing goes unchecked.  torch ops give exact strided extents.
  NARROW lists the ABI arguments whose extent is the rectangle named by the call's own (pointer, leading dimension, rows, columns)
  arguments instead of the whole block: column blocks of one buffer (Fu / GFu / Fi / GFi blocks) are written by different launches.

Check
  Every two accesses on different streams whose extents overlap, one of them a write, must be ordered: the earlier one (in host order)
  must happen before the later one.  A report names both launches (ABI name or aten op) and their streams, the llmrec_b200 source lines
  that issued them, and the buffer, by a reverse map from the engine's attributes (`buffer_names`).
"""
from __future__ import annotations

import bisect
import ctypes as C
import os
import re
import sys
from dataclasses import dataclass

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
HEADER = os.path.join(REPO, "include", "llmrec_b200.h")
PKG_DIR = os.path.join(REPO, "llmrec_b200") + os.sep

READ, WRITE = "r", "w"          # WRITE means read-and-write

# ---- the header -------------------------------------------------------------------------------------------------------------------


@dataclass
class Param:
    name: str
    ctype: str                  # normalised, e.g. "const float * const *"

    @property
    def stars(self):
        return self.ctype.count("*")

    @property
    def base(self):
        """the element type without qualifiers and stars"""
        return " ".join(t for t in self.ctype.split() if t not in ("const", "*"))

    @property
    def pointee_const(self):
        """const-ness of what the first level of indirection points to (`const float*`, `const float* const*`)"""
        return self.ctype.split()[0] == "const"


@dataclass
class Header:
    structs: dict               # typedef name -> [Param] (fields in order)
    functions: dict             # name -> [Param]

    def stream_param(self, fn):
        ps = [p for p in self.functions[fn] if p.ctype == "llmrec_stream_t"]
        return ps[0].name if ps else None


def _norm(ctype):
    return " ".join(ctype.replace("*", " * ").split())


def _decl(text):
    """'const float* const* layers_host' -> Param"""
    m = re.match(r"^(.*?)(\w+)\s*(\[\s*\w*\s*\])?$", text.strip(), re.S)
    return Param(m.group(2), _norm(m.group(1)))


def parse_header(path=HEADER):
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    structs = {}
    for m in re.finditer(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", src, re.S):
        fields = []
        for stmt in m.group(1).split(";"):
            stmt = stmt.strip()
            if not stmt:
                continue
            first, *more = stmt.split(",")
            p = _decl(first)
            fields.append(p)
            base = " ".join(t for t in p.ctype.split() if t != "*")
            fields += [Param(n.strip().lstrip("*").strip(), _norm(base + " *" * n.count("*"))) for n in more]
        structs[m.group(2)] = fields
    body = re.sub(r"typedef[^;]*;", "", re.sub(r"typedef\s+struct\s*\{.*?\}\s*\w+\s*;", "", src, flags=re.S))
    functions = {}
    for m in re.finditer(r"([\w\s\*]+?)\b(llmrec_\w+)\s*\(([^)]*)\)\s*;", body):
        args = m.group(3).strip()
        functions[m.group(2)] = [] if args in ("", "void") else [_decl(a) for a in args.split(",")]
    return Header(structs, functions)


# Length of every host array argument of a stream function: an int, or the name of the argument that holds it ("+1": one more).
_PROJ = [f"llmrec_proj_{k}_group_{t}" for k in ("fwd", "wgrad") for t in ("f32", "bf16", "i8")]
LENGTHS = {
    ("llmrec_spmm_csr_f32", "segs_host"): "nseg",
    ("llmrec_spmm_csr_f32", "tiling_host"): 1,
    ("llmrec_spmm_rows_f32", "seg_host"): 1,
    **{(f, "probs_host"): "n_prob" for f in _PROJ},
    **{(f, p): "n_layers" for f in ("llmrec_fuse_fwd_f32", "llmrec_fuse_fwd_rows_f32") for p in ("layers_host", "ld_layers_host")},
    **{(f, p): "n_sides" for f in ("llmrec_fuse_fwd_f32", "llmrec_fuse_fwd_rows_f32") for p in ("sides_host", "ld_sides_host", "coef_host")},
    **{(f, p): "n_sides" for f in ("llmrec_fuse_bwd_f32", "llmrec_fuse_bwd_rows_f32")
       for p in ("sides_host", "ld_sides_host", "coef_host", "d_sides_host", "ld_dsides_host")},
    ("llmrec_grad_init_f32", "regions_host"): "n_regions",
    ("llmrec_bpr_heads_f32", "heads_host"): "n_heads",
    ("llmrec_bpr_heads_ordered_f32", "heads_host"): "n_heads",
    **{("llmrec_adamw_step_f32", p): "n_tensors" for p in ("p_host", "g_host", "m_host", "v_host", "numel_host")},
    **{("llmrec_explain_f32", p): "n_side" for p in ("side_usr", "ld_side_usr", "side_src", "ld_side_src", "coef")},
    **{("llmrec_explain_f32", p): "n_id" for p in ("id_src", "ld_id")},
    ("llmrec_score_topk_group_f32", "member_rowptr_host"): "n_groups+1",
    ("llmrec_rank1_add_f32", "blocks_host"): "n_blocks",
    ("llmrec_scaled_colsum_f32", "terms_host"): "n_terms",
}

# the flags word of a grouped projection problem and the record type of the row maps that follow the problems (LLMREC_PROJ_ROW_MAP)
ROW_MAP_FLAG = {"llmrec_proj_fwd_problem": "_reserved", "llmrec_proj_wgrad_problem": "accumulate"}
ROW_MAP_BIT = 2
ROW_MAP_RECORD = "llmrec_proj_row_map"

# calls that wait for the stream's earlier work before they return (a copy out of pageable host memory; include/llmrec_b200.h)
HOST_SYNCING = {"llmrec_score_topk_group_f32"}


def length_of(fn, name):
    return LENGTHS.get((fn, name))


def host_array_params(hdr, fn):
    """The pointer parameters of `fn` that are HOST arrays: struct arrays, pointer tables, `_host` names, and the arrays LENGTHS names."""
    out = []
    for p in hdr.functions[fn]:
        if p.stars == 0:
            continue
        if p.stars >= 2 or p.base in hdr.structs or p.name.endswith("_host") or (fn, p.name) in LENGTHS:
            out.append(p)
    return out


def roles(hdr, fn):
    """name -> role description of every pointer parameter of a stream function:
    ("dev", r|w)             a device pointer;
    ("table", r|w)           a host table of device pointers, each with that role;
    ("structs", typedef)     a host array of structs (fields by typedef);
    ("host", None)           host data without device pointers (ld tables, coefficients, row pointers read on the host)."""
    out, host = {}, {p.name for p in host_array_params(hdr, fn)}
    for p in hdr.functions[fn]:
        if p.stars == 0 or p.ctype == "llmrec_stream_t":
            continue
        if p.stars >= 2:
            out[p.name] = ("table", READ if p.pointee_const else WRITE)
        elif p.base in hdr.structs:
            out[p.name] = ("structs", p.base)
        elif p.name in host:
            out[p.name] = ("host", None)
        else:
            out[p.name] = ("dev", READ if p.pointee_const else WRITE)
    return out


def field_roles(hdr, typedef):
    """field name -> r|w for the pointer fields of a header struct"""
    return {f.name: (READ if f.pointee_const else WRITE) for f in hdr.structs[typedef] if f.stars}


# ABI arguments narrowed from their allocation to the rectangle the call names: (function, "array.field" or "param") ->
# (rows, cols, ld) in 4-byte elements, from the call's arguments `a` and the struct element `s`.
#   spmm_csr segments   X is [n_cols x d] at ldx, Y and Z are [n_rows x d] at ldy / ldz: the column blocks of Pi / Fu / Fi / GFu / GFi /
#                       GPi that one launch reads and writes next to blocks of the same buffer other launches touch;
#   grad_init regions   G and X are [n x width] at ldg / ldx: the feat_reg blocks and the zeroed blocks of GFu / GFi;
#   rank1_add blocks    Y is [n x width] at ldy: the column blocks of the hoisted engine's compact Fu / Fi.
NARROW = {
    ("llmrec_spmm_csr_f32", "segs_host.X"): lambda a, s: (a["n_cols"], a["d"], s.ldx),
    ("llmrec_spmm_csr_f32", "segs_host.Y"): lambda a, s: (a["n_rows"], a["d"], s.ldy),
    ("llmrec_spmm_csr_f32", "segs_host.Z"): lambda a, s: (a["n_rows"], a["d"], s.ldz),
    ("llmrec_grad_init_f32", "regions_host.G"): lambda a, s: (s.n, s.width, s.ldg),
    ("llmrec_grad_init_f32", "regions_host.X"): lambda a, s: (s.n, s.width, s.ldx),
    ("llmrec_rank1_add_f32", "blocks_host.Y"): lambda a, s: (s.n, s.width, s.ldy),
}


# ---- extents ------------------------------------------------------------------------------------------------------------------------


@dataclass
class Extent:
    """Bytes of one allocation: `blocks` of rows (start, n_rows, row bytes, ld bytes); key = (space, allocation start)."""
    key: tuple
    blocks: list
    label: str = ""

    def overlaps(self, other):
        if self.key != other.key:
            return False
        return any(_blocks_overlap(a, b) for a in self.blocks for b in other.blocks)


def _uniform_overlap(a0, na, wa, b0, nb, wb, ld):
    """rows [a0 + i ld, + wa), i < na and [b0 + j ld, + wb), j < nb: does any pair intersect?  With D = b0 - a0 and k = j - i the rows
    meet when -D - wb < k ld < wa - D."""
    D = b0 - a0
    k_lo = (-D - wb) // ld + 1
    k_hi = -((D - wa) // ld) - 1
    return max(k_lo, -(na - 1)) <= min(k_hi, nb - 1)


def _blocks_overlap(a, b):
    a0, na, wa, la = a
    b0, nb, wb, lb = b
    if wa <= 0 or wb <= 0 or na <= 0 or nb <= 0:
        return False
    if a0 + (na - 1) * la + wa <= b0 or b0 + (nb - 1) * lb + wb <= a0:
        return False
    if na == 1 and nb == 1:
        return True
    if na == 1 or nb == 1 or la == lb:
        ld = lb if na == 1 else la
        return _uniform_overlap(a0, na, wa, b0, nb, wb, ld)
    if min(na, nb) <= 1 << 16:                                   # different leading dimensions: row by row of the shorter one
        if na > nb:
            a, b = b, a
            a0, na, wa, la = a
            b0, nb, wb, lb = b
        return any(_uniform_overlap(a0 + i * la, 1, wa, b0, nb, wb, lb) for i in range(na))
    return True                                                  # (conservative)


def tensor_extent(t, label=""):
    """Exact strided bytes of a tensor (size-1 and stride-0 dims dropped, contiguous dims merged)."""
    space = "dev" if t.is_cuda else "host"
    key = (space, t.untyped_storage().data_ptr())
    isz = t.element_size()
    start = t.data_ptr()
    dims = [(s, st) for s, st in zip(t.shape, t.stride()) if s > 1 and st != 0]
    if t.numel() == 0:
        return Extent(key, [], label)
    if any(st < 0 for _, st in dims):                            # (envelope)
        lo = start + sum((s - 1) * st for s, st in dims if st < 0) * isz
        hi = start + sum((s - 1) * st for s, st in dims if st > 0) * isz + isz
        return Extent(key, [(lo, 1, hi - lo, hi - lo)], label)
    dims.sort(key=lambda x: -x[1])
    merged = []
    for s, st in dims:
        if merged and merged[-1][1] == s * st:
            merged[-1] = (merged[-1][0] * s, st)
        else:
            merged.append((s, st))
    if merged and merged[-1][1] == 1:
        inner = merged.pop()[0] * isz
    else:
        inner = isz
    if not merged:
        return Extent(key, [(start, 1, inner, inner)], label)
    rows, ld = merged.pop()
    starts = [start]
    for s, st in merged:
        starts = [b + i * st * isz for b in starts for i in range(s)]
        if len(starts) > 4096:
            lo = start
            hi = start + sum((s_ - 1) * st_ for s_, st_ in dims) * isz + isz
            return Extent(key, [(lo, 1, hi - lo, hi - lo)], label)
    return Extent(key, [(b, rows, inner, ld * isz) for b in starts], label)


# ---- accesses, clocks and the check --------------------------------------------------------------------------------------------------

HOST = "host"


@dataclass
class Access:
    idx: int
    name: str                   # ABI function, aten op, or "host write"
    stream: object              # stream handle (int) or HOST
    clock: dict
    reads: list
    writes: list
    where: str

    @property
    def epoch(self):
        return self.clock[self.stream]


@dataclass
class Race:
    a: Access
    b: Access
    ea: Extent
    eb: Extent
    wa: bool                    # a's side of the pair is a write
    wb: bool


class Clocks:
    """Vector clocks: one per stream, one for the host.  Pure bookkeeping (the CPU tests drive it with hand-written traces)."""

    def __init__(self):
        self.vc = {HOST: {HOST: 0}}
        self.events = {}        # id(event) -> (event, clock)
        self.accesses = []
        self.graph_end = {}     # id(graph) -> (graph, clock at the end of its capture)

    @staticmethod
    def _join(a, b):
        for k, v in b.items():
            if a.get(k, 0) < v:
                a[k] = v

    def _stream(self, s):
        c = self.vc.get(s)
        if c is None:
            c = self.vc[s] = {s: 0}
        self._join(c, self.vc[HOST])                              # enqueued after everything the host has waited for
        return c

    def access(self, s, name, reads, writes, where=""):
        c = self.vc[HOST] if s == HOST else self._stream(s)
        c[s] = c.get(s, 0) + 1
        a = Access(len(self.accesses), name, s, dict(c), list(reads), list(writes), where)
        self.accesses.append(a)
        return a

    def record(self, ev, s):
        self.events[id(ev)] = (ev, dict(self._stream(s)))

    def wait(self, ev, s):
        c = self._stream(s)
        rec = self.events.get(id(ev))
        if rec is not None:                                       # a never-recorded event adds no edge
            self._join(c, rec[1])

    def event_sync(self, ev):
        rec = self.events.get(id(ev))
        if rec is not None:
            self._join(self.vc[HOST], rec[1])

    def stream_sync(self, s):
        self._join(self.vc[HOST], self._stream(s))

    def device_sync(self):
        for s, c in list(self.vc.items()):
            if s != HOST:
                self._join(self.vc[HOST], c)

    def capture_end(self, graph, s):
        self.graph_end[id(graph)] = (graph, dict(self._stream(s)))

    def replay(self, graph, s):
        rec = self.graph_end.get(id(graph))
        if rec is not None:
            self._join(self._stream(s), rec[1])

    @staticmethod
    def ordered(a, b):
        """a happens before b"""
        return b.clock.get(a.stream, 0) >= a.epoch

    def races(self, limit=200):
        by_key = {}
        for a in self.accesses:
            for w, exts in ((False, a.reads), (True, a.writes)):
                for e in exts:
                    by_key.setdefault(e.key, []).append((a, w, e))
        out, seen = [], set()
        for items in by_key.values():
            if len({a.stream for a, _, _ in items}) < 2 or not any(w for _, w, _ in items):
                continue
            for i, (a, wa, ea) in enumerate(items):
                for b, wb, eb in items[i + 1:]:
                    if a.stream == b.stream or not (wa or wb):
                        continue
                    x, y, ex, ey, wx, wy = (a, b, ea, eb, wa, wb) if a.idx < b.idx else (b, a, eb, ea, wb, wa)
                    if (x.idx, y.idx) in seen or self.ordered(x, y) or not ex.overlaps(ey):
                        continue
                    seen.add((x.idx, y.idx))
                    out.append(Race(x, y, ex, ey, wx, wy))
                    if len(out) >= limit:
                        return out
        return out


# ---- the recorder on a live process ------------------------------------------------------------------------------------------------


def _where(depth=2):
    """the innermost llmrec_b200 source lines of the current Python stack"""
    f, out = sys._getframe(depth), []
    while f is not None and len(out) < 3:
        fn = f.f_code.co_filename
        if fn.startswith(PKG_DIR):
            out.append(f"{os.path.relpath(fn, REPO)}:{f.f_lineno}")
        f = f.f_back
    return " < ".join(out) or "(outside llmrec_b200)"


def _ptr(v):
    if v is None:
        return 0
    if isinstance(v, int):
        return v
    if isinstance(v, C.c_void_p):
        return v.value or 0
    if hasattr(v, "value") and isinstance(v.value, int):
        return v.value
    raise TypeError(f"not a pointer argument: {v!r}")


def _host_obj(v):
    """the ctypes object behind a host-array argument (byref, array, structure)"""
    return getattr(v, "_obj", v)


class _Blocks:
    """Allocated blocks of the CUDA caching allocator, from torch.cuda.memory_snapshot(), refreshed when the allocator's counters move."""

    def __init__(self, torch):
        self.torch, self.stamp, self.starts, self.ends = torch, None, [], []

    def _refresh(self, force=False):
        st = self.torch.cuda.memory_stats()
        stamp = (st.get("allocation.all.allocated", 0), st.get("allocation.all.freed", 0), st.get("segment.all.allocated", 0))
        if stamp == self.stamp and not force:
            return
        blocks = []
        for seg in self.torch.cuda.memory_snapshot():
            addr = seg["address"]
            for b in seg["blocks"]:
                if b["state"] in ("active_allocated", "active_pending_free"):
                    blocks.append((addr, b["size"]))
                addr += b["size"]
        blocks.sort()
        self.starts, self.ends, self.stamp = [s for s, _ in blocks], [s + n for s, n in blocks], stamp

    def find(self, p):
        for force in (False, True):
            self._refresh(force)
            i = bisect.bisect_right(self.starts, p) - 1
            if i >= 0 and p < self.ends[i]:
                return self.starts[i], self.ends[i] - self.starts[i]
        return None


class _LibProxy:
    def __init__(self, rec, lib):
        self._rec, self._lib = rec, lib

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("llmrec_"):
            return fn
        rec = self._rec

        def call(*args):
            if rec.on:
                rec._abi(name, args)
            rc = fn(*args)
            if rec.on and name in HOST_SYNCING:
                rec.clocks.stream_sync(_ptr(args[-1]))
            return rc
        return call


class Recorder:
    """Install with `install(monkeypatch)` (the patches go away with the monkeypatch); `on` switches recording; `races()` checks."""

    def __init__(self):
        import torch
        self.torch = torch
        self.hdr = parse_header()
        self.clocks = Clocks()
        self.on = False
        self.stream_names = {}
        self._blocks = _Blocks(torch)
        self._mode = None

    # -- installation --
    def install(self, monkeypatch, trainer_module=None):
        import torch
        from llmrec_b200 import _native as N
        rec, ck = self, self.clocks
        monkeypatch.setattr(N, "_lib", _LibProxy(self, N.lib()))
        cur = lambda: torch.cuda.current_stream().cuda_stream
        sid = lambda s: cur() if s is None else s.cuda_stream
        E, S = torch.cuda.Event, torch.cuda.Stream
        ev_record, ev_wait, ev_sync, st_sync, dev_sync = E.record, E.wait, E.synchronize, S.synchronize, torch.cuda.synchronize

        def record(ev, stream=None):
            ev_record(ev, stream)
            if rec.on:
                ck.record(ev, sid(stream))

        def wait(ev, stream=None):
            ev_wait(ev, stream)
            if rec.on:
                ck.wait(ev, sid(stream))

        def esync(ev):
            ev_sync(ev)
            if rec.on:
                ck.event_sync(ev)

        def ssync(st):
            st_sync(st)
            if rec.on:
                ck.stream_sync(st.cuda_stream)

        def dsync(device=None):
            dev_sync(device)
            if rec.on:
                ck.device_sync()

        monkeypatch.setattr(E, "record", record)
        monkeypatch.setattr(E, "wait", wait)
        monkeypatch.setattr(E, "synchronize", esync)
        monkeypatch.setattr(S, "synchronize", ssync)
        monkeypatch.setattr(torch.cuda, "synchronize", dsync)
        G = torch.cuda.CUDAGraph
        g_end, g_replay = G.capture_end, G.replay

        def capture_end(g):
            g_end(g)
            if rec.on:
                ck.capture_end(g, cur())

        def replay(g):
            if rec.on:
                ck.replay(g, cur())
            g_replay(g)

        monkeypatch.setattr(G, "capture_end", capture_end)
        monkeypatch.setattr(G, "replay", replay)
        if trainer_module is not None:
            T = trainer_module.Trainer
            next_slot = T._next_slot

            def staged(tr, need):
                slot = next_slot(tr, need)
                if rec.on:                                        # the host fills the slot from here on
                    ck.access(HOST, "host write", [], [tensor_extent(slot.host, "slot.host")], _where(1))
                return slot

            monkeypatch.setattr(T, "_next_slot", staged)
        self._mode = _aten_mode(self)
        self._mode.__enter__()
        self.main = cur()
        self.stream_names.setdefault(self.main, "main")
        return self

    def uninstall(self):
        if self._mode is not None:
            self._mode.__exit__(None, None, None)
            self._mode = None
        self.on = False

    def name_stream(self, stream, name):
        self.stream_names[stream.cuda_stream if hasattr(stream, "cuda_stream") else stream] = name

    # -- ABI calls --
    def _dev(self, fn, label, p, role, rect=None):
        hit = self._blocks.find(p)
        if hit is None:
            raise AssertionError(f"{fn}: {label} = {p:#x} lies outside every block of the CUDA caching allocator")
        start, size = hit
        if rect is None:
            return Extent(("dev", start), [(start, 1, size, size)], label), role
        rows, cols, ld = (int(x) for x in rect)
        return Extent(("dev", start), [(p, rows, 4 * cols, 4 * ld)], label), role

    def _abi(self, fn, args):
        params = self.hdr.functions[fn]
        if len(args) != len(params):
            raise AssertionError(f"{fn}: called with {len(args)} arguments, the header declares {len(params)}")
        a = {p.name: v for p, v in zip(params, args)}
        sname = self.hdr.stream_param(fn)
        if sname is None:
            for p in params:                                      # host functions never see device memory
                if p.stars == 1 and p.base not in self.hdr.structs:
                    v = _ptr(a[p.name])
                    if v and self._blocks.find(v) is not None:
                        raise AssertionError(f"{fn} runs on the host but {p.name} = {v:#x} is device memory")
            return
        ints = {p.name: int(getattr(a[p.name], "value", a[p.name]) or 0) for p in params if p.stars == 0 and p.ctype != "llmrec_stream_t"}
        acc = []
        for pname, (kind, what) in roles(self.hdr, fn).items():
            v = a[pname]
            if kind == "dev":
                p, nar = _ptr(v), NARROW.get((fn, pname))
                if p:
                    acc.append(self._dev(fn, pname, p, what, nar(ints, None) if nar else None))
                continue
            if kind == "host" or v is None:
                continue
            n = self._length(fn, pname, ints)
            obj = _host_obj(v)
            if kind == "table":
                for i in range(n):
                    p = _ptr(obj[i])
                    if p:
                        acc.append(self._dev(fn, f"{pname}[{i}]", p, what))
                continue
            struct_t, fr = what, field_roles(self.hdr, what)
            elems = [obj] if isinstance(obj, C.Structure) else [obj[i] for i in range(n)]
            for i, s in enumerate(elems):
                for f, role in fr.items():
                    p = _ptr(getattr(s, f))
                    if p:
                        nar = NARROW.get((fn, f"{pname}.{f}"))
                        acc.append(self._dev(fn, f"{pname}[{i}].{f}", p, role, nar(ints, s) if nar else None))
            flag = ROW_MAP_FLAG.get(re.sub(r"_(bf16|i8)$", "", struct_t))
            if flag and any(getattr(s, flag) & ROW_MAP_BIT for s in elems):
                base = C.addressof(obj) + n * C.sizeof(type(elems[0]))
                from llmrec_b200 import _native as N
                maps = (N.ProjRowMap * n).from_address(base)
                mr = field_roles(self.hdr, ROW_MAP_RECORD)
                for i, s in enumerate(elems):
                    if getattr(s, flag) & ROW_MAP_BIT:
                        for f, role in mr.items():
                            p = _ptr(getattr(maps[i], f))
                            if p:
                                acc.append(self._dev(fn, f"row_maps[{i}].{f}", p, role))
        reads = [e for e, r in acc if r == READ]
        writes = [e for e, r in acc if r == WRITE]
        self.clocks.access(_ptr(a[sname]), fn, reads, writes, _where(1))

    @staticmethod
    def _length(fn, pname, ints):
        n = LENGTHS[(fn, pname)]
        if isinstance(n, int):
            return n
        name, _, plus = n.partition("+")
        return ints[name] + int(plus or 0)

    # -- torch ops --
    def _aten(self, func, args, kwargs, out):
        torch = self.torch
        name = func.name()
        if func.is_view or name in _SKIP:
            return
        reads, writes, cuda, host_out = [], [], False, False
        schema = func._schema.arguments
        for i, arg in enumerate(schema):
            v = args[i] if i < len(args) else kwargs.get(arg.name)
            is_w = arg.alias_info is not None and arg.alias_info.is_write
            for t in _tensors(v):
                cuda |= t.is_cuda
                if t.is_cuda or t.is_pinned():
                    (writes if is_w else reads).append(tensor_extent(t, arg.name))
        for t in _tensors(out):
            cuda |= t.is_cuda
            host_out |= not t.is_cuda
            if t.is_cuda or t.is_pinned():
                writes.append(tensor_extent(t, "out"))
        if not cuda:
            return
        s = torch.cuda.current_stream().cuda_stream
        self.clocks.access(s, name, reads, writes, _where(1))
        blocking = not (kwargs.get("non_blocking") or (name == "aten::copy_" and len(args) > 2 and args[2]))
        if name in _SYNCING or (host_out and blocking and name in ("aten::copy_", "aten::_to_copy")) or \
                (name == "aten::copy_" and not args[0].is_cuda and blocking):
            self.clocks.stream_sync(s)

    # -- the check --
    def races(self):
        return self.clocks.races()

    def describe(self, race, names=None):
        def side(a, e, w):
            st = self.stream_names.get(a.stream, "host" if a.stream == HOST else f"stream {a.stream:#x}")
            return f"{a.name} [{st}] {'writes' if w else 'reads'} {e.label} at {a.where}"
        buf = ", ".join((names or {}).get(race.ea.key, [])) or f"allocation {race.ea.key[1]:#x} ({race.ea.key[0]})"
        return f"unordered: {side(race.a, race.ea, race.wa)}  <->  {side(race.b, race.eb, race.wb)}  on {buf}"

    def report(self, races, names=None, limit=12):
        lines = [self.describe(r, names) for r in races[:limit]]
        more = f"\n... {len(races) - limit} more" if len(races) > limit else ""
        return "\n".join(lines) + more


_SKIP = {"aten::empty", "aten::empty_strided", "aten::empty_like", "aten::new_empty", "aten::new_empty_strided", "aten::detach",
         "aten::alias", "aten::lift_fresh", "aten::record_stream", "aten::set_", "aten::resize_", "aten::_has_same_storage_numel",
         "aten::is_pinned", "aten::_pin_memory", "aten::size", "aten::stride", "aten::sym_size", "aten::sym_stride", "aten::dim"}
# ops whose result the host reads before it continues
_SYNCING = {"aten::_local_scalar_dense", "aten::nonzero", "aten::_unique2", "aten::unique_dim", "aten::unique_consecutive",
            "aten::masked_select", "aten::is_nonzero", "aten::equal"}


def _tensors(v):
    import torch
    if isinstance(v, torch.Tensor):
        if v.layout == torch.strided:
            yield v
    elif isinstance(v, (list, tuple)):
        for x in v:
            yield from _tensors(x)


def _aten_mode(rec):
    from torch.utils._python_dispatch import TorchDispatchMode

    class _AtenRecorder(TorchDispatchMode):
        def __torch_dispatch__(self, func, types, args=(), kwargs=None):
            kwargs = kwargs or {}
            out = func(*args, **kwargs)
            if rec.on:
                rec._aten(func, args, kwargs, out)
            return out

    return _AtenRecorder()


# ---- buffer names --------------------------------------------------------------------------------------------------------------------


def buffer_names(**roots):
    """(space, allocation start) -> attribute paths of the tensors found under `roots` (engine, trainer, samplers, ...): attributes of
    llmrec_b200 objects, dict entries and list items, a few levels deep."""
    import torch
    out, seen = {}, set()
    todo = [(name, obj, 0) for name, obj in roots.items()]
    while todo:
        path, obj, depth = todo.pop(0)
        if id(obj) in seen or depth > 5:
            continue
        seen.add(id(obj))
        if isinstance(obj, torch.Tensor):
            if obj.device.type == "meta" or obj.layout != torch.strided:
                continue
            key = ("dev" if obj.is_cuda else "host", obj.untyped_storage().data_ptr())
            if len(out.setdefault(key, [])) < 4:
                out[key].append(path)
            continue
        if isinstance(obj, dict) and len(obj) <= 256:                # (the long ones are id tables of the data loader)
            todo += [(f"{path}[{k!r}]" if not isinstance(k, str) else f"{path}[{k}]", v, depth + 1) for k, v in obj.items()]
        elif isinstance(obj, (list, tuple)) and len(obj) <= 64:
            todo += [(f"{path}[{i}]", v, depth + 1) for i, v in enumerate(obj)]
        elif hasattr(obj, "__dict__") and any(c.__module__.startswith("llmrec_b200") for c in type(obj).__mro__):
            todo += [(f"{path}.{k}", v, depth + 1) for k, v in vars(obj).items()]
    return out
