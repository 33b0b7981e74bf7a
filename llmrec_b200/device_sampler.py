"""Device-side batch sampler (`--device_sampler 1`; SURVEY.md 8f-1): Data.sample() (utility/load_data.py:157-195) and the
augmented-edge step (main.py:216-224) as one kernel that fills the engine's static index buffer, so a replayed training step needs no
host sampler and no H2D copy.  Same distributions as the reference, NOT its RNG streams -- the parity default stays the host replay
(host_native.BatchSampler)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native as N
from . import ops


class DeviceSampler:
    def __init__(self, exist_users, train_rowptr, train_col_sorted, n_items, batch_size, aug_pos, aug_neg, aug_limit, aug_rate, device, seed=0):
        """Raises what the host sampler raises when an exist user has no train item or no possible negative, and ValueError when a train
        row is not sorted ascending: the kernel assumes all three (its binary search and its negative draw)."""
        check_device_sampler_inputs(exist_users, train_rowptr, train_col_sorted, n_items)
        dev = torch.device(device)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)
        self.exist, self.rowptr, self.col = t(exist_users), t(train_rowptr), t(train_col_sorted)
        self.n_items, self.batch = int(n_items), int(batch_size)
        self.n_aug = int(self.batch * aug_rate) if aug_pos is not None else 0          # int(len(users) * rate), main.py:218
        self.aug_pos = t(aug_pos) if aug_pos is not None else None
        self.aug_neg = t(aug_neg) if aug_neg is not None else None
        self.aug_limit = int(aug_limit)
        self.state = torch.tensor([int(seed), 0], dtype=torch.int64, device=dev)       # {seed, step}; the kernel advances step
        self.keys = torch.zeros(max(int(self.exist.numel()), self.batch), dtype=torch.int32, device=dev)

    def fill(self, index_buffer, meta_table):
        """index_buffer: the engine's [4 x cap] int32 buffer; meta_table: [cap + 1, 2] int32 {B', n_keep}.  One launch on the current stream."""
        cap = int(index_buffer.shape[1])
        N.check(N.lib().llmrec_device_sample_batch(
            C.c_void_p(self.exist.data_ptr()), self.exist.numel(), self.batch, C.c_void_p(self.rowptr.data_ptr()), C.c_void_p(self.col.data_ptr()),
            self.n_items, self.n_aug, C.c_void_p(self.aug_pos.data_ptr()) if self.n_aug else None, C.c_void_p(self.aug_neg.data_ptr()) if self.n_aug else None,
            self.aug_pos.numel() if self.n_aug else 0, self.aug_limit, C.c_void_p(meta_table.data_ptr()), cap, C.c_void_p(self.state.data_ptr()),
            C.c_void_p(index_buffer.data_ptr()), C.c_void_p(self.keys.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "device_sample_batch")
        ops._count()


def check_device_sampler_inputs(exist_users, train_rowptr, train_col_sorted, n_items):
    """The precondition of llmrec_device_sample_batch: every exist user has 1 <= deg < n_items, and every train row is sorted ascending."""
    rowptr = np.asarray(train_rowptr, dtype=np.int64)
    col = np.asarray(train_col_sorted)
    exist = np.asarray(exist_users, dtype=np.int64)
    deg = rowptr[exist + 1] - rowptr[exist]
    if (deg <= 0).any():
        raise_sampler_error(2)
    if (deg >= int(n_items)).any():
        raise_sampler_error(3)
    down = np.flatnonzero(col[1:] < col[:-1]) + 1                     # positions whose item is below the one before it
    starts = np.zeros(len(col) + 1, dtype=bool)
    starts[rowptr[:-1][rowptr[:-1] < len(col)]] = True
    if (~starts[down]).any():
        j = int(down[~starts[down]][0])
        u = int(np.searchsorted(rowptr, j, side="right") - 1)
        raise ValueError(f"device sampler: train row {u} is not sorted ascending (items {int(col[j - 1])}, {int(col[j])}); "
                         "the kernel's binary search needs sorted rows")


STATE_ELEMS = 1252                      # LLMREC_REF_SAMPLER_STATE_ELEMS: random key[624], pos, numpy key[624], pos, error, pad
_PY, _NP, _ERR = 0, 625, 1250


def raise_sampler_error(rc):
    """The exception host_native.BatchSampler.draw raises for the same return code."""
    if rc == 4:
        raise KeyError("a sampled user is missing from augmented_sample_dict")
    if rc == 5:
        raise RuntimeError("device batch sampler gave up (rc=5): a rejection loop drew 2^24 words without accepting one")
    raise RuntimeError(f"native batch sampler failed (rc={rc}): a sampled user has no train items or no possible negative")


class ReferenceDeviceSampler:
    """`--device_sampler 2`: the batches of host_native.BatchSampler -- CPython's `random` and numpy's global MT19937 streams, bit for bit --
    drawn on the GPU by one launch (csrc/device_sampler_ref.cu), so it can sit inside a captured step.

    Two ways to use it.  `fill(buffer, meta_table)` draws one batch into `buffer` on the current stream.  A training step uses `attach()`
    instead: the sampler keeps the NEXT batch pre-drawn in a buffer of its own; `step_begin()` copies it into the engine's index buffer and
    draws the one after it on a side stream, beside the step, and `step_end()` joins that stream back at the end of the step.  The draw reads
    only the streams, the train CSR and the augmentation tables, which no step writes, so the step does not wait for it.

    While batches are drawn on the device the device copies of the two streams are the live ones.  `sync_to_host()` writes them back into
    `random` / `np.random` -- with a batch pre-drawn, the streams as they were BEFORE that batch, which is where a host-sampled run stands
    after the batches consumed so far.  `upload_from_host()` goes the other way, in place (a captured launch holds the state's address), and
    draws the pending batch again from the uploaded streams.  `host_is_current`: no batch was consumed since the last of the two, so the
    host streams may still be reseeded and uploaded again.

    A failing draw (a user without train items or without a possible negative, a uid missing from the augmentation tables) cannot raise on
    the device: it sets an error word and every later call draws nothing.  Once a step has consumed the failed batch, the host's next
    synchronisation (`check()`, `sync_to_host()`) raises the host sampler's exception.  Steps run between the failing draw and that check
    train on a placeholder batch and mean nothing; the reference itself raises (or loops forever) at that batch."""

    def __init__(self, exist_users, train_rowptr, train_col, train_col_sorted, n_items, batch_size, aug_pos, aug_neg, aug_limit, aug_rate,
                 device):
        """train_col: the rows in the host sampler's order (Data.csr("train")); train_col_sorted: the same rows sorted ascending"""
        from .host_native import _sample_uses_pool
        dev = self.device = torch.device(device)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)
        self.exist, self.rowptr, self.col, self.col_sorted = t(exist_users), t(train_rowptr), t(train_col), t(train_col_sorted)
        self.n_items, self.batch = int(n_items), int(batch_size)
        n = int(self.exist.numel())
        self.n_aug = int(self.batch * aug_rate) if aug_pos is not None else 0          # int(len(users) * rate), main.py:218
        self.users_pool = self.batch <= n and _sample_uses_pool(n, self.batch)
        self.aug_pool = bool(self.n_aug) and _sample_uses_pool(self.batch, self.n_aug)
        self.aug_pos = t(aug_pos) if self.n_aug else None
        self.aug_neg = t(aug_neg) if self.n_aug else None
        self.aug_limit = int(aug_limit)
        self.state = torch.zeros(STATE_ELEMS, dtype=torch.int32, device=dev)
        self.prev = torch.zeros_like(self.state)        # the streams before the pre-drawn batch
        self.work = torch.zeros(max(int(N.lib().llmrec_device_sample_batch_ref_work(n, self.batch, int(self.users_pool), int(self.aug_pool))), 1),
                                dtype=torch.int32, device=dev)
        self.index_buffer = self.next = None
        self._saved = None
        self.upload_from_host()

    # ---- the two streams ----------------------------------------------------------------------------------------------------------
    @staticmethod
    def host_state():
        """int32[STATE_ELEMS] of the current `random` / `np.random` streams, error word 0."""
        import random
        version, py_state, _ = random.getstate()
        name, np_key, np_pos, _, _ = np.random.get_state()
        if version != 3 or name != "MT19937":
            raise RuntimeError("unexpected random / np.random generator")
        s = np.zeros(STATE_ELEMS, dtype=np.uint32)
        s[_PY:_PY + 625] = py_state
        s[_NP:_NP + 624] = np_key
        s[_NP + 624] = np_pos
        return torch.from_numpy(s.view(np.int32))

    def _consumed(self):
        """the streams after the batches consumed so far"""
        return self.prev if self.next is not None else self.state

    def upload_from_host(self):
        """The device streams := the host's; clears the error word; an attached sampler draws its pending batch again.  In place."""
        self.state.copy_(self.host_state())
        if self.next is not None:
            self._predraw()
        self.host_is_current = True

    def check(self):
        """Raise the host sampler's exception if a consumed batch failed to draw (synchronises)."""
        rc = int(self._consumed()[_ERR])
        if rc:
            raise_sampler_error(rc)

    def sync_to_host(self):
        """`random` / `np.random` := the device streams after the consumed batches (synchronises); raises instead when one of them failed."""
        import random
        s = self._consumed().cpu().numpy()
        if s[_ERR]:
            raise_sampler_error(int(s[_ERR]))
        u = s.view(np.uint32)
        _, _, gauss = random.getstate()
        random.setstate((3, tuple(int(x) for x in u[_PY:_PY + 624]) + (int(s[_PY + 624]),), gauss))
        _, _, _, has_gauss, cached = np.random.get_state()
        np.random.set_state(("MT19937", u[_NP:_NP + 624].copy(), int(s[_NP + 624]), has_gauss, cached))
        self.host_is_current = True

    # ---- one batch into a given buffer ---------------------------------------------------------------------------------------------
    def fill(self, index_buffer, meta_table):
        """index_buffer: a [4 x cap] int32 buffer (rows users / pos / neg / {B', n_keep}); meta_table: [cap + 1, 2] int32 {B', n_keep}.
        One launch on the current stream; the device streams advance by one batch."""
        self.host_is_current = False
        self._launch(index_buffer, meta_table)

    # ---- batches for a training step, pre-drawn beside the step before ------------------------------------------------------------
    def attach(self, index_buffer, meta_table, side_stream=True):
        """Feed the engine's index buffer: draw the first batch now.  side_stream: draw the next batch on a stream of its own (False: on
        the step's stream, after the copy)."""
        self.index_buffer, self.meta_table = index_buffer, meta_table
        self.next = torch.zeros_like(index_buffer)
        self._side = torch.cuda.Stream(self.device) if side_stream and self.device.type == "cuda" else None
        if self._side is not None:
            self._ev_fork, self._ev_done = torch.cuda.Event(), torch.cuda.Event()
        self._predraw()

    def _predraw(self):
        self.prev.copy_(self.state)
        self._launch(self.next, self.meta_table)

    def step_begin(self):
        """The pre-drawn batch -> the index buffer; the next batch is drawn beside the step (inside a capture too)."""
        self.host_is_current = False
        self.index_buffer.copy_(self.next)
        if self._side is None:
            self._predraw()
            return
        main = torch.cuda.current_stream(self.device)
        self._ev_fork.record(main)
        self._side.wait_event(self._ev_fork)
        with torch.cuda.stream(self._side):
            self._predraw()
            self._ev_done.record(self._side)

    def step_end(self):
        if self._side is not None:
            torch.cuda.current_stream(self.device).wait_event(self._ev_done)

    def save(self):
        """Keep what one step_begin changes (the graph warm-up step hands its batch back with `undo`)."""
        self._saved = (self.state.clone(), self.prev.clone(), self.next.clone())

    def undo(self):
        for dst, src in zip((self.state, self.prev, self.next), self._saved):
            dst.copy_(src)
        self._saved = None

    def _launch(self, index_buffer, meta_table):
        cap = int(index_buffer.shape[1])
        ptr = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None
        N.check(N.lib().llmrec_device_sample_batch_ref(
            ptr(self.exist), self.exist.numel(), self.batch, int(self.users_pool), ptr(self.rowptr), ptr(self.col), ptr(self.col_sorted), self.n_items,
            self.n_aug, int(self.aug_pool), ptr(self.aug_pos), ptr(self.aug_neg), self.aug_pos.numel() if self.n_aug else 0, self.aug_limit,
            ptr(meta_table), cap, ptr(self.state), ptr(index_buffer), ptr(self.work), self.work.numel(),
            C.c_void_p(torch.cuda.current_stream().cuda_stream)), "device_sample_batch_ref")
        ops._count()
