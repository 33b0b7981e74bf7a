"""CPU stand-in for the device sampler on the reference's streams (`llmrec_device_sample_batch_ref`, `--device_sampler 2`).  TEST
INFRASTRUCTURE ONLY, like tests/ops_emulator.py, which it leaves unchanged: `install()` patches a test process so that
`ReferenceDeviceSampler` draws each batch with the host C sampler (`llmrec_host_sample_batch`) on the state tensor's two streams, writes
the index buffer and meta row as the kernel does, and keeps the kernel's error word.  The Trainer plumbing around the sampler -- state
uploads and downloads, checkpoints, the warm-up undo -- then runs without a GPU."""
import numpy as np

from llmrec_b200 import _native as N
from llmrec_b200.device_sampler import _ERR, _NP, _PY, ReferenceDeviceSampler


def _launch(self, index_buffer, meta_table):
    s = self.state.numpy()
    B = self.batch
    cap = int(index_buffer.shape[1])
    out = index_buffer.numpy()
    if s[_ERR] == 0:
        work = np.zeros((3, cap), dtype=np.int32)
        py_key, np_key = s[_PY:_PY + 624].view(np.uint32).copy(), s[_NP:_NP + 624].view(np.uint32).copy()
        pos = np.array([s[_PY + 624], s[_NP + 624], 0], dtype=np.int32)
        n = int(self.exist.numel())
        stamp = np.zeros(max(n, 1), dtype=np.int32)
        pool = np.empty(max(n, 2 * B) + 8, dtype=np.int32)
        arr = lambda t: np.ascontiguousarray(t.numpy()) if t is not None else None
        exist, rowptr, col, ap, an = arr(self.exist), arr(self.rowptr), arr(self.col), arr(self.aug_pos), arr(self.aug_neg)
        rc = N.lib().llmrec_host_sample_batch(
            py_key.ctypes.data, pos[0:].ctypes.data, np_key.ctypes.data, pos[1:].ctypes.data, exist.ctypes.data, n, B, int(self.users_pool),
            rowptr.ctypes.data, col.ctypes.data, self.n_items, self.n_aug, int(self.aug_pool),
            ap.ctypes.data if self.n_aug else 0, an.ctypes.data if self.n_aug else 0, ap.shape[0] if self.n_aug else 0, self.aug_limit,
            stamp.ctypes.data, 1, pool.ctypes.data, work.ctypes.data, cap, pos[2:].ctypes.data)
        if rc == 0:
            Bp = int(pos[2])
            out[:3, :Bp] = work[:, :Bp]
            out[3, :2] = meta_table[Bp].numpy()
            s[_PY:_PY + 624], s[_PY + 624] = py_key.view(np.int32), pos[0]
            s[_NP:_NP + 624], s[_NP + 624] = np_key.view(np.int32), pos[1]
            return
        s[_ERR] = rc
    out[:3, :B] = 0                                    # the kernel's placeholder batch: user 0 / item 0, B' = batch
    out[3, :2] = meta_table[B].numpy()


def install():
    ReferenceDeviceSampler._launch = _launch
