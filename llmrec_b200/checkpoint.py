"""Checkpoints of a training run: the file format, the durable write and the validated read.

One file, written with torch.save: a plain dict of CPU tensors and Python scalars / tuples / dicts, no pickled project class, so it loads
with `torch.load(path, weights_only=True)`.  Sections:

  format       1
  model        {reference parameter name: fp32 contiguous tensor}; goes straight into MM_Model.load_state_dict(..., strict=False).  The
               unused batch_norm and the feature tables (constants of the data set, in any --feat_dtype) are not saved.
  optim        m, v ({name: tensor}), state (AdamW's fp64[4] device step block, verbatim), lr, betas, eps, weight_decay
  rng          Python's `random`, numpy's legacy global MT19937 (the streams the host samplers advance), torch's CPU and CUDA generators,
               each as tensors / ints, and the device sampler's {seed, step} when there is one
  loop         where Trainer.train() continues: next epoch, next batch inside it, the epoch's loss accumulators, early-stopping counters
  fingerprint  must: shapes of the data set and the model, a mismatch raises; recorded: the flags a bit-exact resume needs equal, a
               difference is reported to the caller (continuing at another --lr is legitimate)

Writing goes to `path + ".tmp"` in the same directory, is flushed and fsync'ed, and then replaces `path`: a reader never sees a
half-written file and a crash during a save keeps the previous checkpoint.  Reading validates the whole file against the live tensors
before the caller copies anything, so a failed load changes nothing.
"""
from __future__ import annotations

import os
import random

import numpy as np
import torch

FORMAT = 1
SECTIONS = ("model", "optim", "rng", "loop", "fingerprint")
LOOP_KEYS = ("epoch", "batch", "epoch_stats", "best_recall", "stopping_step", "test_ret", "n_interactions")


def engine_tensors(engine):
    """The engine's `state_tensors()`; engines that keep their state per rank have none to offer."""
    if not hasattr(engine, "state_tensors"):
        raise ValueError(f"checkpoints cover the single-GPU engines (engine.HotPath, hoist.HoistedHotPath); {type(engine).__name__} keeps its "
                         "parameters and moments per rank")
    return engine.state_tensors()


def to_host(tensors):
    """name -> contiguous CPU copy.  A view with a leading dimension larger than its width comes out without its padding.  CUDA
    sources are copied asynchronously into pinned memory; the one synchronize at the end completes them all."""
    out, on_device = {}, False
    for k, t in tensors.items():
        t = t.detach()
        h = torch.empty(t.shape, dtype=t.dtype, pin_memory=t.is_cuda)
        h.copy_(t, non_blocking=True)
        on_device |= t.is_cuda
        out[k] = h
    if on_device:
        torch.cuda.synchronize()
    return out


def engine_sections(host, opt):
    """The `model` and `optim` sections from the host copies of `state_tensors()` and the optimizer's hyper-parameters."""
    pick = lambda sec: {k[len(sec) + 1:]: t for k, t in host.items() if k.startswith(sec + "/")}
    return pick("model"), dict(m=pick("m"), v=pick("v"), state=host["state"], lr=float(opt.lr), betas=tuple(float(b) for b in opt.betas),
                               eps=float(opt.eps), weight_decay=float(opt.wd))


def _flat(ck):
    """The inverse of `engine_sections`: the keys of `state_tensors()`."""
    out = {"model/" + k: t for k, t in ck["model"].items()}
    out.update({"m/" + k: t for k, t in ck["optim"]["m"].items()})
    out.update({"v/" + k: t for k, t in ck["optim"]["v"].items()})
    out["state"] = ck["optim"]["state"]
    return out


# ---- the RNG streams ----------------------------------------------------------------------------------------------------------------
# The C host sampler keeps no stream of its own: host_native.BatchSampler.draw advances Python's `random` and numpy's global MT19937 in
# place.  Its `stamp` / `epoch` / `pool` members are scratch and are left out: `stamp[j] == epoch` marks a position as drawn in THIS call,
# `epoch` is new for every call (a fresh sampler starts at 1 over a zeroed stamp array, so no stale mark can match), and `pool` is filled
# before it is read (csrc/host_sampler.cu, py_sample).
def rng_state(device, sampler_state=None):
    """sampler_state: the host copy of DeviceSampler.state ({seed, step}, its whole state) when the batches are drawn on the GPU"""
    version, key, gauss = random.getstate()
    name, np_key, np_pos, has_gauss, cached = np.random.get_state()
    if version != 3 or name != "MT19937":
        raise RuntimeError("unexpected random / np.random generator")
    out = dict(py_key=torch.tensor(key, dtype=torch.int64), py_gauss=gauss, np_key=torch.from_numpy(np_key.astype(np.int64)), np_pos=int(np_pos),
               np_has_gauss=int(has_gauss), np_cached=float(cached), torch_cpu=torch.get_rng_state())
    if device.type == "cuda":
        out["torch_cuda"] = torch.cuda.get_rng_state(device)
    if sampler_state is not None:
        out["device_sampler"] = sampler_state
    return out


def set_rng_state(rng, device, device_sampler=None):
    random.setstate((3, tuple(rng["py_key"].tolist()), rng["py_gauss"]))
    np.random.set_state(("MT19937", rng["np_key"].numpy().astype(np.uint32), rng["np_pos"], rng["np_has_gauss"], rng["np_cached"]))
    torch.set_rng_state(rng["torch_cpu"])
    if device.type == "cuda" and "torch_cuda" in rng:
        torch.cuda.set_rng_state(rng["torch_cuda"], device)
    if device_sampler is not None and "device_sampler" in rng:
        device_sampler.state.copy_(rng["device_sampler"])              # in place: the captured sampler launch reads this address


def _check_rng(rng, path):
    want = dict(py_key=((625,), torch.int64), np_key=((624,), torch.int64), torch_cpu=(None, torch.uint8))
    for k, (shape, dtype) in want.items():
        t = rng.get(k)
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or (shape is not None and tuple(t.shape) != shape):
            raise ValueError(f"{path}: rng/{k} is missing or malformed")
    for k in ("py_gauss", "np_pos", "np_has_gauss", "np_cached"):
        if k not in rng:
            raise ValueError(f"{path}: rng/{k} is missing")
    s = rng.get("device_sampler")
    if s is not None and (not isinstance(s, torch.Tensor) or s.dtype != torch.int64 or tuple(s.shape) != (2,)):
        raise ValueError(f"{path}: rng/device_sampler is malformed")


# ---- write / read -------------------------------------------------------------------------------------------------------------------
def write(path, model, optim, rng, loop, fingerprint):
    payload = dict(format=FORMAT, model=model, optim=optim, rng=rng, loop=loop, fingerprint=fingerprint)
    path = os.fspath(path)
    folder = os.path.dirname(os.path.abspath(path))
    os.makedirs(folder, exist_ok=True)
    tmp = path + ".tmp"
    try:
        with open(tmp, "wb") as f:
            torch.save(payload, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    fd = os.open(folder, os.O_RDONLY)                                  # the rename itself reaches the disk
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def read(path, fingerprint, live):
    """Load and validate `path` against this run: `fingerprint` = dict(must, recorded) of the live Trainer, `live` = its engine's
    `state_tensors()`.  -> (checkpoint dict, the `state_tensors` keys -> saved tensors, ["flag: saved -> now", ...] for the recorded
    fields that differ).  Raises ValueError, before anything of the caller's has been touched."""
    try:
        ck = torch.load(path, map_location="cpu", weights_only=True)
    except FileNotFoundError:
        raise
    except Exception as e:
        raise ValueError(f"{path}: not a readable checkpoint ({type(e).__name__}: {e})") from e
    if not isinstance(ck, dict) or ck.get("format") != FORMAT:
        raise ValueError(f"{path}: checkpoint format {ck.get('format') if isinstance(ck, dict) else None!r}, this version reads format {FORMAT}")
    for sec in SECTIONS:
        if not isinstance(ck.get(sec), dict):
            raise ValueError(f"{path}: section '{sec}' is missing")
    fp = ck["fingerprint"]
    for cls in ("must", "recorded"):
        if not isinstance(fp.get(cls), dict):
            raise ValueError(f"{path}: fingerprint/{cls} is missing")
    for k, want in fingerprint["must"].items():
        if k not in fp["must"]:
            raise ValueError(f"{path}: fingerprint/{k} is missing")
        if fp["must"][k] != want:
            raise ValueError(f"{path}: {k} is {fp['must'][k]!r} in the checkpoint and {want!r} in this run")
    for k in ("m", "v", "state"):
        if k not in ck["optim"]:
            raise ValueError(f"{path}: optim/{k} is missing")
    saved = _flat(ck)
    for k, dst in live.items():
        src = saved.get(k)
        if not isinstance(src, torch.Tensor):
            raise ValueError(f"{path}: tensor '{k}' is missing")
        if tuple(src.shape) != tuple(dst.shape) or src.dtype != dst.dtype:
            raise ValueError(f"{path}: tensor '{k}' is {tuple(src.shape)} {src.dtype}, this run holds {tuple(dst.shape)} {dst.dtype}")
    _check_rng(ck["rng"], path)
    loop = ck["loop"]
    for k in LOOP_KEYS:
        if k not in loop:
            raise ValueError(f"{path}: loop/{k} is missing")
    es = loop["epoch_stats"]
    if not isinstance(es, torch.Tensor) or tuple(es.shape) != (4,) or es.dtype != torch.float32:
        raise ValueError(f"{path}: loop/epoch_stats is malformed")
    now = fingerprint["recorded"]
    diffs = [f"{k}: {fp['recorded'].get(k)!r} -> {v!r}" for k, v in now.items() if fp["recorded"].get(k) != v]
    return ck, saved, diffs
