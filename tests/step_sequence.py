"""One run of consecutive training steps of an engine, every step held to the fp64 step model (tests/step_fp64_model.py), every
AdamW update to its fp64 restatement (tests/fp64_bounds.py), and the full forward after the run to `oracle.llmrec_oracle.forward`.
TEST INFRASTRUCTURE ONLY: tests/test_step_sequence_fp64_gpu.py runs it on the H100 engines, tests/test_step_sequence_fp64_cpu.py on
the emulated ones (tests/ops_emulator.py).  The bounds and their calibration are stated in the GPU test's docstring."""
import numpy as np
import torch

import step_fp64_model as SM
from fp64_bounds import RATIOS, adamw_ref, check, state_ok

def forward_bound(hp, out, tau, rho=SM.RHO):
    """(U, I) bounds from the fp64 forward `out`: tau (|Y_e| + rho (max over e's row of |Y| + sum_t |c_t|)), c_t the fusion weights
    of the side terms (each multiplies a unit row)."""
    c = hp.cfg
    side = 2 * abs(c.model_cat_rate) + abs(c.user_cat_rate) + len(hp.keys) * abs(c.item_cat_rate) if hp.has_feats else 0.0
    lim = lambda Y: tau * (Y.abs() + rho * (Y.abs().amax(dim=1, keepdim=True) + side))
    return lim(out["U"]), lim(out["I"])


def forward_ratio(hp, tau):
    """hp.forward() against the fp64 forward at hp's parameters -> worst |error| / bound over every element of U and I."""
    from oracle import llmrec_oracle as O
    p, f, ui, iu = SM.engine_inputs(hp)
    with torch.no_grad():
        out = O.forward(p, f, ui, iu, SM.oracle_config(hp.cfg))
    U, I = hp.forward()
    worst = 0.0
    for got, want, lim in zip((U, I), (out["U"], out["I"]), forward_bound(hp, out, tau)):
        err = (got.detach().to(want.device, torch.float64) - want).abs()
        ratio = torch.where(torch.isfinite(err), err / lim, torch.full_like(err, float("inf")))      # an unwritten row fails
        worst = max(worst, float(ratio.max()))
    return worst


def opt_tensors(hp):
    """fp32 copies of what `hp.state_tensors()` hands from one step to the next, the step block aside (the emulator's AdamW keeps
    its count in `t`): "model/<name>", "m/<name>", "v/<name>" per optimized parameter."""
    o = hp.opt
    return {f"{sec}/{k}": t.detach().cpu().numpy().copy() for sec, ts in (("model", o.params), ("m", o.m), ("v", o.v))
            for k, t in zip(hp._opt_names, ts)}


def opt_count(opt):
    """AdamW's step count: the device step block of ops.AdamW (state[0]) or the emulator's `t`."""
    st = getattr(opt, "state", None)
    return int(st[0]) if st is not None else int(opt.t)


def check_adamw(hp, pre, k, what):
    """Step k's update: the engine's p, m, v against one fp64 AdamW step from the pre-step fp32 state (`pre`, keys of
    hp.state_tensors()) at step count k with the engine's own gradient; the device step block holds k and its bias corrections.
    -> the worst error / bound."""
    o = hp.opt
    lr, (b1, b2), eps, wd = o.lr, o.betas, o.eps, o.wd
    assert opt_count(o) == k, f"{what}: optimizer step count {opt_count(o)} after step {k}"
    st = getattr(o, "state", None)
    if st is not None:
        s = st.cpu().numpy()
        assert state_ok(s, k, lr, b1, b2), f"{what}: step block {s} after step {k}"
    fam = "adamw " + what
    for name, p, m, v in zip(hp._opt_names, o.params, o.m, o.v):
        refs = adamw_ref(pre["model/" + name], hp.grads[name].detach().cpu().numpy(), pre["m/" + name], pre["v/" + name], k,
                         lr, b1, b2, eps, wd)
        for which, got, (y, b) in zip("pmv", (p, m, v), refs):
            check(got, y, b, fam, f"{what}: step {k} {which} of {name}")
    return RATIOS.pop(fam, 0.0)


def check_row_sets(hp, batch, what, k):
    """The default engine's batch row sets after a step: exactly the distinct users, and the distinct pos | neg items, of the step's
    live triplets (nothing left from an earlier step, nothing from the index buffer's slots past B')."""
    u, p, n = batch
    for rs, want, side in ((hp.batch_u, np.unique(u), "user"), (hp.batch_i, np.unique(np.concatenate([p, n])), "item")):
        cnt = int(rs.count[0])
        got = np.sort(rs.list[:cnt].cpu().numpy())
        assert cnt == want.size and np.array_equal(got, want), \
            f"{what}: step {k} {side} row set holds {cnt} rows, the batch {want.size} ({np.setdiff1d(got, want)[:8]} not in it)"


def step(hp, how, batch):
    """One training step of `how` on the (users, pos, neg) int32 numpy batch: "train_step" (eager), "graphed" (the captured graph;
    the first call warms up and captures) or "buffer" (eager through the index buffer the graph reads, live length in its meta row)."""
    dev = hp.E_u.device
    u, p, n = (torch.from_numpy(x).to(dev) for x in batch)
    if how == "graphed":
        hp.train_step_graphed(u, p, n)
    elif how == "buffer":
        B = int(u.numel())
        gi = hp.index_buffer(B)
        gi[0, :B], gi[1, :B], gi[2, :B] = u, p, n
        gi[3, 0], gi[3, 1] = hp.meta_row(B)
        hp.train_step(gi[0], gi[1], gi[2], gi[3])
    elif how == "train_step":
        hp.train_step(u, p, n)
    else:
        raise ValueError(how)
    if dev.type == "cuda":
        torch.cuda.synchronize()


def run_sequence(hp, batches, tau_name, how, what, row_sets=None, done=None):
    """len(batches) steps of `how`, each checked as the GPU test's docstring states; then the full forward.
    row_sets: check the batch row sets after every step (default: where the engine fuses the batch's rows, the hoisted engine aside).
    done: a list that gets k appended once step k passed every check.
    -> dict(grads=, adamw=, forward=) of the largest error / bound ratios."""
    tau = SM.TAU[tau_name]
    if row_sets is None:
        row_sets = getattr(hp, "demand_fuse", False) and not hasattr(hp, "TU")
    worst = dict(grads=0.0, adamw=0.0)
    for k, batch in enumerate(batches, 1):
        pre = opt_tensors(hp)
        p, f, ui, iu = SM.engine_inputs(hp)
        ref = SM.reference(p, f, ui, iu, SM.oracle_config(hp.cfg), *(torch.from_numpy(x).long() for x in batch), hp.ni)
        del ref.per_head
        SM.check_cuts(ref, tau_name, f"{what} step {k}")
        step(hp, how, batch)
        res = SM.check_grads(ref, hp.grads, tau, what=f"{what} step {k}")
        SM.check_loss(ref, hp.loss, hp.head_out, SM.engine_heads(hp.keys), tau, what=f"{what} step {k}")
        worst["grads"] = max(worst["grads"], max(v[0] for v in res.values()))
        worst["adamw"] = max(worst["adamw"], check_adamw(hp, pre, k, what))
        if row_sets:
            check_row_sets(hp, batch, what, k)
        if done is not None:
            done.append(k)
    worst["forward"] = forward_ratio(hp, tau)
    assert worst["forward"] <= 1.0, f"{what}: forward after {len(batches)} steps at {worst['forward']:.3g} of its bound"
    return worst
