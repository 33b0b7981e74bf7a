"""Torch-CPU stand-ins for the ordered (bit-reproducible) ops of `llmrec_b200.ops`, on top of tests/ops_emulator.py.  TEST INFRASTRUCTURE
ONLY, like that file: `install()` patches a test process so that the engines run with `HotPathConfig.deterministic` on a machine without a
GPU.  Each stand-in implements the order definition of include/llmrec_b200.h literally: one fp32 row add per contribution, in a Python loop."""
import torch

import ops_emulator as base


def scatter_add_rows_ordered(G, idx, Y, scratch=None):   # llmrec_scatter_add_rows_ordered_f32: one fp32 row add per b, ascending
    for b, r in enumerate(idx.long().tolist()):
        if r >= 0:
            Y[r] += G[b]


def bpr_slot_plan(users, pos, neg, meta=None, plan=None):                 # llmrec_bpr_slot_plan: slots sorted by (row, slot)
    B = int(users.numel())
    n = B if meta is None else int(meta[0])
    plan = torch.zeros(6 * B, dtype=torch.int32) if plan is None else plan
    items = torch.stack([pos[:n], neg[:n]], 1).reshape(-1)               # slot 2b = pos[b], 2b + 1 = neg[b]
    for keys, s0, r0 in ((users[:n], 0, B), (items, 2 * B, 4 * B)):
        order = torch.argsort(keys.long(), stable=True)
        plan[s0:s0 + order.numel()] = order.to(torch.int32)
        plan[r0:r0 + order.numel()] = keys[order]
    return plan


def bpr_heads(heads, users, pos, neg, n_keep, regs0_over_bs, out, loss, work, meta=None, ordered=None):      # llmrec_bpr_heads_ordered_f32
    """ordered=None: llmrec_bpr_heads_f32 (the stand-in of ops_emulator).  With a slot plan: the same forward values; each head's
    per-triplet row gradients (that stand-in on one row per triplet) are added one fp32 row at a time -- heads ascending, batch
    positions ascending, pos before neg."""
    if ordered is None:
        return base.bpr_heads(heads, users, pos, neg, n_keep, regs0_over_bs, out, loss, work, meta=meta)
    if meta is not None:
        B, n_keep = int(meta[0]), int(meta[1])
        users, pos, neg = users[:B], pos[:B], neg[:B]
    u, p, n = users.long(), pos.long(), neg.long()
    B = int(u.numel())
    ar = torch.arange(B, dtype=torch.int32)
    for h, (XU, XI, GU, GI, w_mf, w_emb) in enumerate(heads):
        gu, gi = torch.zeros(B, XU.shape[1]), torch.zeros(2 * B, XU.shape[1])
        base.bpr_heads([(XU[u], torch.cat([XI[p], XI[n]]), gu, gi, w_mf, w_emb)], ar, ar, ar + B, n_keep, regs0_over_bs,
                       out[4 * h:4 * h + 4], loss, None)
        for t in range(B):
            if GU is not None:
                GU[u[t]] += gu[t]
            if GI is not None:
                GI[p[t]] += gi[t]
                GI[n[t]] += gi[B + t]


def install():
    """ops_emulator.install() plus the ordered ops."""
    import llmrec_b200.ops as ops
    base.install()
    ops.scatter_add_rows_ordered, ops.bpr_slot_plan, ops.bpr_heads = scatter_add_rows_ordered, bpr_slot_plan, bpr_heads
