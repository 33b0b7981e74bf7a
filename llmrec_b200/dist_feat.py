"""Multi-GPU form of the FULL hot path (side-feature projections + propagation + fusion + the 8 loss heads)  --  SURVEY.md 8e.

Same sharding as dist.ShardedHotPath (users in contiguous row ranges, item-sized activations replicated), plus:
    item feature tables   sharded by contiguous ITEM ranges: rank r stores and projects rows [ilo, ihi) only (the projection is
                          row-local, Models.py:145-150); the projected block Pi [ni x S*d] is all-gathered;
    user feature table    sharded with the users; P_usr stays local;
    linear layers         replicated; every rank forms the weight gradient of its own rows, ONE small all-reduce per tensor.
Exchanges per step (L layers, S = 2 + #attribute tables feature blocks of d columns):
    forward   all-gather Pi | sum_r R_r^T Fu_r [ni x S*d] | sum_r R_r^T P_usr_r [ni x d] | sum_r R_r^T U_l,r [ni x d] per layer
              | the batch's user rows [B' x 4d]
    backward  sum_r R_r^T (su . Gprof_u_r) [ni x d] | sum_r R_r^T (su . gU_l,r) [ni x d] per layer | sum_r R_r^T (su . GFu_r) [ni x S*d]
              | the 8 weight / bias gradients
Item-side gradients that come straight from the loss (heads, feat_reg, fusion) are identical on every rank and are added ONCE,
after the cross-rank sum.  The schedule mirrors engine.HotPath line by line; world size 1 reproduces it.

Status: runs on the H100 at world 1 (tests/test_dist_gpu.py against engine.HotPath; tests/test_dist_fp64_gpu.py holds every
gradient, loss head and AdamW update of five-step runs to the fp64 step model in proj_mode 0 and 2).  World 2 over NCCL is in the
same tests and needs two visible GPUs; on CPU the orchestration runs at world 1/2/3 under gloo with torch stand-ins for the kernels
(tests/test_dist_feat_emulated.py against the oracle, tests/test_dist_fp64_cpu.py against the fp64 step model, even and uneven item
ranges).  No benchmark uses it.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import ops
from .dist import ShardedGraph, owner_local_index, shard_bounds
from .engine import HotPathConfig, PARAM_ORDER
from .sides import SideLayout


class ShardedFeatureHotPath:
    """params: dict name -> fp32 tensor; `user_id_embedding.weight` holds THIS RANK's user rows, everything else is replicated.
    feats_local: dict(image, text, item={key: ...}) with this rank's ITEM rows [item_lo, item_hi) and user = this rank's USER rows."""

    def __init__(self, graph: ShardedGraph, params, feats_local, cfg: HotPathConfig, user_lo: int, item_lo: int, group=None):
        self.g, self.cfg, self.group, self.p, self.f = graph, cfg, group, params, feats_local
        if cfg.deterministic:
            raise ValueError("deterministic steps are not implemented for the sharded engines (their loss heads and row exchanges scatter with float atomics)")
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.E_u, self.E_i = params["user_id_embedding.weight"], params["item_id_embedding.weight"]
        nu, ni, d, L = self.E_u.shape[0], self.E_i.shape[0], cfg.embed_size, cfg.n_layers
        self.nu, self.ni, self.d, self.L = nu, ni, d, L
        self.lo, self.hi = int(user_lo), int(user_lo) + nu
        self.keys = list(feats_local["item"].keys())
        self.sides = SideLayout(self.keys, d)
        S = self.S = self.sides.S
        self.ilo, self.ihi = int(item_lo), int(item_lo) + feats_local["image"].shape[0]
        self.even_items = self.world > 1 and ni % self.world == 0 and (self.ihi - self.ilo) * self.world == ni
        dev = self.E_i.device
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        self.Pi, self.Fu, self.Fi = new(ni, S * d), new(nu, S * d), new(ni, S * d)
        self.P_usr, self.prof_i, self.prof_u = new(nu, d), new(ni, d), new(nu, d)
        self.GFu, self.GFi, self.GP_usr = new(nu, S * d), new(ni, S * d), new(nu, d)
        self.Gprof_i, self.Gprof_u = new(ni, d), new(nu, d)
        self.Ul = [self.E_u] + [new(nu, d) for _ in range(L)]
        self.Il = [self.E_i] + [new(ni, d) for _ in range(L)]
        self.U, self.I = new(nu, d), new(ni, d)
        self.part, self.part_w = new(ni, d), new(ni, S * d)
        self.parts = [new(ni, d), new(ni, d)]
        self.gU, self.gI, self.dIl = new(nu, d), new(ni, d), new(ni, d)
        self.bufU, self.tmpI = new(nu, d), new(ni, d)
        self.grads = {k: torch.zeros_like(v) for k, v in params.items()}
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.loss_local = torch.zeros(1, dtype=torch.float32, device=dev)
        self.n_heads = 3 + len(self.keys)
        self.head_out = torch.zeros(self.n_heads * 4, dtype=torch.float32, device=dev)
        self._B = None
        self.opt = ops.AdamW([params[k] for k in PARAM_ORDER], lr=1e-4)
        self.comm_bytes = 0

    def set_lr(self, lr):
        self.opt.lr = lr

    def blk(self, buf, s):
        return self.sides.blk(buf, s)

    # -- collectives ---------------------------------------------------------------------------------------------------------
    def _allreduce(self, t):
        if self.world > 1:
            dist.all_reduce(t, group=self.group)
            self.comm_bytes += t.numel() * 4

    def _gather_item_rows(self, full):
        """rows [ilo, ihi) of `full` are valid on this rank -> all rows valid everywhere."""
        if self.world == 1:
            return
        if self.even_items:
            dist.all_gather_into_tensor(full, full[self.ilo:self.ihi], group=self.group)
        else:                                                         # uneven item ranges: zero the foreign rows and sum
            full[:self.ilo].zero_(); full[self.ihi:].zero_()
            dist.all_reduce(full, group=self.group)
        self.comm_bytes += full.numel() * 4

    def _item_sum(self, op, segs_src, buf, out, softmax=False):
        """out = [softmax]( si (.) sum over ranks of op . src ): per-rank partial into `buf`, one all-reduce, row scale."""
        op.apply([(x, y, None, False) for x, y in segs_src])
        self._allreduce(buf)
        ops.row_scale_softmax(buf, self.g.si, out, softmax)

    # -- forward (Models.py:145-197) --------------------------------------------------------------------------------------------
    def forward(self):
        g, sd, d, S, L, m = self.g, self.sides, self.d, self.S, self.L, self.cfg.proj_mode
        probs = sd.proj_problems(self.f, self.p, self.Pi[self.ilo:self.ihi], self.P_usr)
        ops.proj_fwd_group([t for t in probs if t[0].shape[0] > 0], d, m)                                  # :145-150, this rank's rows
        self._gather_item_rows(self.Pi)
        g.ui.apply([(self.blk(self.Pi, s), self.blk(self.Fu, s), None, False) for s in range(S)] + [(self.Il[0], self.Ul[1], None, L == 1)])
        self._item_sum(g.iu_raw, [(self.blk(self.Fu, s), self.blk(self.part_w, s)) for s in range(S)], self.part_w, self.Fi)   # :154,157,163
        self._item_sum(g.iu_raw, [(self.P_usr, self.part)], self.part, self.prof_i)                        # :166
        self._item_sum(g.iu_raw, [(self.Ul[1], self.part)], self.part, self.Il[1], L == 1)                 # :175,180
        segs = [(self.prof_i, self.prof_u, None, False)]                                                   # :167
        if L >= 2:
            segs.append((self.Il[1], self.Ul[2], None, L == 2))
        g.ui.apply(segs)
        for l in range(2, L + 1):
            self._item_sum(g.iu_raw, [(self.Ul[l], self.part)], self.part, self.Il[l], l == L)
            if l < L:
                g.ui.apply([(self.Il[l], self.Ul[l + 1], None, l + 1 == L)])
        coefs, su, si = sd.coefs(self.cfg), sd.fused(self.Fu, self.prof_u), sd.fused(self.Fi, self.prof_i)
        ops.fuse_fwd(self.Ul, su, coefs, self.U)                                                           # :185-197
        ops.fuse_fwd(self.Il, si, coefs, self.I)
        self._fuse_args = (coefs, su, si)
        return self.U, self.I

    # -- losses + output gradients (main.py:232-256,330-342,151-165) --------------------------------------------------------------------
    def loss_and_output_grads(self, users, pos, neg):
        c, d = self.cfg, self.d
        B = int(users.numel())
        if self._B != B:
            dev = users.device
            self._B = B
            self.Ub4, self.gUb4 = torch.empty(B, 4 * d, device=dev), torch.empty(B, 4 * d, device=dev)
            self.arange = torch.arange(B, dtype=torch.int32, device=dev)
            self.work = ops.bpr_work(self.n_heads, B, dev)
        n_keep = int((1 - c.prune_loss_drop_rate) * B)
        local = owner_local_index(users, self.lo, self.hi)
        ub = lambda s: self.Ub4[:, s * d:(s + 1) * d]
        gb = lambda s: self.gUb4[:, s * d:(s + 1) * d]
        for s, src in enumerate((self.U, self.blk(self.Fu, 0), self.blk(self.Fu, 1), self.prof_u)):       # owners fill, others zero
            ops.gather_rows(src, local, ub(s))
        self._allreduce(self.Ub4)
        for t in (self.loss, self.loss_local, self.gUb4, self.gU, self.gI, self.GFu, self.GFi, self.Gprof_u, self.Gprof_i):
            t.zero_()
        creg, sd = c.feat_reg_decay / self.ni, self.sides
        ops.sqnorm_grad(sd.reg(self.Fu), sd.reg(self.GFu), creg, False, self.loss_local)                   # this rank's users only
        ops.sqnorm_grad(sd.reg(self.Fi), sd.reg(self.GFi), creg, False, self.loss)                         # replicated
        # the gathered user rows: U | img_u | txt_u | prof_u, so blocks 0 and 1 of Ub4[:, d:] are the image and text rows
        heads = [(ub(0), self.I, gb(0), self.gI, 1.0, 1.0)] + sd.heads(c, self.Ub4[:, d:], ub(3), self.gUb4[:, d:], gb(3), self.Fi, self.GFi)
        ops.bpr_heads(heads, self.arange, pos, neg, n_keep, c.regs0 / c.batch_size, self.head_out, self.loss, self.work)
        for s, dst in enumerate((self.gU, self.blk(self.GFu, 0), self.blk(self.GFu, 1), self.Gprof_u)):   # user-row grads to their owners
            ops.scatter_add_rows(gb(s), local, dst)
        self._allreduce(self.loss_local)
        self.loss += self.loss_local
        return self.loss

    # -- backward ---------------------------------------------------------------------------------------------------------------
    def backward(self):
        g, d, S, L, m = self.g, self.d, self.S, self.L, self.cfg.proj_mode
        G, sd = self.grads, self.sides
        coefs, su, si = self._fuse_args
        dsu, dsi = sd.fused(self.GFu, self.Gprof_u), sd.fused(self.GFi, self.Gprof_i)
        dUl = G["user_id_embedding.weight"]
        ops.fuse_bwd(self.gU, L + 1, dUl, su, coefs, dsu, True)
        ops.fuse_bwd(self.gI, L + 1, self.dIl, si, coefs, dsi, True)
        # prof_u = ui . prof_i  ->  Gprof_i += sum_r R_r^T (su . Gprof_u_r)
        g.uiT_raw.apply([(self.Gprof_u, self.part, None, False)])
        self._allreduce(self.part)
        self.Gprof_i += self.part
        g_cur = self.dIl
        for l in range(L, 0, -1):
            src = ops.row_softmax_bwd(self.Il[l], g_cur, out=self.tmpI) if l == L else g_cur
            segs = [(src, self.bufU, dUl, False)]                                                          # gU_l = dUl + iu^T src (local rows)
            if l == L:
                segs += [(self.blk(self.GFi, s), self.blk(self.GFu, s), self.blk(self.GFu, s), False) for s in range(S)]
                segs.append((self.Gprof_i, self.GP_usr, None, False))
            g.iuT.apply(segs)
            if l == L:
                ops.row_softmax_bwd(self.Ul[l], self.bufU, out=self.bufU)
            dst = self.parts[l & 1]
            g.uiT_raw.apply([(self.bufU, dst, None, False)])                                               # sum_r R_r^T (su . gU_l)
            self._allreduce(dst)
            dst += self.dIl                                                                                # replicated direct part, once
            if l == L:
                g.uiT_raw.apply([(self.blk(self.GFu, s), self.blk(self.part_w, s), None, False) for s in range(S)])
                self._allreduce(self.part_w)                                                               # = GPi (all item rows)
            g_cur = dst
        G["item_id_embedding.weight"].copy_(g_cur)
        # weight gradients: this rank's item rows / user rows, then one all-reduce per tensor.  A rank holds rows of every item table
        # or of none, so dropping the empty tables keeps each dW's first problem the one that does not accumulate
        probs = sd.wgrad_problems(self.f, G, self.part_w[self.ilo:self.ihi], self.GP_usr)
        live = [t for t in probs if t[0].shape[0] > 0]
        for name in ("image_trans", "text_trans", "user_trans", "item_trans"):
            if not any(t[2] is G[name + ".weight"] for t in live):                                        # a rank without rows of that table
                G[name + ".weight"].zero_(); G[name + ".bias"].zero_()
        if live:
            ops.proj_wgrad_group(live, d, m)
        for name in ("image_trans", "text_trans", "user_trans", "item_trans"):
            self._allreduce(G[name + ".weight"])
            self._allreduce(G[name + ".bias"])
        return G

    def train_step(self, users, pos, neg):
        self.forward()
        self.loss_and_output_grads(users, pos, neg)
        self.backward()
        self.opt.step([self.grads[k] for k in PARAM_ORDER])
        return self.loss


def item_shard_bounds(n_items: int, world: int):
    """Item ranges of the feature tables (same contiguous balanced partition as the users')."""
    return shard_bounds(n_items, world)
