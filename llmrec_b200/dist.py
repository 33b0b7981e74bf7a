"""Multi-GPU (one process per GPU, NCCL over NVLink) form of the ID-propagation hot path  --  SURVEY.md 8e.

Sharding.  Users are split into contiguous row ranges, one per rank; rank r keeps
    R_r = R[users_r, :]  as CSR (local user rows x ALL item columns) and CSR(R_r^T) (all items x local users),
    E_u[users_r], its AdamW moments and every user-sized activation;
item-sized tensors ([ni x d]: E_i, I_l, gradients, AdamW moments) are REPLICATED and kept identical on every rank.
Consequences (L layers; the reference has no multi-GPU code, the oracle is 1-GPU == G-GPU equality):
    ui . X      = su (.) R_r X              local  (X = item-sized, replicated)                       no exchange
    iu . Y      = si (.) sum_r R_r^T Y_r    every rank forms its [ni x d] partial, ONE all-reduce,    1 exchange / layer
                                            then scale / softmax (llmrec_row_scale_softmax_f32)
    ui^T . G    = sum_r R_r^T (su (.) G_r)  same exchange in the backward chain                       1 exchange / layer
    iu^T . G    = R_r (si (.) G)            local
    losses      the batch's user rows are summed into a [B' x d] buffer (owners fill, others zero, one tiny
                all-reduce); every rank then evaluates the BPR/prune head redundantly on identical data -> identical
                item gradients without an exchange, user-row gradients scattered to their owners.
Only item-sized data ever crosses NVLink (4 all-reduces of ni*d*4 bytes per step at L = 2); user-sized data never moves.
This is the ID-only configuration (no side-feature tables), the one the 10M x 1M synthetic benchmark uses.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import ops
from .engine import HotPathConfig
from .ops import CsrOperator


def shard_bounds(n: int, world: int):
    """Contiguous, balanced row ranges: rank r owns [b[r], b[r+1])."""
    base, rem = divmod(n, world)
    b = [0]
    for r in range(world):
        b.append(b[-1] + base + (1 if r < rem else 0))
    return b


def owner_local_index(users: torch.Tensor, lo: int, hi: int) -> torch.Tensor:
    """int32 local row of each batch user on this rank, -1 where another rank owns it."""
    u = users.to(torch.int64)
    own = (u >= lo) & (u < hi)
    return torch.where(own, u - lo, torch.full_like(u, -1)).to(torch.int32)


def csr_from_sorted_rows(rows: torch.Tensor, n_rows: int) -> torch.Tensor:
    counts = torch.bincount(rows, minlength=n_rows)
    rp = torch.zeros(n_rows + 1, dtype=torch.int64, device=rows.device)
    rp[1:] = torch.cumsum(counts, 0)
    return rp.to(torch.int32)


def build_shard_csr(u_local: torch.Tensor, items: torch.Tensor, nu_local: int, n_items: int, group=None, solo=False):
    """Device-agnostic part of the shard construction (also exercised on CPU with gloo in tests/test_dist_cpu.py):
    CSR(R_r), CSR(R_r^T) and the (deg + 1e-8)^-1/2 scales; ITEM degrees are summed over ranks."""
    key, _ = torch.sort(u_local.to(torch.int64) * n_items + items.to(torch.int64))
    ul, it = key // n_items, key % n_items
    rowptr_u = csr_from_sorted_rows(ul, nu_local)
    col_u = it.to(torch.int32).contiguous()
    keyt, _ = torch.sort(it * nu_local + ul)
    rowptr_i = csr_from_sorted_rows(keyt // nu_local, n_items)
    col_i = (keyt % nu_local).to(torch.int32).contiguous()
    deg_u = (rowptr_u[1:] - rowptr_u[:-1]).to(torch.float64)
    deg_i = (rowptr_i[1:] - rowptr_i[:-1]).to(torch.float64)
    if not solo and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(deg_i, group=group)                             # item degrees are global
    inv = lambda d: torch.pow(d + 1e-8, -0.5).to(torch.float32)         # main.py:114-118 (never inf with the +1e-8)
    return dict(rowptr_u=rowptr_u, col_u=col_u, rowptr_i=rowptr_i, col_i=col_i, su=inv(deg_u), si=inv(deg_i), nnz=int(key.numel()))


class ShardedGraph:
    """Local shard of the bipartite graph.  u_local/items: int64 edge lists (local user row, global item), unique pairs."""

    def __init__(self, u_local: torch.Tensor, items: torch.Tensor, nu_local: int, n_items: int, group=None, tile_nnz: int = 0, solo=False, pieces: int = 1):
        c = build_shard_csr(u_local, items, nu_local, n_items, group, solo)
        self.nu_local, self.n_items, self.nnz = int(nu_local), int(n_items), c["nnz"]
        self.su, self.si = c["su"], c["si"]
        rowptr_u, col_u, rowptr_i, col_i = c["rowptr_u"], c["col_u"], c["rowptr_i"], c["col_i"]
        self.rowptr_u, self.col_u, self.rowptr_i, self.col_i = rowptr_u, col_u, rowptr_i, col_i
        # ui: rows = local users (row scale su).  iu_raw / uiT_raw: rows = items, partial sums to be all-reduced.
        self.ui = CsrOperator(rowptr_u, col_u, nu_local, n_items, rs=self.su, tile_nnz=tile_nnz)
        self.iu_raw = CsrOperator(rowptr_i, col_i, n_items, nu_local, tile_nnz=tile_nnz)
        w_uiT = self.su[col_i.long()].contiguous()
        self.uiT_raw = CsrOperator(rowptr_i, col_i, n_items, nu_local, vals=w_uiT, plan=self.iu_raw.plan)
        self.iuT = CsrOperator(rowptr_u, col_u, nu_local, n_items, vals=self.si[col_u.long()].contiguous(), plan=self.ui.plan)
        # item-row pieces of the two exchange operators: piece k's all-reduce overlaps the SpMM of piece k+1
        self.pieces = []
        if pieces > 1:
            b = shard_bounds(n_items, pieces)
            for k in range(pieces):
                lo, hi = b[k], b[k + 1]
                rp = rowptr_i[lo:hi + 1].contiguous()
                fwd = CsrOperator(rp, col_i, hi - lo, nu_local, tile_nnz=tile_nnz)
                bwd = CsrOperator(rp, col_i, hi - lo, nu_local, vals=w_uiT, plan=fwd.plan)
                self.pieces.append((lo, hi, fwd, bwd))


class ShardedHotPath:
    """ID-only training step over a ShardedGraph; world size 1 reproduces engine.HotPath(feats=None) exactly."""

    def __init__(self, graph: ShardedGraph, E_u_local: torch.Tensor, E_i: torch.Tensor, cfg: HotPathConfig, user_lo: int, group=None, solo=False,
                 item_sharded: bool = False, demand: bool = False):
        """item_sharded (opt-in, needs n_items % world == 0): the item-side exchanges whose result is only consumed row-wise
        become reduce-scatter -> row-local work on this rank's item range -> all-gather (same bytes on NVLink as the
        all-reduce): the scale/softmax after each forward exchange runs on 1/world of the rows, and the item table's AdamW
        state and update are sharded by item (the updated rows are all-gathered instead of the gradient)."""
        self.g, self.cfg, self.group = graph, cfg, group
        if cfg.deterministic:
            raise ValueError("deterministic steps are not implemented for the sharded engines (their loss heads and row exchanges scatter with float atomics)")
        self.world = dist.get_world_size(group) if (dist.is_initialized() and not solo) else 1
        self.item_sharded = bool(item_sharded) and self.world > 1 and E_i.shape[0] % self.world == 0
        self.E_u, self.E_i = E_u_local, E_i
        self.lo, self.hi = int(user_lo), int(user_lo) + E_u_local.shape[0]
        nu, ni, d, L = E_u_local.shape[0], E_i.shape[0], cfg.embed_size, cfg.n_layers
        self.nu, self.ni, self.d, self.L = nu, ni, d, L
        dev = E_i.device
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        zeros = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)      # layer outputs: demand mode leaves untouched rows readable
        self.Ul = [E_u_local] + [zeros(nu, d) for _ in range(L)]
        self.Il = [E_i] + [zeros(ni, d) for _ in range(L)]
        self.U, self.I = new(nu, d), new(ni, d)
        self.part = new(ni, d)                       # per-rank partial of an item-side product (all-reduced in place)
        self.parts = [self.part, new(ni, d)]         # backward chain ping-pong (the reduced partial IS the next gradient)
        self.gU = new(nu, d)
        self.g_Eu, self.g_Ei = new(nu, d), None
        self.dIl, self.bufU, self.tmpI = new(ni, d), new(nu, d), new(ni, d)
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.head_out = torch.zeros(4, dtype=torch.float32, device=dev)
        self._B = None
        if self.item_sharded:
            rank = dist.get_rank(group)
            per = ni // self.world
            self.ilo, self.ihi = rank * per, (rank + 1) * per
            self.shard = new(per, d)                                       # this rank's rows of a reduced item-side product
            self.opt = ops.AdamW([E_u_local, E_i[self.ilo:self.ihi]], lr=1e-4)
        else:
            self.opt = ops.AdamW([E_u_local, E_i], lr=1e-4)
        self.comm_bytes = 0
        self.item_opt_sharded = False
        # demand-driven training step: the LAST propagation layer reaches the loss only through the batch (U_L on the batch users and
        # on the neighbours of the batch items, I_L on the batch items), so its four products are evaluated on those rows only and the
        # user table's gradient stays row-sparse; every value that is computed is the same sum as in the dense schedule.
        self.demand = bool(demand) and not self.item_sharded and L >= 1 and d in (32, 64, 128)
        if self.demand:
            self.needU = ops.RowSet(nu, dev)        # local users whose U_L row this step reads
            self.batchU = ops.RowSet(nu, dev)       # local batch users (rows of the user table that receive a gradient)
            self.batchI = ops.RowSet(ni, dev)       # batch items (the only non-zero rows of the top-layer item gradient)
            # the LAST exchange of a step yields the gradient of E_i, which only its AdamW update reads: reduce-scatter it, update this rank's
            # 1/G of the item rows (moments sharded too), all-gather the updated rows -- the bytes of the all-reduce, 1/G of the optimizer work
            self.item_opt_sharded = self.world > 1 and ni % self.world == 0
            if self.item_opt_sharded:
                rank = dist.get_rank(group)
                per = ni // self.world
                self.ilo, self.ihi = rank * per, (rank + 1) * per
                self.shard = new(per, d)
                self.opt = ops.AdamW([E_u_local, E_i[self.ilo:self.ihi]], lr=1e-4)

    def set_lr(self, lr):
        self.opt.lr = lr

    def _allreduce(self, t):
        if self.world > 1:
            dist.all_reduce(t, group=self.group)
            self.comm_bytes += t.numel() * 4

    def _reduce_scatter(self, part):
        """self.shard = this rank's item rows of sum over ranks of `part` ([ni x d], equal contiguous row ranges)."""
        dist.reduce_scatter_tensor(self.shard, part, group=self.group)
        self.comm_bytes += part.numel() * 2                                 # accounted like half an all-reduce

    def _all_gather_rows(self, full):
        """every rank's [ilo, ihi) rows of `full` -> all rows, in place."""
        dist.all_gather_into_tensor(full, full[self.ilo:self.ihi], group=self.group)
        self.comm_bytes += full.numel() * 2

    def _exchange(self, which, src, out=None, src_mask=None, overlap=None):
        """self.part = sum over ranks of (item-side operator `which`) . src.  With item-row pieces, the NCCL all-reduce of
        piece k runs on NCCL's stream while the SpMM of piece k+1 runs on the compute stream (NVLink transfer hidden
        behind the gather)."""
        g = self.g
        part = self.part if out is None else out
        if self.world == 1 or not g.pieces:
            (g.iu_raw if which == "iu" else g.uiT_raw).apply([(src, part, None, False)], src_mask=src_mask)
            if overlap is not None and self.world > 1:
                # the NCCL kernels run on NCCL's stream; independent work queued on the compute stream now overlaps the transfer
                work = dist.all_reduce(part, group=self.group, async_op=True)
                self.comm_bytes += part.numel() * 4
                overlap()
                work.wait()
            else:
                self._allreduce(part)
                if overlap is not None:
                    overlap()
            return
        works = []
        for lo, hi, fwd, bwd in g.pieces:
            (fwd if which == "iu" else bwd).apply([(src, part[lo:hi], None, False)], src_mask=src_mask)
            works.append(dist.all_reduce(part[lo:hi], group=self.group, async_op=True))
            self.comm_bytes += (hi - lo) * self.d * 4
        if overlap is not None:
            overlap()
        for w in works:
            w.wait()

    # -- forward (Models.py:169-186) ------------------------------------------------------------------------
    def forward(self, fuse_items=True):
        """fuse_items=False (training): the fused item output I is only needed on the batch's pos/neg rows and is
        produced there by loss_and_output_grads -- the [ni x d] mean over layers is replicated work on every rank."""
        L = self.L
        for l in range(1, L + 1):
            self.g.ui.apply([(self.Il[l - 1], self.Ul[l], None, l == L)])                    # U_l = [softmax] ui . I_{l-1}
            if self.item_sharded:
                self.g.iu_raw.apply([(self.Ul[l], self.part, None, False)])                   # per-rank partial of R^T U_l
                self._reduce_scatter(self.part)
                ops.row_scale_softmax(self.shard, self.g.si[self.ilo:self.ihi], self.Il[l][self.ilo:self.ihi], l == L)
                self._all_gather_rows(self.Il[l])
                continue
            self._exchange("iu", self.Ul[l])                                                  # sum_r R_r^T U_l  (all-reduce)
            ops.row_scale_softmax(self.part, self.g.si, self.Il[l], l == L)                   # I_l = [softmax] si (.) sum
        ops.fuse_fwd(self.Ul, [], [], self.U)                                                 # mean over layers (:185-186)
        if fuse_items:
            ops.fuse_fwd(self.Il, [], [], self.I)
        return self.U, self.I

    # -- loss + output grads ------------------------------------------------------------------------------------
    def loss_and_output_grads(self, users, pos, neg):
        """users: GLOBAL user ids (int32, identical on every rank); pos/neg: item ids.
        Item-side gradients of the loss are ROW-SPARSE (<= 2B' rows): they are kept compact ([2B' x d], indexed by batch
        position) and scatter-added where the dense chain needs them, instead of carrying dense [ni x d] copies."""
        c = self.cfg
        B = int(users.numel())
        if self._B != B:
            dev = users.device
            self._B = B
            self.Ub, self.gUb = torch.empty(B, self.d, device=dev), torch.empty(B, self.d, device=dev)
            self.Ib, self.gIb = torch.empty(2 * B, self.d, device=dev), torch.empty(2 * B, self.d, device=dev)
            self.arange = torch.arange(B, dtype=torch.int32, device=dev)
            self.arange2 = self.arange + B
            self.pn = torch.empty(2 * B, dtype=torch.int32, device=dev)
            self.work = ops.bpr_work(1, B, dev)
        local = owner_local_index(users, self.lo, self.hi)
        ops.gather_rows(self.U, local, self.Ub)                                               # owners fill, others zero
        self._allreduce(self.Ub)
        self.pn[:B].copy_(pos); self.pn[B:].copy_(neg)
        ops.fuse_fwd(self.Il, [], [], self.I, rows=self.pn)                                   # I on the batch rows only
        ops.gather_rows(self.I, self.pn, self.Ib)
        self.loss.zero_(); self.gUb.zero_(); self.gIb.zero_(); self.gU.zero_()
        n_keep = int((1 - c.prune_loss_drop_rate) * B)
        ops.bpr_heads([(self.Ub, self.Ib, self.gUb, self.gIb, 1.0, 1.0)], self.arange, self.arange, self.arange2, n_keep,
                      c.regs0 / c.batch_size, self.head_out, self.loss, self.work)
        ops.scatter_add_rows(self.gUb, local, self.gU)
        self.gIb.mul_(1.0 / (self.L + 1))                                                     # rows of dIl = gI / (L+1)
        return self.loss

    # -- backward chain ---------------------------------------------------------------------------------------------
    def backward(self):
        L = self.L
        ops.fuse_bwd(self.gU, L + 1, self.g_Eu, [], [], [], True)                             # dUl (= grad of E_u) = gU/(L+1)
        self.dIl.zero_()
        ops.scatter_add_rows(self.gIb, self.pn, self.dIl)                                     # dense dIl only feeds the softmax bwd
        g_cur = self.dIl
        grad_Ei = None
        for l in range(L, 0, -1):
            src = ops.row_softmax_bwd(self.Il[l], g_cur, out=self.tmpI) if l == L else g_cur
            self.g.iuT.apply([(src, self.bufU, self.g_Eu, False)])                            # gU_l = dUl + iu^T src   (local rows)
            if l == L:
                ops.row_softmax_bwd(self.Ul[l], self.bufU, out=self.bufU)
            if l == 1 and self.item_sharded:
                # the last exchange yields the gradient of E_i, which only its (sharded) AdamW update reads
                self.g.uiT_raw.apply([(self.bufU, self.part, None, False)])
                self._reduce_scatter(self.part)
                pn = self.pn.to(torch.int64)
                own = (pn >= self.ilo) & (pn < self.ihi)
                ops.scatter_add_rows(self.gIb, torch.where(own, pn - self.ilo, torch.full_like(pn, -1)).to(torch.int32), self.shard)
                grad_Ei = self.shard
                break
            self._exchange("uiT", self.bufU, out=self.parts[l & 1])                           # sum_r R_r^T (su (.) gU_l)
            g_cur = self.parts[l & 1]
            ops.scatter_add_rows(self.gIb, self.pn, g_cur)                                    # gI_{l-1} = sum + dIl (row-sparse addend)
            grad_Ei = g_cur
        self.g_Ei = grad_Ei
        return self.g_Eu, self.g_Ei

    # -- demand-driven step (same results, rows the batch cannot reach are never computed) ---------------------------------
    def _batch_buffers(self, B, dev):
        if getattr(self, "_Bd", None) == B:
            return
        self._Bd = B
        d = self.d
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        self.Ub, self.gUb, self.dUb = new(B, d), new(B, d), new(B, d)
        self.Ib, self.gIb, self.dIb = new(2 * B, d), new(2 * B, d), new(2 * B, d)
        self.Pc, self.sic, self.srcI = new(2 * B, d), new(2 * B, 1), new(2 * B, d)
        self.arange = torch.arange(B, dtype=torch.int32, device=dev)
        self.arange2 = self.arange + B
        self.pn = torch.empty(2 * B, dtype=torch.int32, device=dev)
        self.cnt_pn = torch.full((1,), 2 * B, dtype=torch.int32, device=dev)
        self.work = ops.bpr_work(1, B, dev)

    def _train_step_demand(self, users, pos, neg):
        g, L, c = self.g, self.L, self.cfg
        B = int(users.numel())
        self._batch_buffers(B, users.device)
        local = owner_local_index(users, self.lo, self.hi)
        self.pn[:B].copy_(pos); self.pn[B:].copy_(neg)
        pn = self.pn
        # row sets of this step (device-side, no host sync); built while the first forward exchange is in flight when there is one
        def build_sets():
            self.needU.clear(); self.needU.add_neighbors(g.rowptr_i, g.col_i, pn); self.needU.add_ids(local); self.needU.compact()
            self.batchU.clear(); self.batchU.add_ids(local)
            self.batchI.clear(); self.batchI.add_ids(pn)
        if L < 2:
            build_sets()
        rows, cnt = self.needU.list, self.needU.count
        # ---- forward: layers 1 .. L-1 dense, layer L on the rows the loss can reach ----
        for l in range(1, L):
            g.ui.apply([(self.Il[l - 1], self.Ul[l], None, False)])
            self._exchange("iu", self.Ul[l], overlap=build_sets if l == 1 else None)
            ops.row_scale_softmax(self.part, g.si, self.Il[l], False)
        g.ui.apply_rows((self.Il[L - 1], self.Ul[L], None, True), rows, cnt)                  # U_L = softmax(ui . I_{L-1}) on needU
        g.iu_raw.apply_rows((self.Ul[L], self.part, None, False), pn, self.cnt_pn, cta_per_row=True)   # this rank's partial of R^T U_L on the batch items (hub items: 1e5 neighbours)
        ops.gather_rows(self.part, pn, self.Pc)
        self._allreduce(self.Pc)                                                              # [2B' x d] instead of [ni x d]
        ops.gather_rows(g.si.view(-1, 1), pn, self.sic)
        ops.row_scale_softmax(self.Pc, self.sic.view(-1), self.Pc, True)                      # I_L = softmax(si (.) sum) on the batch items
        ops.assign_rows(self.Pc, pn, self.Il[L])
        # ---- loss head on the batch rows ----
        ops.fuse_fwd(self.Ul, [], [], self.Ub, rows=local, compact=True)                      # owners fill, others zero
        self._allreduce(self.Ub)
        ops.fuse_fwd(self.Il, [], [], self.Ib, rows=pn, compact=True)
        ops.grad_init([(self.gUb, None, 0.0), (self.gIb, None, 0.0)], self.loss)
        n_keep = int((1 - c.prune_loss_drop_rate) * B)
        ops.bpr_heads([(self.Ub, self.Ib, self.gUb, self.gIb, 1.0, 1.0)], self.arange, self.arange, self.arange2, n_keep,
                      c.regs0 / c.batch_size, self.head_out, self.loss, self.work)
        ops.fuse_bwd(self.gUb, L + 1, self.dUb, [], [], [], False)                            # the mean's share of every layer: g / (L+1)
        ops.fuse_bwd(self.gIb, L + 1, self.dIb, [], [], [], False)
        # ---- backward chain ----
        # E_u enters the step only through the mean over layers (U_0): its gradient is dUb on the batch rows, known now.  The dense AdamW
        # pass over the user table (row-sparse gradient) is queued while the first backward exchange is in flight.
        self.opt.advance()
        done = []

        def update_users():
            ops.zero_rows(self.g_Eu, local)
            ops.scatter_add_rows(self.dUb, local, self.g_Eu)
            self.opt.step_tensor(0, self.g_Eu, row_mask=self.batchU.mask)
            done.append(1)
        g_cur = None
        for l in range(L, 0, -1):
            if l == L:
                # the top-layer item gradient lives on the batch items only: softmax backward per batch position on the compact rows
                # (linear in the gradient, so duplicates add up), scattered into the rows of tmpI the source mask lets the gather read
                ops.row_softmax_bwd(self.Pc, self.dIb, out=self.srcI)                         # Pc still holds I_L on the batch rows
                ops.zero_rows(self.tmpI, pn)
                ops.scatter_add_rows(self.srcI, pn, self.tmpI)
                g.iuT.apply_rows((self.tmpI, self.bufU, None, False), rows, cnt, src_mask=self.batchI.mask)   # gU_L on needU (the only rows it reaches)
                ops.scatter_add_rows(self.dUb, local, self.bufU)
                ops.row_softmax_bwd_rows(self.Ul[l], self.bufU, self.bufU, rows, cnt)
                mask = self.needU.mask
            else:
                g.iuT.apply([(g_cur, self.bufU, None, False)])
                ops.scatter_add_rows(self.dUb, local, self.bufU)
                mask = None
            if l == 1 and self.item_opt_sharded:
                g.uiT_raw.apply([(self.bufU, self.parts[1], None, False)], src_mask=mask)      # this rank's partial of the gradient of E_i
                work = dist.reduce_scatter_tensor(self.shard, self.parts[1], group=self.group, async_op=True)
                self.comm_bytes += self.parts[1].numel() * 2
                if not done:
                    update_users()                                                            # overlaps the transfer
                pn64 = pn.to(torch.int64)
                own = (pn64 >= self.ilo) & (pn64 < self.ihi)
                idx = torch.where(own, pn64 - self.ilo, torch.full_like(pn64, -1)).to(torch.int32)
                work.wait()
                ops.scatter_add_rows(self.dIb, idx, self.shard)                               # + dI_0 on this rank's rows
                self.g_Ei = self.shard
                self.opt.step_tensor(1, self.shard)
                self._all_gather_rows(self.E_i)                                               # updated item rows back to every rank
                return self.loss
            if l == L:
                self._exchange("uiT", self.bufU, out=self.parts[l & 1], src_mask=mask, overlap=update_users)
            else:
                self._exchange("uiT", self.bufU, out=self.parts[l & 1])
            g_cur = self.parts[l & 1]
            ops.scatter_add_rows(self.dIb, pn, g_cur)                                         # + dI_{l-1} (row-sparse addend)
        self.g_Ei = g_cur
        if not done:
            update_users()
        self.opt.step_tensor(1, self.g_Ei)
        return self.loss

    def step_grads(self):
        """The gradients the last train_step handed to AdamW -> (this rank's user rows [nu x d], item rows, first item row).
        The demand step's user gradient is row-sparse: AdamW reads g_Eu on the batch rows only, so every other row reads zero here.
        With the item table's optimizer sharded (item_sharded, item_opt_sharded) the item gradient holds this rank's rows [ilo, ihi).
        For tests; it launches nothing inside a step."""
        g_u = self.g_Eu
        if self.demand:
            bits = (self.batchU.mask.to(torch.int64) & 0xffffffff)[:, None] >> torch.arange(32, device=g_u.device)
            keep = (bits & 1).reshape(-1)[:self.nu].bool()
            g_u = torch.where(keep[:, None], g_u, torch.zeros_like(g_u))
        return g_u, self.g_Ei, (self.ilo if (self.item_sharded or self.item_opt_sharded) else 0)

    def train_step(self, users, pos, neg):
        if self.demand:
            return self._train_step_demand(users, pos, neg)
        self.forward(fuse_items=False)
        self.loss_and_output_grads(users, pos, neg)
        self.backward()
        self.opt.step([self.g_Eu, self.g_Ei])
        if self.item_sharded:
            self._all_gather_rows(self.E_i)                                                   # updated item rows back to every rank
        return self.loss


# --------------------------------------------------------------------------------------------------------------------
# synthetic graphs of the large configuration, generated on the device shard by shard
# --------------------------------------------------------------------------------------------------------------------
def synthetic_shard(n_users, n_items, n_edges, rank, world, device, seed=0, zipf_a=0.8):
    """Edges of this rank's users: every user >= 1 edge, item popularity ~ (rank + 16)^-a; duplicates removed.
    Deterministic in (seed, user range) only up to the per-rank generator, i.e. each rank's shard is reproducible."""
    b = shard_bounds(n_users, world)
    lo, hi = b[rank], b[rank + 1]
    nu = hi - lo
    g = torch.Generator(device=device).manual_seed(seed * 1000003 + rank)
    extra = int(round(n_edges * nu / n_users)) - nu
    w = torch.pow(torch.arange(n_items, device=device, dtype=torch.float64) + 16.0, -zipf_a)
    cdf = torch.cumsum(w / w.sum(), 0).to(torch.float32)
    perm = torch.randperm(n_items, device=device, generator=g)
    users = torch.cat([torch.arange(nu, device=device), torch.randint(0, nu, (max(extra, 0),), device=device, generator=g)])
    items = perm[torch.searchsorted(cdf, torch.rand(users.numel(), device=device, generator=g)).clamp_(max=n_items - 1)]
    key = torch.unique(users * n_items + items)
    return key // n_items, key % n_items, lo, hi


def store_shard(path, rank, world, device, split="train"):
    """This rank's slice of a binary CSR interaction store (utility/csr_store.py): users [lo, hi) of the contiguous
    partition, read straight from the memory-mapped arrays (only this rank's pages are touched).
    -> (u_local int64, items int64, lo, hi, n_users, n_items); duplicate (user, item) pairs are removed, as scipy's
    CSR construction of `train_mat` does upstream (main.py:59, 114-118 see a binary matrix)."""
    from .utility import csr_store
    import numpy as np
    meta, rows = csr_store.read(path)
    r = rows[split]
    n_users, n_items = int(meta["n_users"]), int(meta["n_items"])
    b = shard_bounds(n_users, world)
    lo, hi = b[rank], b[rank + 1]
    e0, e1 = int(r.rowptr[lo]), int(r.rowptr[hi])
    counts = np.diff(np.asarray(r.rowptr[lo:hi + 1]))
    u = torch.repeat_interleave(torch.arange(hi - lo, dtype=torch.int64), torch.from_numpy(counts.astype(np.int64)))
    it = torch.from_numpy(np.asarray(r.col[e0:e1]).astype(np.int64))
    key = torch.unique(u.to(device) * n_items + it.to(device))
    return key // n_items, key % n_items, lo, hi, n_users, n_items
