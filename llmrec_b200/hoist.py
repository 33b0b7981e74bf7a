"""Hoisted side-feature mode of the hot path (`--hoist_side 1`; SURVEY.md 8f-3).

With the default flags (Dropout p = 0, mask branch off) every side-feature operand of MM_Model.forward is LINEAR in constant
tables (Models.py:145-167):

    img_u = ui.(X W^T + 1 b^T)          = (ui.X) W^T      + (ui.1) b^T
    img_i = iu.img_u                    = (iu.ui.X) W^T   + (iu.ui.1) b^T          (same for text and the 5 attribute tables)
    prof_i = iu.(X_usr W_u^T + 1 b_u^T) = (iu.X_usr) W_u^T + (iu.1) b_u^T
    prof_u = ui.prof_i                  = (ui.iu.X_usr) W_u^T + (ui.iu.1) b_u^T

so 16 of the 20 propagation products per forward (and their 16 transposes per backward) act on constants.  This engine
precomputes the propagated TABLES once (TU [nu x Kc], TI [ni x Kc], column blocks img | txt | att_0..4 | usr | scales) with the
same SpMM kernel, and a training step then
  * propagates only the ID embeddings (2L + 2L SpMM launches on one [n x d] operand each),
  * gathers the <= B' user rows and <= 2B' item rows of the batch from TU / TI and projects the compact blocks with the grouped
    wgmma kernels (+ the rank-1 bias term scale (x) b),
  * evaluates fusion, the 8 BPR/prune heads and their gradients on compact [B' x .] blocks,
  * takes the weight gradients from the same compact rows, the bias gradients from scaled column sums, and feat_reg
    (main.py:151-156, a sum over ALL rows) with its gradient from one k x k Gram matrix per modality,
  * scatters the batch rows' ID gradients into the dense tables and runs the unchanged dense backward chain + AdamW.
Per step that is ~0.3 GB of HBM traffic instead of ~1.9 GB at netflix scale.  Results equal the default engine up to fp32
reassociation ((ui.X) W^T vs ui.(X W^T)); tests hold both to the same golden tolerances.  Auto-disabled by the caller when
drop_rate > 0 or the mask branch is on (the linearity argument needs dropout to be the identity).
"""
from __future__ import annotations

import torch

from . import feat_int8, ops
from .engine import HotPath, HotPathConfig


class HoistedHotPath(HotPath):
    compact_items = False             # projects gathered rows of the propagated tables, never the full item tables

    def __init__(self, operators, params, feats, cfg: HotPathConfig, graph_scalars):
        """graph_scalars: dict(cu, ci, ru, ri) fp32 CUDA vectors = ui.1, iu.ui.1, ui.iu.1, iu.1 (BipartiteGraph.ones_propagated())."""
        super().__init__(operators, params, feats, cfg)
        if not self.has_feats:
            raise ValueError("hoisting needs side features")
        if cfg.proj_mode == 2:
            raise ValueError("--hoist_side 1 runs on the tensor-core projection kernels (proj_mode 3xtf32 / tf32)")
        self._build_tables(graph_scalars)
        self._compact = None

    # ---- one-time precompute --------------------------------------------------------------------------------------
    def _build_tables(self, gs):
        dev, sd = self.E_u.device, self.sides
        raw = sd.tables(self.feats)
        # the logical widths come from the weights (an int8 table's rows are wider: values, padding and the row scale)
        widths = [int(self.p[w + ".weight"].shape[1]) for w in sd.weights]
        wide = lambda X, w: feat_int8.dequantize(X, w) if X.dtype == torch.int8 else X.float()
        self.col0 = [0]
        for w in widths:
            self.col0.append(self.col0[-1] + w)
        self.widths = widths
        Kc = self.col0[-1] + 32                                   # + one 32-column pad block holding the scale columns
        self.Kc = Kc
        TU = torch.zeros(self.nu, Kc, dtype=torch.float32, device=dev)
        TI = torch.zeros(self.ni, Kc, dtype=torch.float32, device=dev)
        # bf16 / int8 feature tables (--feat_dtype) are widened to fp32 one table at a time for these one-time products; TU / TI stay fp32
        for j, X in enumerate(raw[:-1]):                          # item-side raw tables: TU_s = ui.X, TI_s = iu.TU_s
            c0, w = self.col0[j], widths[j]
            self.ui.apply([(wide(X, w), TU[:, c0:c0 + w], None, False)])
            self.iu.apply([(TU[:, c0:c0 + w], TI[:, c0:c0 + w], None, False)])
        c0, w = self.col0[-2], widths[-1]                          # user table: TI_usr = iu.X_usr (prof_i), TU_usr = ui.TI_usr (prof_u)
        self.iu.apply([(wide(raw[-1], w), TI[:, c0:c0 + w], None, False)])
        self.ui.apply([(TI[:, c0:c0 + w], TU[:, c0:c0 + w], None, False)])
        sc = self.col0[-1]
        TU[:, sc] = gs["cu"]; TU[:, sc + 1] = gs["ru"]             # Fu bias scale, prof_u bias scale
        TI[:, sc] = gs["ci"]; TI[:, sc + 1] = gs["ri"]             # Fi bias scale, prof_i bias scale
        self.TU, self.TI, self.sc = TU, TI, sc
        # Gram matrices of the image / text tables over BOTH sides (feat_reg touches img_i, txt_i, img_u, txt_u): one-time fp64 products
        self.gram = []
        for j in range(len(sd.reg_weights)):
            c0, w = self.col0[j], widths[j]
            A, Bm = TU[:, c0:c0 + w].double(), TI[:, c0:c0 + w].double()
            G = (A.t() @ A + Bm.t() @ Bm).float().contiguous()
            h = (A.t() @ TU[:, sc].double() + Bm.t() @ TI[:, sc].double()).float().contiguous()
            n2 = float((TU[:, sc].double() ** 2).sum() + (TI[:, sc].double() ** 2).sum())
            self.gram.append((G, h, n2))

    def _tab(self, T, j):
        return T[:, self.col0[j]:self.col0[j] + self.widths[j]]

    # ---- full forward (eval, MM_Model.forward): projections of the propagated tables, no side-feature SpMM ------------
    def forward(self):
        d, m, p, S = self.d, self.cfg.proj_mode, self.p, self.S
        probs, r1 = [], []
        for j in range(S):
            W, b = self.sides.param(p, j)
            probs.append((self._tab(self.TU, j), W, None, self.blk(self.Fu, j)))
            probs.append((self._tab(self.TI, j), W, None, self.blk(self.Fi, j)))
            r1 += [(self.blk(self.Fu, j), self.TU[:, self.sc], b), (self.blk(self.Fi, j), self.TI[:, self.sc], b)]
        Wu, bu = self.sides.param(p, S)
        probs += [(self._tab(self.TU, S), Wu, None, self.prof_u), (self._tab(self.TI, S), Wu, None, self.prof_i)]
        r1 += [(self.prof_u, self.TU[:, self.sc + 1], bu), (self.prof_i, self.TI[:, self.sc + 1], bu)]
        probs.sort(key=lambda t: -t[0].shape[1])
        with self._t("proj_fwd"):
            ops.proj_fwd_group(probs, d, m)
            ops.rank1_add(r1)
        self._prop_fwd(with_feats=False)
        self._fuse_fwd()
        return self.U, self.I

    def _fold_in_sources(self, users, R):
        """fold_in reads Pi = X.W^T + b and fold_in_items P_usr = X_usr.W_u^T + b_u, which this engine never materialises (its forward
        projects the propagated tables): one grouped projection per call, of the full item-side tables into the engine's Pi or of
        the user table into its P_usr, which no hoisted step reads.  Fu, which fold_in_items also reads, is written by the forward
        (TU.W^T + cu b^T)."""
        sd, f, p = self.sides, self.feats, self.p
        probs = sd.proj_problems(f, p, Pi=self.Pi) if users else sd.proj_problems(f, p, P_usr=self.P_usr)
        ops.proj_fwd_group(probs, self.d, self.cfg.proj_mode)

    # ---- compact buffers of a training step ---------------------------------------------------------------------------
    def _ensure_compact(self, cap):
        c = self._compact
        if c is not None and c["cap"] == cap:
            return c
        dev, d, S, new = self.E_u.device, self.d, self.S, lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.E_u.device)
        c = dict(cap=cap, Xu=new(cap, self.Kc), Xi=new(2 * cap, self.Kc),
                 Fu=new(cap, S * d), Fi=new(2 * cap, S * d), pu=new(cap, d), pi=new(2 * cap, d),
                 GFu=new(cap, S * d), GFi=new(2 * cap, S * d), Gpu=new(cap, d), Gpi=new(2 * cap, d),
                 U=new(cap, d), I=new(2 * cap, d), gU=new(cap, d), gI=new(2 * cap, d), dU=new(cap, d), dI=new(2 * cap, d),
                 ar=torch.arange(cap, dtype=torch.int32, device=dev), ar2=torch.arange(cap, 2 * cap, dtype=torch.int32, device=dev))
        if self.cfg.deterministic:                                # rank scratch of the two ordered scatters (they may overlap: one each)
            c.update(rank_u=torch.zeros(2 * cap, dtype=torch.int32, device=dev), rank_i=torch.zeros(4 * cap, dtype=torch.int32, device=dev))
        self._compact = c
        return c

    def train_step(self, users, pos, neg, meta=None):
        """users/pos/neg: int32 CUDA index vectors of equal length (capacity-sized with `meta` = {B', n_keep} on the graph path).
        pos and neg must be the two halves of ONE contiguous [2 x cap] block (engine index buffer rows 1-2, or a fresh cat)."""
        if self.opt is None:
            raise RuntimeError("attach an optimizer with set_optimizer() first")
        cfg, d, S, L, p, m, sd = self.cfg, self.d, self.S, self.L, self.p, self.cfg.proj_mode, self.sides
        cap = int(users.numel())
        self.ensure_capacity(max(cap, self.batch_capacity()) if meta is None else cap)
        c = self._ensure_compact(cap)
        if pos.data_ptr() + 4 * cap == neg.data_ptr():
            pn = torch.as_strided(pos, (2 * cap,), (1,))
        else:
            pn = c.setdefault("pn", torch.empty(2 * cap, dtype=torch.int32, device=users.device))
            pn[:cap].copy_(pos); pn[cap:].copy_(neg)
        blk = self.blk
        tab = lambda X, j: X[:, self.col0[j]:self.col0[j] + self.widths[j]]
        g = self.grads
        creg = cfg.feat_reg_decay / self.ni
        reg_names = sd.reg_weights
        det = cfg.deterministic
        # deterministic steps: the compact blocks give every triplet rows of its own, so the heads' only shared destination is Gpu (the
        # attribute heads, folded in head order), and the scatters of dU / dI into the dense tables (a batch repeats users and items)
        # add in ascending batch position
        scatter = (lambda G, idx, Y, key: ops.scatter_add_rows_ordered(G, idx, Y, scratch=c[key])) if det else (lambda G, idx, Y, key: ops.scatter_add_rows(G, idx, Y))

        # ---- branches: ID layers | first touch of the gradient buffers + feat_reg  ||  main: the batch's side-feature rows ----
        def init_branch():
            # feat_reg (main.py:151-156) and its gradient depend on the parameters only (Gram form): they are written FIRST into zeroed
            # weight / bias gradients; the batch terms below accumulate on top
            zero = [(c["gU"], None, 0.0), (c["gI"], None, 0.0), (c["GFu"], None, 0.0), (c["GFi"], None, 0.0), (c["Gpu"], None, 0.0),
                    (c["Gpi"], None, 0.0), (self.dUl, None, 0.0), (self.dIl, None, 0.0)]
            for name in reg_names:
                zero += [(g[name + ".weight"], None, 0.0), (g[name + ".bias"].view(1, -1), None, 0.0)]
            with self._t("grad_init"):
                ops.grad_init(zero, self.loss)
            with self._t("feat_reg"):
                for j, name in enumerate(reg_names):
                    G, h, n2 = self.gram[j]
                    ops.feat_reg_gram(p[name + ".weight"], p[name + ".bias"], G, h, n2, creg, g[name + ".weight"], g[name + ".bias"], self.loss)
            if det:
                self._plan_slots(c["ar"], c["ar"], c["ar2"], meta)

        self._fork(lambda: self._prop_fwd(with_feats=False), lane=0)                          # ID layers (Models.py:169-183)
        self._fork(init_branch, lane=1)
        with self._t("gather"):
            ops.gather_rows(self.TU, users, c["Xu"])
            ops.gather_rows(self.TI, pn, c["Xi"])
        probs, r1 = [], []
        for j in range(S):
            W, b = sd.param(p, j)
            probs += [(tab(c["Xu"], j), W, None, blk(c["Fu"], j)), (tab(c["Xi"], j), W, None, blk(c["Fi"], j))]
            r1 += [(blk(c["Fu"], j), c["Xu"][:, self.sc], b), (blk(c["Fi"], j), c["Xi"][:, self.sc], b)]
        Wu, bu = sd.param(p, S)
        probs += [(tab(c["Xu"], S), Wu, None, c["pu"]), (tab(c["Xi"], S), Wu, None, c["pi"])]
        r1 += [(c["pu"], c["Xu"][:, self.sc + 1], bu), (c["pi"], c["Xi"][:, self.sc + 1], bu)]
        probs.sort(key=lambda t: -t[0].shape[1])
        with self._t("proj_fwd"):
            ops.proj_fwd_group(probs, d, m)                                                   # Models.py:145-167 on the batch's rows
            ops.rank1_add(r1)
        self._join()
        coefs, su, si = sd.coefs(cfg), sd.fused(c["Fu"], c["pu"]), sd.fused(c["Fi"], c["pi"])
        with self._t("fuse_fwd"):
            self._fork(lambda: ops.fuse_fwd(self.Ul, su, coefs, c["U"], rows=users, compact=True))   # :185-197 on the batch's rows
            ops.fuse_fwd(self.Il, si, coefs, c["I"], rows=pn, compact=True)
            self._join()
        # ---- losses + output gradients ----
        heads = [(c["U"], c["I"], c["gU"], c["gI"], 1.0, 1.0)] + sd.heads(cfg, c["Fu"], c["pu"], c["GFu"], c["Gpu"], c["Fi"], c["GFi"])
        n_keep = int((1 - cfg.prune_loss_drop_rate) * cap)
        with self._t("bpr"):
            ops.bpr_heads(heads, c["ar"], c["ar"], c["ar2"], n_keep, cfg.regs0 / cfg.batch_size, self.head_out, self.loss, self._bpr_work, meta=meta,
                          **({"ordered": self._slot_plan} if det else {}))
        # ---- backward: fusion on the compact rows, ID gradients scattered into the dense chain ----
        dsu, dsi = sd.fused(c["GFu"], c["Gpu"]), sd.fused(c["GFi"], c["Gpi"])

        def user_side_bwd():
            ops.fuse_bwd(c["gU"], L + 1, c["dU"], su, coefs, dsu, True)
            scatter(c["dU"], users, self.dUl, "rank_u")                                       # rows past B' carry zero gradients

        with self._t("fuse_bwd"):
            self._fork(user_side_bwd)
            ops.fuse_bwd(c["gI"], L + 1, c["dI"], si, coefs, dsi, True)
            scatter(c["dI"], pn, self.dIl, "rank_i")
            self._join()
        # ---- branch: the dense ID chain  ||  main: weight / bias gradients from the compact rows ----
        self._fork(lambda: self._chain_bwd(with_feats=False), lane=0)
        wg, seen = [], set(reg_names)                             # image / text gradients already hold the feat_reg term
        bias_terms = {}
        for j in list(range(S)) + [S]:
            name = sd.weights[j]
            dYu, dYi = (blk(c["GFu"], j), blk(c["GFi"], j)) if j < S else (c["Gpu"], c["Gpi"])
            scol = self.sc if j < S else self.sc + 1
            wg.append((tab(c["Xu"], j), dYu, g[name + ".weight"], None, name in seen)); seen.add(name)
            wg.append((tab(c["Xi"], j), dYi, g[name + ".weight"], None, True))
            bias_terms.setdefault(name, []).extend([(dYu, c["Xu"][:, scol]), (dYi, c["Xi"][:, scol])])
        def bias_grads():
            for name, terms in bias_terms.items():
                ops.scaled_colsum(terms, g[name + ".bias"], accumulate=name in reg_names)

        with self._t("proj_wgrad"):
            self._fork(bias_grads, lane=1)
            ops.proj_wgrad_group(wg, d, m)
        self._join()
        with self._t("adamw"):
            self.opt.step([self.grads[k] for k in self._opt_names])
        return self.loss

    def loss_and_output_grads(self, users, pos, neg, meta=None):
        raise NotImplementedError("the hoisted engine runs whole steps (train_step); use the default engine for the piecewise API")

    def families(self, users, pos, neg):
        return {"step": lambda: self.train_step(users, pos, neg)}
