"""The fused hot path: forward, losses, backward and AdamW of one LLMRec training step,
scheduled by hand over the sm_90a kernels (no autograd, no host synchronisation).

Follows (reference file:line):  MM_Model.forward  Models.py:127-199 ; bpr_loss / prune_loss /
feat_reg / loss assembly  main.py:330-342,158-165,151-156,273 ; AdamW  main.py:100-104,278.
Default flags (mask off, dropout p = 0); the mask / MAE branch drives the same pieces eagerly from main.Trainer._train_batch_masked.

HBM layout (fp32, row-major):
  Pi  [ni x S*d]  side-feature projections, column blocks  img | txt | att_0..att_4      (S = 2 + #keys)
  Fu  [nu x S*d]  ui . Pi      (img_u | txt_u | att_u)        Fi [ni x S*d]  iu . Fu  (img_i | txt_i | att_i)
  P_usr [nu x d], prof_i [ni x d] = iu . P_usr, prof_u [nu x d] = ui . prof_i
  Ul[l] [nu x d], Il[l] [ni x d]  ID layers (l = 0 is the embedding table itself)
  U [nu x d], I [ni x d]          fused outputs
Every operand that shares a sparsity pattern rides in ONE SpMM launch (segments), so the reference's
20 forward SpMMs are 2L launches (4 at L = 2) and the 20 backward ones 2L + 1.

Schedule: a step is a small DAG, not a chain.  `_fork` / `_join` put independent launches on side streams (event fork / join):
the ID layers beside the projection kernel and the side-feature products, the first touch of the gradient buffers beside the
tail of the forward pass, user- and item-side fusion side by side, the ID backward chain beside the side-feature chain and the
weight-gradient kernel.  Captured, that is ONE CUDA graph with parallel branches (0.84 -> 0.74 ms per step at the netflix shape);
on CPU stand-ins and under the span timer the same launches run in program order.

Batch-row fusion: during training only the loss heads read U / I, at the batch's rows, and they scatter gU / gI into those rows only.
So train_step fuses the batch's rows alone, in both directions.  A branch forked at the start of the step builds two device-side row
sets from the index buffer (`_batch_rows`: users, and pos | neg items, augmented triplets included; a repeated id is one row; only the
first B' entries of a captured step's buffer are live) -- no host sync, one graph for every B'.  The fusion kernels then take the
row list with its device-side count; each listed row runs the same per-row code as the full form, so it gets the same bits.  Off the
batch the full backward would write dUl = dIl = 0 and add an exact zero to GFu / GFi / Gprof_*; `_grad_init(id_grads=True)` zeroes
dUl / dIl instead, and the side-feature gradients already hold their final values.  Rows of U / I outside the batch keep stale values
after a training step: `forward()` (evaluation, MM_Model, the eager mask / MAE branch) fuses every row.  At the netflix shape the two
fusion families drop from 0.041 + 0.081 ms to 0.008 + 0.011 ms (H100 SXM 80 GB HBM3, 700 W; DESIGN §5).

Deterministic steps (`HotPathConfig.deterministic`, off by default): the loss heads' scatter of row gradients is the one launch of the
default 3xTF32 / TF32 step whose float adds land in a schedule-dependent order (a batch repeats users and items, and the attribute heads
share Gprof_u).  When set, the same branch that builds the row sets sorts the batch's slots by (row, slot) (`ops.bpr_slot_plan`, from the
index buffer alone), and the heads gather each destination row in a fixed order -- heads ascending, batch positions ascending, pos before
neg (include/llmrec_b200.h) -- so two runs of a step give the same bits, graph or eager, with or without branches.

Live items: Pi[i] is read only by Fu = ui . Pi, and only when item i is a column of ui; GPi[i] = (ui^T GFu)[i] is an empty row, exactly
zero, when item i has no training edge.  So the projections skip those rows: `_build_live_items` fixes the set of items with a training
edge once (the non-empty rows of ui^T), copies their rows of the item-side tables into compact tables (`fx`), and zeroes Pi once.  The
forward writes compact row r to Pi[live_i[r]] (same bits as the full-table call); the weight gradient pairs compact row r with
GPi[live_i[r]] (dW differs by rounding only; db still sums every row of GPi, so it keeps its bits).  Skipped when every item has an
edge.  At the netflix shape 30 % of the items have none: the two projection families read 372 MB less per step.
"""
from __future__ import annotations

import contextlib
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import ops
from .sides import SideLayout


@dataclass
class HotPathConfig:
    embed_size: int = 64
    n_layers: int = 2                 # len(weight_size)
    model_cat_rate: float = 0.02
    user_cat_rate: float = 2.8
    item_cat_rate: float = 0.005
    aug_mf_rate: float = 0.012
    mm_mf_rate: float = 1e-4
    prune_loss_drop_rate: float = 0.71
    feat_reg_decay: float = 1e-5
    regs0: float = 1e-5
    batch_size: int = 1024
    aug_sample_rate: float = 0.1      # main.py:218: a batch grows by at most int(batch_size * rate) augmented triplets
    proj_mode: int = 0                # ops.PROJ_MODE
    deterministic: bool = False       # loss-head row gradients accumulated in a fixed order instead of with float atomics (bit-reproducible steps)


PARAM_ORDER = ("image_trans.weight", "image_trans.bias", "text_trans.weight", "text_trans.bias",
               "user_trans.weight", "user_trans.bias", "item_trans.weight", "item_trans.bias",
               "user_id_embedding.weight", "item_id_embedding.weight")


def _known_ids(known, m, n, msg):
    """The `known` argument of a fold-in: None (every row -1) or one id in [0, n) or -1 per row -> int64[m]; else ValueError(msg)."""
    kn = np.full(m, -1, dtype=np.int64) if known is None else \
        (known.detach().cpu().numpy() if hasattr(known, "detach") else np.asarray(known)).astype(np.int64).reshape(-1)
    if kn.size != m or (m and (kn.min() < -1 or kn.max() >= n)):
        raise ValueError(msg.format(n=n, m=m))
    return kn


class KernelTimer:
    """CUDA-event timer per kernel family on the current stream (bench.py's roofline leg)."""

    def __init__(self):
        self.spans = []

    @contextlib.contextmanager
    def span(self, name):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        yield
        b.record()
        self.spans.append((name, a, b))

    def totals(self):
        """name -> (total ms, count) ; call after a synchronize."""
        out = {}
        for name, a, b in self.spans:
            t, c = out.get(name, (0.0, 0))
            out[name] = (t + a.elapsed_time(b), c + 1)
        return out


class HotPath:
    """params: dict name -> fp32 CUDA tensor (the live parameter storage, updated in place).
    feats: None (ID-only, the large synthetic config) or dict(image, text, user, item={key: tensor})."""

    compact_items = True              # project the item-side tables on the live items only (`_build_live_items`); off in subclasses
                                      # that never run the full-table projections

    def __init__(self, operators, params, feats, cfg: HotPathConfig):
        self.ui, self.iu, self.uiT, self.iuT = operators
        self.cfg = cfg
        if cfg.deterministic and cfg.proj_mode == 2:
            raise ValueError("deterministic steps need the tensor-core projections (proj_mode 3xtf32 / tf32): the fp32 SIMT weight gradient "
                             "adds its row chunks with float atomics")
        self.p = params
        self.feats = feats
        d, L = cfg.embed_size, cfg.n_layers
        self.E_u, self.E_i = params["user_id_embedding.weight"], params["item_id_embedding.weight"]
        nu, ni = self.E_u.shape[0], self.E_i.shape[0]
        self.nu, self.ni, self.d, self.L = nu, ni, d, L
        dev = self.E_u.device
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        self.has_feats = feats is not None
        self.keys = list(feats["item"].keys()) if self.has_feats else []
        self.sides = SideLayout(self.keys, d) if self.has_feats else None
        S = self.S = self.sides.S if self.has_feats else 0
        self.fx = feats                                                    # what the projection kernels read
        if self.has_feats:
            self.Pi, self.Fu, self.Fi = new(ni, S * d), new(nu, S * d), new(ni, S * d)
            self.P_usr, self.prof_i, self.prof_u = new(nu, d), new(ni, d), new(nu, d)
            self.GPi, self.GFu, self.GFi = new(ni, S * d), new(nu, S * d), new(ni, S * d)
            self.GP_usr, self.Gprof_i, self.Gprof_u = new(nu, d), new(ni, d), new(nu, d)
        self.Ul = [self.E_u] + [new(nu, d) for _ in range(L)]
        self.Il = [self.E_i] + [new(ni, d) for _ in range(L)]
        self.U, self.I = new(nu, d), new(ni, d)
        # gradients
        self.gU, self.gI = new(nu, d), new(ni, d)
        self.dIl = new(ni, d)
        self.bufU, self.bufI, self.tmpI = new(nu, d), new(ni, d), new(ni, d)
        self.grads = {k: torch.zeros_like(v) for k, v in params.items()}
        self.dUl = self.grads["user_id_embedding.weight"]
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.n_heads = (3 + len(self.keys)) if self.has_feats else 1
        self.head_out = torch.zeros(self.n_heads * 4, dtype=torch.float32, device=dev)
        self._bpr_work, self._cap, self._graph = None, 0, None
        self._slot_plan = None            # cfg.deterministic: the step's slot plan (ops.bpr_slot_plan), sized with _bpr_work
        self.pre_step = None              # optional launches replayed in front of every staged step (device-side batch sampler)
        self.pre_step_undo = None         # undoes the side effect of ONE pre_step (the warm-up step before a capture must not consume a batch)
        self.pre_step_save = None         # called before the warm-up's pre_step: keeps what pre_step_undo puts back
        self.post_step = None             # optional launches after every staged step (joins what pre_step forked)
        self.opt = None
        self.timer = None
        # independent launches of a step run as BRANCHES: a side stream forked from / joined into the current one with events, so the
        # captured step is a graph with parallel nodes (LLMREC_BRANCHES=0: one chain; off on CPU stand-ins and under the span timer)
        self.branches = dev.type == "cuda" and os.environ.get("LLMREC_BRANCHES", "1") != "0"
        self._side, self._forked = {}, set()
        self.force_split = False          # tests: run the branch SCHEDULE (split launches) even where nothing can overlap (CPU stand-ins)
        # train_step fuses only the batch's rows, in both directions (`_batch_rows`).  Gated like `branches`: CUDA devices only, so the
        # CPU stand-ins keep running the full-row schedule their emulated ops implement; and only with side features, so the ID-only
        # engine keeps U / I whole after a step -- it is the single-GPU reference the sharded engines are compared with row by row.
        self.demand_fuse = dev.type == "cuda" and self.has_feats
        if self.demand_fuse:
            self.batch_u, self.batch_i = ops.RowSet(nu, dev), ops.RowSet(ni, dev)
            self._batch_max = (0, 0)
        # the live item set: gated like `demand_fuse` (the CPU stand-ins keep the full-table projections); LLMREC_LIVE_ITEMS=0 turns it off
        self.live_i, self.n_live, self._live_pos = None, ni, None
        if self.has_feats and dev.type == "cuda" and self.compact_items and os.environ.get("LLMREC_LIVE_ITEMS", "1") != "0":
            self._build_live_items()

    def _build_live_items(self):
        """Items with a training edge = the non-empty rows of ui^T = the distinct columns of ui.  With some items edgeless: the compact
        item-side tables X[live_i] (the tables' own dtype) become what the projections read, and Pi is zeroed once -- its edgeless rows
        are never written again, and no product reads them.  The full tables stay (the hoisted precompute, the --mask branch and MM_Model
        read them)."""
        dev = self.E_u.device
        rp = self.uiT.rowptr.long()
        live = torch.nonzero(rp[1:] > rp[:-1]).flatten()
        cols = torch.unique(self.ui.col.long())
        if not torch.equal(live.cpu(), cols.cpu()):
            raise RuntimeError("live items: the non-empty rows of ui^T are not the distinct columns of ui")
        n_live = int(live.numel())
        if n_live == self.ni:
            return
        self.live_i, self.n_live = live.to(torch.int32).contiguous(), n_live
        self._live_pos = torch.full((self.ni,), -1, dtype=torch.long, device=dev)
        self._live_pos[live] = torch.arange(n_live, device=dev)
        f = self.feats
        self.fx = dict(image=f["image"][live].contiguous(), text=f["text"][live].contiguous(), user=f["user"],
                       item={k: v[live].contiguous() for k, v in f["item"].items()})
        self.Pi.zero_()

    def refresh_item_feats(self, rows):
        """The full item-side tables were overwritten at `rows` (the --mask branch rewrites attribute rows in place): copy those rows into
        the compact tables the projections read.  A no-op without a live item set."""
        if self.live_i is None:
            return
        rows = rows.to(self._live_pos.device).long()
        pos = self._live_pos[rows]
        keep = pos >= 0
        src, dst = rows[keep], pos[keep]
        for name in ("image", "text"):
            self.fx[name][dst] = self.feats[name][src]
        for k, v in self.feats["item"].items():
            self.fx["item"][k][dst] = v[src]

    def _t(self, name):
        return self.timer.span(name) if self.timer is not None else contextlib.nullcontext()

    # ---- branches -------------------------------------------------------------------------------
    def _fork(self, thunk, lane=0):
        """Run `thunk` on side stream `lane`, ordered after everything enqueued on the current stream so far; `_join` orders the current
        stream behind every lane used since the last join.  Every buffer a branch touches is a persistent engine buffer, so no allocator
        bookkeeping is needed."""
        if not self.branches or self.timer is not None:
            thunk()
            return
        st = self._side.get(lane)
        if st is None:
            st = self._side[lane] = torch.cuda.Stream(device=self.E_u.device)
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            thunk()
        self._forked.add(lane)

    def _opset(self, k):
        """(ui, iu, uiT, iuT) with their own long-row scratch / tickets: launches through set k may overlap launches of the primary set
        and of the other sets."""
        sets = self.__dict__.setdefault("_opsets", {})
        if k not in sets:
            sets[k] = tuple(o.branch() for o in (self.ui, self.iu, self.uiT, self.iuT))
        return sets[k]

    def _join(self, lanes=None):
        for lane in sorted(self._forked if lanes is None else self._forked & set(lanes)):
            torch.cuda.current_stream().wait_stream(self._side[lane])
            self._forked.discard(lane)

    # ---- column-block views ------------------------------------------------------------------
    def blk(self, buf, s):
        d = self.d
        return buf[:, s * d:(s + 1) * d]

    def side_views(self, grads=False):
        """name -> tensor views of the side outputs of the reference's return tuple (Models.py:199); att_i / att_u: key -> view.
        grads: their gradient buffers instead (p_usr has none: its gradient enters `backward` as gp_usr_direct)."""
        if not self.has_feats:
            return {}
        Fu, Fi, P_usr, prof_u, prof_i = ((self.GFu, self.GFi, None, self.Gprof_u, self.Gprof_i) if grads else
                                         (self.Fu, self.Fi, self.P_usr, self.prof_u, self.prof_i))
        b, att = self.blk, self.sides.att
        return dict(img_i=b(Fi, 0), txt_i=b(Fi, 1), img_u=b(Fu, 0), txt_u=b(Fu, 1), p_usr=P_usr, prof_u=prof_u, prof_i=prof_i,
                    att_i=dict(zip(self.keys, att(Fi))), att_u=dict(zip(self.keys, att(Fu))))

    def outputs(self):
        """(output, gradient buffer) pairs in the order of the reference's return tuple (Models.py:199): U, I, img_i, txt_i, img_u,
        txt_u, p_usr, prof_u, prof_i, att_u per key, att_i per key."""
        out = [(self.U, self.gU), (self.I, self.gI)]
        if self.has_feats:
            v, g = self.side_views(), self.side_views(grads=True)
            out += [(v[n], g[n]) for n in ("img_i", "txt_i", "img_u", "txt_u", "p_usr", "prof_u", "prof_i")]
            out += [(v[a][k], g[a][k]) for a in ("att_u", "att_i") for k in self.keys]
        return out

    # ---- forward -------------------------------------------------------------------------------
    def forward(self):
        self._proj_fwd()
        self._prop_fwd()
        self._fuse_fwd()
        return self.U, self.I

    def _proj_fwd(self):
        if self.has_feats:
            with self._t("proj_fwd"):                                                    # compact item tables -> Pi[live_i]
                ops.proj_fwd_group(self.sides.proj_problems(self.fx, self.p, self.Pi, self.P_usr, self.live_i), self.d, self.cfg.proj_mode)

    def _prop_fwd(self, with_feats=None, after_sides=None, with_ids=True, opset=None):
        """with_feats=False: the ID layers only (the hoisted mode propagates no side-feature operand); with_ids=False: the side-feature
        operands only (train_step runs the ID layers as a branch beside the projections).  opset: (ui, iu) to launch through.
        after_sides: called once Fu and Fi exist (after the second product; at once without side features) -- train_step forks the
        first touch of the gradient buffers there."""
        L, S = self.L, self.S
        wf = self.has_feats if with_feats is None else with_feats
        ui, iu = (self.ui, self.iu) if opset is None else opset
        if after_sides is not None and not wf:
            after_sides()
        # step t even: ui (I_{t/2} -> U_{t/2+1});  t odd: iu (U_{(t+1)/2} -> I_{(t+1)/2}); softmax on the last layer
        n_steps = max(2 * L if with_ids else 0, 3 if wf else 0)
        for t in range(n_steps):
            segs = []
            if t % 2 == 0:
                l = t // 2 + 1
                if wf and t == 0:
                    segs += [(self.blk(self.Pi, s), self.blk(self.Fu, s), None, False) for s in range(S)]                # :153,156,162
                if wf and t == 2:
                    segs.append((self.prof_i, self.prof_u, None, False))                                               # :167
                if with_ids and l <= L:
                    segs.append((self.Il[l - 1], self.Ul[l], None, l == L))                                            # :174,178
                with self._t("spmm_fwd"):
                    ui.apply(segs)
            else:
                l = (t + 1) // 2
                if wf and t == 1:
                    segs += [(self.blk(self.Fu, s), self.blk(self.Fi, s), None, False) for s in range(S)]                # :154,157,163
                    segs.append((self.P_usr, self.prof_i, None, False))                                                # :166
                if with_ids and l <= L:
                    segs.append((self.Ul[l], self.Il[l], None, l == L))                                                # :175,180
                with self._t("spmm_fwd"):
                    iu.apply(segs)
                if after_sides is not None and wf and t == 1:
                    after_sides()

    def _batch_rows(self, users, pos, neg, meta=None):
        """Device-side row sets of the step's batch: its users, and its pos | neg items (augmented triplets included); a repeated id is
        one row.  With `meta` only the first B' = meta[0] entries are live (the index buffer's later slots hold earlier batches' ids)."""
        n = None if meta is None else meta[:1]
        self.batch_u.clear()
        self.batch_u.add_ids(users, n)
        self.batch_u.compact()
        self.batch_i.clear()
        self.batch_i.add_ids(pos, n)
        self.batch_i.add_ids(neg, n)
        self.batch_i.compact()
        self._batch_max = (min(self.nu, int(users.numel())), min(self.ni, int(pos.numel()) + int(neg.numel())))

    def _rows_kw(self, batch_rows):
        """Keyword arguments of the user- and item-side fusion: all rows, or the row sets of the last `_batch_rows`."""
        if not batch_rows:
            return {}, {}
        mu, mi = self._batch_max
        return (dict(rows=self.batch_u.list, count=self.batch_u.count, max_rows=mu),
                dict(rows=self.batch_i.list, count=self.batch_i.count, max_rows=mi))

    def _side_coefs(self):
        """fusion weights of the side terms (SideLayout.coefs; none without side features)"""
        return self.sides.coefs(self.cfg) if self.has_feats else []

    def _fuse_fwd(self, batch_rows=False):
        """batch_rows: U / I on the batch's rows only (train_step); the other rows keep whatever they held."""
        coefs, su, si = self._side_coefs(), [], []
        if self.has_feats:
            su, si = self.sides.fused(self.Fu, self.prof_u), self.sides.fused(self.Fi, self.prof_i)
        ku, ki = self._rows_kw(batch_rows)
        with self._t("fuse_fwd"):
            self._fork(lambda: ops.fuse_fwd(self.Ul, su, coefs, self.U, **ku))                                         # :185-197
            ops.fuse_fwd(self.Il, si, coefs, self.I, **ki)
            self._join()
        self._fuse_args = (coefs, su, si)

    # ---- fold-in: one side of the forward for rows given at call time ----------------------------------------------------------
    def fold_in(self, rowptr, col, known=None):
        """-> U_new [m x d]: the fused representation of m users whose histories are the rows of an int CSR over item ids (rowptr[m+1],
        col; `graph.history_matrix` rejects ids outside [0, n_items) and collapses repeats).  known: optional int[m], the trained user id
        of each row or -1.  Reads the item side of the last full `forward()` (Pi, prof_i, Il) and the parameters; writes no buffer a
        training step reads.

        Every user-side quantity of the forward is the user's row of ui = diag(su) R times an item-side tensor (Fu = ui.Pi,
        prof_u = ui.prof_i, Ul[l] = [softmax] ui.Il[l-1]), so with R the new rows and su their (deg + 1e-8)^-1/2 these are ONE SpMM
        launch with S + 1 + L segments, followed by the fusion of the m rows.  Layer 0 is E_u[known] for a trained user; an unknown user
        has no ID embedding, and its layer 0 is a zero row (it enters the mean of the L + 1 layers as 0)."""
        from .graph import history_matrix
        R = history_matrix(rowptr, col, self.ni)
        kn = _known_ids(known, R.shape[0], self.nu, "fold_in: known must hold one trained user id in [0, {n}) or -1 per history ({m})")
        return self._fold_in(True, R, kn)

    def fold_in_items(self, rowptr, col, known=None):
        """-> I_new [m x d]: the fused representation of m items whose interactions are the rows of an int CSR over trained user ids
        (rowptr[m+1], col; `graph.history_matrix` rejects ids outside [0, n_users) and collapses repeats).  known: optional int[m], the
        trained item id of each row or -1.  Reads the user side of the last full `forward()` (Fu, P_usr, Ul) and the parameters; writes
        no buffer a training step reads.

        The mirror of `fold_in`: every item-side quantity of the forward is the item's row of iu = diag(si) R^T times a user-side
        tensor (Fi = iu.Fu, prof_i = iu.P_usr, Il[l] = [softmax] iu.Ul[l]), so with R^T the new rows and si their (deg + 1e-8)^-1/2 these
        are ONE SpMM launch with S + 1 + L segments, followed by the fusion of the m rows.  Layer 0 is E_i[known] for a trained item and
        a zero row for a new one.  The item's own side features enter no term of its row (they reach items only through two hops)."""
        from .graph import history_matrix
        R = history_matrix(rowptr, col, self.nu, what="new items", unit="user id")
        kn = _known_ids(known, R.shape[0], self.ni, "fold_in_items: known must hold one trained item id in [0, {n}) or -1 per item ({m})")
        return self._fold_in(False, R, kn)

    def fold_in_operands(self, rowptr, col, known=None):
        """The per-row operands of `fold_in` before the fusion -> (layers, F, prof, su): the L + 1 layers [m x d] (layer 0 = E_u[known]
        or zeros), the side-feature blocks F [m x S*d] and profile rows prof [m x d] (None without side features) and the row scales su
        fp32 [m] of ui = diag(su) R.  `fold_in` fuses exactly these; explanations split a score over them (recommend.explain)."""
        from .graph import history_matrix
        R = history_matrix(rowptr, col, self.ni)
        kn = _known_ids(known, R.shape[0], self.nu, "fold_in: known must hold one trained user id in [0, {n}) or -1 per history ({m})")
        return self._fold_in_operands(True, R, kn)

    def _fold_in(self, users, R, kn):
        """The fold-in of m new rows of one side (users: R's rows are users over item ids, else items over user ids) with layer-0 ids
        kn: the operands of `_fold_in_operands`, fused."""
        m, d, dev = R.shape[0], self.d, self.E_u.device
        if m == 0:
            return torch.empty(0, d, dtype=torch.float32, device=dev)
        layers, F, prof, _ = self._fold_in_operands(users, R, kn)
        sides = self.sides.fused(F, prof) if self.has_feats else []
        out = torch.empty(m, d, dtype=torch.float32, device=dev)
        ops.fuse_fwd(layers, sides, self._side_coefs(), out)                                                                # :185-197
        return out

    def _fold_in_operands(self, users, R, kn):
        """The one launch of a fold-in: the segments are the other side's S blocks, its profile and its ID layers (softmax on l = L).
        -> (layers [L + 1] of [m x d], F [m x S*d] or None, prof [m x d] or None, the rows' scales fp32 [m])."""
        from .graph import inv_sqrt_degree
        m, d, L, dev = R.shape[0], self.d, self.L, self.E_u.device
        train_op, E = (self.ui, self.E_u) if users else (self.iu, self.E_i)
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a.astype(dt))).to(dev)
        new = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        rs = t(inv_sqrt_degree(R), np.float32)
        if m == 0:
            return [new(0, d) for _ in range(L + 1)], *((new(0, self.S * d), new(0, d)) if self.has_feats else (None, None)), rs
        op = ops.CsrOperator(t(R.indptr, np.int32), t(R.indices, np.int32), m, R.shape[1], rs=rs,
                             tile_nnz=getattr(train_op.plan, "tile_nnz", 0))       # pieces cut as the training operator cuts them
        layers = [new(m, d) for _ in range(L + 1)]
        self._fold_in_sources(users, R)
        segs, F, prof = [], None, None
        if self.has_feats:
            F, prof = new(m, self.S * d), new(m, d)
            src_F, src_prof = (self.Pi, self.prof_i) if users else (self.Fu, self.P_usr)                   # :153-157,162-163,166-167
            segs += [(self.blk(src_F, s), self.blk(F, s), None, False) for s in range(self.S)]
            segs.append((src_prof, prof, None, False))
        src_layers = self.Il[:L] if users else self.Ul[1:]                                                    # :174-180
        segs += [(src_layers[l - 1], layers[l], None, l == L) for l in range(1, L + 1)]
        op.apply(segs)
        ops.gather_rows(E, t(kn, np.int32), layers[0])                          # known -> E row, -1 -> zeros
        return layers, F, prof, rs

    def _fold_in_sources(self, users, R):
        """Bring what a fold-in reads up to date: Pi on the items of R (users), or P_usr (items).  This engine's forward projects
        every user row, but the live items only, leaving Pi's edgeless rows zero, and a history given at call time may hold such an
        item.  Those rows are projected here with the grouped kernels and a row map into Pi's edgeless rows, which no training launch
        reads (no ui column points there)."""
        if not users or self.live_i is None:
            return
        if getattr(self, "_edgeless", None) is None:
            # once: the edgeless item ids and their rows of the item-side tables (the tables' own dtype), as _build_live_items does
            dead = torch.nonzero(self._live_pos < 0).flatten()
            f = self.feats
            self._edgeless = (dead.cpu().numpy(), dead.to(torch.int32).contiguous(),
                              dict(image=f["image"][dead].contiguous(), text=f["text"][dead].contiguous(),
                                   item={k: v[dead].contiguous() for k, v in f["item"].items()}))
        dead_np, dead, x = self._edgeless
        if dead_np.size == 0 or not np.isin(np.unique(R.indices), dead_np, assume_unique=True).any():
            return
        ops.proj_fwd_group(self.sides.proj_problems(x, self.p, Pi=self.Pi, rows=dead), self.d, self.cfg.proj_mode)

    # ---- backward: expects gU, gI and (GFu, GFi, Gprof_u, Gprof_i, GP_usr_direct) filled ---------------
    def backward(self, gp_usr_direct=None, batch_rows=False):
        self._fuse_bwd(batch_rows)
        self._chain_bwd(gp_usr_direct)
        self._wgrad()
        return self.grads

    def _fuse_bwd(self, batch_rows=False):
        """batch_rows: the batch's rows only -- gU / gI are zero on every other row, where the full form writes dUl = dIl = 0 and adds an
        exact zero to GFu / GFi / Gprof_*; `_grad_init(id_grads=True)` has zeroed dUl / dIl instead."""
        L = self.L
        coefs, su, si = self._fuse_args
        dsu, dsi = [], []
        if self.has_feats:
            dsu, dsi = self.sides.fused(self.GFu, self.Gprof_u), self.sides.fused(self.GFi, self.Gprof_i)
        ku, ki = self._rows_kw(batch_rows)
        with self._t("fuse_bwd"):
            self._fork(lambda: ops.fuse_bwd(self.gU, L + 1, self.dUl, su, coefs, dsu, True, **ku))
            ops.fuse_bwd(self.gI, L + 1, self.dIl, si, coefs, dsi, True, **ki)
            self._join()

    def _chain_bwd(self, gp_usr_direct=None, with_feats=None, with_ids=True, opset=None):
        """with_feats=False: the ID chain only; with_ids=False: the side-feature operands only; opset: (uiT, iuT) to launch through."""
        L, S = self.L, self.S
        wf = self.has_feats if with_feats is None else with_feats
        uiT, iuT = (self.uiT, self.iuT) if opset is None else opset
        if wf:
            # prof_u = ui . prof_i  ->  Gprof_i += ui^T Gprof_u
            with self._t("spmm_bwd"):
                uiT.apply([(self.Gprof_u, self.Gprof_i, self.Gprof_i, False)])
        gE_i = self.grads["item_id_embedding.weight"]
        g_cur_I = self.dIl
        for l in range(L, 0, -1):
            if not with_ids and l < L:
                break
            # I_l = [softmax] iu . U_l
            segs = []
            if with_ids:
                if l == L:
                    with self._t("softmax_bwd"):
                        src = ops.row_softmax_bwd(self.Il[l], g_cur_I, out=self.tmpI)
                else:
                    src = g_cur_I
                segs.append((src, self.bufU, self.dUl, False))
            if wf and l == L:
                segs += [(self.blk(self.GFi, s), self.blk(self.GFu, s), self.blk(self.GFu, s), False) for s in range(S)]
                segs.append((self.Gprof_i, self.GP_usr, gp_usr_direct, False))
            with self._t("spmm_bwd"):
                iuT.apply(segs)
            # U_l = [softmax] ui . I_{l-1}
            segs = []
            dst = gE_i if l == 1 else self.bufI
            if with_ids:
                if l == L:
                    with self._t("softmax_bwd"):
                        ops.row_softmax_bwd(self.Ul[l], self.bufU, out=self.bufU)
                segs.append((self.bufU, dst, self.dIl, False))
            if wf and l == L:
                segs += [(self.blk(self.GFu, s), self.blk(self.GPi, s), None, False) for s in range(S)]    # zero rows off the live items
            with self._t("spmm_bwd"):
                uiT.apply(segs)
            g_cur_I = dst

    def _wgrad(self):
        if self.has_feats:
            with self._t("proj_wgrad"):                                                  # compact row r <-> GPi[live_i[r]]
                probs = self.sides.wgrad_problems(self.fx, self.grads, self.GPi, self.GP_usr, self.live_i)
                ops.proj_wgrad_group(probs, self.d, self.cfg.proj_mode)

    # ---- losses + their gradients w.r.t. the forward outputs ---------------------------------------------
    def batch_capacity(self):
        """Largest B' a step of this configuration can see: batch_size sampled + int(batch_size * aug_sample_rate) augmented
        triplets (main.py:217-224), rounded up to a multiple of 8."""
        c = self.cfg
        return (c.batch_size + int(c.batch_size * c.aug_sample_rate) + 7) // 8 * 8

    def ensure_capacity(self, cap):
        """Index buffer [4 x cap] (rows users, pos, neg, meta = {B', n_keep}), the per-B' meta table, the BPR work block and (deterministic
        steps) the slot plan, sized ONCE for a batch capacity: every captured graph reads these addresses, so they are only ever replaced together
        with the graphs (ADVICE r1: a per-B' work buffer freed under a live graph was a use-after-free)."""
        if getattr(self, "_cap", 0) >= cap:
            return
        dev = self.E_u.device
        if getattr(self, "_graph", None) is not None:
            torch.cuda.synchronize()
        self._graph = None
        self._cap = int(cap)
        self._gidx = torch.zeros((4, self._cap), dtype=torch.int32, device=dev)
        keep = [int((1 - self.cfg.prune_loss_drop_rate) * b) for b in range(self._cap + 1)]      # main.py:161-162 (double arithmetic)
        self._meta_table = torch.tensor([[b, k] for b, k in enumerate(keep)], dtype=torch.int32).to(dev)
        self._bpr_work = ops.bpr_work(self.n_heads, self._cap, dev)
        if self.cfg.deterministic:
            self._slot_plan = torch.zeros(6 * self._cap, dtype=torch.int32, device=dev)

    def loss_and_output_grads(self, users, pos, neg, meta=None, init_done=False, plan_done=False):
        """users/pos/neg: int32 CUDA tensors of equal length B' (sampled + augmented triplets) -- or, with `meta` (int32 CUDA
        {B', n_keep}), capacity-sized buffers whose first B' entries are live (the CUDA-graph path).
        init_done: `_grad_init` already ran for this step (train_step forks it beside the tail of the forward pass).
        plan_done: the slot plan of a deterministic step was already built from these index arrays (train_step's row-set branch)."""
        c = self.cfg
        B = int(users.numel())
        self.ensure_capacity(max(B, self.batch_capacity()))
        n_keep = int((1 - c.prune_loss_drop_rate) * B)                     # main.py:161-162 (double arithmetic)
        heads = [(self.U, self.I, self.gU, self.gI, 1.0, 1.0)]                                                        # main.py:232-235
        if self.has_feats:
            heads += self.sides.heads(c, self.Fu, self.prof_u, self.GFu, self.Gprof_u, self.Fi, self.GFi)
        if not init_done:
            self._grad_init()
        with self._t("bpr"):
            if c.deterministic and not plan_done:
                self._plan_slots(users, pos, neg, meta)
            ops.bpr_heads(heads, users, pos, neg, n_keep, c.regs0 / c.batch_size, self.head_out, self.loss, self._bpr_work, meta=meta,
                          **({"ordered": self._slot_plan} if c.deterministic else {}))
        return self.loss

    def _plan_slots(self, users, pos, neg, meta=None):
        ops.bpr_slot_plan(users, pos, neg, meta=meta, plan=self._slot_plan)

    def _grad_init(self, id_grads=False):
        """First touch of every gradient buffer the loss heads accumulate into: the feat_reg gradient c*X on the image/text blocks (its
        value starts the loss, main.py:151-156), zeros elsewhere.  Needs Fu / Fi only, not the fused outputs.
        id_grads: also zero dUl / dIl, which the batch-row fusion backward writes on the batch's rows only."""
        c = self.cfg
        regions = [(self.gU, None, 0.0), (self.gI, None, 0.0)]
        if self.has_feats:
            creg, sd = c.feat_reg_decay / self.ni, self.sides
            regions += [(sd.reg(self.GFu), sd.reg(self.Fu), creg), (sd.reg(self.GFi), sd.reg(self.Fi), creg),
                        (self.Gprof_u, None, 0.0), (self.Gprof_i, None, 0.0)]
            if self.keys:
                regions += [(sd.unreg(self.GFu), None, 0.0), (sd.unreg(self.GFi), None, 0.0)]
        if id_grads:          # last: the loss's partial sums keep their slots, so its fixed-order reduction gives the same bits
            regions += [(self.dUl, None, 0.0), (self.dIl, None, 0.0)]
        with self._t("grad_init"):
            ops.grad_init(regions, self.loss)

    def train_step(self, users, pos, neg, meta=None):
        """forward + losses + backward + AdamW; everything stays on the current stream."""
        if self.opt is None:
            raise RuntimeError("attach an optimizer with set_optimizer() first")
        split = self.has_feats and self.timer is None and (self.branches or self.force_split)
        demand, det = self.demand_fuse, self.cfg.deterministic
        if det:
            self.ensure_capacity(max(int(users.numel()), self.batch_capacity()))     # the slot plan is filled before the heads size anything
        if demand or det:
            # the batch's row sets and the slot plan of a deterministic step depend on the indices only: a branch from the start of the step,
            # joined before the fusion
            def index_branch():
                if demand:
                    self._batch_rows(users, pos, neg, meta)
                if det:
                    self._plan_slots(users, pos, neg, meta)

            self._fork(index_branch, lane=1)
        grad_init = lambda: self._grad_init(id_grads=demand)
        if split:
            # the ID layers do not depend on the projections: they run as a branch (through operators with their own long-row scratch)
            # beside the projection kernel and the side-feature products; the first touch of the gradient buffers follows on the branch.
            # (Giving the two single-operand user-profile products a lane of their own was measured: no gain, removed.)
            ids = self._opset(0)
            if getattr(self, "_ev_ids", None) is None and self.branches:
                self._ev_ids = torch.cuda.Event()

            def id_layers():
                self._prop_fwd(with_feats=False, opset=ids[:2])
                if self.branches:
                    self._ev_ids.record()                                    # on the branch

            self._fork(id_layers, lane=0)
            self._proj_fwd()
            self._prop_fwd(with_ids=False, after_sides=lambda: self._fork(grad_init, lane=0))
            if self.branches:
                torch.cuda.current_stream().wait_event(self._ev_ids)         # the item-side fusion below reads Il; grad_init may still run
        else:
            self._proj_fwd()
            self._prop_fwd(after_sides=lambda: self._fork(grad_init))        # branch: runs beside the remaining products and the fusion
        self._join([1])                                                      # the row sets
        self._fuse_fwd(batch_rows=demand)                                    # joins
        self._join()
        self.loss_and_output_grads(users, pos, neg, meta, init_done=True, plan_done=det)
        if split:
            self._fuse_bwd(batch_rows=demand)
            self._fork(lambda: self._chain_bwd(with_feats=False, opset=ids[2:]), lane=0)    # ID chain
            self._chain_bwd(with_ids=False)                                                  # side-feature operands
            self._wgrad()
            self._join()
        else:
            self.backward(batch_rows=demand)
        with self._t("adamw"):
            self.opt.step([self.grads[k] for k in self._opt_names])
        return self.loss

    def families(self, users, pos, neg):
        """name -> thunk launching one kernel family of the step (bench.py times each from its own CUDA graph).  The fusion families run
        as train_step runs them: with the batch-row fusion, on the row sets of this batch (built here, outside the timed thunks), and
        the loss heads with the first touch of dUl / dIl that this fusion needs."""
        fuse_fwd, fuse_bwd = self._fuse_fwd, self._fuse_bwd
        loss_heads = lambda: self.loss_and_output_grads(users, pos, neg)
        if self.demand_fuse:
            self._batch_rows(users, pos, neg)
            fuse_fwd, fuse_bwd = (lambda: self._fuse_fwd(batch_rows=True)), (lambda: self._fuse_bwd(batch_rows=True))
            loss_heads = lambda: (self._grad_init(id_grads=True), self.loss_and_output_grads(users, pos, neg, init_done=True))
        f = {"spmm_fwd": self._prop_fwd, "fuse_fwd": fuse_fwd, "loss_heads": loss_heads,
             "fuse_bwd": fuse_bwd, "spmm_bwd": self._chain_bwd, "adamw": lambda: self.opt.step([self.grads[k] for k in self._opt_names])}
        if self.has_feats:
            f.update(proj_fwd=self._proj_fwd, proj_wgrad=self._wgrad)
        return f

    # ---- CUDA-graph replay of the whole step -----------------------------------------------------------
    def index_buffer(self, need):
        """The static [4 x cap] int32 buffer the captured step reads: rows users / pos / neg, row 3 = {B', n_keep, ...}."""
        self.ensure_capacity(max(int(need), self.batch_capacity()))
        return self._gidx

    def meta_row(self, B):
        """(B', n_keep) for the host side of a staging buffer (same double arithmetic as main.py:161-162)."""
        return int(B), int((1 - self.cfg.prune_loss_drop_rate) * B)

    def replay_staged(self):
        """Replay the captured step on whatever the index buffer holds (Trainer copies a pinned staging slot straight into it).
        ONE graph serves every batch length: the kernels take B' and n_keep from row 3 of the buffer."""
        if getattr(self, "_graph", None) is None:
            cap = self._cap
            u, p, n, meta = self._gidx[0], self._gidx[1], self._gidx[2], self._gidx[3]
            torch.cuda.synchronize()
            held = self._gidx.clone()
            if not getattr(self, "_warm", False):
                # one eager step at full capacity sizes every lazily allocated scratch buffer; its parameter update is undone
                snap = self._snapshot_state()
                self._gidx[3, :2].copy_(self._meta_table[cap])
                if self.pre_step_save is not None:
                    self.pre_step_save()
                if self.pre_step is not None:
                    self.pre_step()
                self.train_step(u, p, n, meta)
                if self.post_step is not None:
                    self.post_step()
                self._restore_state(snap)
                if self.pre_step is not None and self.pre_step_undo is not None:
                    self.pre_step_undo()
                self._gidx.copy_(held)
                self._warm = True
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                if self.pre_step is not None:
                    self.pre_step()
                self.train_step(u, p, n, meta)
                if self.post_step is not None:
                    self.post_step()
            self._graph = g
        self._graph.replay()
        return self.loss

    def train_step_graphed(self, users, pos, neg):
        """Same as train_step, replayed from the CUDA graph (the ~40 launches of a step cost more host time than device time at
        netflix scale).  users/pos/neg: int32 CUDA tensors of length B'; they are copied into the static index buffer."""
        B = int(users.numel())
        gi = self.index_buffer(B)
        gi[0, :B].copy_(users, non_blocking=True)
        gi[1, :B].copy_(pos, non_blocking=True)
        gi[2, :B].copy_(neg, non_blocking=True)
        gi[3, :2].copy_(self._meta_table[B], non_blocking=True)
        return self.replay_staged()

    def state_tensors(self):
        """name -> live tensor, everything one training step hands to the next: "model/<name>", "m/<name>", "v/<name>" per optimized
        parameter (the reference's parameter names) and "state", AdamW's device-side fp64 step block.  The graph warm-up's undo and
        the checkpoints (checkpoint.py) both go through this one list."""
        o = self.opt
        out = {}
        for sec, tensors in (("model", o.params), ("m", o.m), ("v", o.v)):
            out.update({sec + "/" + k: t for k, t in zip(self._opt_names, tensors)})
        out["state"] = o.state
        return out

    def load_state(self, src):
        """Copy `src` (name -> tensor, the keys of `state_tensors`) INTO the live tensors.  In place on purpose: a captured graph, the
        optimizer's pointer tables and the compact live-item tables hold these addresses, so rebinding a tensor would fork the state.
        Nothing derived from the parameters outlives a step, so nothing else needs a refresh: the W hi/lo split scratch (keyed by W's
        address, ops.proj_fwd_group) is rewritten by every projection launch; the hoisted engine's TU / TI / Gram tables and the
        compact live-item tables are functions of the constant feature tables alone; MM_Model.hot_path keys its engine by the
        embedding table's address, which a copy keeps; U / I and every activation are recomputed by the next forward."""
        for k, dst in self.state_tensors().items():
            dst.copy_(src[k])

    def _snapshot_state(self):
        return {k: t.clone() for k, t in self.state_tensors().items()}

    _restore_state = load_state

    def set_optimizer(self, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01):
        names = [k for k in PARAM_ORDER if k in self.p and (self.has_feats or k.endswith("embedding.weight"))]
        self._opt_names = names
        self.opt = ops.AdamW([self.p[k] for k in names], lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        return self.opt
