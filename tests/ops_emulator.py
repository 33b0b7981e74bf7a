"""Torch-CPU stand-ins for the subset of `llmrec_b200.ops` that the engines (engine.HotPath, dist.ShardedHotPath) call.  TEST INFRASTRUCTURE ONLY: it lets the host-side orchestration of those engines -- buffer
ping-pong, exchange structure, index arithmetic, optimizer sharding -- run under world-size-2 gloo on a machine without
a GPU.  The product never imports this file; `install()` monkeypatches a test process.  Semantics follow
include/llmrec_b200.h, each function naming the entry point it stands in for."""
import torch
import torch.distributed as dist


class CsrOperator:
    """llmrec_spmm_csr_f32:  Y = epi(diag(rs) . P(vals) . diag(cs) . X) + Z,  epi = row softmax when flagged."""

    def __init__(self, rowptr, col, n_rows, n_cols, vals=None, rs=None, cs=None, tile_nnz=0, plan=None):
        self.rowptr, self.col, self.vals, self.rs, self.cs = rowptr.long(), col.long(), vals, rs, cs
        self.n_rows, self.n_cols, self.nnz = int(n_rows), int(n_cols), int(col.numel())
        self.plan = plan if plan is not None else object()
        assert self.rowptr.numel() == self.n_rows + 1

    def branch(self):                                    # own long-row scratch on the device; nothing to copy here
        return self

    def apply_rows(self, seg, rows, count, max_rows=None, src_mask=None, cta_per_row=False):          # llmrec_spmm_rows_f32: listed rows only
        X, Y, Z, sm = seg
        full = torch.empty_like(Y)
        self.apply([(X if src_mask is None else _masked_rows(X, src_mask), full, Z, sm)])
        r = rows[:int(count[0])].long()
        r = r[r >= 0]
        Y[r] = full[r]

    def apply(self, segs, src_mask=None):
        if src_mask is not None:                         # clear bit = that source row is promised to be zero and must not be read
            segs = [(_masked_rows(X, src_mask), Y, Z, sm) for X, Y, Z, sm in segs]
        rp = self.rowptr
        rows = torch.repeat_interleave(torch.arange(self.n_rows), rp[1:] - rp[:-1])
        e = torch.arange(int(rp[0]), int(rp[-1]))
        c = self.col[e]
        w = torch.ones(e.numel()) if self.vals is None else self.vals[e].clone()
        if self.cs is not None:
            w = w * self.cs[c]
        for X, Y, Z, sm in segs:
            assert X.shape[0] == self.n_cols and Y.shape[0] == self.n_rows
            acc = torch.zeros(self.n_rows, X.shape[1]).index_add_(0, rows, X[c] * w[:, None])
            if self.rs is not None:
                acc = acc * self.rs[:, None]
            if sm:
                acc = torch.softmax(acc, dim=-1)
            if Z is not None:
                acc = acc + Z
            Y.copy_(acc)


def _bits(mask, n):
    w = mask.to(torch.int64) & 0xffffffff
    return ((w[:, None] >> torch.arange(32)) & 1).reshape(-1)[:n].bool()


def _masked_rows(X, src_mask):
    """poison the rows a source mask excludes: a correct kernel never reads them"""
    keep = _bits(src_mask, X.shape[0])
    return torch.where(keep[:, None], X, torch.full_like(X, float("nan"))).nan_to_num(0.0) if False else torch.where(keep[:, None], X, torch.zeros_like(X))


class RowSet:                                            # llmrec_mark_neighbors / llmrec_mark_ids / llmrec_compact_mask
    def __init__(self, n, device):
        self.n = int(n)
        self.mask = torch.zeros((self.n + 31) // 32 + 1, dtype=torch.int32)
        self.list = torch.zeros(max(self.n, 1), dtype=torch.int32)
        self.count = torch.zeros(1, dtype=torch.int32)
        self._set = set()

    def clear(self):
        self._set = set(); self.mask.zero_(); self.count.zero_()

    def _sync(self):
        m = torch.zeros(self.mask.numel() * 32, dtype=torch.int64)
        if self._set:
            m[torch.tensor(sorted(self._set))] = 1
        words = (m.view(-1, 32) << torch.arange(32)).sum(1)
        self.mask.copy_(torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32))

    def add_neighbors(self, rowptr, col, rows):
        rp, c = rowptr.long(), col.long()
        for r in rows.long().tolist():
            if r >= 0:
                self._set.update(c[rp[r]:rp[r + 1]].tolist())
        self._sync()

    def add_ids(self, ids, n=None):                   # llmrec_mark_ids / llmrec_mark_ids_rows: ids[0 .. min(n[0], len(ids)))
        live = ids.long() if n is None else ids.long()[:int(n[0])]
        self._set.update(i for i in live.tolist() if i >= 0)
        self._sync()

    def compact(self):
        ids = sorted(self._set, reverse=True)            # any order is allowed
        self.list[:len(ids)] = torch.tensor(ids, dtype=torch.int32) if ids else torch.zeros(0, dtype=torch.int32)
        self.count[0] = len(ids)


def row_softmax_bwd_rows(S, dS, out, rows, count, max_rows=None):       # llmrec_row_softmax_bwd_rows_f32
    r = rows[:int(count[0])].long()
    out[r] = S[r] * (dS[r] - (S[r] * dS[r]).sum(-1, keepdim=True))
    return out


def zero_rows(Y, idx):                                   # llmrec_zero_rows_f32
    i = idx.long()
    Y[i[i >= 0]] = 0.0


def assign_rows(G, idx, Y):                              # llmrec_assign_rows_f32
    i = idx.long()
    Y[i[i >= 0]] = G[i >= 0]


def fill(t, v):                                          # llmrec_fill_f32
    t.fill_(v)


def row_scale_softmax(X, scale, out, softmax):           # llmrec_row_scale_softmax_f32
    y = X * scale[:, None] if scale is not None else X.clone()
    out.copy_(torch.softmax(y, dim=-1) if softmax else y)
    return out


def row_softmax_bwd(S, dS, out=None):                    # llmrec_row_softmax_bwd_f32
    r = S * (dS - (S * dS).sum(-1, keepdim=True))
    if out is None:
        return r
    out.copy_(r)
    return out


def _unit(x):
    return x / x.norm(dim=1, keepdim=True).clamp_min(1e-12)           # F.normalize(x, p=2, dim=1)


def _live_rows(rows, count, max_rows):
    """rows[0 .. min(count[0], max_rows)), entries < 0 skipped (the device-count row-list forms)"""
    mx = rows.numel() if max_rows is None else min(int(max_rows), rows.numel())
    r = rows[:min(int(count[0]), mx)].long()
    return r[r >= 0]


def fuse_fwd(layers, sides, coefs, out, rows=None, compact=False, count=None, max_rows=None):   # llmrec_fuse_fwd_f32 / _rows_f32
    if count is not None:
        rows = _live_rows(rows, count, max_rows)
    if compact:                                          # layers at rows[b]; sides and out are compact [len(rows) x d] blocks
        r = rows.long()
        m = sum(l[r.clamp(min=0)] for l in layers) / len(layers)
        for x, c in zip(sides, coefs):
            m = m + c * _unit(x)
        out.copy_(torch.where((r >= 0)[:, None], m, torch.zeros_like(m)))          # a negative entry = not mine: zeros
        return out
    m = sum(layers) / len(layers)
    for x, c in zip(sides, coefs):
        m = m + c * _unit(x)
    if rows is None:
        out.copy_(m)
    else:
        out[rows.long()] = m[rows.long()]
    return out


def rank1_add(blocks):                                   # llmrec_rank1_add_f32
    for Y, sc, b in blocks:
        Y += sc[:, None] * b[None, :]


def scaled_colsum(terms, out, accumulate=False):         # llmrec_scaled_colsum_f32
    t = sum(((G * sc[:, None]) if sc is not None else G).sum(0) for G, sc in terms)
    out.copy_(out + t if accumulate else t)


def feat_reg_gram(W, b, G, h, n2, c, dW, db, loss):      # llmrec_feat_reg_gram_f32
    WG, Wh = W @ G, W @ h
    loss += 0.5 * c * ((WG * W).sum() + 2 * (b * Wh).sum() + n2 * (b * b).sum())
    dW += c * (WG + b[:, None] * h[None, :])
    db += c * (Wh + n2 * b)


def fuse_bwd(g, n_layers, d_layer, sides, coefs, d_sides, accumulate, rows=None, count=None, max_rows=None):   # llmrec_fuse_bwd_f32 / _rows_f32
    assert rows is None or count is not None
    r = slice(None) if count is None else _live_rows(rows, count, max_rows)     # the row-list form writes the listed rows only
    if d_layer is not None:
        d_layer[r] = g[r] / n_layers
    for x, c, dx in zip(sides, coefs, d_sides):
        y = _unit(x[r])
        t = c * (g[r] - y * (y * g[r]).sum(1, keepdim=True)) / x[r].norm(dim=1, keepdim=True).clamp_min(1e-12)
        dx[r] = dx[r] + t if accumulate else t


def proj_fwd_group(problems, d, mode=0):                 # llmrec_proj_fwd_group_f32
    for X, W, b, out in problems:
        out.copy_(X @ W.t() + (b if b is not None else 0.0))


def proj_wgrad_group(problems, d, mode=0):               # llmrec_proj_wgrad_group_f32
    for X, dY, dW, db, acc in problems:
        gw, gb = dY.t() @ X, dY.sum(0)
        dW.copy_(dW + gw if acc else gw)
        if db is not None:
            db.copy_(db + gb if acc else gb)


def sqnorm_grad(X, G, c, accumulate, loss):              # llmrec_sqnorm_grad_f32
    loss += c * 0.5 * X.pow(2).sum()
    if G is not None:
        G.copy_(G + c * X if accumulate else c * X)


def gather_rows(X, idx, out):                            # llmrec_gather_rows_f32: idx < 0 -> zeros
    i = idx.long()
    out.copy_(torch.where((i >= 0)[:, None], X[i.clamp(min=0)], torch.zeros(1)))
    return out


def scatter_add_rows(G, idx, Y):                         # llmrec_scatter_add_rows_f32: idx < 0 skipped
    i = idx.long()
    keep = i >= 0
    Y.index_add_(0, i[keep], G[keep])


def bpr_work(n_heads, B, device):
    return torch.zeros(1)


def grad_init(regions, loss):                            # llmrec_grad_init_f32
    loss.zero_()
    for G, X, c in regions:
        if X is None:
            G.zero_()
        else:
            G.copy_(c * X)
            loss += c * 0.5 * X.pow(2).sum()


def bpr_heads(heads, users, pos, neg, n_keep, regs0_over_bs, out, loss, work, meta=None):      # llmrec_bpr_heads_f32
    if meta is not None:                                 # capacity-sized index buffers: the live length and n_keep come from `meta`
        B, n_keep = int(meta[0]), int(meta[1])
        users, pos, neg = users[:B], pos[:B], neg[:B]
    u, p, n = users.long(), pos.long(), neg.long()
    for h, (XU, XI, GU, GI, w_mf, w_emb) in enumerate(heads):
        a = XU[u].clone().requires_grad_(True)
        b = XI[p].clone().requires_grad_(True)
        c = XI[n].clone().requires_grad_(True)
        maxi = torch.nn.functional.logsigmoid((a * b).sum(1) - (a * c).sum(1) + 1e-8)
        keep = torch.argsort(maxi.detach(), stable=True)[:n_keep]
        mf = -maxi[keep].mean()
        emb = regs0_over_bs * (1 / (2 * a.pow(2).sum() + 1e-8) + 1 / (2 * b.pow(2).sum() + 1e-8) + 1 / (2 * c.pow(2).sum() + 1e-8))
        (w_mf * mf + w_emb * emb).backward()
        if GU is not None:
            GU.index_add_(0, u, a.grad)
        if GI is not None:
            GI.index_add_(0, p, b.grad)
            GI.index_add_(0, n, c.grad)
        loss += (w_mf * mf + w_emb * emb).detach()
        out[4 * h:4 * h + 3] = torch.tensor([float(mf), float(emb), float(n_keep)])


def score_topk(U, I, users, mask_rowptr, mask_col, K, mode=0, want_vals=False):     # llmrec_score_topk_f32
    """exact fp32 scores, train items excluded, ties -> lowest item id, -1 past the last candidate"""
    u = users.long()
    S = U[u] @ I.t()
    rp = mask_rowptr.long()
    rows = torch.repeat_interleave(torch.arange(rp.numel() - 1), rp[1:] - rp[:-1])
    dense = torch.zeros(rp.numel() - 1, I.shape[0], dtype=torch.bool)
    dense[rows, mask_col.long()] = True
    S = S.masked_fill(dense[u], float("-inf"))
    val, idx = torch.sort(S, dim=1, descending=True, stable=True)
    val, idx = val[:, :K], idx[:, :K].to(torch.int32)
    idx = torch.where(torch.isinf(val), torch.full_like(idx, -1), idx)
    return (idx, val) if want_vals else idx


def topk_hits(idx, users, truth_rowptr, truth_col):      # llmrec_topk_hits
    rp, col = truth_rowptr.long(), truth_col.long()
    out = torch.zeros(idx.shape, dtype=torch.uint8)
    for b, u in enumerate(users.long().tolist()):
        truth = set(col[rp[u]:rp[u + 1]].tolist())
        out[b] = torch.tensor([1 if int(i) in truth else 0 for i in idx[b].tolist()], dtype=torch.uint8)
    return out


class AdamW:                                             # llmrec_adamw_advance + llmrec_adamw_step_f32 (torch.optim.AdamW defaults)
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01):
        self.params, self.lr, self.betas, self.eps, self.wd = list(params), lr, betas, eps, weight_decay
        self.m = [torch.zeros_like(p) for p in self.params]
        self.v = [torch.zeros_like(p) for p in self.params]
        self.t = 0

    def advance(self):
        self.t += 1

    def step_tensor(self, i, grad, row_mask=None):
        if row_mask is not None:
            grad = torch.where(_bits(row_mask, grad.shape[0])[:, None], grad, torch.zeros_like(grad))
        self._update(self.params[i], grad, self.m[i], self.v[i])

    def _update(self, p, g, m, v):
        """adam1 of csrc/adamw.cu: fp32 hyper-parameters (1 - beta formed from fp32 beta), the step size and bias correction the
        advance kernel forms in double, rounded to fp32"""
        f = lambda x: torch.tensor(x, dtype=torch.float32)
        b1, b2, eps = f(self.betas[0]), f(self.betas[1]), f(self.eps)
        step = f(self.lr / (1 - self.betas[0] ** self.t))
        bc2s = f((1 - self.betas[1] ** self.t) ** 0.5)
        p.mul_(f(1) - f(self.lr) * f(self.wd))
        m.add_((1 - b1) * (g - m))
        v.copy_(v * b2 + (1 - b2) * g * g)
        p.sub_(step * (m / (v.sqrt() / bc2s + eps)))

    def step(self, grads, row_masks=None):
        self.t += 1
        if row_masks is not None:                        # llmrec_adamw_step_rows_f32: g is read on the flagged rows only
            grads = [g if mk is None else torch.where(_bits(mk, g.shape[0])[:, None], g, torch.zeros_like(g)) for g, mk in zip(grads, row_masks)]
        for p, g, m, v in zip(self.params, grads, self.m, self.v):
            self._update(p, g, m, v)


def install():
    """Patch llmrec_b200.ops / llmrec_b200.dist in THIS process; add gloo stand-ins for the two NCCL-only collectives."""
    import sys
    import llmrec_b200.ops as ops
    import llmrec_b200.dist as D
    me = sys.modules[__name__]
    import llmrec_b200.graph as G
    for name in ("CsrOperator", "RowSet", "row_softmax_bwd_rows", "zero_rows", "assign_rows", "fill", "row_scale_softmax", "row_softmax_bwd", "fuse_fwd", "fuse_bwd", "gather_rows", "scatter_add_rows",
                 "bpr_work", "bpr_heads", "grad_init", "rank1_add", "scaled_colsum", "feat_reg_gram", "AdamW", "proj_fwd_group", "proj_wgrad_group", "sqnorm_grad", "score_topk", "topk_hits"):
        setattr(ops, name, getattr(me, name))
    D.CsrOperator = CsrOperator
    G.CsrOperator = CsrOperator

    class _Done:
        def wait(self):
            return True

    def reduce_scatter_tensor(out, inp, group=None, async_op=False):
        t = inp.clone()
        dist.all_reduce(t, group=group)
        r, n = dist.get_rank(group), out.shape[0]
        out.copy_(t[r * n:(r + 1) * n])
        return _Done() if async_op else None

    def all_gather_into_tensor(out, inp, group=None):
        parts = [torch.empty_like(inp) for _ in range(dist.get_world_size(group))]
        dist.all_gather(parts, inp.clone(), group=group)
        out.copy_(torch.cat(parts))

    D.dist.reduce_scatter_tensor = reduce_scatter_tensor
    D.dist.all_gather_into_tensor = all_gather_into_tensor
