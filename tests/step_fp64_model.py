"""fp64 restatement of one whole training step: every loss head, its gradient with respect to every parameter, and the bound an
engine's step gradients are held to.  TEST INFRASTRUCTURE ONLY.

The forward is `oracle.llmrec_oracle.forward`, run in float64 on any device.  The operators are built from an engine's own binary
CSR and its fp32 scales su / si, promoted to fp64, so the reference restates the operation the engine computes, not the reference
project's float64 normalisation.  Feature tables enter at their exact values (fp32 as stored, bf16 widened, int8 through
`feat_int8.dequantize`); W and b at their fp32 values.

Heads: "mf" and "emb" of the ID head (main.py:232-235), "img" and "txt" (x mm_mf_rate), one "aug:<key>" per attribute key
(x aug_mf_rate), "feat" (feat_reg, main.py:151-156) and, in the mask branch, "restore" (x att_re_rate, main.py:258-271).  Each
head's gradient is its own `autograd.grad`, so the bound below can weigh each head by its own size.  With feats=None the step is
the ID-only configuration of dist.ShardedHotPath (no feature tables, params = the two ID tables): `id_forward`, heads "mf" / "emb".

Kept sets: each BPR head keeps the n_keep = int((1 - rate) * B') smallest maxi (stable argsort, ties to the lower position, as the
kernel).  `StepRef.cuts[head]` = (gap, need): the fp64 gap of x = <u, p> - <u, n> + 1e-8 between the largest kept and the
smallest dropped row (maxi = logsigmoid(x) is increasing in x, and at the loud rates the cut often lies where maxi ~ -1e-15, so the
gap is measured before the sigmoid), and the largest change of x an engine's rounding can make at those two rows,
TAU_CUT * (1 + sum_k |u_k| (|p_k| + |n_k|)).  A test asserts
gap > need first, so an engine cannot have kept another set; with seeded batches that is a property of the inputs, not a flake.

The bound.  For element e of parameter theta, with g_e the fp64 gradient and g^_e the engine's:

    |g^_e - g_e| <= tau * (M_e + rho * max over e's row of M)

    M   = sum over heads h of |g_h|                     (every parameter)
        + sum_h |dY_h|^T |X|    (projection weights: dY_h = head h's gradient at that layer's output, X its feature table)
        + sum_h sum_rows |dY_h| (projection biases)

Why this form.  The engine computes each head's contribution with fp32 (or TF32) arithmetic whose relative error is bounded by
the size of that contribution, not by the size of the sum: the main head's share of item_trans is 2.4e-3 of the aug heads' at the
default rates, so a bound on |g| alone would hide it, and a bound on max|g| of the tensor would hide every small element.  Summing
|g_h| gives each head's own scale.  A weight gradient is dY^T X summed over 10^4 rows with cancellation: its rounding is relative
to sum |dY||X| (the magnitude test_live_items_gpu.py uses), which may exceed |dW| by orders of magnitude.  rho * rowmax covers the
absolute error an element inherits from the other elements of its row through the chain (the softmax and the normalisations mix
the d columns of a row; the SpMM chain mixes rows of one sign pattern into another).

tau, per projection arithmetic (the rest of the step is fp32 in every mode):
  TAU["fp32"]   = 2e-5  fp32 SIMT projections (proj_mode 2).  The fp32 oracle reaches 0.15 of it on the tiny set and 0.4 at the
                        netflix shape; the emulated engines stay below it.
  TAU["3xtf32"] = 4e-4  3xTF32 (proj_mode 0) and bf16 / int8 tables on the 3-term W.  The ID-embedding gradients inherit the forward's
                        projection error through U / I, and the kernels are specified to 5e-5 of |Y| per output
                        (test_tc_exactness_gpu.py's fingerprint), 16x the error of an exact 3xTF32 split: scaling the TF32
                        calibration below by that error gives 3e-4.  On the H100 the engines reach up to 6.7 x 2e-5 at the netflix
                        shape (an exact truncating 3xTF32 split, emulated on CPU, reaches 0.28 x 2e-5).
  TAU["tf32"]   = 2e-2  plain TF32 (proj_mode 1): the tensor cores truncate fp32 operands to 10 mantissa bits; the fp32 oracle with
                        truncated TF32 projections (`reference(..., proj="tf32-rz")`) reaches 0.31 of it at the netflix shape, and
                        the H100 engines the same.
RHO = 0.1: the fp32 oracle's ID-embedding errors reach 5e-7 of their row's largest M (a row's elements share the softmax and the
normalisations), which tau * rho covers with 4x to spare at TAU["fp32"].  The mutations of tests/test_step_grads_fp64_cpu.py exceed
the bound by 2e3 or more at TAU["fp32"], so each is still rejected at TAU["tf32"].

Structure: an element whose fp64 gradient is exactly zero (an ID row outside the batch's L-hop neighbourhood, an item or user with
no edge that the batch does not name) must be exactly zero in the engine.
"""
from __future__ import annotations

import dataclasses
import unittest.mock
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from llmrec_b200 import feat_int8
from oracle import llmrec_oracle as O

TAU = {"fp32": 2e-5, "3xtf32": 4e-4, "tf32": 2e-2}
RHO = 0.1
TAU_CUT = {"fp32": 2e-5, "3xtf32": 5e-5, "tf32": 2e-3}

PROJ = {"image_trans": "image", "text_trans": "text", "user_trans": "user", "item_trans": "item"}


def oracle_config(cfg) -> O.OracleConfig:
    """The OracleConfig of an engine's HotPathConfig (same rates, L = n_layers)."""
    return O.OracleConfig(embed_size=cfg.embed_size, weight_size=(cfg.embed_size,) * cfg.n_layers, batch_size=cfg.batch_size,
                          regs0=cfg.regs0, model_cat_rate=cfg.model_cat_rate, user_cat_rate=cfg.user_cat_rate,
                          item_cat_rate=cfg.item_cat_rate, aug_mf_rate=cfg.aug_mf_rate, mm_mf_rate=cfg.mm_mf_rate,
                          prune_loss_drop_rate=cfg.prune_loss_drop_rate, feat_reg_decay=cfg.feat_reg_decay)


def sparse64(op, device=None) -> torch.Tensor:
    """fp64 sparse COO of an engine CsrOperator Y = diag(rs) P(vals) diag(cs) X (the kernels' operator, or its CPU stand-in)."""
    dev = torch.device(device) if device is not None else op.rowptr.device
    rp, col = op.rowptr.long().to(dev), op.col.long().to(dev)
    rows = torch.repeat_interleave(torch.arange(op.n_rows, device=dev), rp[1:] - rp[:-1])
    v = torch.ones(col.numel(), dtype=torch.float64, device=dev)
    if op.vals is not None:
        v = v * op.vals.to(dev, torch.float64)
    if op.rs is not None:
        v = v * op.rs.to(dev, torch.float64)[rows]
    if op.cs is not None:
        v = v * op.cs.to(dev, torch.float64)[col]
    return torch.sparse_coo_tensor(torch.stack([rows, col]), v, (op.n_rows, op.n_cols)).coalesce()


def widen(X, k=None, device=None) -> torch.Tensor:
    """A feature table at its exact value in fp64 (int8: the table of logical width k)."""
    if X.dtype == torch.int8:
        X = feat_int8.dequantize(X, k)
    return X.to(device if device is not None else X.device, torch.float64)


def engine_inputs(hp, device=None):
    """(params, feats, ui, iu) in fp64 of an engine as it stands: the parameters of the NEXT step, its full feature tables."""
    dev = torch.device(device) if device is not None else hp.E_u.device
    p = {k: v.detach().to(dev, torch.float64) for k, v in hp.p.items()}
    k_of = lambda name: int(hp.p[name + ".weight"].shape[1])
    f = hp.feats
    feats = dict(image=widen(f["image"], k_of("image_trans"), dev), text=widen(f["text"], k_of("text_trans"), dev),
                 user=widen(f["user"], k_of("user_trans"), dev),
                 item={k: widen(v, k_of("item_trans"), dev) for k, v in f["item"].items()})
    return p, feats, sparse64(hp.ui, dev), sparse64(hp.iu, dev)


def id_forward(params, ui, iu, cfg: O.OracleConfig) -> dict:
    """The ID-only forward: the propagation and layer mean of `oracle.llmrec_oracle.forward` (Models.py:172-186) with no side term."""
    e_u, e_i = params["user_id_embedding.weight"], params["item_id_embedding.weight"]
    us, its = [e_u], [e_i]
    L = cfg.n_ui_layers
    for l in range(L):
        e_u = torch.mm(ui, e_i)
        if l == L - 1:
            e_u = torch.softmax(e_u, dim=-1)
        e_i = torch.mm(iu, e_u)
        if l == L - 1:
            e_i = torch.softmax(e_i, dim=-1)
        us.append(e_u); its.append(e_i)
    return dict(U=torch.mean(torch.stack(us), dim=0), I=torch.mean(torch.stack(its), dim=0))


@dataclass
class StepRef:
    loss: float                     # total
    parts: dict                     # head -> fp64 loss value of that head, rate included
    head_out: dict                  # head -> (mf, emb) as the kernel's out slots hold them (rate excluded)
    grads: dict                     # name -> fp64 gradient, summed over the heads
    per_head: dict                  # head -> name -> fp64 gradient
    mag: dict                       # name -> M of the bound
    cuts: dict                      # BPR head -> (gap of x at the cut, 1 + sum |u| (|p| + |n|) over the two rows at the cut)
    n_keep: int
    B: int


def _tf32(x, rnd):
    """x cut to TF32 (10 explicit mantissa bits): rounded to nearest (ties away from zero), or truncated (rnd=False)"""
    b = x.detach().contiguous().view(torch.int32)
    return ((b + 0x1000 if rnd else b) & ~0x1FFF).view(torch.float32)


def _linear_as(proj):
    """F.linear with the forward arithmetic of a tensor-core mode on fp32 operands, accumulated in fp32: "tf32" (operands cut to TF32)
    or "3xtf32" (X and W split into TF32 hi + lo, the lo * lo product dropped); suffix "-rz" truncates the cut instead of rounding
    it.  Its gradient is the exact product's: the weight-gradient kernels' error is the |dY|^T |X| term of the bound."""
    mode, rnd = proj.split("-") if "-" in proj else (proj, "rn")
    rnd = rnd == "rn"

    def lin(x, W, b=None):
        if mode == "tf32":
            y = _tf32(x, rnd) @ _tf32(W, rnd).t()
        else:
            xh, wh = _tf32(x, rnd), _tf32(W, rnd)
            xl, wl = _tf32(x.detach() - xh, rnd), _tf32(W.detach() - wh, rnd)
            y = xh @ wh.t() + (xh @ wl.t() + xl @ wh.t())
        exact = torch.matmul(x, W.t())
        y = exact + (y - exact).detach()              # the forward's value, the exact product's gradient
        return y if b is None else y + b
    return lin


def reference(params, feats, ui, iu, cfg: O.OracleConfig, users, pos, neg, n_items, drop=None, restore=None, dtype=torch.float64, proj=None, drop_heads=(), n_keep=None, reg_div=None, feat_div=None, detach_last=False, softmax_identity=False):
    """One step's losses and gradients at `params` (fp64 leaves are made here).  users / pos / neg: the B' triplets (lists or int
    tensors).  drop: the dropout masks of the mask branch (O.forward's order); restore: dict(rate, dec, raw_user, raw_items, i_mask,
    u_mask, alpha, kind) for the restoration head.  dtype=float32 gives the fp32 oracle (calibration); proj="3xtf32" / "tf32" gives it
    the projection arithmetic of those tensor-core modes.

    feats=None: the ID-only step (`id_forward`, the "mf" and "emb" heads only).

    The remaining keywords are mutations of the step, for the tests that show the bound can see them: drop_heads (head names
    left out), n_keep (instead of int((1 - rate) * B')), reg_div (instead of cfg.batch_size), feat_div (instead of n_items),
    detach_last (the last triplet's rows get no gradient from any BPR head), softmax_identity (the last layer's softmax Jacobian
    replaced by the identity)."""
    dev = next(iter(params.values())).device
    cast = lambda t: t.to(dev, dtype)
    P = {k: cast(v).detach().requires_grad_(True) for k, v in params.items()}
    X = None if feats is None else \
        dict(image=cast(feats["image"]), text=cast(feats["text"]), user=cast(feats["user"]), item={k: cast(v) for k, v in feats["item"].items()})
    ui_, iu_ = cast(ui), cast(iu)
    dr = None if drop is None else [cast(m) for m in drop]
    idx = lambda a: torch.as_tensor(a, dtype=torch.long).to(dev)
    u, p, n = idx(users), idx(pos), idx(neg)
    if proj is not None:                 # the fp32 oracle with the projections of a tensor-core mode (calibration)
        assert dtype == torch.float32
        with unittest.mock.patch.object(F, "linear", _linear_as(proj)):
            return reference(params, feats, ui, iu, cfg, users, pos, neg, n_items, drop, restore, dtype, None, drop_heads, n_keep,
                             reg_div, feat_div, detach_last, softmax_identity)
    B = int(u.numel())
    keep_n = int((1 - cfg.prune_loss_drop_rate) * B) if n_keep is None else int(n_keep)
    fwd = (lambda: id_forward(P, ui_, iu_, cfg)) if X is None else (lambda: O.forward(P, X, ui_, iu_, cfg, drop=dr))
    if softmax_identity:                 # softmax's value, the identity as its Jacobian (O.forward calls torch.softmax on layer L only)
        sm = torch.softmax
        fake = lambda x, dim=-1: x + (sm(x, dim=dim) - x).detach()
        with unittest.mock.patch.object(torch, "softmax", fake):
            out = fwd()
    else:
        out = fwd()

    def rows(T, ix):
        G = T[ix]
        return torch.cat([G[:-1], G[-1:].detach()]) if detach_last else G

    cuts = {}

    def bpr(name, XU, XI):
        a, b, c = rows(XU, u), rows(XI, p), rows(XI, n)
        x = (a * b).sum(1) - (a * c).sum(1) + 1e-8
        maxi = F.logsigmoid(x)
        order = torch.argsort(maxi.detach().cpu(), stable=True).to(dev)
        if 0 < keep_n < B:
            s = x.detach()[order]
            mag = ((a.detach().abs() * (b.detach().abs() + c.detach().abs())).sum(1))[order[keep_n - 1:keep_n + 1]].max()
            cuts[name] = (float(s[keep_n] - s[keep_n - 1]), 1 + float(mag))
        mf = -maxi[order[:keep_n]].mean()
        reg = 1.0 / (2 * (a ** 2).sum() + 1e-8) + 1.0 / (2 * (b ** 2).sum() + 1e-8) + 1.0 / (2 * (c ** 2).sum() + 1e-8)
        emb = cfg.regs0 * reg / (cfg.batch_size if reg_div is None else reg_div)
        return mf, emb

    losses, head_out = {}, {}
    mf, emb = bpr("mf", out["U"], out["I"])
    losses["mf"], losses["emb"] = mf, emb
    head_out["mf"] = (float(mf), float(emb))
    if X is None:                        # the ID-only step: no side heads, no projections
        for h in drop_heads:
            losses.pop(h)
        names = list(P)
        grads = {k: torch.zeros_like(P[k]) for k in names}
        per_head, mag = {}, {k: torch.zeros_like(P[k]) for k in names}
        for h, L in losses.items():
            g = torch.autograd.grad(L, [P[k] for k in names], retain_graph=True)
            per_head[h] = {k: gg.detach() for k, gg in zip(names, g)}
            for k in names:
                grads[k] += per_head[h][k]; mag[k] += per_head[h][k].abs()
        return StepRef(loss=sum(float(L) for L in losses.values()), parts={h: float(L) for h, L in losses.items()}, head_out=head_out,
                       grads=grads, per_head=per_head, mag=mag, cuts=cuts, n_keep=keep_n, B=B)
    for name, su, si in (("img", "img_u", "img_i"), ("txt", "txt_u", "txt_i")):
        m, e = bpr(name, out[su], out[si])
        losses[name] = cfg.mm_mf_rate * m
        head_out[name] = (float(m), float(e))
    for k in out["att_i"]:
        m, e = bpr("aug:" + k, out["prof_u"], out["att_i"][k])
        losses["aug:" + k] = cfg.aug_mf_rate * m
        head_out["aug:" + k] = (float(m), float(e))
    sq = lambda x: 0.5 * (x ** 2).sum()
    fr = (sq(out["img_i"]) + sq(out["txt_i"]) + sq(out["img_u"]) + sq(out["txt_u"])) / (n_items if feat_div is None else feat_div)
    losses["feat"] = cfg.feat_reg_decay * fr
    if restore is not None:
        r = restore
        dec = {k: cast(v) for k, v in r["dec"].items()}
        losses["restore"] = r["rate"] * O.restoration_loss(out, dec, cast(r["raw_user"]), {k: cast(v) for k, v in r["raw_items"].items()},
                                                           idx(r["i_mask"]), idx(r["u_mask"]), alpha=r.get("alpha", 2), kind=r.get("kind", "sce"))
    for h in drop_heads:
        losses.pop(h)

    names = list(P)
    keys = list(out["att_u"])
    # projection outputs: the total gradient at img_u / txt_u / att_u / p_usr, pulled back through ui (and the dropout mask)
    mids = [out["img_u"], out["txt_u"]] + [out["att_u"][k] for k in keys] + [out["p_usr"]]
    uiT = ui_.t().coalesce()
    per_head, dY = {}, {}
    for h, L in losses.items():
        g = torch.autograd.grad(L, [P[k] for k in names] + mids, retain_graph=True, allow_unused=True)
        per_head[h] = {k: (gg.detach() if gg is not None else torch.zeros_like(P[k])) for k, gg in zip(names, g[:len(names)])}
        gm = [gg.detach() if gg is not None else torch.zeros_like(mm) for gg, mm in zip(g[len(names):], mids)]
        y = [torch.sparse.mm(uiT, x) for x in gm[:-1]] + [gm[-1]]          # img_u = ui.P_img, att_u = ui.P_att, p_usr itself
        if dr is not None:
            y = [y[0] * dr[0], y[1] * dr[1]] + [yy * dr[3 + j] for j, yy in enumerate(y[2:-1])] + [y[-1] * dr[2]]
        dY[h] = dict(image_trans=[(y[0], X["image"])], text_trans=[(y[1], X["text"])],
                     item_trans=[(yy, X["item"][k]) for yy, k in zip(y[2:-1], keys)], user_trans=[(y[-1], X["user"])])
    grads = {k: sum(per_head[h][k] for h in per_head) for k in names}
    mag = {k: sum(per_head[h][k].abs() for h in per_head) for k in names}
    for layer in PROJ:
        for h in dY:
            for y, x in dY[h][layer]:
                mag[layer + ".weight"] = mag[layer + ".weight"] + y.abs().t() @ x.abs()
                mag[layer + ".bias"] = mag[layer + ".bias"] + y.abs().sum(0)
    total = sum(float(L) for L in losses.values())
    return StepRef(loss=total, parts={h: float(L) for h, L in losses.items()}, head_out=head_out, grads=grads, per_head=per_head,
                   mag=mag, cuts=cuts, n_keep=keep_n, B=B)


def allowed(ref: StepRef, name, tau, rho=RHO):
    """The elementwise bound of the module docstring for parameter `name`."""
    M = ref.mag[name]
    row = M.abs().amax(dim=-1, keepdim=True) if M.dim() == 2 else M.abs().max()
    return tau * (M + rho * row)


def grad_excess(ref: StepRef, grads, tau, rho=RHO):
    """name -> (worst |g^ - g| / allowed, number of elements over the bound, number of structural zeros broken)."""
    res = {}
    for k, g in ref.grads.items():
        got = grads[k].detach().to(g.device, torch.float64)
        err = (got - g).abs()
        lim = allowed(ref, k, tau, rho)
        zero = g == 0
        ratio = torch.where(zero, torch.zeros_like(err), err / lim.clamp_min(1e-300))
        res[k] = (float(ratio.max()), int((ratio > 1).sum()), int((zero & (got != 0)).sum()))
    return res


def check_grads(ref: StepRef, grads, tau, rho=RHO, what=""):
    """Assert the bound on every element of every parameter's gradient and the structural zeros."""
    res = grad_excess(ref, grads, tau, rho)
    bad = {k: v for k, v in res.items() if v[1] or v[2]}
    assert not bad, f"{what}: (worst err / bound, elements over, nonzero where fp64 is exactly zero) {bad}"
    return res


def check_cuts(ref: StepRef, mode="fp32", what=""):
    """Every BPR head's kept set is the same for any engine within the bound: the fp64 gap at the cut exceeds what rounding moves."""
    thin = {h: (gap, TAU_CUT[mode] * mag) for h, (gap, mag) in ref.cuts.items() if not gap > TAU_CUT[mode] * mag}
    assert not thin, f"{what}: kept-set cut thinner than the rounding bound (gap, need) {thin}"


def check_loss(ref: StepRef, loss, head_out, heads, tau, what=""):
    """hp.loss against the fp64 total, and each head's (mf, emb, kept) slots of head_out; heads: the head names in engine order.
    Bound: tau * (sum of |head losses| + 1e-6) for the total, tau * (|value| + 1e-6) per slot."""
    tot = sum(abs(v) for v in ref.parts.values())
    assert abs(float(loss) - ref.loss) <= tau * (tot + 1e-6), f"{what}: loss {float(loss)} vs {ref.loss}"
    ho = head_out.detach().double().cpu().view(-1, 4)
    for i, h in enumerate(heads):
        mf, emb = ref.head_out[h]
        assert abs(float(ho[i, 0]) - mf) <= tau * (abs(mf) + 1e-6), f"{what}: head {h} mf {float(ho[i, 0])} vs {mf}"
        assert abs(float(ho[i, 1]) - emb) <= tau * (abs(emb) + 1e-30), f"{what}: head {h} emb {float(ho[i, 1])} vs {emb}"
        assert int(ho[i, 2]) == ref.n_keep, f"{what}: head {h} kept {int(ho[i, 2])} vs {ref.n_keep}"


def engine_heads(keys):
    """The order of the engine's BPR heads (head_out rows): ID, image, text, one per attribute key."""
    return ["mf", "img", "txt"] + ["aug:" + k for k in keys]


def loud(cfg):
    """A legitimate flag setting under which every head carries a visible share of some parameter's gradient (the default rates
    make the emb head 1e-10 of every gradient and the ID head's share of item_trans 2e-3)."""
    return dataclasses.replace(cfg, regs0=1e4, mm_mf_rate=0.7, aug_mf_rate=0.9, feat_reg_decay=0.8, item_cat_rate=0.3, user_cat_rate=1.3,
                               model_cat_rate=0.4)
